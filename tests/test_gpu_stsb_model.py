"""STS-B-DIR's sentence-pair model on the H100 (imbalanced-regression_b200/{rnn,models}.py, csrc/lstm.cu,
csrc/pair_encoder.cu) against float64 (oracle/stsb_ref.py).

Bounds:
- Recurrent forward step, one launch, on the same bf16 operands.  The GEMM accumulates K = Hp exact bf16 products in
  fp32: |error| <= K 2^-24 sum_k |h_k w_k|.  Adding the bf16 projection (exact) and the fp32 bias (the sum
  b_ih + b_hh is rounded once) adds 2^-24 (|x| + |b|) per rounding, so each pre-activation is within
  e_a = (K + 4) 2^-24 (sum |h w| + |x| + |b|).  sigmoid and tanh have slopes <= 1 and fp32 expf / tanhf are within a few
  ulps, so an activated gate is within e_a + 2^-20, and c = f c' + i g within e_c = (e_a,f + 2^-20) |c'| +
  e_a,i + e_a,g + 2^-19 (1 + |c'|).  h = o tanh(c) is within e_a,o + e_c + 2^-19 before its rounding to bf16 (2^-8 |h|).
- Recurrent backward step: dh = dgates' . W_hh + dy with the same GEMM bound (K = 4Hp).  The cell backward is a few
  fp32 products of values in [-1, 1] times dh / dc (relative 2^-20 each), then rounding to bf16: relative 2^-8 plus
  (e_dh + 2^-20 |dc|) times the gate factors.
- Whole layer backward (dirb200_lstm_layer_bwd): the steps are deterministic, so the layer must give the bits of its
  steps launched one at a time for s = T-1 .. 0; each step is then held to the step bound above given the dg[s + 1] and
  dc it read (teacher forcing, so errors do not compound through the bound).
- Inference forward (save = 0): the same arithmetic as save = 1 on two ping-pong state slots, so the same bits.
- Max-pool and pair features: the maximum of fp32 products is exact, so u and v equal torch's max in fp32 bit for bit,
  and the backward scatter is one fp32 expression rounded to bf16, equal to the same expression in torch.
- The whole model (no teacher forcing): the native error must be within 8 x the difference between the float64 oracle
  on the exact fp32 parameters and on bf16-rounded parameters and embeddings (the operands the kernels see); the
  native path also rounds h, the projection and (backward) the gate gradients to bf16 at every step, a perturbation of
  the same order as rounding the operands.  Gradients: relative Frobenius error <= 5e-2 (bf16 gate gradients, relative
  2^-9 each, accumulated through at most T = 9 recurrent steps).
The file reruns itself with DIRB200_SMS=7."""
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24


def _dev():
    return torch.device("cuda", 0)


def pad64(n):
    return (n + 63) // 64 * 64


def gate_perm(H, Hp):
    """interleaved column n of one direction -> torch gate row, or -1"""
    n = torch.arange(4 * Hp)
    u = (n // 64) * 16 + n % 16
    g = (n % 64) // 16
    return torch.where(u < H, g * H + u, torch.full_like(n, -1))


def prep(H, din, blocks, Dp, seed, scale=0.3):
    import _lib
    g = torch.Generator().manual_seed(seed)
    Hp = pad64(H)
    w = []
    for _ in range(2):
        w += [torch.randn(4 * H, din, generator=g) * scale, torch.randn(4 * H, H, generator=g) * scale,
              torch.randn(4 * H, generator=g) * scale, torch.randn(4 * H, generator=g) * scale]
    w = [t.to(_dev()) for t in w]
    out = [torch.full((8 * Hp, Dp), float("nan"), dtype=torch.bfloat16, device=_dev()),
           torch.full((Dp, 8 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev()),
           torch.full((2, 4 * Hp, Hp), float("nan"), dtype=torch.bfloat16, device=_dev()),
           torch.full((2, Hp, 4 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev()),
           torch.full((2, 4 * Hp), float("nan"), device=_dev())]
    _lib.call("dirb200_lstm_prep_weights", *[_lib.ptr(t) for t in w], H, din, blocks, Hp, Dp,
              *[_lib.ptr(t) for t in out], None)
    return w, out


def lens_for(M, T, seed):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(1, T + 1, (M,), generator=g)
    lens[0] = T
    if M > 1:
        lens[1] = 1
    return lens.to(torch.int32)


@pytest.mark.parametrize("H,din,blocks", [(20, 24, 1), (100, 200, 2), (1500, 300, 1)])
def test_prep_weights_layout_and_round_trip(H, din, blocks):
    """The re-layout puts torch's gate rows at the interleaved columns (bf16 round to nearest), zero padding; the
    gradient scatter is its exact inverse in fp32."""
    import _lib
    Hp = pad64(H)
    Dp = pad64(din // blocks) * blocks
    w, (wih, wihT, whh, whhT, bias) = prep(H, din, blocks, Dp, 1)
    perm = gate_perm(H, Hp).to(_dev())
    real = din // blocks
    j = torch.arange(Dp, device=_dev())
    jb, jk = j // (Dp // blocks), j % (Dp // blocks)
    icol = torch.where(jk < real, jb * real + jk, torch.full_like(j, -1))
    for d in range(2):
        w_ih, w_hh, b_ih, b_hh = w[4 * d: 4 * d + 4]
        want = torch.zeros(4 * Hp, Dp, device=_dev())
        ok = (perm[:, None] >= 0) & (icol[None, :] >= 0)
        want[ok] = w_ih[perm.clamp(min=0)][:, icol.clamp(min=0)][ok]
        assert torch.equal(wih[d * 4 * Hp:(d + 1) * 4 * Hp], want.bfloat16())
        assert torch.equal(wihT[:, d * 4 * Hp:(d + 1) * 4 * Hp], want.bfloat16().t())
        want = torch.zeros(4 * Hp, Hp, device=_dev())
        want[perm >= 0, :H] = w_hh[perm[perm >= 0]]
        assert torch.equal(whh[d], want.bfloat16()) and torch.equal(whhT[d], want.bfloat16().t())
        bw = torch.zeros(4 * Hp, device=_dev())
        bw[perm >= 0] = (b_ih + b_hh)[perm[perm >= 0]]
        assert torch.equal(bias[d], bw)
    # scatter(fp32 padded grads built from the reference layout) == the reference layout, bit for bit
    dwih = torch.zeros(8 * Hp, Dp, device=_dev())
    dwhh = torch.zeros(2, 4 * Hp, Hp, device=_dev())
    db = torch.zeros(8 * Hp, device=_dev())
    for d in range(2):
        w_ih, w_hh, b_ih, _ = w[4 * d: 4 * d + 4]
        ok = (perm[:, None] >= 0) & (icol[None, :] >= 0)
        blk = torch.zeros(4 * Hp, Dp, device=_dev())
        blk[ok] = w_ih[perm.clamp(min=0)][:, icol.clamp(min=0)][ok]
        dwih[d * 4 * Hp:(d + 1) * 4 * Hp] = blk
        dwhh[d][perm >= 0, :H] = w_hh[perm[perm >= 0]]
        db[d * 4 * Hp:(d + 1) * 4 * Hp][perm >= 0] = b_ih[perm[perm >= 0]]
    g = [torch.full_like(t, float("nan")) for t in w]
    _lib.call("dirb200_lstm_scatter_grads", _lib.ptr(dwih), _lib.ptr(dwhh), _lib.ptr(db), H, din, blocks, Hp, Dp,
              *[_lib.ptr(t) for t in g], None)
    for d in range(2):
        assert torch.equal(g[4 * d], w[4 * d]) and torch.equal(g[4 * d + 1], w[4 * d + 1])
        assert torch.equal(g[4 * d + 2], w[4 * d + 2]) and torch.equal(g[4 * d + 3], w[4 * d + 2])


def _act(a):
    i, f, g, o = a.chunk(4, -1)
    return torch.sigmoid(i), torch.sigmoid(f), torch.tanh(g), torch.sigmoid(o)


def _check_fwd_step(xproj, whh, bias, lens, h, c, gates, y, s, H):
    """Step s's outputs (h / c slot s + 1, gates, y at the step's time) against float64 from the state the
    step read (h / c slot s), within the bounds of the module docstring."""
    M, Hp = h.shape[2], h.shape[3]
    rows = torch.arange(M, device=_dev())
    active = s < lens.long()
    for d in range(2):
        tau = torch.where(active, torch.full_like(rows, s) if d == 0 else lens.long() - 1 - s, torch.full_like(rows, s))
        W = whh[d].double()
        hp = h[d, s].double()
        x = xproj[tau, rows, d].double()
        b = bias[d].double()
        a = hp @ W.t() + x + b
        ea = (Hp + 4) * U * ((hp.abs() @ W.abs().t()) + x.abs() + b.abs())
        # to the interleaved gate blocks
        a4 = a.view(M, Hp // 16, 4, 16)
        e4 = ea.view(M, Hp // 16, 4, 16)
        i, f, gg, o = [torch.sigmoid(a4[:, :, 0]), torch.sigmoid(a4[:, :, 1]), torch.tanh(a4[:, :, 2]),
                       torch.sigmoid(a4[:, :, 3])]
        cp = c[d, s].double().view(M, Hp // 16, 16)
        cn = f * cp + i * gg
        hn = o * torch.tanh(cn)
        eg = e4 + 2.0 ** -20
        ec = eg[:, :, 1] * cp.abs() + eg[:, :, 0] + eg[:, :, 2] + 2.0 ** -19 * (1 + cp.abs())
        eh = eg[:, :, 3] + ec + 2.0 ** -19 + 2.0 ** -8 * hn.abs()
        cg = c[d, s + 1].double().view(M, Hp // 16, 16)
        hg = h[d, s + 1].double().view(M, Hp // 16, 16)
        act = active[:, None, None]
        assert torch.all(~act | ((cg - cn).abs() <= ec)), (d, (cg - cn).abs().max().item())
        assert torch.all(~act | ((hg - hn).abs() <= eh)), (d, (hg - hn).abs().max().item())
        ga = gates[d, s].double().view(M, Hp // 16, 4, 16)
        want = torch.stack([i, f, gg, o], 2)
        assert torch.all(~act[..., None] | ((ga - want).abs() <= eg)), d
        # inert rows: zero state; padded units exactly 0; y written once at tau
        assert torch.all(act | (cg == 0)) and torch.all(act | (hg == 0))
        assert torch.all(c[d, s + 1, :, H:] == 0) and torch.all(h[d, s + 1, :, H:] == 0)
        yv = y[tau, rows, d * Hp:(d + 1) * Hp]
        assert torch.equal(yv, h[d, s + 1])


@pytest.mark.parametrize("H,M,s", [(1500, 256, 3), (20, 1, 0), (20, 3, 2), (100, 130, 4), (100, 130, 0)])
def test_fwd_step_one_launch(H, M, s):
    import _lib
    T = 6
    Hp = pad64(H)
    _, (_, _, whh, _, bias) = prep(H, 64, 1, 64, 2)
    perm = gate_perm(H, Hp).to(_dev())
    lens = lens_for(M, T, 3).to(_dev())
    g = torch.Generator(device=_dev()).manual_seed(4)
    xproj = (torch.randn(T, M, 2, 4 * Hp, device=_dev(), generator=g)).bfloat16()
    xproj[..., perm < 0] = 0
    h = torch.full((2, T + 1, M, Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
    c = torch.full((2, T + 1, M, Hp), float("nan"), device=_dev())
    h[:, s] = 0
    c[:, s] = 0
    if s > 0:
        h[:, s, :, :H] = (torch.rand(2, M, H, device=_dev(), generator=g) * 2 - 1).bfloat16()
        c[:, s, :, :H] = torch.randn(2, M, H, device=_dev(), generator=g)
    gates = torch.full((2, T, M, 4 * Hp), float("nan"), device=_dev())
    y = torch.full((T, M, 2 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
    _lib.call("dirb200_lstm_fwd_step", _lib.ptr(xproj), _lib.ptr(whh), _lib.ptr(bias), _lib.ptr(lens), T, M, Hp, 1, s,
              _lib.ptr(h), _lib.ptr(c), _lib.ptr(gates), _lib.ptr(y), None)
    torch.cuda.synchronize()
    _check_fwd_step(xproj, whh, bias, lens, h, c, gates, y, s, H)
    rows = torch.arange(M, device=_dev())
    active = s < lens.long()
    written = torch.zeros(T, M, dtype=torch.bool, device=_dev())
    written[torch.full((M,), s, device=_dev()), rows] = True
    tau_r = torch.where(active, lens.long() - 1 - s, torch.full_like(rows, s))
    written_r = torch.zeros(T, M, dtype=torch.bool, device=_dev())
    written_r[tau_r, rows] = True
    assert torch.all(torch.isnan(y[..., :Hp].float()).all(-1) == ~written)
    assert torch.all(torch.isnan(y[..., Hp:].float()).all(-1) == ~written_r)


def test_layer_fwd_teacher_forced_full_size():
    """dirb200_lstm_layer_fwd at T = 40, M = 256, H = 1500 (one launch per step): every step's state, gates and output
    against float64 from the state the native step read (teacher forcing), ragged lengths, both directions."""
    import _lib
    T, M, H = 40, 256, 1500
    Hp = pad64(H)
    _, (_, _, whh, _, bias) = prep(H, 64, 1, 64, 13)
    perm = gate_perm(H, Hp).to(_dev())
    lens = lens_for(M, T, 14).to(_dev())
    g = torch.Generator(device=_dev()).manual_seed(15)
    xproj = torch.randn(T, M, 2, 4 * Hp, device=_dev(), generator=g).bfloat16()
    xproj[..., perm < 0] = 0
    h = torch.full((2, T + 1, M, Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
    c = torch.full((2, T + 1, M, Hp), float("nan"), device=_dev())
    gates = torch.full((2, T, M, 4 * Hp), float("nan"), device=_dev())
    y = torch.full((T, M, 2 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
    _lib.call("dirb200_lstm_layer_fwd", _lib.ptr(xproj), _lib.ptr(whh), _lib.ptr(bias), _lib.ptr(lens), T, M, Hp, 1,
              _lib.ptr(h), _lib.ptr(c), _lib.ptr(gates), _lib.ptr(y), None)
    torch.cuda.synchronize()
    assert torch.all(h[:, 0] == 0) and torch.all(c[:, 0] == 0)
    for s in range(T):
        _check_fwd_step(xproj, whh, bias, lens, h, c, gates, y, s, H)
    assert not torch.isnan(y.float()).any()
    mask = torch.arange(T, device=_dev())[:, None] < lens.long()[None, :]
    assert torch.all(y[~mask] == 0)


@pytest.mark.parametrize("H,M,s", [(1500, 256, 2), (20, 1, 5), (20, 3, 2), (100, 130, 0), (100, 130, 5)])
def test_bwd_step_one_launch(H, M, s):
    import _lib
    T = 6
    Hp = pad64(H)
    _, (_, _, _, whhT, _) = prep(H, 64, 1, 64, 5)
    perm = gate_perm(H, Hp).to(_dev())
    lens = lens_for(M, T, 6).to(_dev())
    g = torch.Generator(device=_dev()).manual_seed(7)
    gates = torch.rand(2, T, M, 4 * Hp, device=_dev(), generator=g)
    gates.view(2, T, M, Hp // 16, 4, 16)[..., 2, :] = gates.view(2, T, M, Hp // 16, 4, 16)[..., 2, :] * 2 - 1
    c = torch.randn(2, T + 1, M, Hp, device=_dev(), generator=g)
    dy = (torch.randn(T, M, 2 * Hp, device=_dev(), generator=g)).bfloat16()
    # padded units hold what the forward leaves there: gates (1/2, 1/2, 0, 1/2), c = 0, and a zero output gradient
    gp = gates.view(2, T, M, Hp // 16, 4, 16)[:, :, :, H // 16:]
    pu = (torch.arange(Hp // 16 * 16, device=_dev()).view(Hp // 16, 16)[H // 16:] >= H)
    for k, val in enumerate((0.5, 0.5, 0.0, 0.5)):
        gk = gp[..., k, :]
        gk[..., pu] = val
    c[..., H:] = 0
    dy.view(T, M, 2, Hp)[..., H:] = 0
    dg = torch.full((2, T, M, 4 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
    dgt = torch.full((T, M, 8 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
    dc = torch.full((2, 2, M, Hp), float("nan"), device=_dev())
    act_next = (s + 1 < lens.long())
    if s + 1 < T:
        dg[:, s + 1] = (torch.randn(2, M, 4 * Hp, device=_dev(), generator=g) * 0.1).bfloat16()
        dg[:, s + 1][:, ~act_next] = 0
        dg[:, s + 1][..., perm < 0] = 0
        dc[:, (s + 1) & 1] = torch.randn(2, M, Hp, device=_dev(), generator=g)
        dc[:, (s + 1) & 1][:, ~act_next] = 0
        dc[..., H:] = 0
    dc_in = dc[:, (s + 1) & 1].clone()
    _lib.call("dirb200_lstm_bwd_step", _lib.ptr(whhT), _lib.ptr(dy), _lib.ptr(gates), _lib.ptr(c), _lib.ptr(lens), T,
              M, Hp, s, _lib.ptr(dc), _lib.ptr(dg), _lib.ptr(dgt), None)
    torch.cuda.synchronize()
    _check_bwd_step(whhT, dy, gates, c, lens, dg, dgt, dc_in if s + 1 < T else None, dc[:, s & 1], s, H)


def _check_bwd_step(whhT, dy, gates, c, lens, dg, dgt, dc_in, dc_out, s, H):
    """Step s's outputs (dg[:, s], its time-order copy in dgt, the carried dc) against float64 from what the step read
    (dg[:, s + 1] and dc_in, the dc slot (s + 1) & 1 before the step; None at s = T - 1), within the bounds of the
    module docstring.  Inert rows and padded units get exact zeros."""
    T, M, Hp = dg.shape[1], dg.shape[2], whhT.shape[1]
    perm = gate_perm(H, Hp).to(_dev())
    rows = torch.arange(M, device=_dev())
    active = s < lens.long()
    for d in range(2):
        tau = torch.where(active, torch.full_like(rows, s) if d == 0 else lens.long() - 1 - s, torch.full_like(rows, s))
        if s + 1 < T:
            A = dg[d, s + 1].double()
            W = whhT[d].double()
            dh = A @ W.t()
            edh = (4 * Hp + 4) * U * (A.abs() @ W.abs().t())
            dcn = dc_in[d].double()
        else:
            dh = torch.zeros(M, Hp, dtype=torch.float64, device=_dev())
            edh = torch.zeros_like(dh)
            dcn = torch.zeros_like(dh)
        dh = dh + dy[tau, rows, d * Hp:(d + 1) * Hp].double()
        ga = gates[d, s].double().view(M, Hp // 16, 4, 16)
        i, f, gg, o = ga[:, :, 0], ga[:, :, 1], ga[:, :, 2], ga[:, :, 3]
        sh = (M, Hp // 16, 16)
        dh, edh, dcn = dh.view(sh), edh.view(sh), dcn.view(sh)
        cp, cn = c[d, s].double().view(sh), c[d, s + 1].double().view(sh)
        tc = torch.tanh(cn)
        dct = dcn + dh * o * (1 - tc * tc)
        want = torch.stack([dct * gg * i * (1 - i), dct * cp * f * (1 - f), dct * i * (1 - gg * gg),
                            dh * tc * o * (1 - o)], 2)
        e = (edh + 2.0 ** -18 * (dh.abs() + dcn.abs() + 1))[:, :, None, :] * (1 + cp.abs()[:, :, None, :])
        e = e + 2.0 ** -8 * want.abs()
        got = dg[d, s].double().view(M, Hp // 16, 4, 16)
        act = active[:, None, None, None]
        assert torch.all(~act | ((got - want).abs() <= e)), (d, (got - want).abs().max().item())
        assert torch.all(act | (got == 0))
        assert torch.all(got.view(M, 4 * Hp)[:, perm < 0] == 0)
        gt = dgt[tau, rows, d * 4 * Hp:(d + 1) * 4 * Hp]
        assert torch.equal(gt, dg[d, s])
        dcp = dc_out[d].double().view(sh)
        edc = (edh + 2.0 ** -19 * (dh.abs() + dcn.abs() + 1)) * (1 + cp.abs())
        assert torch.all(~active[:, None, None] | ((dcp - dct * f).abs() <= edc)), (d, s)
        assert torch.all(active[:, None, None] | (dcp == 0))
        assert torch.all(dc_out[d, :, H:] == 0)


def _same_bits(a, b):
    """Bit-for-bit equality, NaN fill included."""
    it = {2: torch.int16, 4: torch.int32}[a.element_size()]
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(a.view(it), b.view(it))


def _layer_fwd(T, M, H, seed):
    """dirb200_lstm_layer_fwd (save = 1) on random xproj (zero at padded gate columns) and weights at torch's init
    scale 1 / sqrt(H), so the gates and cells are those of a working layer rather than saturated ones.  Every output
    buffer is prefilled with NaN (gates stay NaN at inert rows).  Returns (whh, whhT, bias), lens and
    (xproj, h, c, gates, y)."""
    import _lib
    Hp = pad64(H)
    _, (_, _, whh, whhT, bias) = prep(H, 64, 1, 64, seed, scale=H ** -0.5)
    perm = gate_perm(H, Hp).to(_dev())
    lens = lens_for(M, T, seed + 1).to(_dev())
    g = torch.Generator(device=_dev()).manual_seed(seed + 2)
    xproj = torch.randn(T, M, 2, 4 * Hp, device=_dev(), generator=g).bfloat16()
    xproj[..., perm < 0] = 0
    nan = float("nan")
    h = torch.full((2, T + 1, M, Hp), nan, dtype=torch.bfloat16, device=_dev())
    c = torch.full((2, T + 1, M, Hp), nan, device=_dev())
    gates = torch.full((2, T, M, 4 * Hp), nan, device=_dev())
    y = torch.full((T, M, 2 * Hp), nan, dtype=torch.bfloat16, device=_dev())
    _lib.call("dirb200_lstm_layer_fwd", _lib.ptr(xproj), _lib.ptr(whh), _lib.ptr(bias), _lib.ptr(lens), T, M, Hp, 1,
              _lib.ptr(h), _lib.ptr(c), _lib.ptr(gates), _lib.ptr(y), None)
    return (whh, whhT, bias), lens, (xproj, h, c, gates, y)


def _layer_bwd_teacher_forced(T, M, H, seed):
    """dirb200_lstm_layer_bwd (s = T-1 .. 0 in one call) on gates and c from a native forward and a random bf16 dy
    (zero at padded units and at t >= len):
    - its dg, dg_time and final two-slot dc equal those of dirb200_lstm_bwd_step run for s = T-1 .. 0 on fresh NaN
      buffers, bit for bit (the step order, the range of s, the dc carry);
    - every step is within _check_bwd_step's bound, given the dg[s + 1] and dc slot it read;
    - dg and dg_time are written everywhere, dg_time exactly zero at t >= len and at padded gate columns."""
    import _lib
    Hp = pad64(H)
    (_, whhT, _), lens, (_, h, c, gates, _) = _layer_fwd(T, M, H, seed)
    perm = gate_perm(H, Hp).to(_dev())
    mask = torch.arange(T, device=_dev())[:, None] < lens.long()[None, :]        # [T, M]: t < len
    g = torch.Generator(device=_dev()).manual_seed(seed + 3)
    dy = torch.randn(T, M, 2, Hp, device=_dev(), generator=g).bfloat16()
    dy[..., H:] = 0
    dy[~mask] = 0
    dy = dy.view(T, M, 2 * Hp)

    def bufs():
        nan = float("nan")
        return (torch.full((2, 2, M, Hp), nan, device=_dev()),
                torch.full((2, T, M, 4 * Hp), nan, dtype=torch.bfloat16, device=_dev()),
                torch.full((T, M, 8 * Hp), nan, dtype=torch.bfloat16, device=_dev()))

    common = (_lib.ptr(whhT), _lib.ptr(dy), _lib.ptr(gates), _lib.ptr(c), _lib.ptr(lens), T, M, Hp)
    dc, dg, dgt = bufs()
    _lib.call("dirb200_lstm_layer_bwd", *common, _lib.ptr(dc), _lib.ptr(dg), _lib.ptr(dgt), None)
    dc1, dg1, dgt1 = bufs()
    dcs = {}
    for s in reversed(range(T)):
        _lib.call("dirb200_lstm_bwd_step", *common, s, _lib.ptr(dc1), _lib.ptr(dg1), _lib.ptr(dgt1), None)
        dcs[s] = dc1.clone()
    torch.cuda.synchronize()
    assert _same_bits(dg, dg1) and _same_bits(dgt, dgt1) and _same_bits(dc, dc1)
    for s in range(T):
        _check_bwd_step(whhT, dy, gates, c, lens, dg1, dgt1, dcs[s + 1][:, (s + 1) & 1] if s + 1 < T else None,
                        dcs[s][:, s & 1], s, H)
    assert not torch.isnan(dg.float()).any() and not torch.isnan(dgt.float()).any()
    d4 = dgt.view(T, M, 2, 4 * Hp)
    assert torch.all(d4[~mask] == 0) and torch.all(d4[..., perm < 0] == 0)


def test_layer_bwd_teacher_forced_full_size():
    _layer_bwd_teacher_forced(40, 256, 1500, 16)


@pytest.mark.parametrize("T,M,H", [(1, 10, 20), (6, 1, 20), (7, 130, 100), (5, 33, 64)],
                         ids=["T1", "M1", "M130-H100", "H64"])
def test_layer_bwd_teacher_forced_small(T, M, H):
    """T = 1 (no recurrent product, one dc slot never written), a single row, two row tiles with a ragged second, and
    H = 64 (no padded unit)."""
    _layer_bwd_teacher_forced(T, M, H, 17)


@pytest.mark.parametrize("T,M,H", [(40, 256, 1500), (39, 256, 1500), (7, 10, 20), (8, 10, 20)],
                         ids=["full-even", "full-odd", "small-odd", "small-even"])
def test_layer_fwd_inference_equals_saved(T, M, H):
    """save = 0 (two ping-pong h / c slots, no gates) gives the save = 1 output bit for bit; its slots end holding the
    saved run's slots T and T - 1, each at its own parity; a gates buffer passed in is not touched."""
    import _lib
    (whh, _, bias), lens, (xproj, h, c, gates, y) = _layer_fwd(T, M, H, 18)
    Hp = pad64(H)
    nan = float("nan")
    h2 = torch.full((2, 2, M, Hp), nan, dtype=torch.bfloat16, device=_dev())
    c2 = torch.full((2, 2, M, Hp), nan, device=_dev())
    gates2 = torch.full_like(gates, nan)
    y2 = torch.full_like(y, nan)
    _lib.call("dirb200_lstm_layer_fwd", _lib.ptr(xproj), _lib.ptr(whh), _lib.ptr(bias), _lib.ptr(lens), T, M, Hp, 0,
              _lib.ptr(h2), _lib.ptr(c2), _lib.ptr(gates2), _lib.ptr(y2), None)
    torch.cuda.synchronize()
    assert not torch.isnan(y.float()).any()
    assert _same_bits(y2, y)
    for p in range(2):
        slot = T if T % 2 == p else T - 1
        assert _same_bits(h2[:, p], h[:, slot]) and _same_bits(c2[:, p], c[:, slot]), p
    assert torch.isnan(gates2).all()


def test_col_sum_deterministic_and_exact_order():
    import _lib
    g = torch.Generator(device=_dev()).manual_seed(8)
    x = torch.randn(1000, 320, device=_dev(), generator=g).bfloat16()
    out = torch.empty(320, device=_dev())
    _lib.call("dirb200_col_sum_bf16", _lib.ptr(x), 1000, 320, _lib.ptr(out), None)
    # the documented order: 8 phases of rows r = p (mod 8) summed in order, then the phases in order
    want = torch.zeros(8, 320, device=_dev())
    for r in range(1000):
        want[r % 8] += x[r].float()
    w = want[0].clone()
    for p in range(1, 8):
        w += want[p]
    assert torch.equal(out, w)


def test_pair_maxpool_exact_ties_and_scatter():
    import _lib
    B, T, H = 5, 7, 20
    Hp = 64
    M = 2 * B
    lens = lens_for(M, T, 9).to(_dev())
    g = torch.Generator(device=_dev()).manual_seed(10)
    y = torch.randn(T, M, 2 * Hp, device=_dev(), generator=g).bfloat16()
    y[2:4, :, 3] = 1.5                      # ties in column 3 (t = 2 and 3), within every row with len > 3
    mask = torch.arange(T, device=_dev())[:, None] < lens.long()[None, :]
    y = y * mask[..., None]
    cols = torch.cat([torch.arange(H), Hp + torch.arange(H)]).to(_dev())
    for dmul in (None, (torch.rand(M, T, 2 * H, device=_dev(), generator=g) > 0.2).float() / 0.8):
        feat = torch.empty(B, 8 * H, device=_dev())
        arg = torch.empty(M, 2 * H, dtype=torch.int32, device=_dev())
        _lib.call("dirb200_pair_maxpool_fwd", _lib.ptr(y), _lib.ptr(lens), _lib.ptr(dmul), B, T, H, Hp,
                  _lib.ptr(feat), _lib.ptr(arg), None)
        v = y[:, :, cols].float().permute(1, 0, 2)          # [M, T, 2H]
        if dmul is not None:
            v = v * dmul
        v = v.masked_fill(~mask.t()[..., None], float("-inf"))
        mx = v.max(1).values
        first = (v == mx[:, None, :]).int().argmax(1)      # first maximal t
        assert torch.equal(arg.long(), first)
        u, w = mx[:B], mx[B:]
        assert torch.equal(feat, torch.cat([u, w, (u - w).abs(), u * w], 1))
        gf = torch.randn(B, 8 * H, device=_dev(), generator=g)
        gf[:, 4 * H:6 * H][0] = 1.0
        dy = torch.full((T, M, 2 * Hp), float("nan"), dtype=torch.bfloat16, device=_dev())
        _lib.call("dirb200_pair_maxpool_bwd", _lib.ptr(gf), _lib.ptr(feat), _lib.ptr(arg), _lib.ptr(dmul), B, T, H, Hp,
                  _lib.ptr(dy), None)
        G = 2 * H
        sg = torch.sign(u - w)
        du = gf[:, :G] + sg * gf[:, 2 * G:3 * G] + w * gf[:, 3 * G:]
        dv = gf[:, G:2 * G] - sg * gf[:, 2 * G:3 * G] + u * gf[:, 3 * G:]
        d = torch.cat([du, dv])
        if dmul is not None:
            d = d * torch.gather(dmul, 1, first[:, None, :]).squeeze(1)
        want = torch.zeros(T, M, 2 * Hp, device=_dev())
        r = torch.arange(M, device=_dev())[:, None].expand(M, G)
        want[first, r, cols[None, :].expand(M, G)] = d
        assert torch.equal(dy, want.bfloat16())


def test_embed_gather_exact_and_grad_deterministic():
    import _lib
    V, D, Dp, T, M = 37, 24, 64, 6, 10
    lens = lens_for(M, T, 11).to(_dev())
    g = torch.Generator(device=_dev()).manual_seed(12)
    ids = torch.randint(1, V, (M, T), device=_dev(), generator=g)
    emb = torch.randn(V, D, device=_dev(), generator=g)
    dmul = (torch.rand(M, T, D, device=_dev(), generator=g) > 0.2).float() / 0.8
    x = torch.full((T, M, Dp), float("nan"), dtype=torch.bfloat16, device=_dev())
    _lib.call("dirb200_embed_gather", _lib.ptr(ids), _lib.ptr(lens), _lib.ptr(emb), _lib.ptr(dmul), V, M, T, D, Dp,
              _lib.ptr(x), None)
    mask = (torch.arange(T, device=_dev())[None, :] < lens.long()[:, None])
    want = torch.zeros(T, M, Dp, device=_dev())
    want[..., :D] = (emb[ids] * dmul * mask[..., None]).permute(1, 0, 2)
    assert torch.equal(x, want.bfloat16())
    dx = torch.randn(T, M, Dp, device=_dev(), generator=g).bfloat16()
    outs = []
    for _ in range(2):
        dw = torch.full((V, D), float("nan"), device=_dev())
        _lib.call("dirb200_embed_grad", _lib.ptr(ids), _lib.ptr(lens), _lib.ptr(dx), _lib.ptr(dmul), V, M, T, D, Dp,
                  -1, _lib.ptr(dw), None)
        outs.append(dw)
    # a padding row gets no gradient (F.embedding's padding_idx); the other rows are unchanged
    pad = int(ids[0, 0])
    dwp = torch.full((V, D), float("nan"), device=_dev())
    _lib.call("dirb200_embed_grad", _lib.ptr(ids), _lib.ptr(lens), _lib.ptr(dx), _lib.ptr(dmul), V, M, T, D, Dp, pad,
              _lib.ptr(dwp), None)
    keep = torch.arange(V, device=_dev()) != pad
    assert torch.all(dwp[pad] == 0) and torch.equal(dwp[keep], outs[0][keep])
    assert torch.equal(outs[0], outs[1])
    contrib = (dx[..., :D].double().permute(1, 0, 2) * dmul.double() * mask[..., None])
    ref = torch.zeros(V, D, dtype=torch.float64, device=_dev()).index_add_(0, ids.reshape(-1),
                                                                           contrib.reshape(-1, D))
    n = torch.zeros(V, device=_dev()).index_add_(0, ids.reshape(-1), mask.reshape(-1).float())
    bound = (n[:, None].double() + 1) * U * torch.zeros(V, D, dtype=torch.float64, device=_dev()).index_add_(
        0, ids.reshape(-1), contrib.abs().reshape(-1, D))
    assert torch.all((outs[0].double() - ref).abs() <= bound + 1e-30)


# ---------------------------------------------------------------- the model
class _Vocab:
    def __init__(self, V):
        self.V = V
        self._padding_token = '@@PADDING@@'

    def get_vocab_size(self, ns):
        return self.V

    def get_token_index(self, tok):
        return 0


class _Task:
    name = 'sts-b'

    def __init__(self):
        self.calls = 0

    def scorer(self, logits, labels):
        self.calls += 1


def _args(**kw):
    a = dict(d_word=24, n_layers_highway=0, glove=1, train_words=0, d_hid=20, n_layers_enc=2, dropout=0.2, fds=0,
             bucket_num=50, bucket_start=0, start_update=0, start_smooth=1, fds_kernel='gaussian', fds_ks=5,
             fds_sigma=2, fds_mmt=0.9, cuda=0, loss='mse', huber_beta=0.5)
    a.update(kw)
    return SimpleNamespace(**a)


def _build(seed=0, V=37, **kw):
    from models import build_model
    torch.manual_seed(seed)
    args = _args(**kw)
    embs = torch.randn(V, args.d_word) * 0.5
    return build_model(args, _Vocab(V), embs, [_Task()]), args


def _batch(B=5, T1=7, T2=9, V=37, seed=1):
    g = torch.Generator().manual_seed(seed)
    l1 = torch.randint(1, T1 + 1, (B,), generator=g)
    l2 = torch.randint(1, T2 + 1, (B,), generator=g)
    l1[0], l1[1], l2[0], l2[2] = T1, 1, T2, 1
    s1 = torch.randint(1, V, (B, T1), generator=g) * (torch.arange(T1)[None] < l1[:, None])
    s2 = torch.randint(1, V, (B, T2), generator=g) * (torch.arange(T2)[None] < l2[:, None])
    label = torch.rand(B, 1, generator=g) * 5
    return s1.to(_dev()), s2.to(_dev()), label.to(_dev())


def _oracle_params(model, dtype, bf16=False):
    enc = model.pair_encoder
    rnd = (lambda t: t.detach().bfloat16().to(dtype)) if bf16 else (lambda t: t.detach().to(dtype))
    p = {"emb": rnd(enc._text_field_embedder.token_embedder_words.weight).cpu(),
         "lstm": {k: rnd(v).cpu() for k, v in enc._phrase_layer._module.named_parameters()}}
    if bf16:       # the bias enters the kernels as the fp32 sum b_ih + b_hh
        for k in list(p["lstm"]):
            if k.startswith("bias"):
                p["lstm"][k] = getattr(enc._phrase_layer._module, k).detach().to(dtype).cpu()
    return p


def _oracle_feature(p, s1, s2, drops=None, arg=None):
    from oracle import stsb_ref
    B, T1 = s1.shape
    T2 = s2.shape[1]
    T = max(T1, T2)
    ids = torch.cat([torch.nn.functional.pad(s1, (0, T - T1)), torch.nn.functional.pad(s2, (0, T - T2))]).cpu()
    lens = torch.cat([(s1 != 0).sum(1), (s2 != 0).sum(1)]).cpu()
    de = do = None
    if drops is not None:
        pad = lambda m, t: torch.nn.functional.pad(m, (0, 0, 0, T - t))
        m1e, m2e, m1o, m2o = [m.cpu().to(p["emb"].dtype) for m in drops]
        de = torch.cat([pad(m1e, T1), pad(m2e, T2)])
        do = torch.cat([pad(m1o, T1), pad(m2o, T2)])
    return stsb_ref.forward(p, ids, lens, B, de, do, arg=arg)


@pytest.mark.parametrize("train,train_words", [(False, 1), (True, 1), (True, 0)],
                         ids=["eval", "train", "train-frozen-emb"])
def test_model_feature_and_grads_vs_float64(train, train_words):
    """Feature within 8x the bf16-operand sensitivity of the float64 oracle; every LSTM gradient (and the trainable
    embedding's) within 5e-2 relative Frobenius error.  Frozen embeddings: no embedding gradient."""
    model, _ = _build(train_words=train_words)
    model.train(train)
    s1, s2, label = _batch()
    feat = model.pair_encoder({'words': s1}, {'words': s2})
    drops = model.pair_encoder.last_dropout if train else None
    p64 = _oracle_params(model, torch.float64)
    for v in [p64["emb"], *p64["lstm"].values()]:
        v.requires_grad_(True)
    ref = _oracle_feature(p64, s1, s2, drops)
    refb = _oracle_feature(_oracle_params(model, torch.float64, bf16=True), s1, s2, drops)
    err = (feat.double().cpu() - ref.detach()).abs().max().item()
    sens = (refb - ref).abs().max().item()
    assert err <= 8 * sens + 1e-6, (err, sens)
    # gradients: the float64 max taken at the native argmax (bf16 near-ties may pick another t than float64 would)
    arg = feat.grad_fn.saved_tensors[1].cpu()
    ref = _oracle_feature(p64, s1, s2, drops, arg=arg)
    gf = torch.randn(feat.shape, generator=torch.Generator().manual_seed(3), dtype=torch.float64)
    feat.backward(gf.float().to(_dev()))
    (ref * gf).sum().backward()
    lstm = model.pair_encoder._phrase_layer._module
    for k, v in p64["lstm"].items():
        got = getattr(lstm, k).grad.double().cpu()
        rel = (got - v.grad).norm() / v.grad.norm()
        assert rel <= 5e-2, (k, rel.item())
    w = model.pair_encoder._text_field_embedder.token_embedder_words.weight
    if not train_words:
        assert w.grad is None
        return
    ge = w.grad.double().cpu()
    assert (ge - p64["emb"].grad).norm() / p64["emb"].grad.norm() <= 5e-2
    assert torch.all(ge[0] == 0)            # the padding row


def test_fixture_parity_loose():
    """The native model loaded with the reference model's state_dict (tests/golden/stsb_model.npz: the reference's own
    models.py / fds.py / loss.py, FDS smoothing active at epoch 1, dropout 0): feature, smoothed embs, logits, every
    loss kind and every gradient, loosely (bf16 operands and activations: 3e-2 of the largest value for the feature
    and logits, 5e-2 relative Frobenius error for the gradients)."""
    import numpy as np
    z = np.load(os.path.join(ROOT, "tests", "golden", "stsb_model.npz"))
    s1, s2 = torch.from_numpy(z["s1"]).to(_dev()), torch.from_numpy(z["s2"]).to(_dev())
    label, weight = torch.from_numpy(z["label"]).to(_dev()), torch.from_numpy(z["weight"]).to(_dev())
    near = lambda got, want, tol=3e-2: np.abs(got - want).max() <= tol * np.abs(want).max()
    for kind in ("mse", "l1", "focal_mse", "focal_l1", "huber"):
        model, _ = _build(fds=1, train_words=1, dropout=0.0, loss=kind)
        model.load_state_dict({k: torch.from_numpy(np.asarray(z["p:" + k])) for k in model.state_dict()}, strict=True)
        model.train()
        seen = {}
        model.pair_encoder.register_forward_hook(lambda m, i, o: seen.__setitem__("f", o.detach().clone()))
        out = model(_Task(), 1, {'words': s1}, {'words': s2}, label=label, weight=weight)
        assert abs(out['loss'].item() - float(z[f"loss_{kind}"])) <= 3e-2 * abs(float(z[f"loss_{kind}"])), kind
        if kind != "mse":
            continue
        assert near(seen["f"].cpu().numpy(), z["feature"])
        assert near(out['embs'].detach().cpu().numpy(), z["embs"])
        assert near(out['logits'].detach().cpu().numpy(), z["logits"])
        out['loss'].backward()
        for n, p in model.named_parameters():
            want = z["g:" + n]
            got = p.grad.cpu().numpy()
            assert np.linalg.norm(got - want) <= 5e-2 * np.linalg.norm(want), n


def test_model_forward_loss_fds_and_adam_step():
    """MultiTaskModel.forward: out keys, loss = weighted mse of logits vs label / 5, FDS smoothing path, embs feeding
    FDSSTSB.update_running_stats, one optim.Adam step changes every trainable parameter."""
    import optim
    model, _ = _build(fds=1)
    model.train()
    s1, s2, label = _batch()
    task = _Task()
    out = model(task, 1, {'words': s1}, {'words': s2}, label=label, weight=torch.ones_like(label))
    assert set(out) == {'embs', 'labels', 'logits', 'loss'} and task.calls == 1
    lin = getattr(model, 'sts-b_pred_layer')
    want = ((out['logits'] - label / 5) ** 2).mean()
    assert abs(out['loss'].item() - want.item()) <= 1e-5 * abs(want.item()) + 1e-7
    model.FDS.update_last_epoch_stats(1)
    model.FDS.update_running_stats(out['embs'].detach(), label.view(-1), 1)
    out = model(task, 2, {'words': s1}, {'words': s2}, label=label, weight=None)
    opt = optim.Adam([p for p in model.parameters() if p.requires_grad], lr=1e-3)
    before = {n: p.detach().clone() for n, p in model.named_parameters() if p.requires_grad}
    opt.zero_grad()
    out['loss'].backward()
    opt.step()
    for n, p in model.named_parameters():
        if p.requires_grad:
            assert torch.isfinite(p).all() and not torch.equal(p.detach(), before[n]), n
    assert lin.weight.grad is not None


def test_retrain_fc_launches_no_lstm_backward():
    import _lib
    model, _ = _build()
    for n, p in model.named_parameters():
        p.requires_grad_(n.startswith('sts-b_pred_layer'))
    model.train()
    s1, s2, label = _batch()
    out = model(_Task(), 0, {'words': s1}, {'words': s2}, label=label)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    out['loss'].backward()
    torch.cuda.synchronize()
    assert _lib.launch_count() - n0 <= 2        # the regressor's backward only
    assert all(p.grad is None for n, p in model.named_parameters() if not n.startswith('sts-b_pred_layer'))


def test_determinism_and_row_independence():
    model, _ = _build(train_words=1, dropout=0.0)
    model.train()
    s1, s2, label = _batch(B=6)
    outs = []
    for _ in range(2):
        model.zero_grad()
        f = model.pair_encoder(s1, s2)
        f.sum().backward()
        outs.append((f.detach().clone(), [p.grad.clone() for p in model.pair_encoder.parameters()]))
    assert torch.equal(outs[0][0], outs[1][0])
    assert all(torch.equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))
    # row 2 alone (trimmed to its own lengths) gives the same feature bits
    l1, l2 = int((s1[2] != 0).sum()), int((s2[2] != 0).sum())
    f1 = model.pair_encoder(s1[2:3, :l1], s2[2:3, :l2])
    assert torch.equal(f1[0], outs[0][0][2])


def test_matches_cudnn_packed_lstm():
    """The native BiLSTM against torch's packed cuDNN LSTM in fp32 on the same fp32 parameters (eval, one sentence
    batch): within the bf16 bound above measured against the float64 oracle, plus the fp32 path's own error."""
    model, _ = _build(dropout=0.0)
    model.eval()
    s1, s2, _ = _batch()
    feat = model.pair_encoder(s1, s2)
    lstm = model.pair_encoder._phrase_layer._module
    ref = torch.nn.LSTM(24, 20, 2, bidirectional=True, batch_first=True).to(_dev())
    ref.load_state_dict(lstm.state_dict())
    emb = model.pair_encoder._text_field_embedder.token_embedder_words.weight
    encs = []
    for s in (s1, s2):
        L = (s != 0).sum(1)
        pk = torch.nn.utils.rnn.pack_padded_sequence(emb[s], L.cpu(), batch_first=True, enforce_sorted=False)
        with torch.no_grad():
            o, _ = ref(pk)
        o, _ = torch.nn.utils.rnn.pad_packed_sequence(o, batch_first=True, total_length=s.shape[1])
        o = o.masked_fill(~(torch.arange(s.shape[1], device=_dev())[None] < L[:, None])[..., None], float("-inf"))
        encs.append(o.max(1).values)
    u, v = encs
    want = torch.cat([u, v, (u - v).abs(), u * v], 1)
    p64 = _oracle_params(model, torch.float64)
    sens = (_oracle_feature(_oracle_params(model, torch.float64, bf16=True), s1, s2) -
            _oracle_feature(p64, s1, s2)).abs().max().item()
    assert (feat - want).abs().max().item() <= 8 * sens + 1e-5


def test_state_dict_keys_and_refusals():
    model, _ = _build(fds=1)
    keys = set(model.state_dict())
    lstm_keys = {f"pair_encoder._phrase_layer._module.{n}_l{k}{s}" for k in range(2) for s in ("", "_reverse")
                 for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")}
    assert lstm_keys <= keys
    assert "pair_encoder._text_field_embedder.token_embedder_words.weight" in keys
    assert {"sts-b_pred_layer.weight", "sts-b_pred_layer.bias"} <= keys
    s1, s2, label = _batch()
    bad = s1.clone()
    bad[3] = 0
    with pytest.raises(ValueError, match="zero-length"):
        model.pair_encoder(bad, s2)


@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_stsb_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process)."""
    if os.environ.get("DIRB200_STSB_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_STSB_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
