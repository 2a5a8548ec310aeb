"""The ResNet runner's batched kernels against float64, one launch at a time and in place on the runner.

Each runs over a descriptor table, and only the runner (csrc/resnet_runner.cu) launches it:
  prep_weights_all_kernel    every conv weight -> bf16 fprop [co][tap][c] and dgrad [c][tap][co] operands (FastDiv
                             index arithmetic); the stem -> its 256-wide space-to-depth operand.  Bit-exact: round to
                             nearest even, formed on the integer bits.
  wgrad_reduce_all_kernel    grads[w_off ..] += the sum of each conv's split-K partials, [co][(r, s, c)] -> [co][c][r][s]
                             (stem: the space-to-depth taps, the padding channel dropped).  A sum of splits + 1 terms in
                             any order: |got - (G0 + S)| <= (splits + 1) u (|G0| + sum |p|), S the float64 sum.
  bn_eval_coeffs_all_kernel  scale = gamma rsqrt(var + eps), shift = beta - mean scale: rsqrtf is within 2 ulp, so the
                             scale is within 2^-21 relative and |shift - ref| <= u |shift| + 2^-20 |mean scale|.
u = 2^-24.  Standalone, through the "Test aids: the runner's batched kernels" of include/dirb200.h: jobs at unaligned
offsets with NaN guards around every output, at ResNet-50's conv forms and at divisors and filter shapes it does not
have.  In place, through dirb200_resnet_peek_conv: every conv operand after a training forward, every stage's writes
into a caller-owned gradient buffer, every conv's weight gradient against its own partials, every BatchNorm's eval
coefficients.  The whole file runs a second time with DIRB200_SMS=7 (other split factors, many grid-stride passes)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF = torch.bfloat16
F64 = torch.float64
NAN_BF16 = 0x7FC0


class PrepJob(ctypes.Structure):
    _fields_ = [("w_off", ctypes.c_int64), ("cout", ctypes.c_int), ("cin", ctypes.c_int), ("kh", ctypes.c_int),
                ("kw", ctypes.c_int), ("stem", ctypes.c_int), ("w_fprop", ctypes.c_void_p), ("w_dgrad", ctypes.c_void_p)]


class ReduceJob(ctypes.Structure):
    _fields_ = [("partial", ctypes.c_void_p), ("w_off", ctypes.c_int64), ("splits", ctypes.c_int), ("cout", ctypes.c_int),
                ("cin", ctypes.c_int), ("kh", ctypes.c_int), ("kw", ctypes.c_int), ("stem", ctypes.c_int)]


class BnJob(ctypes.Structure):
    _fields_ = [("c", ctypes.c_int), ("gamma_off", ctypes.c_int64), ("beta_off", ctypes.c_int64),
                ("rm_off", ctypes.c_int64), ("rv_off", ctypes.c_int64), ("scale", ctypes.c_void_p),
                ("shift", ctypes.c_void_p)]


class ConvPeek(ctypes.Structure):
    _fields_ = [("w_fprop", ctypes.c_void_p), ("w_dgrad", ctypes.c_void_p), ("partial", ctypes.c_void_p),
                ("scale", ctypes.c_void_p), ("shift", ctypes.c_void_p), ("w_off", ctypes.c_int64)] + \
               [(k, ctypes.c_int) for k in ("cout", "cin", "kh", "kw", "stride", "pad", "stem", "splits")]


def lib():
    import _lib
    import _convlib, resnet  # noqa: F401  (register the conv-stack / runner bindings)
    return _lib


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def dev_view(ptr, n, typestr):
    """A torch view of n elements of device memory at ptr ('<f4' fp32, '<i2' bf16 bits)."""
    class _A:
        __cuda_array_interface__ = dict(shape=(n,), typestr=typestr, data=(ptr, False), version=2)
    return torch.as_tensor(_A(), device=DEV)


def bf16_bits(w):
    """fp32 -> bf16 bits by round to nearest even, written out on the integer bits (no NaN inputs): add 0x7FFF plus the
    kept part's lowest bit, keep the high half.  Subnormals round like any other value, overflow goes to infinity."""
    b = w.detach().contiguous().view(torch.int32).to(torch.int64) & 0xFFFFFFFF
    r = (b + 0x7FFF + ((b >> 16) & 1)) >> 16
    return torch.where(r >= 32768, r - 65536, r).to(torch.int16)


# the stem's space-to-depth operand (csrc/conv_api.cu): k = (r', s', ph, pw, c4) -> tap r = 2 r' + ph - 1,
# s = 2 s' + pw - 1 of the 3x7x7 filter, or no tap (c4 = 3, r or s outside 0 .. 6)
def stem_maps():
    k = np.arange(256)
    rp, sp, ph, pw, c = k >> 6, (k >> 4) & 3, (k >> 3) & 1, (k >> 2) & 1, k & 3
    r, s = 2 * rp + ph - 1, 2 * sp + pw - 1
    valid = (c < 3) & (r >= 0) & (s >= 0) & (r < 7) & (s < 7)
    src = np.where(valid, (c * 7 + r) * 7 + s, -1)             # operand column k <- weight index (c, r, s)
    inv = np.full(147, -1)
    inv[src[valid]] = k[valid]                                 # weight index -> its one operand column
    assert (inv >= 0).all()
    return src, inv


STEM_SRC, STEM_INV = stem_maps()


def stem_operand_ref(w):
    """w fp32 [cout][3][7][7] -> bf16 bits [cout][256] (zero where no tap exists), from the mapping above."""
    w = w.detach().reshape(w.shape[0], 147)
    src = torch.from_numpy(STEM_SRC).to(w.device)
    op = torch.where(src >= 0, w[:, src.clamp(min=0)], torch.zeros((), device=w.device))
    return bf16_bits(op)


def tricky_f32(n, g):
    """fp32 values over a wide exponent range with every bf16 rounding case: exact ties (low half 0x8000), one below and
    one above, plus signed zeros, infinities, subnormals and FLT_MAX."""
    x = torch.randn(n, generator=g, device=DEV) * torch.exp2(torch.randint(-40, 40, (n,), generator=g, device=DEV).float())
    b = x.view(torch.int32)
    sel = torch.randint(0, 8, (n,), generator=g, device=DEV)
    hi = b & -65536
    b = torch.where(sel == 0, hi | 0x8000, torch.where(sel == 1, hi | 0x7FFF, torch.where(sel == 2, hi | 0x8001, b)))
    x = b.view(torch.float32).clone()
    special = torch.tensor([0.0, -0.0, float("inf"), -float("inf"), 1e-40, -3e-39, 3.4028235e38, -3.39e38],
                           device=DEV)
    idx = torch.randint(0, n, (min(n, 64),), generator=g, device=DEV)
    x[idx] = special[torch.arange(idx.numel(), device=DEV) % special.numel()]
    return x


# ------------------------------------------------------------------------------------------------ prep_weights_all
# (cout, cin, kh, kw, stem)
PREP_FORMS = [
    (64, 3, 7, 7, 1),                                                          # stem
    (64, 64, 1, 1, 0), (256, 64, 1, 1, 0), (64, 256, 1, 1, 0), (128, 256, 1, 1, 0), (512, 128, 1, 1, 0),
    (128, 512, 1, 1, 0), (256, 512, 1, 1, 0), (1024, 256, 1, 1, 0), (256, 1024, 1, 1, 0), (512, 1024, 1, 1, 0),
    (2048, 512, 1, 1, 0), (512, 2048, 1, 1, 0), (1024, 512, 1, 1, 0), (2048, 1024, 1, 1, 0),   # 1x1 and downsample
    (64, 64, 3, 3, 0), (128, 128, 3, 3, 0), (256, 256, 3, 3, 0), (512, 512, 3, 3, 0),           # 3x3 (strided too)
    (192, 320, 1, 1, 0), (320, 576, 3, 3, 0), (576, 192, 1, 1, 0),            # divisors ResNet-50 does not have
    (64, 192, 5, 5, 0), (192, 64, 7, 7, 0), (128, 64, 3, 5, 0), (96, 3, 7, 7, 0),   # 5x5, non-stem 7x7, 3x5 taps
    (7, 5, 3, 3, 0), (1, 1, 1, 1, 0), (1, 2048, 1, 1, 0), (2048, 1, 1, 1, 0), (64, 3, 7, 7, 1),
]


def test_prep_weights_all_is_bit_exact_and_writes_only_its_jobs():
    L = lib()
    g = gen(1)
    rng = np.random.RandomState(1)
    jobs, metas = [], []
    p_off = f_off = d_off = 0
    for i, (co, ci, kh, kw, stem) in enumerate(PREP_FORMS):
        p_off += int(rng.randint(1, 40))                         # unaligned, with a gap before every job
        f_off += int(rng.randint(1, 40))
        n = co * ci * kh * kw
        nf = co * 256 if stem else n
        dg = not stem and i % 3 != 2                             # every third non-stem job has no dgrad operand
        if dg:
            d_off += int(rng.randint(1, 40))
        metas.append((co, ci, kh, kw, stem, p_off, f_off, d_off if dg else None))
        p_off += n
        f_off += nf
        if dg:
            d_off += n
    params = tricky_f32(p_off + 17, g)
    wf = torch.full((f_off + 33,), NAN_BF16, dtype=torch.int16, device=DEV)
    wd = torch.full((d_off + 33,), NAN_BF16, dtype=torch.int16, device=DEV)
    for co, ci, kh, kw, stem, po, fo, do in metas:
        jobs.append(PrepJob(po, co, ci, kh, kw, stem, wf.data_ptr() + 2 * fo,
                            None if do is None else wd.data_ptr() + 2 * do))
    arr = (PrepJob * len(jobs))(*jobs)
    L.call("dirb200_prep_weights_all", L.ptr(params), arr, len(jobs), L.stream_ptr())
    torch.cuda.synchronize()
    f_seen = torch.zeros(wf.numel(), dtype=torch.bool, device=DEV)
    d_seen = torch.zeros(wd.numel(), dtype=torch.bool, device=DEV)
    for co, ci, kh, kw, stem, po, fo, do in metas:
        w = params[po:po + co * ci * kh * kw].view(co, ci, kh, kw)
        if stem:
            ref = stem_operand_ref(w).reshape(-1)
            got = wf[fo:fo + ref.numel()]
            assert torch.equal(got, ref), ("stem", co, (got != ref).sum().item())
            # the single-conv API forms the same operand
            one = torch.empty(co * 256, dtype=torch.int16, device=DEV)
            L.call("dirb200_conv_prep_weights", L.ptr(w.contiguous()), co, 3, 7, 7, 1, L.ptr(one), None,
                   L.stream_ptr())
            assert torch.equal(one, ref)
            f_seen[fo:fo + ref.numel()] = True
            continue
        ref = bf16_bits(w.permute(0, 2, 3, 1).contiguous()).reshape(-1)
        got = wf[fo:fo + ref.numel()]
        assert torch.equal(got, ref), ((co, ci, kh, kw), (got != ref).sum().item())
        f_seen[fo:fo + ref.numel()] = True
        if do is not None:
            ref = bf16_bits(w.permute(1, 2, 3, 0).contiguous()).reshape(-1)
            got = wd[do:do + ref.numel()]
            assert torch.equal(got, ref), ("dgrad", (co, ci, kh, kw), (got != ref).sum().item())
            d_seen[do:do + ref.numel()] = True
    # nothing outside the jobs was written (the guards keep their NaN bits)
    assert (wf[~f_seen] == NAN_BF16).all()
    assert (wd[~d_seen] == NAN_BF16).all()


# ------------------------------------------------------------------------------------------------ wgrad_reduce_all
# (splits, cout, cin, kh, kw, stem): every tail length of the 4-chain loop, totals that are not a multiple of 256 and
# ones larger than the grid (2 x SMs x 256 per pass)
REDUCE_JOBS = [
    (1, 64, 64, 1, 1, 0), (2, 7, 5, 3, 3, 0), (3, 64, 64, 3, 3, 0), (4, 256, 64, 1, 1, 0), (5, 128, 128, 3, 3, 0),
    (6, 3, 1, 1, 1, 0), (7, 320, 192, 3, 3, 0), (8, 100, 3, 3, 5, 0), (9, 512, 512, 3, 3, 0), (13, 1000, 1, 1, 1, 0),
    (33, 2048, 512, 1, 1, 0), (3, 64, 3, 7, 7, 1), (13, 64, 3, 7, 7, 1), (33, 8, 3, 7, 7, 1),
]


def rand_partials(splits, n, g):
    """Mixed signs and magnitudes over 2^-12 .. 2^12, and exact cancellations between the first two splits."""
    p = torch.randn(splits, n, generator=g, device=DEV) * torch.exp2(
        torch.randint(-12, 13, (splits, n), generator=g, device=DEV).float())
    if splits >= 2:
        cancel = torch.rand(n, generator=g, device=DEV) < 0.3
        p[1] = torch.where(cancel, -p[0], p[1])
    return p.contiguous()


def reduce_ref(partial, splits, co, ci, kh, kw, stem):
    """float64 (S, sum |p|) in the weight layout [co][c][r][s]."""
    p = partial.view(splits, co, -1).to(F64)
    s, a = p.sum(0), p.abs().sum(0)
    if stem:
        inv = torch.from_numpy(STEM_INV).to(DEV)
        return s[:, inv].reshape(-1), a[:, inv].reshape(-1)
    perm = lambda t: t.view(co, kh, kw, ci).permute(0, 3, 1, 2).reshape(-1)
    return perm(s), perm(a)


def check_reduced(got, g0, s, a, splits, what):
    got, g0 = got.to(F64), g0.to(F64)
    err = (got - (g0 + s)).abs()
    bound = (splits + 1) * U * (g0.abs() + a)
    bad = ~(err <= bound)
    assert not bad.any(), (what, bad.sum().item(), (err - bound).max().item())


def test_wgrad_reduce_all_against_float64():
    L = lib()
    g = gen(2)
    rng = np.random.RandomState(2)
    metas, parts = [], []
    off = 0
    for splits, co, ci, kh, kw, stem in REDUCE_JOBS:
        off += int(rng.randint(1, 62))
        n = co * ci * kh * kw
        metas.append((splits, co, ci, kh, kw, stem, off))
        parts.append(rand_partials(splits, co * (256 if stem else ci * kh * kw), g))
        off += n
    total = off + 29
    inside = torch.zeros(total, dtype=torch.bool, device=DEV)
    for splits, co, ci, kh, kw, stem, o in metas:
        inside[o:o + co * ci * kh * kw] = True
    g0 = torch.randn(total, generator=g, device=DEV) * torch.exp2(
        torch.randint(-8, 9, (total,), generator=g, device=DEV).float())
    g0[~inside] = float("nan")
    jobs = (ReduceJob * len(metas))(*[ReduceJob(p.data_ptr(), o, sp, co, ci, kh, kw, st)
                                      for p, (sp, co, ci, kh, kw, st, o) in zip(parts, metas)])
    outs = []
    for _ in range(2):
        grads = g0.clone()
        L.call("dirb200_wgrad_reduce_all", jobs, len(metas), L.ptr(grads), L.stream_ptr())
        outs.append(grads)
    torch.cuda.synchronize()
    # two identical calls, identical bits
    assert torch.equal(outs[0].view(torch.int32), outs[1].view(torch.int32))
    grads = outs[0]
    assert grads[~inside].isnan().all(), "a job wrote outside its weights"
    for p, (splits, co, ci, kh, kw, stem, o) in zip(parts, metas):
        n = co * ci * kh * kw
        s, a = reduce_ref(p, splits, co, ci, kh, kw, stem)
        check_reduced(grads[o:o + n], g0[o:o + n], s, a, splits, (splits, co, ci, kh, kw, stem))


# (n, h, w, cin, cout, k, stride, pad, stem)
WGRAD_CONVS = [(2, 16, 16, 64, 128, 3, 1, 1, 0), (4, 14, 14, 256, 64, 1, 2, 0, 0), (2, 32, 32, 3, 64, 7, 2, 3, 1),
               (8, 28, 28, 128, 128, 3, 1, 1, 0)]


@pytest.mark.parametrize("shape", WGRAD_CONVS, ids=lambda s: "x".join(map(str, s)))
def test_wgrad_reduce_all_matches_the_single_conv_reduce(shape):
    """dirb200_conv_wgrad (GEMM partials, then its own per-layer reduce, accumulating) and the batched reduce over the
    partials it left in its workspace: both within the float64 bound, and within that bound of each other."""
    L = lib()
    n, h, w, ci, co, k, st, pd, stem = shape
    g = gen(3)
    if stem:
        x = torch.randn(n, h // 2, w // 2, 16, generator=g, device=DEV).to(BF)   # nonzero padding channel: dropped
        ho, wo, K = h // 2, w // 2, 256
    else:
        x = torch.randn(n, h, w, ci, generator=g, device=DEV).to(BF)
        ho, wo, K = (h + 2 * pd - k) // st + 1, (w + 2 * pd - k) // st + 1, k * k * ci
    dy = torch.randn(n, ho, wo, co, generator=g, device=DEV).to(BF)
    nbytes = L.raw("dirb200_conv_wgrad_workspace_bytes")(n, h, w, ci, co, k, k, st, pd, stem)
    splits = nbytes // (K * co * 4)
    assert splits >= 1 and nbytes == splits * K * co * 4
    ws = torch.zeros(nbytes // 4, device=DEV)
    nw = co * ci * k * k
    g0 = torch.randn(nw, generator=g, device=DEV)
    single = g0.clone()
    L.call("dirb200_conv_wgrad", L.ptr(x), L.ptr(dy), L.ptr(single), L.ptr(ws), nbytes, n, h, w, ci, co, k, k, st, pd,
           stem, 1, L.stream_ptr())
    batched = g0.clone()
    jobs = (ReduceJob * 1)(ReduceJob(ws.data_ptr(), 0, splits, co, ci, k, k, stem))
    L.call("dirb200_wgrad_reduce_all", jobs, 1, L.ptr(batched), L.stream_ptr())
    s, a = reduce_ref(ws, splits, co, ci, k, k, stem)
    check_reduced(single, g0, s, a, splits, "single-conv reduce")
    check_reduced(batched, g0, s, a, splits, "batched reduce")
    bound = (splits + 1) * U * (g0.to(F64).abs() + a)
    assert ((single.to(F64) - batched.to(F64)).abs() <= bound).all()


# ------------------------------------------------------------------------------------------------ bn_eval_coeffs_all
EPS = float(np.float32(1e-5))


def bn_stats_tricky(c, g):
    gamma = torch.randn(c, generator=g, device=DEV) * 2            # negative gammas
    beta = torch.randn(c, generator=g, device=DEV)
    rm = torch.randn(c, generator=g, device=DEV) * torch.exp2(torch.randint(-6, 7, (c,), generator=g, device=DEV).float())
    rv = torch.rand(c, generator=g, device=DEV) * 4
    sel = torch.randint(0, 6, (c,), generator=g, device=DEV)
    rv = torch.where(sel == 0, torch.zeros(()), torch.where(sel == 1, rv * 1e20, rv))     # var = 0 and large var
    rv[0] = 0.0
    return gamma, beta, rm, rv


def check_bn_eval(scale, shift, gamma, beta, rm, rv, what):
    g, b, m, v = (t.to(F64) for t in (gamma, beta, rm, rv))
    sc = g / torch.sqrt(v + EPS)
    sh = b - m * sc
    e_sc = (scale.to(F64) - sc).abs()
    assert (e_sc <= 2.0 ** -21 * sc.abs()).all(), (what, "scale", (e_sc / sc.abs()).max().item())
    e_sh = (shift.to(F64) - sh).abs()
    assert (e_sh <= U * sh.abs() + 2.0 ** -20 * (m * sc).abs()).all(), (what, "shift")


def test_bn_eval_coeffs_all_against_float64():
    L = lib()
    g = gen(4)
    cs = [64, 100, 2048, 256, 100, 64]                   # jobs below max_c, tails that are not a multiple of 256
    per = [bn_stats_tricky(c, g) for c in cs]
    # params: [gamma | gap | beta] per job; running: [mean | gap | var]; outputs: NaN gaps between the jobs
    params, running, jobs, outs = [], [], [], []
    po = ro = 0
    out_len = sum(c + 7 for c in cs) + 7
    scale = torch.full((out_len,), float("nan"), device=DEV)
    shift = torch.full((out_len,), float("nan"), device=DEV)
    oo = 7
    for c, (ga, be, m, v) in zip(cs, per):
        params += [torch.full((3,), float("nan"), device=DEV), ga, torch.full((5,), float("nan"), device=DEV), be]
        running += [torch.full((1,), float("nan"), device=DEV), m, torch.full((2,), float("nan"), device=DEV), v]
        jobs.append(BnJob(c, po + 3, po + 3 + c + 5, ro + 1, ro + 1 + c + 2, scale.data_ptr() + 4 * oo,
                          shift.data_ptr() + 4 * oo))
        outs.append(oo)
        po += 3 + c + 5 + c
        ro += 1 + c + 2 + c
        oo += c + 7
    params, running = torch.cat(params), torch.cat(running)
    arr = (BnJob * len(jobs))(*jobs)
    L.call("dirb200_bn_eval_coeffs_all", arr, len(jobs), L.ptr(params), L.ptr(running), EPS, L.stream_ptr())
    torch.cuda.synchronize()
    seen = torch.zeros(out_len, dtype=torch.bool, device=DEV)
    for c, o, (ga, be, m, v) in zip(cs, outs, per):
        check_bn_eval(scale[o:o + c], shift[o:o + c], ga, be, m, v, c)
        seen[o:o + c] = True
    assert scale[~seen].isnan().all() and shift[~seen].isnan().all()


# ------------------------------------------------------------------------------------------------ in place
def conv_table(layers, H, W):
    """Every conv of the runner in its build order: (block, conv, weight name, BN prefix, cin, cout, k, stride, pad,
    input h, input w, stem)."""
    out = [(-1, 0, "conv1.weight", "bn1.", 3, 64, 7, 2, 3, H, W, 1)]
    h, w = (H // 2 - 1) // 2 + 1, (W // 2 - 1) // 2 + 1
    inpl, bi = 64, 0
    for li, nb in enumerate(layers):
        pl = 64 << li
        for b in range(nb):
            s = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
            out += [(bi, 0, pre + "conv1.weight", pre + "bn1.", inpl, pl, 1, 1, 0, h, w, 0),
                    (bi, 1, pre + "conv2.weight", pre + "bn2.", pl, pl, 3, s, 1, h, w, 0),
                    (bi, 2, pre + "conv3.weight", pre + "bn3.", pl, pl * 4, 1, 1, 0, ho, wo, 0)]
            if b == 0 and (s != 1 or inpl != pl * 4):
                out.append((bi, 3, pre + "downsample.0.weight", pre + "downsample.1.", inpl, pl * 4, 1, s, 0, h, w, 0))
            inpl, h, w, bi = pl * 4, ho, wo, bi + 1
    return out


def make_model(layers):
    from resnet import ResNet, Bottleneck
    torch.manual_seed(0)
    return ResNet(Bottleneck, list(layers)).to(DEV).train()


def peek_conv(L, net, block, conv):
    out = ConvPeek()
    L.call("dirb200_resnet_peek_conv", net, block, conv, ctypes.byref(out))
    return out


def wgrad_splits(L, n, cv):
    _, _, _, _, ci, co, k, s, p, h, w, stem = cv
    plan = (ctypes.c_int * 7)()
    L.call("dirb200_conv_plan", n, h, w, ci, co, k, k, s, p, stem, 2, plan)
    return plan[4]


def check_operands(L, m, net, table):
    flat = m.flat_parameters()
    named = dict(m.named_parameters())
    for cv in table:
        block, conv, name, _, ci, co, k, s, p, _, _, stem = cv
        pk = peek_conv(L, net, block, conv)
        assert (pk.cout, pk.cin, pk.kh, pk.kw, pk.stride, pk.pad, pk.stem) == (co, ci, k, k, s, p, stem), name
        assert pk.w_off == (named[name].data_ptr() - flat.data_ptr()) // 4, name
        w = flat[pk.w_off:pk.w_off + co * ci * k * k].view(co, ci, k, k)
        if stem:
            assert pk.w_dgrad is None
            got = dev_view(pk.w_fprop, co * 256, "<i2")
            assert torch.equal(got, stem_operand_ref(w).reshape(-1)), name
            continue
        got = dev_view(pk.w_fprop, w.numel(), "<i2")
        assert torch.equal(got, bf16_bits(w.permute(0, 2, 3, 1).contiguous()).reshape(-1)), name
        got = dev_view(pk.w_dgrad, w.numel(), "<i2")
        assert torch.equal(got, bf16_bits(w.permute(1, 2, 3, 0).contiguous()).reshape(-1)), name


CASES = [((3, 4, 6, 3), 16, 64, 64, False), ((3, 4, 6, 3), 4, 224, 224, False), ((2, 2, 1, 1), 16, 64, 64, False),
         ((3, 4, 6, 3), 2, 228, 304, True)]


@pytest.mark.parametrize("layers,n,h,w,blocks", CASES, ids=["r50_b16_64", "r50_b4_224", "shallow_b16_64",
                                                              "nyud2_encoder_b2_228x304"])
def test_runner_kernels_in_place(layers, n, h, w, blocks):
    L = lib()
    m = make_model(layers)
    shape = (n, 3, h, w)
    net = m._net(shape)
    table = conv_table(layers, h, w)
    nconv = len(table)
    assert nconv == 1 + sum(3 * nb + 1 for nb in layers)
    flat, running = m.flat_parameters(), m._flat["running"]
    npar = L.raw("dirb200_resnet_param_count")(net)
    nst = L.raw("dirb200_resnet_num_stages")(net)
    g = gen(5)
    x = torch.randn(shape, generator=g, device=DEV)
    ranges = []
    for stage in range(nst + 1):
        lo, hi = ctypes.c_int64(), ctypes.c_int64()
        L.call("dirb200_resnet_stage_param_range", net, stage, ctypes.byref(lo), ctypes.byref(hi))
        ranges.append((lo.value, hi.value))
    assert ranges[0][0] == 0 and ranges[-1][1] == npar
    assert all(ranges[i][1] == ranges[i + 1][0] for i in range(nst))
    # the recorded split factors are the ones the wgrad GEMM uses for that conv
    for cv in table:
        assert peek_conv(L, net, cv[0], cv[1]).splits == wgrad_splits(L, n, cv), cv[2]
    grads = torch.empty(npar, device=DEV)
    for it in range(2):               # eager, then the captured graphs of the forward and of every backward stage
        if blocks:
            outs = m._run_forward_blocks(x, training=True)
        else:
            m._run_forward(x, training=True)
        torch.cuda.synchronize()
        check_operands(L, m, net, table)
        g0 = torch.randn(npar, generator=g, device=DEV) * torch.exp2(
            torch.randint(-6, 7, (npar,), generator=g, device=DEV).float())
        grads.copy_(g0)
        d_enc = torch.randn(n, 2048, generator=g, device=DEV) * 1e-2
        for stage in range(nst, -1, -1):
            before = grads.clone()
            if blocks:
                db = None if stage == 0 else (torch.randn(outs[stage - 1].shape, generator=g, device=DEV) * 1e-3).to(BF)
                L.call("dirb200_resnet_backward_blocks_stage", net, stage, L.ptr(db), L.ptr(flat), L.ptr(grads),
                       L.stream_ptr())
            else:
                L.call("dirb200_resnet_backward_stage", net, stage, L.ptr(d_enc), L.ptr(flat), L.ptr(grads),
                       L.stream_ptr())
            lo, hi = ranges[stage]
            changed = (grads.view(torch.int32) != before.view(torch.int32)).nonzero().flatten()
            assert changed.numel() > 0, stage
            # nothing outside the stage's own slice, so no finished slice, is touched
            assert changed.min().item() >= lo and changed.max().item() < hi, (stage, lo, hi, changed.min().item(),
                                                                              changed.max().item())
        torch.cuda.synchronize()
        for cv in table:
            block, conv, name, _, ci, co, k, _, _, _, _, stem = cv
            pk = peek_conv(L, net, block, conv)
            K = 256 if stem else k * k * ci
            part = dev_view(pk.partial, pk.splits * co * K, "<f4")
            s, a = reduce_ref(part, pk.splits, co, ci, k, k, stem)
            nw = co * ci * k * k
            check_reduced(grads[pk.w_off:pk.w_off + nw], g0[pk.w_off:pk.w_off + nw], s, a, pk.splits, (it, name))
            del part, s, a
    # eval forward: every BatchNorm's folded coefficients from the flat parameters and running statistics
    named, bufs = dict(m.named_parameters()), dict(m.named_buffers())
    with torch.no_grad():
        for cv in table:
            pre = cv[3]
            c = named[pre + "weight"].numel()
            ga, be, rm, rv = bn_stats_tricky(c, g)
            named[pre + "weight"].copy_(ga)
            named[pre + "bias"].copy_(be)
            bufs[pre + "running_mean"].copy_(rm)
            bufs[pre + "running_var"].copy_(rv)
        if blocks:
            m._run_forward_blocks(x, training=False)
        else:
            m._run_forward(x, training=False)
    torch.cuda.synchronize()
    for cv in table:
        pk, pre = peek_conv(L, net, cv[0], cv[1]), cv[3]
        c = cv[5]
        check_bn_eval(dev_view(pk.scale, c, "<f4"), dev_view(pk.shift, c, "<f4"), named[pre + "weight"],
                      named[pre + "bias"], bufs[pre + "running_mean"], bufs[pre + "running_var"], pre)
    assert bufs["bn1.running_var"].data_ptr() == running.data_ptr() + 4 * 64


def test_peek_conv_refuses_bad_indices():
    L = lib()
    m = make_model((2, 2, 1, 1))
    net = m._net((2, 3, 64, 64))
    out = ConvPeek()

    def refused(block, conv, msg):
        rc = L.raw("dirb200_resnet_peek_conv")(net, block, conv, ctypes.byref(out))
        assert rc == -1 and msg in L.last_error(), (block, conv, rc, L.last_error())

    refused(-2, 0, "bad block")
    refused(6, 0, "bad block")
    refused(-1, 1, "bad conv")
    refused(0, 4, "bad conv")
    refused(0, -1, "bad conv")
    refused(1, 3, "no downsample")         # layer1.1 is an identity block
    peek_conv(L, net, 0, 3)                  # layer1.0 has one


def test_whole_file_with_few_sms():
    """This file again with the grids capped at 7 SMs (DIRB200_SMS is read once per process): other split-K factors,
    and the grid-stride loops of the reduce run many passes."""
    if os.environ.get("DIRB200_SMS"):
        pytest.skip("already running under DIRB200_SMS")
    e = dict(os.environ)
    e["DIRB200_SMS"] = "7"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
