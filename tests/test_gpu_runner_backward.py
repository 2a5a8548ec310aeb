"""The ResNet runner's backward pass in place, element by element, against float64.  dirb200_resnet_set_backward_tap
copies the transient gradients of one block (or the stem) right after the launch that produces each of them, and
dirb200_resnet_peek_backward / _peek_bn_coef read them back.  Every check is teacher-forced: it is fed the runner's own
tensors, taken from where the reference network routes them (forward inputs through dirb200_resnet_peek / _peek_conv,
gradients through the taps of the producing launch), never from a pointer the runner reports.  u = 2^-24.

  average-pool backward  the last block's incoming gradient, bit for bit: bf16(fl32(d_enc x fl32(1 / hw))).
  stored dz              identity blocks, bit for bit: bf16(mask fl32(gA + gB [+ g3])) in the kernel's order (dz_ref of
                         test_gpu_layer_kernels.py); gB a compact gradient is placed at the even pixels.
  BN backward            for every BatchNorm (stem, conv1 / 2 / 3, downsample): float64 S0 = sum dz, S1 = sum dz y over
                         the tapped operands, with dz the unrounded fp32 mask (gA + gB) of a downsample block, the
                         stored dz of an identity block, g [fl32(y scale + shift) > 0] after a conv (g: the tapped
                         dgrad output).  |S - S_ref| <= L u sum |term|, L the fp32 chain of the path this run takes:
                         the dgrad epilogue's (chain_length) where dirb200_conv_plan says fuses_bn_moments, else
                         bn_bwd_reduce's (rows per row lane + lanes + 2, with the fewest CTAs its grid can have).  That
                         error is carried into A, B, C (plus one fp32 rounding each) and into dgamma, dbeta, checked as
                         grads - g0 (bn_bwd_coeffs accumulates).
  dy of every conv       bit for bit: bf16(fmaf(A, dz, fmaf(B, y, C))) with the runner's own coefficients, so that apply
                         errors and coefficient errors are told apart; the bound 2^-8 |ref| + 2 u (|A dz| + |B y| + |C|)
                         of test_gpu_layer_kernels.py is reported.
  every dgrad output     the float64 transposed conv of the tapped dy with the conv's own bf16 dgrad operand, per
                         element within 2^-8 |ref| + (1 + 2^-8) KAPPA(k^2 cout) A (test_gpu_conv.py); the compact
                         downsample gradient on its strided grid, the full stride-2 one exactly 0 where no tap reaches.
  every weight gradient  the split-K partials the last backward left against float64 sum x dy (x: the conv's forward
                         input as the reference routes it; the stem: x rounded to bf16 at 7x7 / stride 2 / pad 3), within
                         the wgrad bound of test_gpu_conv.py; grads - g0 against their sum by check_reduced.
  max-pool backward      gA + gB through the stored argmax (maxpool_bwd_ref); pixels no window picks exactly 0.
  chaining               block b's incoming gA / gB are bit-identical to block b+1's nA and its nB (downsample) or dz
                         (identity); the stem's to block 0's.  Valid across backwards: there are no float atomics.
  multi-scale            a gradient on all four outputs, and one on layer2's only: g3 enters only the last block of its
                         group, the topmost gradient enters as gA, stages above it write nothing and leave their grads
                         slice bit-identical to g0.
  graph replay           per case the untapped backward before the tapped ones (eager, then captured) and after them (a
                         replay) give a flat gradient bit-identical to every tapped one: the taps perturb nothing.

Cases: ResNet-50 at 16 x 64^2, 4 x 224^2 and 256 x 224^2 (at 224^2 every stride-2 downsample gradient is compact),
(2, 2, 1, 1) at 16 x 64^2, ResNet-18 at 4 x 64^2 and 256 x 224^2 (its layer1.0 is an identity block: the max-pool
backward's second gradient is that block's stored dz), (1, 1, 1, 1) basic, and the NYUD2 multi-scale encoder at 1 and 8 x
228 x 304 (maps 57 x 76, 29 x 38, 15 x 19: every stride-2 downsample gradient takes the full parity-class form).  At
batch 256 a subset of the blocks is tapped: the stem, layer1.0 (ResNet-50: the stride-1 downsample block; ResNet-18: an
identity block feeding the max pool), the last block of layer1 (identity, receives the compact gradient), layer2.0 (a
stride-2 downsample block) and the last block.  The whole file runs again in subprocesses with DIRB200_SMS=7,
DIRB200_GRAPH=0 and DIRB200_FUSED_BWD_MOMENTS=0 (every BN backward through bn_bwd_reduce)."""
import ctypes
import gc
import os
import time

import pytest
import torch

from test_gpu_conv import BF16_U, KAPPA
from test_gpu_conv_epilogues import chain_length, expected_rows, num_sms
from test_gpu_layer_kernels import dz_ref, lanes, maxpool_bwd_ref
from test_gpu_runner_forward import (BUDGET, SLACK, by_block, conv_input, fma32, forward, lib, peek_u8, randomize_bn,
                                     raw_y, rerun, row_chunks, zbits)
from test_gpu_runner_kernels import check_reduced, conv_table, dev_view, make_model, peek_conv, reduce_ref

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
BF = torch.bfloat16
F64 = torch.float64
NO_TAP = -2


def conv2d_input(*a, **k):
    """float64 transposed conv by torch's own GEMM path: cuDNN may pick its algorithm by the free memory of the moment,
    and not every algorithm keeps the per-element accuracy the bounds below rely on."""
    with torch.backends.cudnn.flags(enabled=False):
        return torch.nn.grad.conv2d_input(*a, **k)


def conv2d_weight(*a, **k):
    with torch.backends.cudnn.flags(enabled=False):
        return torch.nn.grad.conv2d_weight(*a, **k)

# tap selectors (include/dirb200.h, dirb200_resnet_peek_backward)
GA, GB, G3, DZ, DY_TAIL, DY_DS, DG_TAIL, DY_PRE, DG_C2, DY_C1, NA, NB, POOL, DY_STEM = range(14)

WORST = {}


def note(kind, err, bound):
    r = (err / bound.clamp_min(1e-300)).max().item() if err.numel() else 0.0
    WORST[kind] = max(WORST.get(kind, 0.0), r)


def fused_moments():
    return os.environ.get("DIRB200_FUSED_BWD_MOMENTS", "1")[:1] != "0"


def tap(c, which):
    """[rows, channels] bf16 view of a tapped tensor of the last backward, or None when it was not written."""
    ptr, rows, ch = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_int()
    rc = c.L.raw("dirb200_resnet_peek_backward")(c.net, which, ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch))
    if rc != 0:
        assert "not written" in c.L.last_error(), c.L.last_error()
        return None
    return dev_view(ptr.value, rows.value * ch.value, "<i2").view(BF).view(rows.value, ch.value)


def same_bits(a, b):
    return a is not None and b is not None and a.shape == b.shape and torch.equal(a.view(torch.int16), b.view(torch.int16))


def out_hw(cv):
    _, _, _, _, _, _, k, s, p, h, w, _ = cv
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


def nchw(t, b, h, w):
    """float64 NCHW images b of the NHWC rows t."""
    return t[b.start * h * w:b.stop * h * w].view(-1, h, w, t.shape[1]).permute(0, 3, 1, 2).double()


def img_chunks(n, per_image):
    step = max(1, BUDGET // per_image)
    for b0 in range(0, n, step):
        yield slice(b0, min(n, b0 + step))


def offset(c, t):
    return (t.data_ptr() - c.flat.data_ptr()) // 4


# ------------------------------------------------------------------------------------------------ BatchNorm backward
def reduce_chain(rows, ch):
    """fp32 chain of one bn_bwd_reduce column sum: rows per row lane with the fewest CTAs the grid can have (one per SM
    or one per 16 rows per lane), plus the in-CTA combine."""
    ln = lanes(ch)
    nb = max(1, min(-(-rows // (ln * 16)), num_sms()))
    return -(-rows // (nb * ln)) + ln + 2


def dgrad_chain(c, cv, rows):
    """Chain of the moments the dgrad of cv accumulates for the BN before it, or None when that dgrad does not fuse them."""
    _, _, _, _, ci, co, k, s, p, h, w, _ = cv
    a = (ctypes.c_int * 7)()
    c.L.call("dirb200_conv_plan", c.n, h, w, ci, co, k, k, s, p, 0, 1, a)
    if not (fused_moments() and a[6]):
        return None
    m_tiles = -(-rows // 128)
    n_tiles = ci // a[0]
    return chain_length((expected_rows(m_tiles, n_tiles), n_tiles, a[0], 1), m_tiles)


def check_bn(c, cv, S0, S1, A0, A1, Lc, rows, tag):
    """A, B, C and the accumulated dgamma / dbeta of cv's BatchNorm from float64 moments carrying L u sum |term|.
    Returns the runner's coefficients [3][c] (fp32)."""
    block, conv, name, pre = cv[:4]
    co = cv[5]
    mp, ip, cp = ctypes.c_void_p(), ctypes.c_void_p(), ctypes.c_void_p()
    c.L.call("dirb200_resnet_peek_bn_stats", c.net, block, conv, ctypes.byref(mp), ctypes.byref(ip))
    c.L.call("dirb200_resnet_peek_bn_coef", c.net, block, conv, ctypes.byref(cp))
    mu, is_ = dev_view(mp.value, co, "<f4").double(), dev_view(ip.value, co, "<f4").double()
    coef = dev_view(cp.value, 3 * co, "<f4").view(3, co)
    gw, gb = c.named[pre + "weight"], c.named[pre + "bias"]
    ga = gw.double()
    n = float(rows)
    d0, d1 = Lc * U * A0, Lc * U * A1
    dg = is_ * (S1 - mu * S0)
    ddg = is_ * (d1 + mu.abs() * d0)
    ref = [ga * is_, -ga * is_ * is_ * dg / n, ga * is_ * (mu * is_ * dg / n - S0 / n)]
    bnd = [U * ref[0].abs(),
           ga.abs() * is_ * is_ * ddg / n + U * ref[1].abs(),
           ga.abs() * is_ * (mu.abs() * is_ * ddg / n + d0 / n) + U * ref[2].abs()]
    for i, kind in enumerate(("bn coef A", "bn coef B", "bn coef C")):
        e, b = (coef[i].double() - ref[i]).abs(), SLACK * bnd[i] + 1e-30
        note(kind, e, b)
        assert (e <= b).all(), f"{tag} {name}: {kind} worst excess {(e - b).max().item():.3e} (L = {Lc})"
    for kind, p, d, dd in (("dgamma", gw, dg, ddg), ("dbeta", gb, S0, d0)):
        o = offset(c, p)
        g0 = c.g0[o:o + co].double()
        r = g0 + d
        e, b = (c.grads[o:o + co].double() - r).abs(), SLACK * (dd + U * d.abs() + U * r.abs()) + 1e-30
        note(kind, e, b)
        assert (e <= b).all(), f"{tag} {name}: {kind} (grads - g0) worst excess {(e - b).max().item():.3e}"
    return coef


def check_dy(dy, dz_of, y, coef, tag):
    """dy = bf16(fmaf(A, dz, fmaf(B, y, C))) bit for bit (dz_of(q): the fp32 dz the apply forms for rows q)."""
    assert dy is not None and dy.shape == y.shape, tag
    A, B, C = coef[0], coef[1], coef[2]
    for q in row_chunks(y.shape[0], y.shape[1]):
        dz = dz_of(q)
        ref = fma32(dz, A, fma32(y[q], B, C)).to(BF)
        bad = zbits(dy[q]) != zbits(ref)
        assert not bad.any(), f"{tag}: {int(bad.sum())} of {bad.numel()} elements differ from the fp32 apply"
        ad, by = A.double() * dz.double(), B.double() * y[q].double()
        r64 = ad + by + C.double()
        note("dy", (dy[q].double() - r64).abs(), 2.0 ** -8 * r64.abs() + 2 * U * (ad.abs() + by.abs() + C.double().abs()))


def conv_bn(c, cv, g, dy, dgrad_cv, tag):
    """The BN backward of a conv followed by BN + ReLU: g the tapped gradient of its activation, dy the tapped output."""
    y = raw_y(c.L, c.net, cv)
    pk = peek_conv(c.L, c.net, cv[0], cv[1])
    sc, sh = dev_view(pk.scale, cv[5], "<f4"), dev_view(pk.shift, cv[5], "<f4")
    assert g is not None and g.shape == y.shape, (tag, cv[2])
    rows, ch = y.shape
    z = torch.zeros((), device=DEV)
    dz_of = lambda q: torch.where(fma32(y[q], sc, sh) > 0, g[q].float(), z)
    S0, S1, A0, A1 = (torch.zeros(ch, dtype=F64, device=DEV) for _ in range(4))
    for q in row_chunks(rows, ch):
        dz = dz_of(q).double()
        t = dz * y[q].double()
        S0 += dz.sum(0); A0 += dz.abs().sum(0); S1 += t.sum(0); A1 += t.abs().sum(0)
    Lc = dgrad_chain(c, dgrad_cv, rows) if dgrad_cv is not None else None
    if Lc is None:
        Lc = reduce_chain(rows, ch)
    coef = check_bn(c, cv, S0, S1, A0, A1, Lc, rows, tag)
    check_dy(dy, dz_of, y, coef, f"{tag} {cv[2]} dy")


# ------------------------------------------------------------------------------------------------ convolutions
def dgrad_weight(c, cv):
    """The conv's own bf16 dgrad operand [cin][k][k][cout] as a float64 [cout][cin][k][k] filter."""
    _, _, _, _, ci, co, k, _, _, _, _, _ = cv
    pk = peek_conv(c.L, c.net, cv[0], cv[1])
    return dev_view(pk.w_dgrad, ci * k * k * co, "<i2").view(BF).view(ci, k, k, co).permute(3, 0, 1, 2).double()


def check_dgrad(c, cv, dy, got, tag):
    _, _, name, _, ci, co, k, s, p, h, w, _ = cv
    ho, wo = out_hw(cv)
    hh, ww, ss = h, w, s
    assert got is not None and dy is not None, (tag, name)
    if s == 2 and got.shape[0] == c.n * ho * wo:
        # the compact gradient of a stride-2 1x1 downsample: a plain 1x1 dgrad over the strided grid
        assert k == 1 and p == 0 and h % 2 == 0 and w % 2 == 0, (tag, name)
        hh, ww, ss = ho, wo, 1
        c.forms.add("compact")
    elif s == 2 and k == 1:
        c.forms.add("full stride-2 1x1")
    assert got.shape == (c.n * hh * ww, ci) and dy.shape == (c.n * ho * wo, co), (tag, name, got.shape, dy.shape)
    wt = dgrad_weight(c, cv)
    for b in img_chunks(c.n, max(ci * hh * ww, co * ho * wo) * 2):
        d = nchw(dy, b, ho, wo)
        shape = (b.stop - b.start, ci, hh, ww)
        ref = conv2d_input(shape, wt, d, stride=ss, padding=p)
        A = conv2d_input(shape, wt.abs(), d.abs(), stride=ss, padding=p)
        g = nchw(got, b, hh, ww)
        err = (g - ref).abs()
        bound = BF16_U * ref.abs() + (1 + BF16_U) * KAPPA(k * k * co) * A
        note("dgrad", err, bound)
        bad = ~(err <= bound)
        assert not bad.any(), f"{tag} {name} dgrad: {int(bad.sum())} of {bad.numel()} elements over the bound"
        assert (g[A == 0] == 0).all(), f"{tag} {name} dgrad: a pixel no tap reaches is not 0"
        del ref, A, g, d


def check_wgrad(c, cv, dy, tag):
    """The conv's split-K partials against float64 sum x dy, and grads - g0 against their sum."""
    block, conv, name, _, ci, co, k, s, p, h, w, stem = cv
    ho, wo = out_hw(cv)
    assert dy is not None and dy.shape == (c.n * ho * wo, co), (tag, name)
    pk = peek_conv(c.L, c.net, block, conv)
    src = conv_input(c.L, c.net, c.x, cv)
    ref = torch.zeros(co, ci, k, k, dtype=F64, device=DEV)
    A = torch.zeros_like(ref)
    for b in img_chunks(c.n, max(ci * k * k * ho * wo, ci * h * w, co * ho * wo)):
        xin, d = src(b), nchw(dy, b, ho, wo)
        ref += conv2d_weight(xin, ref.shape, d, stride=s, padding=p)
        A += conv2d_weight(xin.abs(), ref.shape, d.abs(), stride=s, padding=p)
        del xin, d
    K = 256 if stem else k * k * ci
    part = dev_view(pk.partial, pk.splits * co * K, "<f4")
    S, Sa = reduce_ref(part, pk.splits, co, ci, k, k, stem)
    per_split = -(-(-(-(c.n * ho * wo) // 64)) // pk.splits) * 64
    kw = KAPPA(per_split) + pk.splits * U
    err, bound = (S - ref.reshape(-1)).abs(), kw * A.reshape(-1)
    note("wgrad", err, bound)
    bad = ~(err <= bound)
    assert not bad.any(), f"{tag} {name} wgrad: {int(bad.sum())} of {bad.numel()} weights over the bound"
    nw = co * ci * k * k
    check_reduced(c.grads[pk.w_off:pk.w_off + nw], c.g0[pk.w_off:pk.w_off + nw], S, Sa, pk.splits, (tag, name))


# ------------------------------------------------------------------------------------------------ one block
def check_block(c, bi, tag):
    convs = c.blk[bi]
    tail, pre = (1, 0) if c.basic else (2, 1)
    T, M, C1, D = convs[tail], convs[pre], convs[0], convs.get(3)
    oh, ow = out_hw(T)
    rows, ch = c.n * oh * ow, T[5]
    gA, gB, g3 = tap(c, GA), tap(c, GB), tap(c, G3)
    assert gA is not None and gA.shape == (rows, ch), tag
    g2m = None
    t = dict(g1=gA, mask=peek_u8(c.L, c.net, bi), g3=g3)
    if gB is not None:
        if gB.shape[0] == rows:
            g2m, t["g2"] = "dense", gB
        else:
            assert gB.shape == (c.n * (oh // 2) * (ow // 2), ch) and oh % 2 == 0 and ow % 2 == 0, tag
            e = torch.zeros(c.n, oh, ow, ch, dtype=BF, device=DEV)
            e[:, ::2, ::2] = gB.view(c.n, oh // 2, ow // 2, ch)
            g2m, t["g2e"] = "compact", e.view(rows, ch)
            c.forms.add("compact gB")
    if g3 is not None:
        c.forms.add("g3")
    # ---- block output: stored dz (identity) and the tail / downsample BatchNorms
    yT = raw_y(c.L, c.net, T)
    yD = raw_y(c.L, c.net, D) if D else None
    dzs = tap(c, DZ)
    assert (dzs is None) == (D is not None), tag
    z = torch.zeros(ch, dtype=F64, device=DEV)
    S0, A0, S1, A1, S2, A2 = (z.clone() for _ in range(6))
    for q in row_chunks(rows, ch):
        dz = dz_ref(t, q, "bits", g2m, g3 is not None, ch)
        if dzs is not None:
            ref = dz.to(BF)
            bad = dzs[q].view(torch.int16) != ref.view(torch.int16)
            assert not bad.any(), f"{tag}: {int(bad.sum())} stored dz differ"
            dz = dzs[q].float()
        dz = dz.double()
        t1 = dz * yT[q].double()
        S0 += dz.sum(0); A0 += dz.abs().sum(0); S1 += t1.sum(0); A1 += t1.abs().sum(0)
        if D:
            t2 = dz * yD[q].double()
            S2 += t2.sum(0); A2 += t2.abs().sum(0)
    Lc = reduce_chain(rows, ch)
    coefT = check_bn(c, T, S0, S1, A0, A1, Lc, rows, tag)
    if dzs is not None:
        dz_of = lambda q: dzs[q].float()
    else:
        dz_of = lambda q: dz_ref(t, q, "bits", g2m, False, ch)
    dyT = tap(c, DY_TAIL)
    check_dy(dyT, dz_of, yT, coefT, f"{tag} {T[2]} dy")
    if D:
        coefD = check_bn(c, D, S0, S2, A0, A2, Lc, rows, tag)
        dyD = tap(c, DY_DS)
        check_dy(dyD, dz_of, yD, coefD, f"{tag} {D[2]} dy")
    else:
        assert tap(c, DY_DS) is None and tap(c, NB) is None, tag
    # ---- tail conv, then the pre-tail conv's BN
    check_wgrad(c, T, dyT, tag)
    g_pre = tap(c, DG_TAIL)
    check_dgrad(c, T, dyT, g_pre, tag)
    dy_pre = tap(c, DY_PRE)
    conv_bn(c, M, g_pre, dy_pre, T, tag)
    check_wgrad(c, M, dy_pre, tag)
    if c.basic:
        assert tap(c, DG_C2) is None and tap(c, DY_C1) is None, tag
        dy1 = dy_pre
    else:
        g1 = tap(c, DG_C2)
        check_dgrad(c, M, dy_pre, g1, tag)
        dy1 = tap(c, DY_C1)
        conv_bn(c, C1, g1, dy1, M, tag)
        check_wgrad(c, C1, dy1, tag)
    nA = tap(c, NA)
    check_dgrad(c, C1, dy1, nA, tag)
    nB = None
    if D:
        check_wgrad(c, D, dyD, tag)
        nB = tap(c, NB)
        check_dgrad(c, D, dyD, nB, tag)
    return gA, gB, nA, nB if D else dzs


def check_stem(c, tag):
    cv = c.blk[-1][0]
    ph, pw = (c.h // 2 - 1) // 2 + 1, (c.w // 2 - 1) // 2 + 1
    gA, gB = tap(c, GA), tap(c, GB)
    assert gA is not None and gA.shape == (c.n * ph * pw, 64), tag
    idx = peek_u8(c.L, c.net, -1)
    g = tap(c, POOL)
    assert g is not None and g.shape == (c.n * (c.h // 2) * (c.w // 2), 64), tag
    for b in img_chunks(c.n, 4 * (c.h // 2) * (c.w // 2) * 64):
        r = slice(b.start * ph * pw, b.stop * ph * pw)
        ref, bound, cnt = maxpool_bwd_ref(gA[r].view(-1, ph, pw, 64), None if gB is None else gB[r].view(-1, ph, pw, 64),
                                          idx[r].view(-1, ph, pw, 64), c.h // 2, c.w // 2)
        got = g[b.start * (c.h // 2) * (c.w // 2):b.stop * (c.h // 2) * (c.w // 2)].reshape(-1)
        assert (got[cnt == 0].view(torch.int16) == 0).all(), f"{tag}: a pixel that is no window's argmax is not 0"
        err = (got.double() - ref).abs()
        note("max-pool backward", err, bound)
        assert (err <= bound).all(), f"{tag} max-pool backward: {int((err > bound).sum())} pixels over the bound"
    dy = tap(c, DY_STEM)
    conv_bn(c, cv, g, dy, None, tag)
    check_wgrad(c, cv, dy, tag)
    return gA, gB


# ------------------------------------------------------------------------------------------------ cases
class Ctx:
    pass


def backward(c, tap_block, d_blocks):
    c.L.call("dirb200_resnet_set_backward_tap", c.net, tap_block)
    c.grads.copy_(c.g0)
    for stage in range(c.nst, -1, -1):
        if d_blocks is not None:
            db = d_blocks[stage - 1] if stage else None
            c.L.call("dirb200_resnet_backward_blocks_stage", c.net, stage, c.L.ptr(db), c.L.ptr(c.flat),
                     c.L.ptr(c.grads), c.L.stream_ptr())
        else:
            c.L.call("dirb200_resnet_backward_stage", c.net, stage, c.L.ptr(c.d_enc), c.L.ptr(c.flat), c.L.ptr(c.grads),
                     c.L.stream_ptr())
    torch.cuda.synchronize()
    return c.grads.clone()


def run_backwards(c, d_blocks, taps, top, tag):
    """Untapped backwards (eager, captured), one tapped backward per block of `taps` (descending), an untapped replay."""
    ends = {sum(c.layers[:s + 1]) - 1: s + 1 for s in range(c.nst)}           # last block of layer group -> stage
    stage_of = lambda bi: next(s + 1 for s in range(c.nst) if bi < sum(c.layers[:s + 1]))
    flat0 = backward(c, NO_TAP, d_blocks)
    assert same_bits(flat0, backward(c, NO_TAP, d_blocks)), f"{tag}: two untapped backwards differ"
    later = None              # (block, its nA, its nB or dz) of the block tapped before
    for bi in taps:
        flat = backward(c, bi, d_blocks)
        assert same_bits(flat, flat0), f"{tag}: the backward tapped at block {bi} changed the flat gradient"
        btag = f"{tag} block {bi}"
        if bi >= 0 and top is not None and stage_of(bi) > top:
            # above the first gradient of a multi-scale backward: nothing ran
            assert all(tap(c, s) is None for s in range(14)), f"{btag}: a stage without a gradient wrote something"
            later = None
            continue
        if bi < 0:
            gA, gB = check_stem(c, btag)
            nxt = (gA, gB)
        else:
            gA, gB, nA, nBdz = check_block(c, bi, btag)
            nxt = (nA, nBdz)
            if d_blocks is None and bi == len(c.blk) - 2:
                # average-pool backward of d_enc
                hw = gA.shape[0] // c.n
                inv = torch.tensor(1.0 / hw, dtype=torch.float32, device=DEV)
                ref = (c.d_enc * inv).to(BF).view(c.n, 1, -1).expand(c.n, hw, -1).reshape(gA.shape)
                assert same_bits(gA, ref), f"{btag}: the average-pool backward differs"
            if d_blocks is not None:
                s = ends.get(bi)
                if s is not None and s == top:
                    assert same_bits(gA, d_blocks[s - 1].reshape(gA.shape)), f"{btag}: gA is not the group gradient"
                    assert tap(c, G3) is None, btag
                elif s is not None and d_blocks[s - 1] is not None:
                    assert same_bits(tap(c, G3), d_blocks[s - 1].reshape(gA.shape)), f"{btag}: g3 is not the group gradient"
                else:
                    assert tap(c, G3) is None, f"{btag}: g3 entered a block that does not end a layer group"
        if later is not None and later[0] == bi + 1:
            assert same_bits(gA, later[1]), f"{btag}: gA is not block {bi + 1}'s nA"
            assert same_bits(gB, later[2]), f"{btag}: gB is not block {bi + 1}'s nB / dz"
        later = (bi, *[t.clone() for t in nxt]) if bi >= 0 else None
    c.L.call("dirb200_resnet_set_backward_tap", c.net, NO_TAP)
    assert same_bits(flat0, backward(c, NO_TAP, d_blocks)), f"{tag}: the untapped backward after the taps differs"
    if top is not None and top < c.nst:
        # the stages above the first gradient did nothing: their slice of the flat gradient is still g0
        lo, hi = ctypes.c_int64(), ctypes.c_int64()
        c.L.call("dirb200_resnet_stage_param_range", c.net, top + 1, ctypes.byref(lo), ctypes.byref(hi))
        npar = c.L.raw("dirb200_resnet_param_count")(c.net)
        assert torch.equal(flat0[lo.value:npar].view(torch.int32), c.g0[lo.value:npar].view(torch.int32)), \
            f"{tag}: a stage above the first gradient changed its gradients"

CASES = [((3, 4, 6, 3), 0, 16, 64, 64, False), ((3, 4, 6, 3), 0, 4, 224, 224, False),
         ((2, 2, 1, 1), 0, 16, 64, 64, False), ((2, 2, 2, 2), 1, 4, 64, 64, False), ((1, 1, 1, 1), 1, 16, 64, 64, False),
         ((3, 4, 6, 3), 0, 1, 228, 304, True), ((3, 4, 6, 3), 0, 8, 228, 304, True),
         ((2, 2, 2, 2), 1, 256, 224, 224, False), ((3, 4, 6, 3), 0, 256, 224, 224, False)]
IDS = ["r50_b16_64", "r50_b4_224", "shallow_b16_64", "r18_b4_64", "basic1111_b16_64", "nyud2_encoder_b1_228x304",
       "nyud2_encoder_b8_228x304", "r18_b256_224", "r50_b256_224"]


def subset(layers):
    """stem, layer1.0, the last block of layer1, layer2.0, the last block (descending)."""
    return sorted({0, layers[0] - 1, layers[0], sum(layers) - 1}, reverse=True) + [-1]


@pytest.mark.parametrize("layers,basic,n,h,w,blocks", CASES, ids=IDS)
def test_backward_in_place(layers, basic, n, h, w, blocks):
    torch.cuda.reset_peak_memory_stats()
    c = Ctx()
    c.L, c.layers, c.basic, c.n, c.h, c.w = lib(), layers, bool(basic), n, h, w
    c.m = make_model(layers, c.basic)
    c.net = c.m._net((n, 3, h, w))
    table = conv_table(layers, h, w, c.basic)
    c.blk = by_block(table)
    c.named = dict(c.m.named_parameters())
    c.flat = c.m.flat_parameters()
    c.nst = c.L.raw("dirb200_resnet_num_stages")(c.net)
    c.forms = set()
    npar = c.L.raw("dirb200_resnet_param_count")(c.net)
    g = torch.Generator(device=DEV).manual_seed(n + h + w + len(layers) + basic)
    t0 = time.time()
    randomize_bn(c.m, table, g, running=False)
    c.x = torch.randn(n, 3, h, w, generator=g, device=DEV)
    outs = forward(c.m, c.x, blocks, True)
    torch.cuda.synchronize()
    # the flat gradient starts from a non-zero g0 spread over exponents: every "accumulates" claim is tested
    c.g0 = torch.zeros(c.flat.numel(), device=DEV)
    c.g0[:npar] = torch.randn(npar, generator=g, device=DEV) * torch.exp2(
        torch.randint(-6, 7, (npar,), generator=g, device=DEV).float())
    c.grads = torch.empty_like(c.g0)
    taps = subset(layers) if n >= 256 else list(range(sum(layers) - 1, -2, -1))
    if blocks:
        c.d_enc = None
        rnd = lambda s: (torch.randn(outs[s].shape, generator=g, device=DEV) * 1e-3).to(BF)
        run_backwards(c, [rnd(s) for s in range(4)], taps, 4, "all four outputs")
        run_backwards(c, [None, rnd(1), None, None], taps, 2, "layer2's output only")
    else:
        c.d_enc = torch.randn(n, c.L.raw("dirb200_resnet_feature_dim")(c.net), generator=g, device=DEV) * 1e-2
        run_backwards(c, None, taps, None, "d_enc")
    # a tap on a block that does not exist is refused; switching off works without a net change
    assert c.L.raw("dirb200_resnet_set_backward_tap")(c.net, sum(layers)) == -1 and "bad block" in c.L.last_error()
    ptr, rows, ch = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_int()
    rc = c.L.raw("dirb200_resnet_peek_backward")(c.net, 0, ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch))
    assert rc == -1 and "no backward tap" in c.L.last_error(), c.L.last_error()
    # the wiring forms the case is there for were met
    want = {"full stride-2 1x1", "g3"} if blocks else {"compact gB", "compact"}
    assert want <= c.forms, (want, c.forms)
    peak = torch.cuda.max_memory_allocated() / 2 ** 30
    free = torch.cuda.mem_get_info()[0] / 2 ** 30
    # the net (and its tap buffers) goes now, not whenever the model is collected
    c.m._free_nets()
    del c
    gc.collect()
    torch.cuda.empty_cache()
    print(f"\nbackward {IDS[CASES.index((layers, basic, n, h, w, blocks))]}: {time.time() - t0:.1f} s, "
          f"torch peak {peak:.1f} GiB, {free:.1f} GiB free with the net, {len(taps)} taps; worst error / bound so far: " + ", ".join(f"{k} {v:.3f}" for k, v in WORST.items()))


RERUN_VARS = ("DIRB200_SMS", "DIRB200_GRAPH", "DIRB200_FUSED_BWD_MOMENTS")


@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}, {"DIRB200_GRAPH": "0"}, {"DIRB200_FUSED_BWD_MOMENTS": "0"}],
                         ids=["sms7", "no_graphs", "bn_bwd_reduce_pass"])
def test_whole_file_rerun(env):
    """This file again in a fresh process (the switches are read once per process): grids capped at 7 SMs (other
    split factors, long chains), eager launches only, every BN backward through the separate bn_bwd_reduce pass."""
    if any(os.environ.get(k) for k in RERUN_VARS):
        pytest.skip("already a rerun")
    rerun(env, "-k", "not rerun", path=os.path.abspath(__file__))
