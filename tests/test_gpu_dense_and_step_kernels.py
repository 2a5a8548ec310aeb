"""The up-sampling and channel-copy kernels of csrc/dense_ops.cu, the regressor head (avgpool, linear1) and the optimizer
kernels (adam, sgd, grad_clip) of csrc/nn_kernels.cu, one launch at a time through the C ABI, against float64 references
computed on the GPU.  Outputs are prefilled with NaN, so every element must be written.  u = 2^-24.

  upsample_bilinear_fwd   out = Wy . x . Wx^T per image and channel, with Wy [ho x h], Wx [wo x w] built from a Python
                          restatement of the align_corners=False index rule (src_index, pinned to F.interpolate in
                          tests/test_dense_and_step_kernels_cpu.py).  upsample_lerp rounds hx = 1 - lx, each product
                          lx*v and ly*bot, and each of its three fmas: a term w_y w_x v passes through at most 4
                          roundings, so |out - ref| <= 2^-8 |ref| + (1 + 2^-8) 4u A, A the same interpolation of |x|
                          (the 2^-8 terms: the bf16 store).
  upsample_bilinear_bwd   dx = Wy^T . dy . Wx.  Each weight wy * wx carries <= 5 roundings (1 - ly, the sum of the two
                          candidate weights, once per axis, and their product) and the fma chain over the T = nnz(Wy
                          column) * nnz(Wx column) gathered terms adds T, so |dx - ref| <= 2^-8 |ref| + (1 + 2^-8)
                          (T + 5) u sum |w dy|.  Two runs are bit-identical; an image's dx depends on its own dy only.
  copy_channels           bit-exact, channels outside [dst_off, dst_off + c) of a sentinel-filled destination unchanged;
                          cat_channels / split_channels forward and backward, uncovered gradient channels exactly 0.
  avgpool_fwd             hw - 1 adds, the rounded 1/hw and the product: |enc - ref| <= (hw + 2) u sum |x| / hw.
  avgpool_bwd             bit-exact: bf16(fp32(g) * fp32(1/hw)).
  linear1_fwd             ceil(d/256) fmas per thread, a 5-level warp tree, the serial sum over 8 warps and the bias:
                          |pred - ref| <= (ceil(d/256) + 14) u (sum |x w| + |b|).
  linear1_bwd             dx bit-exact fp32(g w); dw within n u sum |g x| (fma chain over n); dbias within n u sum |g|.
  adam / sgd              teacher-forced: step t starts from the kernel's own state after step t - 1.  The moments
                          (m, v, momentum buffer) are bounded by the roundings on each term's path times the sum of the
                          absolute values of the terms; the parameter against the update formed from the kernel's own
                          moments, within u |p'| + k u |delta|.
  grad_clip_coef          the norm within (L / 2 + 1) u of |scale| ||g||, L the per-thread fp32 chain of the grid the entry
                          point launches; the coefficient bit-exact from the kernel's own norm.

Every bound is multiplied by 1.001 for the second-order terms.  The whole file runs a second time with DIRB200_SMS=7
(few CTAs: the grid-stride loops iterate many times)."""
import math
import os
import subprocess
import sys
import types

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
SLACK = 1.001
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
BF = torch.bfloat16
BENCH_PARAMS = 23_510_081          # the flat parameter buffer of the IMDB-WIKI benchmark's ResNet-50 (n mod 4 = 1)


def lib():
    import _lib
    import resnet  # noqa: F401  (registers the linear1 / optimizer entry points)
    return _lib


def num_sms():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = int(os.environ.get("DIRB200_SMS", "0") or 0)
    return cap if 0 < cap < sms else sms


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def bits(t):
    return t.view(torch.int16)


def rand_bf16(shape, g, lo=2.0 ** -8, hi=6.0):
    """bf16 normal values, |x| in [lo, hi] or exactly 0."""
    x = torch.randn(*shape, generator=g, device=DEV).clamp_(-hi, hi)
    x = torch.where(x.abs() < lo, torch.zeros((), device=DEV), x)
    return x.to(BF)


def nan_bf16(*shape):
    return torch.full(shape, float("nan"), dtype=BF, device=DEV)


def nan_f32(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def check(name, got, ref, bound):
    ok = (got.double() - ref).abs() <= bound            # NaN (never written) fails
    if not ok.all():
        i = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.numel()} elements outside the bound, first at {i}: "
                             f"got {got[tuple(i)].item()!r}, ref {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3e}")


def check_bits(name, got, ref):
    bad = bits(got) != bits(ref) if got.dtype == BF else got.view(torch.int32) != ref.view(torch.int32)
    assert not bad.any(), f"{name}: {int(bad.sum())} elements differ, first at {bad.nonzero()[0].tolist()}"


# ------------------------------------------------------------------------------------------------------- up-sampling
def src_index(in_size, out_size):
    """(i0, i1, lambda) of every output position under F.upsample(..., mode='bilinear', align_corners=False), restated:
    scale = fp32(in) / fp32(out); s = fp32 of float64(o + 0.5) * float64(scale) - 0.5 (the product of two fp32 values
    and the subtraction are exact in float64 at these magnitudes, so this is the fp32 fma); s clamped at 0;
    i0 = floor(s) clamped to in - 1; i1 = i0 + (i0 < in - 1); lambda = s - i0 (exact)."""
    scale = np.float32(in_size) / np.float32(out_size)
    s = ((np.arange(out_size, dtype=np.float64) + 0.5) * np.float64(scale) - 0.5).astype(np.float32)
    s = np.maximum(s, np.float32(0))
    i0 = np.minimum(np.floor(s).astype(np.int64), in_size - 1)
    i1 = i0 + (i0 < in_size - 1)
    return i0, i1, s - i0.astype(np.float32)


def interp_matrix(in_size, out_size):
    """float64 [out, in]: row o holds 1 - lambda at i0 and lambda at i1 (summed where i0 == i1)."""
    i0, i1, lam = src_index(in_size, out_size)
    W = np.zeros((out_size, in_size))
    o = np.arange(out_size)
    lam = lam.astype(np.float64)
    np.add.at(W, (o, i0), 1.0 - lam)
    np.add.at(W, (o, i1), lam)
    return W


def up_apply(Wy, Wx, x):
    """[n, h, w, c] -> [n, ho, wo, c]: Wy . x . Wx^T per image and channel (float64)."""
    return torch.einsum("pw,nowc->nopc", Wx, torch.einsum("oh,nhwc->nowc", Wy, x))


def up_adjoint(Wy, Wx, dy):
    """[n, ho, wo, c] -> [n, h, w, c]: Wy^T . dy . Wx (float64)."""
    return torch.einsum("pw,nhpc->nhwc", Wx, torch.einsum("oh,nopc->nhpc", Wy, dy))


# (n, h, w, c, ho, wo)
UP_SHAPES = [
    # D's up-projections at 228 x 304 (batch 2)
    (2, 8, 10, 1024, 15, 19), (2, 15, 19, 512, 29, 38), (2, 29, 38, 256, 57, 76), (2, 57, 76, 128, 114, 152),
    # MFF's four branches to 114 x 152
    (2, 57, 76, 256, 114, 152), (2, 29, 38, 512, 114, 152), (2, 15, 19, 1024, 114, 152), (2, 8, 10, 2048, 114, 152),
    # batch 8 at 114 x 152: more work than grid1d's 32 CTAs per SM, so the grid-stride loop iterates
    (8, 57, 76, 128, 114, 152), (8, 57, 76, 256, 114, 152),
    (3, 15, 19, 64, 15, 19),                 # same size
    (2, 37, 41, 8, 7, 5),                    # non-integer down-sampling, ratios 5.3 and 8.2
    (2, 12, 9, 24, 5, 4),                    # non-integer down-sampling, c = 24
    (2, 1, 1, 8, 13, 17), (2, 13, 17, 8, 1, 1),
    (2, 1, 20, 16, 5, 33), (3, 7, 1, 8, 14, 1),   # one axis of size 1
    (1, 5, 7, 24, 11, 9),
]


def up_id(s):
    n, h, w, c, ho, wo = s
    return f"{n}x{h}x{w}x{c}-to-{ho}x{wo}"


def up_weights(h, w, ho, wo):
    Wy = torch.tensor(interp_matrix(h, ho), dtype=F64, device=DEV)
    Wx = torch.tensor(interp_matrix(w, wo), dtype=F64, device=DEV)
    return Wy, Wx


def run_up_bwd(dy, shape):
    L = lib()
    n, h, w, c, ho, wo = shape
    dx = nan_bf16(n, h, w, c)
    L.call("dirb200_upsample_bilinear_bwd", L.ptr(dy), n, h, w, c, ho, wo, L.ptr(dx), L.stream_ptr())
    torch.cuda.synchronize()
    return dx


@pytest.mark.parametrize("shape", UP_SHAPES, ids=[up_id(s) for s in UP_SHAPES])
def test_upsample_bilinear_fwd_bwd_per_element(shape):
    L = lib()
    n, h, w, c, ho, wo = shape
    g = gen(sum(shape))
    Wy, Wx = up_weights(h, w, ho, wo)

    x = rand_bf16((n, h, w, c), g)
    out = nan_bf16(n, ho, wo, c)
    L.call("dirb200_upsample_bilinear_fwd", L.ptr(x), n, h, w, c, ho, wo, L.ptr(out), L.stream_ptr())
    torch.cuda.synchronize()
    ref = up_apply(Wy, Wx, x.double())
    A = up_apply(Wy, Wx, x.double().abs())
    check("upsample fwd", out, ref, 2.0 ** -8 * ref.abs() + (1 + 2.0 ** -8) * 4 * U * SLACK * A)
    del ref, A

    dy = rand_bf16((n, ho, wo, c), g)
    dx = run_up_bwd(dy, shape)
    ref = up_adjoint(Wy, Wx, dy.double())
    M = up_adjoint(Wy, Wx, dy.double().abs())
    T = ((Wy != 0).sum(0)[:, None] * (Wx != 0).sum(0)[None, :]).to(F64)[None, :, :, None]
    check("upsample bwd", dx, ref, 2.0 ** -8 * ref.abs() + (1 + 2.0 ** -8) * (T + 5) * U * SLACK * M)
    del ref, M

    # deterministic: a second run gives the same bits; an image's dx depends on its own dy only
    check_bits("upsample bwd, second run", run_up_bwd(dy, shape), dx)
    if n > 1:
        dy2 = dy.clone()
        dy2[0] = rand_bf16((ho, wo, c), g)
        dx2 = run_up_bwd(dy2, shape)
        check_bits("upsample bwd, images 1.. with image 0's dy changed", dx2[1:], dx[1:])
        assert (bits(dx2[0]) != bits(dx[0])).any()


# ------------------------------------------------------------------------------------------------------ channel copy
def sentinel(shape, seed):
    """destination filler: bf16 values drawn at 7x the scale of the copied ones, so a channel the copy should have
    written, or should have left alone, shows"""
    return rand_bf16(shape, gen(seed), lo=0.0, hi=1e4) * 7


def copy_into(src, src_off, dst, dst_off, c):
    """dirb200_copy_channels over every pixel of src / dst ([..., channels]); returns dst's state before the call."""
    L = lib()
    before = dst.clone()
    pixels = src.numel() // src.shape[-1]
    L.call("dirb200_copy_channels", L.ptr(src), src.shape[-1], src_off, L.ptr(dst), dst.shape[-1], dst_off, c, pixels,
           L.stream_ptr())
    torch.cuda.synchronize()
    return before


def check_copy(src, src_off, dst, dst_off, c, before, tag):
    check_bits(f"{tag}: copied channels", dst[..., dst_off:dst_off + c], src[..., src_off:src_off + c])
    check_bits(f"{tag}: channels below the range", dst[..., :dst_off], before[..., :dst_off])
    check_bits(f"{tag}: channels above the range", dst[..., dst_off + c:], before[..., dst_off + c:])


# (pixel dims, source widths, destination width, source offsets, destination offsets, widths copied)
COPY_CASES = [
    ("mff_concat_4x16_to_64", (8, 114, 152), [(16, 0, 64, 16 * i, 16) for i in range(4)]),
    ("r_input_64_64_to_128", (8, 114, 152), [(64, 0, 128, 0, 64), (64, 0, 128, 64, 64)]),
    ("paired_conv_split_16_16_of_64", (8, 114, 152), [(64, 0, 16, 0, 16), (64, 16, 16, 0, 16)]),
    ("conv1_2_pad_16_48_and_split_16", (8, 57, 76), [(16, 0, 64, 0, 16), (48, 0, 64, 16, 48), (64, 0, 16, 0, 16)]),
    ("strided_middle", (3, 5, 7), [(40, 8, 72, 24, 24), (24, 16, 24, 8, 8)]),
    ("grid_stride_256", (8, 114, 152), [(256, 0, 512, 256, 256)]),
]


@pytest.mark.parametrize("dims,copies", [c[1:] for c in COPY_CASES], ids=[c[0] for c in COPY_CASES])
def test_copy_channels_sentinel(dims, copies):
    g = gen(len(copies) + dims[1])
    for k, (cs, soff, cd, doff, c) in enumerate(copies):
        src = rand_bf16(dims + (cs,), g)
        dst = sentinel(dims + (cd,), 100 + k)
        before = copy_into(src, soff, dst, doff, c)
        check_copy(src, soff, dst, doff, c, before, f"copy {k} ({cs}[{soff}:{soff + c}] -> {cd}[{doff}:])")


def test_copy_channels_zero_pixels_launches_nothing():
    L = lib()
    src = rand_bf16((4, 16), gen(1))
    dst = sentinel((4, 32), 2)
    before = dst.clone()
    n0 = L.launch_count()
    L.call("dirb200_copy_channels", L.ptr(src), 16, 0, L.ptr(dst), 32, 8, 16, 0, L.stream_ptr())
    torch.cuda.synchronize()
    assert L.launch_count() == n0
    check_bits("pixels = 0", dst, before)


@pytest.mark.parametrize("dims,widths", [((8, 114, 152), (16, 16, 16, 16)), ((8, 114, 152), (64, 64)),
                                         ((8, 57, 76), (16, 48)), ((2, 3, 5), (8, 24, 16))],
                         ids=["mff_concat", "r_input", "conv1_2_zero_pad", "small"])
def test_cat_channels_fwd_bwd_bit_exact(dims, widths):
    import dense_ops as D
    g = gen(sum(widths))
    parts = [rand_bf16(dims + (c,), g).requires_grad_(True) for c in widths]
    out = D.cat_channels(parts)
    check_bits("cat forward", out, torch.cat([p.detach() for p in parts], -1))
    dy = rand_bf16(dims + (sum(widths),), g)
    grads = torch.autograd.grad(out, parts, dy)
    off = 0
    for k, (gr, c) in enumerate(zip(grads, widths)):
        check_bits(f"cat backward, part {k}", gr, dy[..., off:off + c])
        off += c


def poison_free_block(shape):
    """Leave a NaN-filled block of this size in the caching allocator, so that an uninitialised allocation of the same
    size shows as NaN rather than as whatever zeros happened to be there."""
    t = torch.full(shape, float("nan"), dtype=BF, device=DEV)
    del t


@pytest.mark.parametrize("dims,total,sizes", [((8, 114, 152), 64, (16, 16)), ((8, 57, 76), 64, (16,)),
                                              ((8, 114, 152), 128, (64, 64)), ((2, 3, 5), 40, (8, 24))],
                         ids=["paired_conv_16_16_of_64", "conv1_2_16_of_64", "covering_64_64", "covering_8_24"])
def test_split_channels_fwd_bwd_bit_exact(dims, total, sizes):
    import dense_ops as D
    g = gen(total + len(sizes))
    y = rand_bf16(dims + (total,), g).requires_grad_(True)
    outs = D.split_channels(y, sizes)
    off = 0
    for k, (o, c) in enumerate(zip(outs, sizes)):
        check_bits(f"split forward, part {k}", o, y.detach()[..., off:off + c])
        off += c
    covered = off
    gs = [rand_bf16(dims + (c,), g) for c in sizes]
    poison_free_block(dims + (total,))
    (dy,) = torch.autograd.grad(outs, y, gs)
    off = 0
    for k, (gr, c) in enumerate(zip(gs, sizes)):
        check_bits(f"split backward, part {k}", dy[..., off:off + c], gr)
        off += c
    assert (bits(dy[..., covered:]) == 0).all(), "split backward: a dropped channel's gradient is not exactly 0"
    if len(sizes) == 1:
        return

    # a None gradient (an output that reached no loss, with gradient materialisation off): its channels are 0
    ctx = types.SimpleNamespace(dims=dims + (total,), sizes=sizes)
    none_at = len(sizes) - 1
    poison_free_block(dims + (total,))
    (dy,) = D._SplitFn.backward(ctx, *[None if k == none_at else gr for k, gr in enumerate(gs)])[:1]
    torch.cuda.synchronize()
    off = 0
    for k, (gr, c) in enumerate(zip(gs, sizes)):
        if k == none_at:
            assert (bits(dy[..., off:off + c]) == 0).all(), "split backward: a None gradient's channels are not 0"
        else:
            check_bits(f"split backward with a None gradient, part {k}", dy[..., off:off + c], gr)
        off += c
    assert (bits(dy[..., covered:]) == 0).all()


# --------------------------------------------------------------------------------------------------- regressor head
# (n, hw, c): the benchmark's 7x7x2048 at batch 256; one image; one pixel; c = 8; an uneven map
POOL_CASES = [(256, 49, 2048), (1, 49, 2048), (3, 1, 64), (5, 7, 8), (2, 12 * 16, 64)]


@pytest.mark.parametrize("n,hw,c", POOL_CASES, ids=[f"{n}x{hw}x{c}" for n, hw, c in POOL_CASES])
def test_avgpool_fwd_bwd(n, hw, c):
    L = lib()
    g = gen(n + hw + c)
    x = rand_bf16((n, hw, c), g)
    enc = nan_f32(n, c)
    L.call("dirb200_avgpool_fwd", L.ptr(x), n, hw, c, L.ptr(enc), L.stream_ptr())
    torch.cuda.synchronize()
    xd = x.double()
    check("avgpool fwd", enc, xd.sum(1) / hw, (hw + 2) * U * SLACK * xd.abs().sum(1) / hw)

    genc = torch.randn(n, c, generator=g, device=DEV)
    dx = nan_bf16(n, hw, c)
    L.call("dirb200_avgpool_bwd", L.ptr(genc), n, hw, c, L.ptr(dx), L.stream_ptr())
    torch.cuda.synchronize()
    inv = torch.tensor(np.float32(1) / np.float32(hw), device=DEV)
    check_bits("avgpool bwd", dx, (genc * inv).to(BF)[:, None, :].expand(n, hw, c))


# (n, d): the benchmark's regressor; one row; d not a multiple of 256; d below one CTA; d = 8
LINEAR_CASES = [(256, 2048), (1, 2048), (7, 1000), (3, 100), (256, 8)]


@pytest.mark.parametrize("n,d", LINEAR_CASES, ids=[f"{n}x{d}" for n, d in LINEAR_CASES])
def test_linear1_fwd_bwd(n, d):
    L = lib()
    g = gen(n + d)
    x = torch.randn(n, d, generator=g, device=DEV)
    w = torch.randn(d, generator=g, device=DEV)
    b = torch.randn(1, generator=g, device=DEV)
    pred = nan_f32(n)
    L.call("dirb200_linear1_fwd", L.ptr(x), L.ptr(w), L.ptr(b), n, d, L.ptr(pred), L.stream_ptr())
    torch.cuda.synchronize()
    xd, wd, bd = x.double(), w.double(), b.double()
    mag = xd.abs() @ wd.abs() + bd.abs()
    check("linear1 fwd", pred, xd @ wd + bd, (-(-d // 256) + 14) * U * SLACK * mag)

    gp = torch.randn(n, generator=g, device=DEV)
    gd = gp.double()
    for with_dx in (True, False):
        dx = nan_f32(n, d) if with_dx else None
        dw, db = nan_f32(d), nan_f32(1)
        L.call("dirb200_linear1_bwd", L.ptr(gp), L.ptr(x), L.ptr(w), n, d, L.ptr(dx), L.ptr(dw), L.ptr(db),
               L.stream_ptr())
        torch.cuda.synchronize()
        tag = "linear1 bwd" + ("" if with_dx else " (dx = NULL)")
        if with_dx:
            check_bits(f"{tag} dx", dx, gp[:, None] * w[None, :])
        check(f"{tag} dw", dw, gd @ xd, n * U * SLACK * (gd.abs() @ xd.abs()))
        check(f"{tag} dbias", db, gd.sum().view(1), n * U * SLACK * gd.abs().sum().view(1))


# ------------------------------------------------------------------------------------------------------- optimizers
def step_inputs(n, g, scale=1.0):
    """randn of n elements with +-1e3 * scale in the elements past the last full float4 (a dropped tail shows)"""
    t = torch.randn(n, generator=g, device=DEV) * scale
    tail = n - n % 4
    t[tail:] = torch.where(t[tail:] < 0, -1e3, 1e3) * scale
    return t


def clip_coef(grads, n, grad_scale, max_norm, ws):
    """out = [coef, norm] of dirb200_grad_clip_coef (NaN-prefilled)"""
    L = lib()
    out = nan_f32(2)
    L.call("dirb200_grad_clip_coef", L.ptr(grads), n, grad_scale, max_norm, L.ptr(ws), ws.numel(), L.ptr(out),
           L.stream_ptr())
    torch.cuda.synchronize()
    return out


def clip_ws():
    return torch.zeros(lib().raw("dirb200_grad_clip_workspace_bytes")(), dtype=torch.uint8, device=DEV)


def effective_scale(g, n, grad_scale, clip, ws):
    """(clip_coef buffer or None, float64 grad_scale * coef): with clipping, max_norm is half the gradient's norm"""
    if not clip:
        return None, float(np.float32(grad_scale))
    norm = float(g.double().norm()) * grad_scale
    out = clip_coef(g, n, grad_scale, 0.5 * norm, ws)
    coef = out[:1].clone()
    assert 0.4 < float(coef) < 0.6
    return coef, float(np.float32(grad_scale)) * float(coef)


# (n, grad_scale, weight_decay, clip)
ADAM_CASES = [(1, 0.5, 0.0, False), (2, 1.0, 0.0, True), (3, 0.5, 0.0, True), (5, 0.5, 0.0, False),
              (4099, 0.5, 0.0, True), (4099, 1.0, 1e-2, False), (BENCH_PARAMS, 0.5, 0.0, True)]


@pytest.mark.parametrize("n,grad_scale,wd,clip", ADAM_CASES,
                         ids=[f"n{n}-scale{s}-wd{w}-{'clip' if c else 'noclip'}" for n, s, w, c in ADAM_CASES])
def test_adam_step_teacher_forced(n, grad_scale, wd, clip):
    """m' = fma(b1, m, (1 - b1) gr) and v' = fma(b2, v, (1 - b2) gr gr) with gr = g * scale [+ wd p]: the g term of m'
    passes through <= 5 roundings (scale * coef, g * scale, the decay fma, the product, the fma), that of v' through
    <= 9 (the three of gr twice, two products, the fma).  p' = p - (lr / bc1) (m' / (sqrt(v') / sqrt(bc2) + eps)) from
    the kernel's own m', v': the update delta carries <= 8 roundings (bc1, lr / bc1, sqrt(bc2), sqrt, the division by
    it, + eps, m' / denom, the product), the subtraction one more relative to p'."""
    L = lib()
    g = gen(n % 10007 + int(grad_scale * 10) + int(wd * 1e3) + clip)
    lr, b1, b2, eps = 1e-3, 0.9, 0.999, 1e-8
    f = lambda v: float(np.float32(v))
    lr_, b1_, b2_, eps_, wd_ = f(lr), f(b1), f(b2), f(eps), f(wd)
    p = step_inputs(n, g, 0.1)
    m = 0.01 * torch.randn(n, generator=g, device=DEV)
    v = 1e-4 * torch.rand(n, generator=g, device=DEV)
    ws = clip_ws()
    for step in (1, 2, 3):
        gr = step_inputs(n, g)
        coef, s = effective_scale(gr, n, grad_scale, clip, ws)
        p0, m0, v0, gd = p.double(), m.double(), v.double(), gr.double()
        L.call("dirb200_adam_step", L.ptr(p), L.ptr(gr), L.ptr(m), L.ptr(v), n, lr, b1, b2, eps, wd, step,
               grad_scale, L.ptr(coef), L.stream_ptr())
        torch.cuda.synchronize()
        gs, dp = gd * s, wd_ * p0
        tag = f"step {step}"
        check(f"{tag} m", m, b1_ * m0 + (1 - b1_) * (gs + dp),
              SLACK * U * (abs(b1_) * m0.abs() + 5 * (1 - b1_) * (gs.abs() + dp.abs())))
        check(f"{tag} v", v, b2_ * v0 + (1 - b2_) * (gs + dp) ** 2,
              SLACK * U * (b2_ * v0 + 9 * (1 - b2_) * (gs.abs() + dp.abs()) ** 2))
        md, vd = m.double(), v.double()
        delta = lr_ / (1 - b1_ ** step) * md / (vd.sqrt() / math.sqrt(1 - b2_ ** step) + eps_)
        ref = p0 - delta
        check(f"{tag} p", p, ref, SLACK * U * (ref.abs() + 8 * delta.abs()))
        del p0, m0, v0, gd, gs, dp, md, vd, delta, ref


# (n, grad_scale, weight_decay, momentum, clip); every case starts with first_step = 1 over a non-zero buffer
SGD_CASES = [(5, 0.5, 1e-4, 0.9, False), (4099, 1.0, 0.0, 0.9, True), (3, 0.5, 0.0, 0.0, False),
             (2, 1.0, 1e-4, 0.9, False), (1, 0.5, 1e-4, 0.0, True), (4099, 0.5, 1e-4, 0.9, False),
             (BENCH_PARAMS, 0.5, 1e-4, 0.9, True)]


@pytest.mark.parametrize("n,grad_scale,wd,momentum,clip", SGD_CASES,
                         ids=[f"n{n}-scale{s}-wd{w}-mom{mo}-{'clip' if c else 'noclip'}" for n, s, w, mo, c in SGD_CASES])
def test_sgd_step_teacher_forced(n, grad_scale, wd, momentum, clip):
    """gr = g * scale [+ wd p] (scale * coef, the product and the decay fma: 3 roundings), buf' = gr at first_step
    (the ABI's contract, whatever the buffer holds) else fma(momentum, buf, gr): buf' within 4u of the sum of its
    terms' absolute values.  p' = p - lr * buf' from the kernel's own buf' (with momentum 0, from the float64 gr)."""
    L = lib()
    g = gen(n % 10007 + int(grad_scale * 10) + int(wd * 1e4) + int(momentum * 10) + clip)
    lr = 0.05
    f = lambda v: float(np.float32(v))
    lr_, wd_, mom_ = f(lr), f(wd), f(momentum)
    p = step_inputs(n, g)
    buf = torch.randn(n, generator=g, device=DEV) if momentum else None
    ws = clip_ws()
    for step in (1, 2, 3):
        first = int(step == 1)
        gr = step_inputs(n, g, 0.1)
        coef, s = effective_scale(gr, n, grad_scale, clip, ws)
        p0, gd = p.double(), gr.double()
        b0 = buf.double() if momentum else None
        L.call("dirb200_sgd_step", L.ptr(p), L.ptr(gr), L.ptr(buf), n, lr, momentum, wd, first, grad_scale,
               L.ptr(coef), L.stream_ptr())
        torch.cuda.synchronize()
        gs, dp = gd * s, wd_ * p0
        tag = f"step {step} (first_step = {first})"
        if momentum:
            ref_b = gs + dp + (0.0 if first else mom_ * b0)
            mag = 4 * (gs.abs() + dp.abs()) + (0.0 if first else mom_ * b0.abs())
            check(f"{tag} buf", buf, ref_b, SLACK * U * mag)
            upd = lr_ * buf.double()
            ref = p0 - upd
            check(f"{tag} p", p, ref, SLACK * U * (ref.abs() + upd.abs()))
        else:
            upd = lr_ * (gs + dp)
            ref = p0 - upd
            check(f"{tag} p", p, ref, SLACK * U * (ref.abs() + 4 * lr_ * (gs.abs() + dp.abs())))
        del p0, gd, b0, gs, dp, upd, ref


def clip_chain(n):
    """per-thread fp32 chain length of dirb200_grad_clip_coef: its grid is grid1d(n / 4 + 1, 256, 4) capped at 1024
    CTAs; each grid-stride iteration folds one float4 (4 fmas), block 0's threads add one tail element each"""
    n4 = n // 4
    grid = min(max(1, min(-(-(n4 + 1) // 256), 4 * num_sms())), 1024)
    return 4 * -(-n4 // (grid * 256)) + 1


@pytest.mark.parametrize("grad_scale", (1.0, 0.5))
@pytest.mark.parametrize("n", (1, 2, 3, 5, 4099, BENCH_PARAMS))
def test_grad_clip_coef_three_calls_one_workspace(n, grad_scale):
    """Three calls on one workspace (its ticket must be reset by each): a gradient whose norm the coefficient clips,
    a zero gradient (coefficient exactly 1) and one under max_norm (coefficient 1).  The sum of squares is within L u
    of float64 (L = clip_chain), so the norm within (L / 2 + 1) u; the coefficient min(1, max_norm / (norm + 1e-6)) is
    formed in fp32 from the kernel's own norm, bit for bit."""
    g = gen(n % 10007 + int(grad_scale * 10))
    ws = clip_ws()
    Lc = clip_chain(n)
    grads = step_inputs(n, g)
    norm_ref = float(grads.double().norm()) * grad_scale
    for k, (gr, max_norm) in enumerate(((grads, 0.25 * norm_ref), (torch.zeros(n, device=DEV), 1.0),
                                        (step_inputs(n, g), 1e9))):
        out = clip_coef(gr, n, grad_scale, max_norm, ws)
        norm, coef = float(out[1]), float(out[0])
        ref = float(gr.double().norm()) * grad_scale
        assert abs(norm - ref) <= SLACK * (Lc / 2 + 1) * U * ref, (k, norm, ref, Lc)
        want = np.float32(max_norm) / (np.float32(norm) + np.float32(1e-6))
        want = min(np.float32(1), want)
        assert np.float32(coef).tobytes() == want.tobytes(), (k, coef, want)
        if k == 0:
            assert 0.2 < coef < 0.3
        else:
            assert coef == 1.0
        if k == 1:
            assert norm == 0.0


# ------------------------------------------------------------------------------------------------------------ few SMs
def test_dense_and_step_kernels_with_seven_sms():
    """This file again with the grids capped at 7 SMs (DIRB200_SMS is read once per process): the grid-stride loops of
    the up-sampling, copy, pooling and optimizer kernels iterate many times, and the clip's per-thread chains grow."""
    if os.environ.get("DIRB200_SMS"):
        pytest.skip("already running under DIRB200_SMS")
    e = dict(os.environ)
    e["DIRB200_SMS"] = "7"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
