"""GPU parity of the wgmma implicit-GEMM convolutions (fprop / dgrad / wgrad) against float64 convolutions of the
same bf16-rounded operands, element by element.

fprop and dgrad store bf16: every output must lie within  2^-8 |ref| + (1 + 2^-8) KAPPA(K) A  of the float64 result
ref, where A is the same convolution of |operands| (the abs-conv) and KAPPA(K) the fp32 accumulation error of a K-long
dot product (below).  A bound relative to the tensor maximum would let a conv that is wrong only on its
small-magnitude outputs pass.  wgrad is fp32 end to end: |dw - ref| <= KAPPA(pixels per split) A + splits 2^-24 A."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24            # fp32 unit round-off
BF16_U = 2.0 ** -8        # bf16 unit round-off (8-bit significand, round to nearest)


def KAPPA(K):
    """fp32 accumulation error per unit of the abs-conv for a K-long reduction on the wgmma path: K / 16 k16 steps,
    each one rounding of the running fp32 accumulator (the bf16 products are exact), plus up to 16 roundings of the
    sums inside one step: (K / 16 + 16) * 2^-24."""
    return (K / 16 + 16) * U


def nhwc_bf16(t):      # NCHW fp32 -> NHWC bf16 contiguous
    return t.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)


def to_nchw_f32(t):
    return t.float().permute(0, 3, 1, 2).contiguous()


def to_nchw_f64(t):
    return t.double().permute(0, 3, 1, 2).contiguous()


def check_elementwise(what, got, ref, A, bound):
    """|got - ref| <= bound everywhere; reports the worst |got - ref| / A (the measured accumulation error)."""
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                     # NaN (an output never written) counts as over the bound
    ratio = (err / A.clamp_min(1e-300)).max().item()
    assert not bad.any(), (f"{what}: {int(bad.sum())} of {bad.numel()} elements over the bound; worst excess "
                           f"{(err - bound).max().item():.3e}, max |err| / A {ratio:.3e}")
    return ratio


def check_bf16_out(what, got_nhwc, ref, A, K):
    return check_elementwise(what, to_nchw_f64(got_nhwc), ref, A,
                             BF16_U * ref.abs() + (1 + BF16_U) * KAPPA(K) * A)


def run_conv(n, h, w, cin, cout, k, stride, pad, seed=0, check_dgrad=True, device_rng=False):
    import _lib, _convlib  # noqa: F401
    g = torch.Generator(device=DEV if device_rng else "cpu").manual_seed(seed)   # device_rng: full-size tensors
    gdev = DEV if device_rng else "cpu"
    x = torch.randn(n, cin, h, w, generator=g, device=gdev).to(DEV)
    wt = (torch.randn(cout, cin, k, k, generator=g, device=gdev) / (cin * k * k) ** 0.5).to(DEV)
    xb = nhwc_bf16(x)
    xr = to_nchw_f64(xb)                                  # bf16-rounded x as float64 NCHW
    wr = wt.to(torch.bfloat16).double()
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    st = _lib.stream_ptr()
    wf = torch.empty(cout, k, k, cin, dtype=torch.bfloat16, device=DEV)
    wd = torch.empty(cin, k, k, cout, dtype=torch.bfloat16, device=DEV)
    _lib.call("dirb200_conv_prep_weights", _lib.ptr(wt), cout, cin, k, k, 0, _lib.ptr(wf), _lib.ptr(wd), st)
    assert torch.equal(wf, wt.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16))
    assert torch.equal(wd, wt.permute(1, 2, 3, 0).contiguous().to(torch.bfloat16))
    y = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    shape = (n, h, w, cin, cout, k, k, stride, pad)
    _lib.call("dirb200_conv_fprop", _lib.ptr(xb), _lib.ptr(wf), _lib.ptr(y), *shape, 0, st)
    ref = F.conv2d(xr, wr, stride=stride, padding=pad)
    A = F.conv2d(xr.abs(), wr.abs(), stride=stride, padding=pad)
    worst = {"fprop": check_bf16_out("fprop", y, ref, A, k * k * cin)}
    del ref, A, y

    dy = torch.randn(n, cout, ho, wo, generator=g, device=gdev).to(DEV)
    dyb = nhwc_bf16(dy)
    dyr = to_nchw_f64(dyb)
    del dy, x
    if check_dgrad:
        dx = torch.full((n, h, w, cin), float("nan"), dtype=torch.bfloat16, device=DEV)
        _lib.call("dirb200_conv_dgrad", _lib.ptr(dyb), _lib.ptr(wd), _lib.ptr(dx), *shape, st)
        ref_dx = torch.nn.grad.conv2d_input(xr.shape, wr, dyr, stride=stride, padding=pad)
        A_dx = torch.nn.grad.conv2d_input(xr.shape, wr.abs(), dyr.abs(), stride=stride, padding=pad)
        worst["dgrad"] = check_bf16_out("dgrad", dx, ref_dx, A_dx, k * k * cout)
        del ref_dx, A_dx, dx

    nbytes = _lib.raw("dirb200_conv_wgrad_workspace_bytes")(*shape, 0)
    splits = nbytes // (k * k * cin * cout * 4)
    kblocks = -(-(n * ho * wo) // 64)
    per_split = -(-kblocks // splits) * 64               # pixels one split-K partial sums
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    dw = torch.full((cout, cin, k, k), float("nan"), dtype=torch.float32, device=DEV)
    _lib.call("dirb200_conv_wgrad", _lib.ptr(xb), _lib.ptr(dyb), _lib.ptr(dw), _lib.ptr(ws), nbytes, *shape, 0, 0, st)
    ref_dw = torch.nn.grad.conv2d_weight(xr, wr.shape, dyr, stride=stride, padding=pad)
    A_dw = torch.nn.grad.conv2d_weight(xr.abs(), wr.shape, dyr.abs(), stride=stride, padding=pad)
    kw_ = KAPPA(per_split) + splits * U                  # + the fp32 sum over the splits
    worst["wgrad"] = check_elementwise("wgrad", dw, ref_dw, A_dw, kw_ * A_dw)
    # accumulate mode: dw (already within the bound) + a second copy, one more fp32 rounding
    _lib.call("dirb200_conv_wgrad", _lib.ptr(xb), _lib.ptr(dyb), _lib.ptr(dw), _lib.ptr(ws), nbytes, *shape, 0, 1, st)
    check_elementwise("wgrad accumulate", dw, 2 * ref_dw, A_dw, 2 * kw_ * A_dw + U * 2 * ref_dw.abs())
    torch.cuda.synchronize()
    print("conv", shape, "max |err| / A:", {kk: f"{v:.2e}" for kk, v in worst.items()})
    return worst


@pytest.mark.parametrize("cfg", [
    # n, h, w, cin, cout, k, stride, pad      (every distinct conv form of ResNet-50, small spatial sizes)
    (2, 8, 8, 64, 64, 1, 1, 0),        # layer1 1x1
    (2, 8, 8, 64, 256, 1, 1, 0),       # expand 1x1, BN=128 tiles x2
    (2, 8, 8, 256, 64, 1, 1, 0),       # reduce 1x1, 4 k-blocks
    (2, 8, 8, 64, 64, 3, 1, 1),        # layer1 3x3
    (2, 8, 8, 128, 128, 3, 2, 1),      # strided 3x3
    (2, 8, 8, 256, 512, 1, 2, 0),      # strided 1x1 downsample
    (3, 7, 7, 512, 512, 3, 1, 1),      # ragged M (147 pixels), many k-blocks (72)
    (1, 14, 14, 1024, 256, 1, 1, 0),   # 16 k-blocks > ring depth
    (4, 7, 7, 512, 2048, 1, 1, 0),     # 16 n-tiles
    (5, 9, 11, 64, 128, 3, 2, 1),      # odd sizes, non-square
    (75, 14, 14, 256, 256, 3, 1, 1),   # im2col TMA: 115 m-tiles, several tiles per CTA
    (64, 28, 28, 512, 256, 1, 1, 0),   # tiled TMA: 392 m-tiles, 8 k-blocks
    (64, 14, 14, 256, 1024, 1, 1, 0),  # 8 n-tiles, several tiles per CTA
    (3, 12, 20, 64, 64, 3, 1, 1),      # non-square
    (5, 7, 9, 64, 64, 3, 1, 1),
    (4, 56, 56, 64, 64, 3, 1, 1),      # the layer1 shape
    (1, 6, 60, 64, 64, 3, 1, 1),
    (2, 5, 100, 64, 64, 3, 1, 1),
    # 5x5 / stride 1 / pad 2: the NYUD2 decoder and refinement convolutions (nyud2-dir/models/modules.py:11-20,154-160)
    (2, 12, 16, 128, 128, 5, 1, 2),    # R.conv0 / conv1 form: 25 taps x 2 channel blocks = 50 k-blocks
    (3, 9, 11, 64, 128, 5, 1, 2),      # odd sizes
    (1, 24, 32, 128, 64, 5, 1, 2),     # up-projection form (Cout < Cin)
    (2, 8, 8, 256, 256, 5, 1, 2),      # 100 k-blocks
])
def test_conv_forms(cfg):
    run_conv(*cfg)


@pytest.mark.parametrize("cfg,device_rng", [
    # the BiLSTM's GEMMs (imbalanced-regression_b200/rnn.py) as the 1x1 convs over an n = 1, h = T, w = M "image" they
    # run as: Cout = 8 Hp gate columns (both directions), K = T M = 10 240 pixels in wgrad
    ((1, 40, 256, 320, 12288, 1, 1, 0), True),    # layer 0's projection, W_ih wgrad, dx: d_word 300 pads to 320, so
                                                  # dgrad's N = 320 runs in 64-wide tiles
    ((1, 40, 256, 3072, 12288, 1, 1, 0), True),   # layer 1 (input 2 Hp = 3072)
    ((1, 40, 256, 1536, 6144, 1, 1, 0), True),    # the W_hh wgrad of one direction (K = Hp, N = 4 Hp)
    ((1, 9, 10, 64, 512, 1, 1, 0), False),        # the small model (H 20, T 9, M 10): 90 pixels, a ragged k-block
], ids=["lstm-l0", "lstm-l1", "lstm-whh", "lstm-small"])
def test_conv_lstm_forms(cfg, device_rng):
    run_conv(*cfg, seed=4, device_rng=device_rng)


def test_conv_layer1_full_batch_shape():
    # a BASELINE-size layer: batch 32 of the 56x56x64 3x3 (M = 100 352 rows, 784 tiles)
    run_conv(32, 56, 56, 64, 64, 3, 1, 1, seed=1)


def test_conv_nyud2_refinement_shape():
    # BASELINE config 4 geometry at batch 1: the 5x5 128 -> 128 conv of nyud2-dir's R module on a 240 x 320 map
    run_conv(1, 240, 320, 128, 128, 5, 1, 2, seed=2, device_rng=True)


def test_stem_conv_and_s2d():
    import _lib, _convlib  # noqa: F401
    g = torch.Generator(device="cpu").manual_seed(3)
    n, h, w, cout = 3, 32, 32, 64
    x = torch.randn(n, 3, h, w, generator=g).to(DEV)
    wt = (torch.randn(cout, 3, 7, 7, generator=g) / 147 ** 0.5).to(DEV)
    st = _lib.stream_ptr()
    xs = torch.empty(n, h // 2, w // 2, 16, dtype=torch.bfloat16, device=DEV)
    _lib.call("dirb200_input_to_s2d", _lib.ptr(x), n, h, w, _lib.ptr(xs), st)
    ref_s2d = torch.zeros(n, h // 2, w // 2, 16, device=DEV)
    for ph in range(2):
        for pw in range(2):
            for c in range(3):
                ref_s2d[..., (ph * 2 + pw) * 4 + c] = x[:, c, ph::2, pw::2]
    assert torch.equal(xs, ref_s2d.to(torch.bfloat16))
    wf = torch.empty(cout, 256, dtype=torch.bfloat16, device=DEV)
    _lib.call("dirb200_conv_prep_weights", _lib.ptr(wt), cout, 3, 7, 7, 1, _lib.ptr(wf), None, st)
    shape = (n, h, w, 3, cout, 7, 7, 2, 3)
    y = torch.full((n, h // 2, w // 2, cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    _lib.call("dirb200_conv_fprop", _lib.ptr(xs), _lib.ptr(wf), _lib.ptr(y), *shape, 1, st)
    xr, wr = x.to(torch.bfloat16).double(), wt.to(torch.bfloat16).double()
    ref = F.conv2d(xr, wr, stride=2, padding=3)
    A = F.conv2d(xr.abs(), wr.abs(), stride=2, padding=3)
    check_bf16_out("stem fprop", y, ref, A, 256)       # the 4x4x16 space-to-depth GEMM: K = 256
    dy = torch.randn(n, cout, h // 2, w // 2, generator=g).to(DEV)
    dyb = nhwc_bf16(dy)
    nbytes = _lib.raw("dirb200_conv_wgrad_workspace_bytes")(*shape, 1)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    dw = torch.full((cout, 3, 7, 7), float("nan"), dtype=torch.float32, device=DEV)
    _lib.call("dirb200_conv_wgrad", _lib.ptr(xs), _lib.ptr(dyb), _lib.ptr(dw), _lib.ptr(ws), nbytes, *shape, 1, 0, st)
    dyr = to_nchw_f64(dyb)
    ref_dw = torch.nn.grad.conv2d_weight(xr, wr.shape, dyr, stride=2, padding=3)
    A_dw = torch.nn.grad.conv2d_weight(xr.abs(), wr.shape, dyr.abs(), stride=2, padding=3)
    splits = nbytes // (cout * 256 * 4)
    per_split = -(-(-(-(n * (h // 2) * (w // 2)) // 64)) // splits) * 64
    check_elementwise("stem wgrad", dw, ref_dw, A_dw, (KAPPA(per_split) + splits * U) * A_dw)
