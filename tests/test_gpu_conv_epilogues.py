"""The fused BatchNorm epilogues of the implicit-GEMM convolution, one launch at a time (the test-aid entry points of
include/dirb200.h), against float64 references computed on the GPU:

  a. fprop BN statistics: per-CTA rows of sum y / sum y^2 of the STORED bf16 y, reduced by the StatLayout rule;
  b. bn_finalize over those rows: mean, invstd, scale, shift and the running-statistics update;
  c. the folded-BN inference epilogue: relu(conv*s + h), conv*s + h, relu(bf16(conv*s + h) + residual);
  d. the BN-backward moments of a stride-1 dgrad (S0 = sum dz, S1 = sum dz*y, dz = dx * [y*scale + shift > 0]) and
     bn_bwd_coeffs over them.

Sums are bounded by the fp32 chain the kernel has: |S - S_ref| <= L * 2^-24 * sum |term| with L = 16 staged rows
+ the tiles one CTA walks + 3 for the combine of the eight per-warp slots.

Sum-of-squares cancellation in bn_finalize (var = S1 / n - mean^2): on an H100 80GB HBM3 at a 700 W power limit the
worst relative invstd error over the channels with |mean| / std > 8 (ratios up to 11.9) was 5.9e-8, about one fp32
rounding (the `invstd` lines this file prints with -s).

The whole file runs a second time with DIRB200_SMS=7 (few CTAs, uneven CTA counts per column tile, many tiles per
CTA, and fewer CTAs than column tiles at Cout = 2048)."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24                     # fp32 unit round-off
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# n, h, w, cin, cout, k, stride, pad
SHAPES = [
    (1, 5, 5, 64, 64, 3, 1, 1),         # 25 output rows: the second consumer warpgroup has no valid row
    (1, 8, 8, 64, 128, 1, 1, 0),        # 64 output rows
    (3, 7, 7, 512, 512, 3, 1, 1),       # ragged M, BN = 128, im2col
    (4, 7, 7, 512, 2048, 1, 1, 0),      # 16 n-tiles, tiled TMA
    (2, 9, 9, 128, 320, 1, 1, 0),       # BN = 64, 5 n-tiles (do not divide the grid)
    (16, 28, 28, 128, 128, 3, 1, 1),    # many tiles per CTA
    (5, 9, 11, 64, 128, 3, 2, 1),       # strided: statistics and affine only
    (2, 12, 16, 128, 128, 5, 1, 2),     # 5x5
]
BIG = (256, 56, 56, 64, 64, 3, 1, 1)    # the longest per-CTA chains of the batch-256 benchmark
STEM = (4, 64, 64, 3, 64, 7, 2, 3)
# dgrad moments: stride 1, N = cin in a dgrad
MOMENT_SHAPES = [s for s in SHAPES if s[6] == 1] + [
    (4, 14, 14, 64, 64, 3, 1, 1),
    (4, 14, 14, 256, 64, 1, 1, 0),
    (2, 7, 7, 2048, 512, 1, 1, 0),
    (3, 7, 7, 256, 256, 3, 1, 1),
]


def ids(shapes):
    return ["x".join(map(str, s)) for s in shapes]


def lib():
    import _lib, _convlib  # noqa: F401
    return _lib


def num_sms():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = int(os.environ.get("DIRB200_SMS", "0") or 0)
    return cap if 0 < cap < sms else sms


def plan_bn(shape, op, stem=0):
    n, h, w, cin, cout, k, s, p = shape
    a = (ctypes.c_int * 7)()
    L = lib()
    assert L.raw("dirb200_conv_plan")(n, h, w, cin, cout, k, k, s, p, stem, op, a) == 0, L.last_error()
    return a[0]


def out_hw(shape):
    n, h, w, cin, cout, k, s, p = shape
    return (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1


def make_weights(shape, seed):
    """fp32 [Cout][Cin][k][k] weights and the two bf16 GEMM operands."""
    n, h, w, cin, cout, k, s, p = shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    wt = torch.randn(cout, cin, k, k, generator=g, device=DEV) / (cin * k * k) ** 0.5
    L = lib()
    st = L.stream_ptr()
    wf = torch.empty(cout, k, k, cin, dtype=torch.bfloat16, device=DEV)
    wd = torch.empty(cin, k, k, cout, dtype=torch.bfloat16, device=DEV)
    L.call("dirb200_conv_prep_weights", L.ptr(wt), cout, cin, k, k, 0, L.ptr(wf), L.ptr(wd), st)
    return wt, wf, wd


def named_rows(lay, c, nrows):
    """[nrows, c] bool: the rows the layout names for each channel (conv.cuh, StatLayout)."""
    rows, n_tiles, bn, group = lay
    named = torch.zeros(nrows, c, dtype=torch.bool, device=DEV)
    for j in range((c + bn - 1) // bn):
        k = 0
        while (j + k * n_tiles) * group < rows:
            for r in range(group):
                q = (j + k * n_tiles) * group + r
                if q < rows:
                    named[q, j * bn:(j + 1) * bn] = True
            k += 1
    return named


def reduce_rows(partial, lay, c):
    """float64 sums of slots 0 / 1 over the named rows; asserts every named element was written and nothing else was."""
    named = named_rows(lay, c, partial.shape[0])
    for slot in (0, 1):
        v = partial[:, slot, :]
        assert torch.isfinite(v[named]).all(), f"slot {slot}: a row the layout names was not written"
        assert torch.isnan(v[~named]).all(), f"slot {slot}: an element outside the layout was written"
    z = torch.zeros((), dtype=torch.float64, device=DEV)
    s0 = torch.where(named, partial[:, 0, :].double(), z).sum(0)
    s1 = torch.where(named, partial[:, 1, :].double(), z).sum(0)
    return s0, s1


def chain_length(lay, m_tiles):
    """fp32 chain of one column sum: 16 staged rows, the tiles of the busiest CTA, 3 levels of the 8-slot combine."""
    rows, n_tiles, bn, group = lay
    ctas_per_ntile = rows // n_tiles            # the last n-tile has the fewest CTAs
    tiles_per_cta = -(-m_tiles // ctas_per_ntile)
    return 16 + tiles_per_cta + 3


def expected_rows(m_tiles, n_tiles):
    return max(min(m_tiles * n_tiles, num_sms()), n_tiles)


# ------------------------------------------------------------------------------------------------- a + b: statistics
def const_channel_input(shape, seed):
    """NHWC input whose channel 0 is held at 1, so that weights of one sign on it give output channels a large mean
    relative to their spread."""
    n, h, w, cin, cout, k, s, p = shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n, h, w, cin, generator=g, device=DEV)
    x[..., 0] = 1.0
    return x


def set_mean_ratios(wt, ratios):
    """Weights on input channel 0 (held at 1): output channel co gets an offset of ratio[co] x its spread (one sign
    per channel)."""
    cout, cin, kh, kw = wt.shape
    spread = wt[:, 1:].float().pow(2).sum(dim=(1, 2, 3)).sqrt()
    wt[:, 0] = (ratios * spread / (kh * kw))[:, None, None]
    return wt


def run_stats(shape, seed, stem=False):
    L = lib()
    n, h, w, cin, cout, k, s, p = shape
    ho, wo = out_hw(shape)
    g = torch.Generator(device=DEV).manual_seed(seed)
    wt = torch.randn(cout, cin, k, k, generator=g, device=DEV) / (cin * k * k) ** 0.5
    ratios = torch.tensor([0.0, 3.0, 10.0], device=DEV).repeat(cout // 3 + 1)[:cout]
    wt = set_mean_ratios(wt, ratios)
    st = L.stream_ptr()
    if stem:
        x = torch.randn(n, 3, h, w, generator=g, device=DEV)
        x[:, 0] = 1.0
        xin = torch.empty(n, h // 2, w // 2, 16, dtype=torch.bfloat16, device=DEV)
        L.call("dirb200_input_to_s2d", L.ptr(x), n, h, w, L.ptr(xin), st)
        wf = torch.empty(cout, 256, dtype=torch.bfloat16, device=DEV)
        L.call("dirb200_conv_prep_weights", L.ptr(wt), cout, 3, 7, 7, 1, L.ptr(wf), None, st)
    else:
        xin = const_channel_input(shape, seed).to(torch.bfloat16)
        wf = wt.permute(0, 2, 3, 1).contiguous().to(torch.bfloat16)
    nrows = max(num_sms(), cout // 64)
    partial = torch.full((nrows, 2, cout), float("nan"), dtype=torch.float32, device=DEV)
    y = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.bfloat16, device=DEV)
    lay = (ctypes.c_int * 4)()
    L.call("dirb200_conv_fprop_bn_stats", L.ptr(xin), L.ptr(wf), L.ptr(y), n, h, w, cin, cout, k, k, s, p,
           1 if stem else 0, L.ptr(partial), lay, st)
    torch.cuda.synchronize()
    lay = tuple(lay)
    pixels = n * ho * wo
    m_tiles = -(-pixels // 128)
    bn = plan_bn(shape, 0, 1 if stem else 0)
    assert lay == (expected_rows(m_tiles, cout // bn), cout // bn, bn, 1), lay
    return y.reshape(pixels, cout), partial, lay, m_tiles


def check_stats(y, partial, lay, m_tiles):
    c = y.shape[1]
    s0, s1 = reduce_rows(partial, lay, c)
    yd = y.double()
    ref0, ref1 = yd.sum(0), (yd * yd).sum(0)
    Lc = chain_length(lay, m_tiles)
    b0 = Lc * U * yd.abs().sum(0)
    b1 = Lc * U * (yd * yd).sum(0)
    e0, e1 = (s0 - ref0).abs(), (s1 - ref1).abs()
    assert (e0 <= b0).all(), f"sum y: worst channel err {(e0 - b0).max().item():.3e} over the bound (L = {Lc})"
    assert (e1 <= b1).all(), f"sum y^2: worst channel err {(e1 - b1).max().item():.3e} over the bound (L = {Lc})"
    return Lc


def check_finalize(y, partial, lay, Lc, tag):
    L = lib()
    rows, c = y.shape
    g = torch.Generator(device=DEV).manual_seed(c + rows)
    gamma = 1.0 + 0.5 * torch.randn(c, generator=g, device=DEV)
    beta = 0.5 * torch.randn(c, generator=g, device=DEV)
    rm0 = torch.randn(c, generator=g, device=DEV)
    rv0 = torch.rand(c, generator=g, device=DEV) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    outs = [torch.full((c,), float("nan"), device=DEV) for _ in range(4)]
    lay_host = (ctypes.c_int * 4)(*lay)
    eps, mom = 1e-5, 0.1
    L.call("dirb200_bn_finalize_layout", L.ptr(partial), lay_host, rows, c, L.ptr(gamma), L.ptr(beta), eps, mom,
           L.ptr(rm), L.ptr(rv), *[L.ptr(o) for o in outs], L.stream_ptr())
    torch.cuda.synchronize()
    mean, invstd, scale, shift = [o.double() for o in outs]
    yd = y.double()
    n = float(rows)
    m = yd.mean(0)
    var = ((yd - m) ** 2).mean(0)
    r_invstd = 1.0 / torch.sqrt(var + torch.tensor(eps, dtype=torch.float32).double())
    ga, be = gamma.double(), beta.double()
    # error of the kernel's sums (a) carried through m = S0 / n and var = S1 / n - m^2
    dm = Lc * U * yd.abs().sum(0) / n
    dvar = Lc * U * (yd * yd).sum(0) / n + 2 * m.abs() * dm + dm * dm
    slack = 1.0 + 1e-3
    # outputs are fp32: one more rounding each (scale and shift: their fp32 arithmetic, two / three roundings)
    b_mean = slack * (dm + U * m.abs()) + 1e-30
    rel_is = 0.5 * dvar / (var + eps)
    b_invstd = slack * r_invstd * (rel_is + U)
    r_scale = ga * r_invstd
    b_scale = slack * r_scale.abs() * (rel_is + 3 * U)
    r_shift = be - m * r_scale
    b_shift = slack * ((dm + U * m.abs()) * r_scale.abs() + m.abs() * b_scale + 2 * U * (m * r_scale).abs()
                       + U * r_shift.abs()) + 1e-30
    for name, got, ref, b in (("mean", mean, m, b_mean), ("invstd", invstd, r_invstd, b_invstd),
                              ("scale", scale, r_scale, b_scale), ("shift", shift, r_shift, b_shift)):
        e = (got - ref).abs()
        assert (e <= b).all(), f"{name}: worst excess {(e - b).max().item():.3e}"
    # running statistics: momentum and 1 - momentum as the fp32 values the kernel uses
    mo = float(torch.tensor(mom, dtype=torch.float32))
    om = float(torch.tensor(1.0, dtype=torch.float32) - torch.tensor(mom, dtype=torch.float32))
    r_rm = om * rm0.double() + mo * m
    unb = var * n / (n - 1)
    r_rv = om * rv0.double() + mo * unb
    b_rm = slack * (mo * dm + 4 * U * (om * rm0.double().abs() + mo * m.abs()))
    b_rv = slack * (mo * dvar * n / (n - 1) + 4 * U * (om * rv0.double().abs() + mo * unb.abs()))
    assert ((rm.double() - r_rm).abs() <= b_rm).all(), "running_mean"
    assert ((rv.double() - r_rv).abs() <= b_rv).all(), "running_var"
    # accuracy where the sum-of-squares form cancels: |mean| / std = 10
    ratio = m.abs() / var.sqrt()
    hi = ratio > 8
    if hi.any():
        worst = ((invstd - r_invstd).abs() / r_invstd)[hi].max().item()
        print(f"invstd {tag}: worst relative error {worst:.3e} over {int(hi.sum())} channels with |mean|/std > 8 "
              f"(max ratio {ratio.max().item():.1f})")


@pytest.mark.parametrize("shape", SHAPES + [BIG], ids=ids(SHAPES + [BIG]))
def test_fprop_bn_stats_and_finalize(shape):
    y, partial, lay, m_tiles = run_stats(shape, seed=sum(shape))
    Lc = check_stats(y, partial, lay, m_tiles)
    check_finalize(y, partial, lay, Lc, "x".join(map(str, shape)))


def test_stem_bn_stats_and_finalize():
    y, partial, lay, m_tiles = run_stats(STEM, seed=5, stem=True)
    Lc = check_stats(y, partial, lay, m_tiles)
    check_finalize(y, partial, lay, Lc, "stem")


# ------------------------------------------------------------------------------------------------- c: folded BN
# kappa: fp32 accumulation error of one output per unit of the abs-conv A = conv(|x|, |w|).  The K-long dot product is
# K / 16 wgmma k16 steps, each one fp32 rounding of the running accumulator (products exact), plus up to 16 roundings
# inside a step: |acc - exact| <= (K / 16 + 16) * 2^-24 * A.
def kappa(K):
    return (K / 16 + 16) * U


def f64_conv(x_nhwc, wt, stride, pad):
    return F.conv2d(x_nhwc.double().permute(0, 3, 1, 2), wt.double(), stride=stride, padding=pad).permute(0, 2, 3, 1)


def candidates(ref, err, post):
    """The range of bf16 results an fp32 value within `err` of `ref` can give after `post` (monotone, applied in
    fp32): every result lies in [lo, hi]; lo == hi where the whole interval rounds to one bf16 value."""
    lo = post((ref - err).float()).to(torch.bfloat16)
    hi = post((ref + err).float()).to(torch.bfloat16)
    return lo, hi


@pytest.mark.parametrize("shape", SHAPES, ids=ids(SHAPES))
def test_fprop_affine_epilogue(shape):
    L = lib()
    n, h, w, cin, cout, k, s, p = shape
    ho, wo = out_hw(shape)
    wt, wf, _ = make_weights(shape, seed=sum(shape) + 1)
    g = torch.Generator(device=DEV).manual_seed(sum(shape) + 2)
    x = torch.randn(n, h, w, cin, generator=g, device=DEV).to(torch.bfloat16)
    wq = wt.to(torch.bfloat16).float()
    ref = f64_conv(x, wq, s, p)
    A = f64_conv(x.abs(), wq.abs(), s, p)
    kap = kappa(k * k * cin)
    # negative and positive scales: the ReLU cuts channels in both directions
    sign = torch.where(torch.arange(cout, device=DEV) % 2 == 0, 1.0, -1.0)
    scale = sign * (0.5 + torch.rand(cout, generator=g, device=DEV))
    shift = 0.5 * torch.randn(cout, generator=g, device=DEV)
    res = torch.randn(n, ho, wo, cout, generator=g, device=DEV).to(torch.bfloat16)
    aff = ref * scale.double() + shift.double()
    # fp32 accumulator error through the fma, plus the fma's own rounding (doubled: margin for the interval ends)
    err = 2 * (scale.double().abs() * kap * A + U * aff.abs()) + 1e-30
    st = L.stream_ptr()
    forms = [("relu(conv*s+h)", None, 1), ("conv*s+h", None, 0), ("relu(q(conv*s+h)+res)", res, 1)]
    for name, r, relu in forms:
        out = torch.full((n, ho, wo, cout), float("nan"), dtype=torch.bfloat16, device=DEV)
        L.call("dirb200_conv_fprop_affine", L.ptr(x), L.ptr(wf), L.ptr(out), n, h, w, cin, cout, k, k, s, p,
               L.ptr(scale), L.ptr(shift), L.ptr(r), relu, st)
        torch.cuda.synchronize()
        if r is None:
            post = torch.relu if relu else (lambda t: t)
            lo, hi = candidates(aff, err, post)
        else:
            # the BN output is rounded to bf16 first (the staging tile), then the fp32 sum with the residual
            qlo, qhi = candidates(aff, err, lambda t: t)
            lo = torch.relu(qlo.float() + r.float()).to(torch.bfloat16)
            hi = torch.relu(qhi.float() + r.float()).to(torch.bfloat16)
        # every step is monotone in the fp32 accumulator, so the output lies between the results of the interval ends;
        # where those agree (most outputs) it must be exactly that bf16 value
        ok = (out >= lo) & (out <= hi)
        amb = (lo != hi).float().mean().item()
        print(f"affine {name} {shape}: {amb:.3f} of the outputs lie within the error bound of a rounding boundary")
        assert ok.all(), (f"{name}: {int((~ok).sum())} of {ok.numel()} outputs outside the bound "
                          f"(ambiguous fraction {amb:.2e}); first bad channel {int((~ok).nonzero()[0, -1])}")
        assert amb < 0.9, f"{name}: the error bound leaves almost every output ambiguous"


# ------------------------------------------------------------------------------------------------- d: dgrad moments
def moment_inputs(shape, seed):
    """y_prev [pixels][cin] with channel means at 0, 3 or 10 of their spread, power-of-two BN scales and shifts that
    put a tenth of each channel's elements exactly on the ReLU threshold y*scale + shift == 0."""
    n, h, w, cin, cout, k, s, p = shape
    g = torch.Generator(device=DEV).manual_seed(seed)
    rows = n * h * w
    ratios = torch.tensor([0.0, 3.0, 10.0], device=DEV).repeat(cin // 3 + 1)[:cin]
    y = (ratios + torch.randn(rows, cin, generator=g, device=DEV)).to(torch.bfloat16)
    # the threshold value of each channel: one of its own elements, planted at a tenth of the rows
    y0 = y[rows // 2].clone()
    tie = torch.rand(rows, cin, generator=g, device=DEV) < 0.1
    y = torch.where(tie, y0.expand(rows, cin), y)
    exp = torch.randint(-2, 3, (cin,), generator=g, device=DEV).float()
    sign = torch.where(torch.arange(cin, device=DEV) % 2 == 0, 1.0, -1.0)
    scale = sign * torch.exp2(exp)
    shift = -(y0.float() * scale)               # exact: y0 is bf16, scale a power of two
    return y, scale, shift, tie


@pytest.mark.parametrize("shape", MOMENT_SHAPES + [BIG], ids=ids(MOMENT_SHAPES + [BIG]))
def test_dgrad_bn_moments_and_coeffs(shape):
    L = lib()
    n, h, w, cin, cout, k, s, p = shape
    ho, wo = out_hw(shape)
    a = (ctypes.c_int * 7)()
    assert L.raw("dirb200_conv_plan")(n, h, w, cin, cout, k, k, s, p, 0, 1, a) == 0
    if a[6] == 0:
        pytest.skip("this dgrad form carries no BN moments under the current switches")
    wt, _, wd = make_weights(shape, seed=sum(shape) + 3)
    g = torch.Generator(device=DEV).manual_seed(sum(shape) + 4)
    dy = torch.randn(n, ho, wo, cout, generator=g, device=DEV).to(torch.bfloat16)
    y, scale, shift, tie = moment_inputs(shape, sum(shape) + 5)
    rows = n * h * w
    st = L.stream_ptr()
    dx_plain = torch.full((n, h, w, cin), float("nan"), dtype=torch.bfloat16, device=DEV)
    L.call("dirb200_conv_dgrad", L.ptr(dy), L.ptr(wd), L.ptr(dx_plain), n, h, w, cin, cout, k, k, s, p, st)
    dx = torch.full((n, h, w, cin), float("nan"), dtype=torch.bfloat16, device=DEV)
    nrows = max(num_sms(), cin // 64)
    partial = torch.full((nrows, 2, cin), float("nan"), dtype=torch.float32, device=DEV)
    lay = (ctypes.c_int * 4)()
    L.call("dirb200_conv_dgrad_bn_moments", L.ptr(dy), L.ptr(wd), L.ptr(dx), n, h, w, cin, cout, k, k, s, p,
           L.ptr(y), L.ptr(scale), L.ptr(shift), L.ptr(partial), lay, st)
    torch.cuda.synchronize()
    lay = tuple(lay)
    m_tiles = -(-rows // 128)
    bn = plan_bn(shape, 1)
    assert lay == (expected_rows(m_tiles, cin // bn), cin // bn, bn, 1), lay
    # the fused epilogue stores the same dx as the plain dgrad
    assert torch.equal(dx.view(torch.int16), dx_plain.view(torch.int16)), "dx differs from dirb200_conv_dgrad"
    s0, s1 = reduce_rows(partial, lay, cin)
    # float64 reference from the STORED dx; the mask is exactly the kernel's fmaf mask (y*scale is exact in float64,
    # adding shift cannot change the sign), ties (== 0) are masked out
    gd = dx.reshape(rows, cin).double()
    yd = y.double()
    mask = (yd * scale.double() + shift.double()) > 0
    assert (~mask[tie]).all()
    dz = torch.where(mask, gd, torch.zeros((), dtype=torch.float64, device=DEV))
    r0, r1 = dz.sum(0), (dz * yd).sum(0)
    Lc = chain_length(lay, m_tiles)
    d0 = Lc * U * dz.abs().sum(0)
    d1 = Lc * U * (dz * yd).abs().sum(0)
    e0, e1 = (s0 - r0).abs(), (s1 - r1).abs()
    tie_g = torch.where(tie, gd, torch.zeros((), dtype=torch.float64, device=DEV)).abs().sum(0)
    assert (e0 <= d0).all(), (f"S0 = sum dz: worst excess {(e0 - d0).max().item():.3e} "
                              f"(the planted ties carry sum |g| up to {tie_g.max().item():.3e})")
    assert (e1 <= d1).all(), f"S1 = sum dz*y: worst excess {(e1 - d1).max().item():.3e}"

    # bn_bwd_coeffs over those rows
    mean = yd.mean(0).float()
    invstd = (1.0 / torch.sqrt(yd.var(0, unbiased=False) + 1e-5)).float()
    gamma = 1.0 + 0.5 * torch.randn(cin, generator=g, device=DEV)
    gg0 = torch.randn(cin, generator=g, device=DEV)
    gb0 = torch.randn(cin, generator=g, device=DEV)
    gg, gb = gg0.clone(), gb0.clone()
    coef = torch.full((3, cin), float("nan"), device=DEV)
    L.call("dirb200_bn_bwd_coeffs_layout", L.ptr(partial), (ctypes.c_int * 4)(*lay), rows, cin, L.ptr(mean),
           L.ptr(invstd), L.ptr(gamma), L.ptr(gg), L.ptr(gb), L.ptr(coef), st)
    torch.cuda.synchronize()
    nn_, mu, is_, ga = float(rows), mean.double(), invstd.double(), gamma.double()
    dg = is_ * (r1 - mu * r0)
    ddg = is_ * (d1 + mu.abs() * d0)
    ref = [ga * is_, -ga * is_ * is_ * dg / nn_, ga * is_ * (mu * is_ * dg / nn_ - r0 / nn_)]
    bnd = [U * ref[0].abs(),
           ga.abs() * is_ * is_ * ddg / nn_ + U * ref[1].abs(),
           ga.abs() * is_ * (mu.abs() * is_ * ddg / nn_ + d0 / nn_) + U * ref[2].abs()]
    slack = 1.0 + 1e-3
    for i in range(3):
        e = (coef[i].double() - ref[i]).abs()
        b = slack * bnd[i] + 1e-30
        assert (e <= b).all(), f"coef row {i}: worst excess {(e - b).max().item():.3e}"
    r_gg, r_gb = gg0.double() + dg, gb0.double() + r0
    b_gg = slack * (ddg + U * dg.abs() + U * r_gg.abs()) + 1e-30
    b_gb = slack * (d0 + U * r0.abs() + U * r_gb.abs()) + 1e-30
    assert ((gg.double() - r_gg).abs() <= b_gg).all(), "grad_gamma"
    assert ((gb.double() - r_gb).abs() <= b_gb).all(), "grad_beta"


# ------------------------------------------------------------------------------------------------- few SMs
def test_epilogues_with_seven_sms():
    """This file again with the persistent grids capped at 7 CTAs (DIRB200_SMS is read once per process)."""
    if os.environ.get("DIRB200_SMS"):
        pytest.skip("already running under DIRB200_SMS")
    e = dict(os.environ)
    e["DIRB200_SMS"] = "7"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=e, cwd=ROOT, capture_output=True, text=True, timeout=1200)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
