"""The HBM-bound BatchNorm / pooling layer kernels of csrc/nn_kernels.cu, one launch at a time (the "Test aids: BatchNorm
/ pooling layer kernels" of include/dirb200.h), in every template form, against float64 references computed on the GPU;
and the standalone dirb200_bn_train_fwd / _bwd at the NYUD2 decoder's shapes.

  bn_apply (6 forms)         bit-exact: out = bf16(relu(fl32(y*s + h) [+ res] [+ fl32(ry*rs + rh)])), mask bits of the
                             stored out.  The operands are drawn so that float64 y*s + h is exact (product and shift
                             exponents within 20 of each other, or a zero term), so its fp32 rounding is the kernel's fmaf.
  bn_bwd_reduce (12 forms)   stored dz bit-exact; S0 = sum dz, S1 = sum dz*y, S2 = sum dz*y2 within L * u * sum |term|,
                             L = ceil(rows / (nblocks * lanes)) + lanes + 2 (the per-thread chain, then the serial combine
                             of the row lanes); every element of partial[nblocks][K][c] written, nothing beyond it.
  bn_bwd_coeffs              A, B, C, dgamma, dbeta against float64 from the same partial rows; accumulates.
  bn_bwd_apply (9 forms)     |dy - ref| <= 2^-8 |ref| + 2u (|A dz| + |B y| + |C|); stored dz bit-exact.
  bn_relu_maxpool_fwd        bit-exact values and first-maximum argmax, with planted ties.
  maxpool_bwd                |dx - ref| <= 2^-8 |ref| + 4u sum |terms|; pixels that are no window's argmax exactly 0.

u = 2^-24.  The whole file runs a second time with DIRB200_SMS=7 (few CTAs, long per-thread chains)."""
import ctypes
import math
import os
import subprocess
import sys

import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
BF = torch.bfloat16

# (rows, c, (h, w) of the maps the rows tile, for the compact-gradient forms; None: not even)
SHAPES = [
    (3, 8, None),                    # fewer rows than the 256 row lanes of c = 8
    (1, 2048, None),                 # one row, one lane
    (2 * 8 * 10, 2048, (8, 10)),     # NYUD2 layer4 map
    (8 * 15 * 19, 1024, None),       # NYUD2 layer3 map (odd)
    (4 * 29 * 38, 512, None),        # NYUD2 layer2 map
    (2 * 57 * 76, 256, None),        # NYUD2 layer1 map
    (2 * 120 * 160, 64, (120, 160)),
    (4 * 56 * 56, 256, (56, 56)),
    (12347, 16, None),               # prime row count: tails of every unrolled loop
    (4099, 128, None),
]
BIG = (256 * 56 * 56, 256, (56, 56))   # the batch-256 benchmark's largest block-output layers


def sid(s):
    return f"{s[0]}x{s[1]}" + (f"-{s[2][0]}x{s[2][1]}" if s[2] else "")


def lib():
    import _lib
    return _lib


def num_sms():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    cap = int(os.environ.get("DIRB200_SMS", "0") or 0)
    return cap if 0 < cap < sms else sms


def lanes(c):
    return 256 // (c // 8)


def chunks(rows, c):
    step = max(1, (1 << 23) // c)
    for r0 in range(0, rows, step):
        yield slice(r0, min(rows, r0 + step))


def bits(t):
    return t.view(torch.int16)


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def rand_bf16(shape, g, lo=2.0 ** -8, hi=6.0):
    """bf16 normal values, |x| in [lo, hi] or exactly 0 (keeps every product within the exact-fma exponent range)."""
    x = torch.randn(*shape, generator=g, device=DEV).clamp_(-hi, hi)
    x = torch.where(x.abs() < lo, torch.zeros((), device=DEV), x)
    return x.to(BF)


def rand_affine(c, g):
    """fp32 scale in +-[0.5, 1.5), shift in +-[2^-6, 1): with |y| in [2^-8, 6] the exponents of y*s and h differ by <= 20."""
    sgn = lambda: torch.where(torch.rand(c, generator=g, device=DEV) < 0.5, -1.0, 1.0)
    scale = sgn() * (0.5 + torch.rand(c, generator=g, device=DEV))
    shift = sgn() * (2.0 ** -6 + torch.rand(c, generator=g, device=DEV) * (1 - 2.0 ** -6))
    return scale, shift


def fma32(y, s, h):
    """fl32(y*s + h) as the kernel's fmaf forms it; asserts that float64 y*s + h is exact."""
    p = y.double() * s.double()
    hd = h.double().expand_as(p)
    _, ep = torch.frexp(p)
    _, eh = torch.frexp(hd)
    ok = (p == 0) | (hd == 0) | ((ep - eh).abs() <= 20)
    assert ok.all(), "operand draw: y*s + h is not exact in float64"
    return (p + hd).float()


def pack_mask(pos):
    """[rows, c] bool -> [rows, c/8] uint8, bit j = channel 8g + j."""
    rows, c = pos.shape
    w = (1 << torch.arange(8, device=DEV, dtype=torch.int32))
    return (pos.view(rows, c // 8, 8).int() * w).sum(-1).to(torch.uint8)


def unpack_mask(m, c):
    rows = m.shape[0]
    sh = torch.arange(8, device=DEV, dtype=torch.int32)
    return ((m.int()[:, :, None] >> sh) & 1).bool().reshape(rows, c)


# ------------------------------------------------------------------------------------------------------------ bn_apply
APPLY_FORMS = [(res, resy, mask) for res, resy in ((0, 0), (1, 0), (0, 1)) for mask in (0, 1)]


def run_bn_apply(shape, forms, seed):
    L = lib()
    rows, c, _ = shape
    g = gen(seed)
    y = rand_bf16((rows, c), g)
    r = rand_bf16((rows, c), g)
    sc, sh = rand_affine(c, g)
    rs, rh = rand_affine(c, g)
    st = L.stream_ptr()
    for res, resy, want_mask in forms:
        for relu in ((1,) if (res or resy or want_mask) else (0, 1)):
            ref = torch.empty(rows, c, dtype=BF, device=DEV)
            for q in chunks(rows, c):
                a = fma32(y[q], sc, sh)
                if res:
                    a = a + r[q].float()
                if resy:
                    a = a + fma32(r[q], rs, rh)
                ref[q] = (torch.relu(a) if relu else a).to(BF)
            ref_mask = pack_mask(ref.float() > 0)
            if want_mask:
                # each of the four channel pairs of a mask byte appears with only its even and with only its odd
                # channel positive
                pos = (ref.float() > 0).view(rows * (c // 8), 4, 2)
                if rows * c >= 1024:
                    assert (pos[..., 0] & ~pos[..., 1]).any(0).all() and (~pos[..., 0] & pos[..., 1]).any(0).all()
            out = torch.full((rows, c), float("nan"), dtype=BF, device=DEV)
            mask = ~ref_mask if want_mask else None        # a byte the kernel does not write cannot match
            L.call("dirb200_layer_bn_apply", L.ptr(y), L.ptr(sc), L.ptr(sh), L.ptr(r if res else None),
                   L.ptr(r if resy else None), L.ptr(rs if resy else None), L.ptr(rh if resy else None), relu, rows, c,
                   L.ptr(out), L.ptr(mask), st)
            torch.cuda.synchronize()
            tag = f"res={res} res_y={resy} mask={want_mask} relu={relu}"
            bad = bits(out) != bits(ref)
            assert not bad.any(), f"{tag}: {int(bad.sum())} outputs differ, first at {bad.nonzero()[0].tolist()}"
            if want_mask:
                bad = mask != ref_mask
                assert not bad.any(), f"{tag}: {int(bad.sum())} mask bytes differ, first at {bad.nonzero()[0].tolist()}"


@pytest.mark.parametrize("shape", SHAPES, ids=[sid(s) for s in SHAPES])
def test_bn_apply_forms_bit_exact(shape):
    run_bn_apply(shape, APPLY_FORMS, seed=shape[0] + shape[1])


def test_bn_apply_block_output_forms_benchmark_size():
    run_bn_apply(BIG, [(1, 0, 1), (0, 1, 1)], seed=11)


# ------------------------------------------------------------------------------------------------------- BN backward
# (mode, g2, y2, write_dz, g3): mode 'y' = mask from fma(y, scale, shift), 'bits' = stored mask, 'none' = no mask
REDUCE_FORMS = [
    ("y", None, 0, 0, 0), ("none", None, 0, 0, 0),
    ("bits", None, 0, 0, 0), ("bits", None, 1, 0, 0), ("bits", None, 0, 1, 0),
    ("bits", "dense", 0, 0, 0), ("bits", "dense", 1, 0, 0), ("bits", "dense", 0, 1, 0),
    ("bits", "compact", 0, 0, 0), ("bits", "compact", 0, 1, 0),
    ("bits", "dense", 0, 1, 1), ("bits", "compact", 0, 1, 1),
]
APPLY_BWD_FORMS = [
    ("none", None, 0, 0), ("y", None, 0, 0),
    ("bits", None, 0, 0), ("bits", None, 1, 0), ("bits", None, 0, 1),
    ("bits", "dense", 0, 0), ("bits", "dense", 1, 0), ("bits", "dense", 0, 1),
    ("bits", "compact", 0, 1),
]


def fname(f):
    mode, g2m, y2, dz = f[:4]
    s = f"mask={mode}" + (f" g2={g2m}" if g2m else "") + (" y2" if y2 else "") + (" dz" if dz else "")
    return s + (" g3" if len(f) > 4 and f[4] else "")


def bwd_inputs(shape, seed):
    """Every operand a BN-backward form can take.  The mask-from-y coefficients are powers of two with a shift that puts
    a tenth of each channel's elements exactly on the threshold y*s + h == 0."""
    rows, c, hw = shape
    g = gen(seed)
    t = dict(g1=rand_bf16((rows, c), g), g2=rand_bf16((rows, c), g), g3=rand_bf16((rows, c), g),
             y=rand_bf16((rows, c), g), y2=rand_bf16((rows, c), g))
    y0 = t["y"][rows // 2].clone()
    tie = torch.rand(rows, c, generator=g, device=DEV) < 0.1
    t["y"] = torch.where(tie, y0.expand(rows, c), t["y"])
    sign = torch.where(torch.arange(c, device=DEV) % 2 == 0, 1.0, -1.0)
    t["scale"] = sign * torch.exp2(torch.randint(-2, 3, (c,), generator=g, device=DEV).float())
    t["shift"] = -(y0.float() * t["scale"])
    t["mask"] = torch.randint(0, 256, (rows, c // 8), generator=g, device=DEV, dtype=torch.int32).to(torch.uint8)
    if hw:
        h, w = hw
        n = rows // (h * w)
        t["g2c"] = rand_bf16((n * (h // 2) * (w // 2), c), g)
        e = torch.zeros(n, h, w, c, dtype=BF, device=DEV)
        e[:, ::2, ::2] = t["g2c"].view(n, h // 2, w // 2, c)
        t["g2e"] = e.view(rows, c)      # the compact gradient at the even pixels, zero elsewhere
    return t


def dz_ref(t, q, mode, g2m, g3, c):
    """fp32 dz of rows q: mask * (g1 [+ g2] [+ g3]), added in the kernel's order."""
    g = t["g1"][q].float()
    if g2m:
        g = g + t["g2e" if g2m == "compact" else "g2"][q].float()
    if g3:
        g = g + t["g3"][q].float()
    if mode == "y":
        keep = (t["y"][q].double() * t["scale"].double() + t["shift"].double()) > 0
    elif mode == "bits":
        keep = unpack_mask(t["mask"][q], c)
    else:
        return g
    return torch.where(keep, g, torch.zeros((), device=DEV))


def reduce_args(t, form, shape, dz_out, partial, nblk):
    L = lib()
    rows, c, hw = shape
    mode, g2m, y2, _, g3 = form
    g2 = t["g2c"] if g2m == "compact" else (t["g2"] if g2m else None)
    h2, w2 = hw if g2m == "compact" else (0, 0)
    return (L.ptr(t["g1"]), L.ptr(g2), L.ptr(t["g3"] if g3 else None), L.ptr(t["y"]), L.ptr(t["y2"] if y2 else None),
            L.ptr(t["scale"] if mode == "y" else None), L.ptr(t["shift"] if mode == "y" else None),
            L.ptr(t["mask"] if mode == "bits" else None), rows, c, h2, w2, L.ptr(dz_out), L.ptr(partial),
            ctypes.byref(nblk), L.stream_ptr())


def run_reduce(t, form, shape):
    """One bn_bwd_reduce launch; returns the partial rows (checked for coverage), nblocks and the float64 sums / bounds."""
    L = lib()
    rows, c, _ = shape
    mode, g2m, y2, wdz, g3 = form
    K = 3 if y2 else 2
    cap = 4 * num_sms()
    partial = torch.full((cap + 2, K, c), float("nan"), device=DEV)
    dz = torch.full((rows, c), float("nan"), dtype=BF, device=DEV) if wdz else None
    nblk = ctypes.c_int(-1)
    L.call("dirb200_layer_bn_bwd_reduce", *reduce_args(t, form, shape, dz, partial, nblk))
    torch.cuda.synchronize()
    nb = nblk.value
    assert 1 <= nb <= cap, nb
    assert torch.isfinite(partial[:nb]).all(), "a partial row element was not written"
    assert torch.isnan(partial[nb:]).all(), "an element beyond partial[nblocks][K][c] was written"
    s = torch.zeros(K, c, dtype=F64, device=DEV)
    a = torch.zeros(K, c, dtype=F64, device=DEV)
    for q in chunks(rows, c):
        d = dz_ref(t, q, mode, g2m, g3, c)
        if wdz:
            db = d.to(BF)
            bad = bits(dz[q]) != bits(db)
            assert not bad.any(), f"{fname(form)}: {int(bad.sum())} stored dz differ, first at {bad.nonzero()[0].tolist()}"
            d = db.float()
        d = d.double()
        terms = [d, d * t["y"][q].double()] + ([d * t["y2"][q].double()] if y2 else [])
        for k, x in enumerate(terms):
            s[k] += x.sum(0)
            a[k] += x.abs().sum(0)
    Lc = -(-rows // (nb * lanes(c))) + lanes(c) + 2
    got = partial[:nb].double().sum(0)
    err = (got - s).abs()
    bound = Lc * U * a
    for k in range(K):
        assert (err[k] <= bound[k]).all(), (f"{fname(form)}: slot {k} worst excess {(err[k] - bound[k]).max().item():.3e} "
                                            f"(L = {Lc}, nblocks = {nb})")
    return partial, nb, s, a, Lc


def check_coeffs(partial, nb, K, gslot, rows, c, s, a, Lc, seed):
    """bn_bwd_coeffs over the rows of a reduce launch, against float64 from the same rows."""
    L = lib()
    g = gen(seed)
    mean = torch.randn(c, generator=g, device=DEV)
    invstd = 0.5 + torch.rand(c, generator=g, device=DEV)
    gamma = 1.0 + 0.5 * torch.randn(c, generator=g, device=DEV)
    gg0 = torch.randn(c, generator=g, device=DEV)
    gb0 = torch.randn(c, generator=g, device=DEV)
    gg, gb = gg0.clone(), gb0.clone()
    coef = torch.full((3, c), float("nan"), device=DEV)
    L.call("dirb200_layer_bn_bwd_coeffs", L.ptr(partial), nb, K, gslot, rows, c, L.ptr(mean), L.ptr(invstd),
           L.ptr(gamma), L.ptr(gg), L.ptr(gb), L.ptr(coef), L.stream_ptr())
    torch.cuda.synchronize()
    p = partial[:nb].double()
    db, s1 = p[:, 0].sum(0), p[:, gslot].sum(0)
    # float64 re-association of the partial sums, relative to the magnitudes involved
    ad, a1 = p[:, 0].abs().sum(0), p[:, gslot].abs().sum(0)
    n, mu, is_, ga = float(rows), mean.double(), invstd.double(), gamma.double()
    dg = is_ * (s1 - mu * db)
    mdg = is_ * (a1 + mu.abs() * ad)
    ref = [ga * is_, -ga * is_ * is_ * dg / n, ga * is_ * (mu * is_ * dg / n - db / n)]
    mag = [ga.abs() * is_, ga.abs() * is_ ** 2 * mdg / n, ga.abs() * is_ * (mu.abs() * is_ * mdg / n + ad / n)]
    for i in range(3):
        e = (coef[i].double() - ref[i]).abs()
        b = 1.001 * U * ref[i].abs() + 2.0 ** -40 * mag[i] + 1e-30
        assert (e <= b).all(), f"K={K} gslot={gslot}: coef row {i} worst excess {(e - b).max().item():.3e}"
    for name, got, g0, d, m in (("grad_gamma", gg, gg0, dg, mdg), ("grad_beta", gb, gb0, db, ad)):
        r = g0.double() + d
        b = 1.001 * U * (d.abs() + r.abs()) + 2.0 ** -40 * m + 1e-30
        e = (got.double() - r).abs()
        assert (e <= b).all(), f"K={K} gslot={gslot}: {name} worst excess {(e - b).max().item():.3e} (accumulated?)"
    # the reduce kernel's own sums agree with float64 to the chain bound; the coefficients' dgamma then does too
    assert ((db - s[0]).abs() <= Lc * U * a[0]).all()


@pytest.mark.parametrize("shape", SHAPES, ids=[sid(s) for s in SHAPES])
def test_bn_bwd_reduce_forms_and_coeffs(shape):
    rows, c, hw = shape
    t = bwd_inputs(shape, seed=rows + 3 * c)
    for form in REDUCE_FORMS:
        if form[1] == "compact" and not hw:
            continue
        partial, nb, s, a, Lc = run_reduce(t, form, shape)
        if form == ("bits", "dense", 1, 0, 0):          # downsample block: both BNs' coefficients from one reduce
            for gslot in (1, 2):
                check_coeffs(partial, nb, 3, gslot, rows, c, s, a, Lc, seed=rows + gslot)
        if form == ("bits", None, 0, 1, 0):
            check_coeffs(partial, nb, 2, 1, rows, c, s, a, Lc, seed=rows + 7)


def test_bn_bwd_reduce_block_output_forms_benchmark_size():
    t = bwd_inputs(BIG, seed=12)
    for form in (("bits", "compact", 0, 1, 0), ("bits", "dense", 1, 0, 0), ("bits", "compact", 0, 1, 1)):
        run_reduce(t, form, BIG)


def run_bwd_apply(t, form, shape, seed):
    L = lib()
    rows, c, hw = shape
    mode, g2m, y2, wdz = form
    g = gen(seed)
    coef = torch.stack([0.5 + torch.rand(c, generator=g, device=DEV), 0.1 * torch.randn(c, generator=g, device=DEV),
                        0.1 * torch.randn(c, generator=g, device=DEV)])
    coef2 = torch.stack([0.5 + torch.rand(c, generator=g, device=DEV), 0.1 * torch.randn(c, generator=g, device=DEV),
                         0.1 * torch.randn(c, generator=g, device=DEV)])
    nan = lambda: torch.full((rows, c), float("nan"), dtype=BF, device=DEV)
    dy, dy2, dz = nan(), (nan() if y2 else None), (nan() if wdz else None)
    g2 = t["g2c"] if g2m == "compact" else (t["g2"] if g2m else None)
    h2, w2 = hw if g2m == "compact" else (0, 0)
    L.call("dirb200_layer_bn_bwd_apply", L.ptr(t["g1"]), L.ptr(g2), L.ptr(t["y"]), L.ptr(coef),
           L.ptr(t["y2"] if y2 else None), L.ptr(coef2 if y2 else None),
           L.ptr(t["scale"] if mode == "y" else None), L.ptr(t["shift"] if mode == "y" else None),
           L.ptr(t["mask"] if mode == "bits" else None), rows, c, h2, w2, L.ptr(dy), L.ptr(dy2), L.ptr(dz),
           L.stream_ptr())
    torch.cuda.synchronize()
    for q in chunks(rows, c):
        d = dz_ref(t, q, mode, g2m, False, c)
        if wdz:
            bad = bits(dz[q]) != bits(d.to(BF))
            assert not bad.any(), f"{fname(form)}: {int(bad.sum())} stored dz differ, first at {bad.nonzero()[0].tolist()}"
        d = d.double()
        for name, out, cf, yy in (("dy", dy, coef, t["y"]), ("dy2", dy2, coef2, t["y2"])):
            if out is None:
                continue
            A, B, C = cf.double()
            ad, by = A * d, B * yy[q].double()
            ref = ad + by + C
            bound = 2.0 ** -8 * ref.abs() + 2 * U * (ad.abs() + by.abs() + C.abs())
            e = (out[q].double() - ref).abs()
            ok = e <= bound                  # NaN (never written) fails
            assert ok.all(), (f"{fname(form)}: {name} {int((~ok).sum())} elements outside the bound, first at row "
                              f"{q.start + int((~ok).nonzero()[0, 0])}")


@pytest.mark.parametrize("shape", SHAPES, ids=[sid(s) for s in SHAPES])
def test_bn_bwd_apply_forms(shape):
    rows, c, hw = shape
    t = bwd_inputs(shape, seed=rows + 5 * c)
    for i, form in enumerate(APPLY_BWD_FORMS):
        if form[1] == "compact" and not hw:
            continue
        run_bwd_apply(t, form, shape, seed=rows + i)


def test_bn_bwd_apply_block_output_forms_benchmark_size():
    t = bwd_inputs(BIG, seed=13)
    for i, form in enumerate((("bits", "dense", 1, 0), ("none", None, 0, 0), ("bits", "compact", 0, 1))):
        run_bwd_apply(t, form, BIG, seed=i)


# ------------------------------------------------------------------------------------------------------------- pooling
POOL_SHAPES = [(2, 114, 152, 64), (3, 18, 22, 64), (2, 15, 19, 16), (1, 2, 2, 8), (5, 6, 4, 128)]
BIG_STEM = (256, 112, 112, 64)


def pool_inputs(shape, seed):
    """Stem pre-activations with planted ties: channel 4k + 0 is driven below zero everywhere (every window ties at 0,
    so the first valid position must win), channel 4k + 1 holds coarse values (duplicated bf16 maxima)."""
    n, h, w, c = shape
    g = gen(seed)
    y = rand_bf16((n, h, w, c), g)
    cls = torch.arange(c, device=DEV) % 4
    coarse = (torch.randn(n, h, w, c, generator=g, device=DEV) * 2).round() / 2
    y = torch.where(cls == 1, coarse.clamp(-4, 4).to(BF), y)
    sc, sh = rand_affine(c, g)
    sc = torch.where(cls == 0, sc.abs(), torch.where(cls == 1, torch.ones((), device=DEV), sc))
    sh = torch.where(cls == 0, torch.full((), -64.0, device=DEV), torch.where(cls == 1, torch.zeros((), device=DEV), sh))
    return y, sc, sh


def pool_ref(act):
    """3x3 / stride 2 / pad 1 max pool of act [n, h, w, c] (float): values and r*3 + s of the FIRST maximum."""
    n, h, w, c = act.shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    p = torch.full((n, h + 3, w + 3, c), float("-inf"), device=DEV)
    p[:, 1:h + 1, 1:w + 1] = act
    win = torch.stack([p[:, r:r + 2 * ho:2, s:s + 2 * wo:2] for r in range(3) for s in range(3)], -1)
    val, idx = win.max(-1, keepdim=True)
    first = (win == val).int().argmax(-1)            # argmax of a 0/1 tensor returns the first 1
    return val[..., 0], first


def run_pool_fwd(shape, seed, img_chunk=16):
    L = lib()
    n, h, w, c = shape
    ho, wo = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    y, sc, sh = pool_inputs(shape, seed)
    out = torch.full((n, ho, wo, c), float("nan"), dtype=BF, device=DEV)
    idx = torch.full((n, ho, wo, c), 255, dtype=torch.uint8, device=DEV)
    L.call("dirb200_layer_bn_relu_maxpool_fwd", L.ptr(y), L.ptr(sc), L.ptr(sh), n, h, w, c, L.ptr(out), L.ptr(idx),
           L.stream_ptr())
    torch.cuda.synchronize()
    for b0 in range(0, n, img_chunk):
        b = slice(b0, min(n, b0 + img_chunk))
        act = torch.relu(fma32(y[b].reshape(-1, c), sc, sh)).to(BF).float().view(-1, h, w, c)
        val, first = pool_ref(act)
        bad = bits(out[b]) != bits(val.to(BF))
        assert not bad.any(), f"pool values: {int(bad.sum())} differ, first at {bad.nonzero()[0].tolist()}"
        bad = idx[b].long() != first
        assert not bad.any(), (f"pool argmax: {int(bad.sum())} differ, first at {bad.nonzero()[0].tolist()} "
                               f"(channel class {int(bad.nonzero()[0, -1]) % 4})")
    # the planted ties are there: channel 0 of the corner window ties everywhere, first valid position (1, 1) wins
    assert int(idx[0, 0, 0, 0]) == 4
    return idx


def check_pool_bwd(shape, idx, seed, with_g2, img_chunk=16):
    L = lib()
    n, h, w, c = shape
    ho, wo = idx.shape[1], idx.shape[2]
    g = gen(seed)
    g1 = rand_bf16((n, ho, wo, c), g)
    g2 = rand_bf16((n, ho, wo, c), g) if with_g2 else None
    dx = torch.full((n, h, w, c), float("nan"), dtype=BF, device=DEV)
    L.call("dirb200_layer_maxpool_bwd", L.ptr(g1), L.ptr(g2), L.ptr(idx), n, h, w, c, L.ptr(dx), L.stream_ptr())
    torch.cuda.synchronize()
    yo = torch.arange(ho, device=DEV).view(1, ho, 1, 1)
    xo = torch.arange(wo, device=DEV).view(1, 1, wo, 1)
    ch = torch.arange(c, device=DEV).view(1, 1, 1, c)
    multi = 0
    for b0 in range(0, n, img_chunk):
        b = slice(b0, min(n, b0 + img_chunk))
        nb = b.stop - b.start
        k = idx[b].long()
        iy, ix = 2 * yo - 1 + k // 3, 2 * xo - 1 + k % 3
        assert ((iy >= 0) & (iy < h) & (ix >= 0) & (ix < w)).all()
        im = torch.arange(nb, device=DEV).view(nb, 1, 1, 1)
        flat = (((im * h + iy) * w + ix) * c + ch).reshape(-1)
        gv = g1[b].double() + (g2[b].double() if with_g2 else 0.0)
        ga = g1[b].double().abs() + (g2[b].double().abs() if with_g2 else 0.0)
        size = nb * h * w * c
        ref = torch.zeros(size, dtype=F64, device=DEV).index_add_(0, flat, gv.reshape(-1))
        mag = torch.zeros(size, dtype=F64, device=DEV).index_add_(0, flat, ga.reshape(-1))
        cnt = torch.zeros(size, dtype=torch.int32, device=DEV).index_add_(0, flat, torch.ones_like(flat, dtype=torch.int32))
        got = dx[b].reshape(-1)
        zero = cnt == 0
        assert (bits(got)[zero] == 0).all(), "a pixel that is no window's argmax is not exactly 0"
        e = (got.double() - ref).abs()
        ok = e <= 2.0 ** -8 * ref.abs() + 4 * U * mag
        assert ok.all(), f"maxpool_bwd (g2={with_g2}): {int((~ok).sum())} pixels outside the bound"
        multi += int((cnt > 1).sum())
    if ho * wo >= 4:
        assert multi > 0, "no pixel is the argmax of several windows"


@pytest.mark.parametrize("shape", POOL_SHAPES, ids=["x".join(map(str, s)) for s in POOL_SHAPES])
def test_bn_relu_maxpool_fwd_and_maxpool_bwd(shape):
    idx = run_pool_fwd(shape, seed=sum(shape))
    n, h, w, c = shape
    if h % 2 == 0 and w % 2 == 0:
        for with_g2 in (False, True):
            check_pool_bwd(shape, idx, seed=sum(shape) + with_g2, with_g2=with_g2)


def test_stem_pool_benchmark_size():
    idx = run_pool_fwd(BIG_STEM, seed=21)
    check_pool_bwd(BIG_STEM, idx, seed=22, with_g2=True)


# -------------------------------------------------------------------------------------- standalone BN entry points
# NYUD2 decoder BatchNorms at batch 8 (228x304 input): MFF branches (16) and output (64), R (128) at 114x152; the D
# module (1024 at 8x10) and its up-projections (512 / 256 at 15x19 / 29x38); c = 8 on few rows.
STANDALONE = [(8 * 114 * 152, 16), (8 * 114 * 152, 64), (8 * 114 * 152, 128), (8 * 8 * 10, 1024), (8 * 15 * 19, 512),
              (8 * 29 * 38, 256), (2 * 7 * 9, 8)]


def stats_nblocks(y, rows, c):
    """The CTA count of the statistics launch the forward makes (the aid runs the same dispatch)."""
    L = lib()
    part = torch.empty(4 * num_sms() + 2, 2, c, device=DEV)
    nb = ctypes.c_int(-1)
    L.call("dirb200_layer_bn_stats", L.ptr(y), rows, c, L.ptr(part), ctypes.byref(nb), L.stream_ptr())
    return nb.value


@pytest.mark.parametrize("relu", (1, 0))
@pytest.mark.parametrize("rows,c", STANDALONE, ids=[f"{r}x{c}" for r, c in STANDALONE])
def test_bn_train_fwd_bwd_standalone(rows, c, relu):
    L = lib()
    g = gen(rows + c + relu)
    ratios = torch.tensor([0.0, 3.0, 10.0], device=DEV).repeat(c // 3 + 1)[:c]
    spread = torch.exp2(torch.randint(-3, 3, (c,), generator=g, device=DEV).float())
    y = ((ratios + torch.randn(rows, c, generator=g, device=DEV)) * spread).to(BF)
    gamma = 1.0 + 0.5 * torch.randn(c, generator=g, device=DEV)
    beta = 0.5 * torch.randn(c, generator=g, device=DEV)
    rm0, rv0 = torch.randn(c, generator=g, device=DEV), torch.rand(c, generator=g, device=DEV) + 0.5
    rm, rv = rm0.clone(), rv0.clone()
    eps, mom = 1e-5, 0.1
    ws = torch.empty(L.raw("dirb200_bn_workspace_bytes")(c), dtype=torch.uint8, device=DEV)
    out = torch.full((rows, c), float("nan"), dtype=BF, device=DEV)
    smean, sinv = torch.full((c,), float("nan"), device=DEV), torch.full((c,), float("nan"), device=DEV)
    ss = torch.full((2, c), float("nan"), device=DEV)
    st = L.stream_ptr()
    L.call("dirb200_bn_train_fwd", L.ptr(y), rows, c, L.ptr(gamma), L.ptr(beta), eps, mom, L.ptr(rm), L.ptr(rv), relu,
           L.ptr(out), L.ptr(smean), L.ptr(sinv), L.ptr(ss), L.ptr(ws), st)
    nb = stats_nblocks(y, rows, c)
    torch.cuda.synchronize()
    n = float(rows)
    yd = y.double()
    m = yd.mean(0)
    var = ((yd - m) ** 2).mean(0)
    e32 = float(torch.tensor(eps, dtype=torch.float32))
    r_is = 1.0 / torch.sqrt(var + e32)
    Lc = -(-rows // (nb * lanes(c))) + lanes(c) + 2
    slack = 1.001
    dm = Lc * U * yd.abs().sum(0) / n
    dvar = Lc * U * (yd * yd).sum(0) / n + 2 * m.abs() * dm + dm * dm
    b_mean = slack * (dm + U * m.abs()) + 1e-30
    b_is = slack * r_is * (0.5 * dvar / (var + e32) + U)
    assert ((smean.double() - m).abs() <= b_mean).all(), "save_mean"
    assert ((sinv.double() - r_is).abs() <= b_is).all(), "save_invstd"
    ratio = m.abs() / var.sqrt()
    hi = ratio > 8
    worst = ((sinv.double() - r_is).abs() / r_is)[hi].max().item() if hi.any() else float("nan")
    print(f"bn_train_fwd {rows}x{c}: worst relative invstd error {worst:.3e} over {int(hi.sum())} channels with "
          f"|mean|/std > 8 (bound {(b_is / r_is)[hi].max().item() if hi.any() else 0:.1e})")
    # running statistics: 1e-6 relative plus what the sums' error carries into them
    mo, om = float(torch.tensor(mom, dtype=torch.float32)), float(1 - torch.tensor(mom, dtype=torch.float32))
    r_rm, r_rv = om * rm0.double() + mo * m, om * rv0.double() + mo * var * n / max(n - 1, 1)
    assert ((rm.double() - r_rm).abs() <= 1e-6 * r_rm.abs() + mo * dm).all(), "running_mean"
    assert ((rv.double() - r_rv).abs() <= 1e-6 * r_rv.abs() + mo * dvar * n / max(n - 1, 1)).all(), "running_var"
    # output: bf16 rounding of the float64 BatchNorm plus the error of scale / shift (carried from invstd and the mean)
    ga, be = gamma.double(), beta.double()
    r_sc = ga * r_is
    b_sc = slack * (ga.abs() * b_is + U * r_sc.abs())
    r_sh = be - m * r_sc
    b_sh = slack * (r_sc.abs() * b_mean + m.abs() * b_sc + 2 * U * ((m * r_sc).abs() + r_sh.abs()))
    for q in chunks(rows, c):
        pre = yd[q] * r_sc + r_sh
        ref = torch.relu(pre) if relu else pre
        e_aff = yd[q].abs() * b_sc + b_sh + U * ((yd[q] * r_sc).abs() + r_sh.abs())
        e = (out[q].double() - ref).abs()
        ok = e <= 2.0 ** -8 * ref.abs() + (1 + 2.0 ** -8) * e_aff
        assert ok.all(), f"bn_train_fwd out: {int((~ok).sum())} elements outside the bound"

    # ---- backward, from the forward's saved statistics and scale / shift
    go = rand_bf16((rows, c), g)
    gg0, gb0 = torch.randn(c, generator=g, device=DEV), torch.randn(c, generator=g, device=DEV)
    gg, gb = gg0.clone(), gb0.clone()
    dx = torch.full((rows, c), float("nan"), dtype=BF, device=DEV)
    L.call("dirb200_bn_train_bwd", L.ptr(go), L.ptr(y), rows, c, L.ptr(gamma), L.ptr(smean), L.ptr(sinv), L.ptr(ss),
           relu, L.ptr(gg), L.ptr(gb), L.ptr(dx), L.ptr(ws), st)
    # the reduction's CTA count (same dispatch as the entry point's)
    part = torch.empty(4 * num_sms() + 2, 2, c, device=DEV)
    nbk = ctypes.c_int(-1)
    L.call("dirb200_layer_bn_bwd_reduce", L.ptr(go), None, None, L.ptr(y), None, L.ptr(ss[0] if relu else None),
           L.ptr(ss[1] if relu else None), None, rows, c, 0, 0, None, L.ptr(part), ctypes.byref(nbk), st)
    torch.cuda.synchronize()
    sc, sh = ss[0].double(), ss[1].double()
    keep = (yd * sc + sh > 0) if relu else torch.ones_like(yd, dtype=torch.bool)
    dz = torch.where(keep, go.double(), torch.zeros((), dtype=F64, device=DEV))
    S0, S1 = dz.sum(0), (dz * yd).sum(0)
    Lb = -(-rows // (nbk.value * lanes(c))) + lanes(c) + 2
    d0, d1 = Lb * U * dz.abs().sum(0), Lb * U * (dz * yd).abs().sum(0)
    mu, is_ = smean.double(), sinv.double()
    dg = is_ * (S1 - mu * S0)
    ddg = is_ * (d1 + mu.abs() * d0)
    A, B, C = ga * is_, -ga * is_ * is_ * dg / n, ga * is_ * (mu * is_ * dg / n - S0 / n)
    bA = U * A.abs()
    bB = ga.abs() * is_ * is_ * ddg / n + U * B.abs()
    bC = ga.abs() * is_ * (mu.abs() * is_ * ddg / n + d0 / n) + U * C.abs()
    r_gg, r_gb = gg0.double() + dg, gb0.double() + S0
    assert ((gg.double() - r_gg).abs() <= slack * (ddg + U * dg.abs() + U * r_gg.abs()) + 1e-30).all(), "grad_gamma"
    assert ((gb.double() - r_gb).abs() <= slack * (d0 + U * S0.abs() + U * r_gb.abs()) + 1e-30).all(), "grad_beta"
    for q in chunks(rows, c):
        ad, by = A * dz[q], B * yd[q]
        ref = ad + by + C
        bound = 2.0 ** -8 * ref.abs() + slack * (2 * U * (ad.abs() + by.abs() + C.abs()) + bA * dz[q].abs()
                                                 + bB * yd[q].abs() + bC)
        ok = (dx[q].double() - ref).abs() <= bound
        assert ok.all(), f"bn_train_bwd dx: {int((~ok).sum())} elements outside the bound"


# ------------------------------------------------------------------------------------------------------------ few SMs
def test_layer_kernels_with_seven_sms():
    """This file again with the grids capped at 7 SMs (DIRB200_SMS is read once per process): few CTAs, so long
    per-thread row chains and few partial rows."""
    if os.environ.get("DIRB200_SMS"):
        pytest.skip("already running under DIRB200_SMS")
    e = dict(os.environ)
    e["DIRB200_SMS"] = "7"
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
