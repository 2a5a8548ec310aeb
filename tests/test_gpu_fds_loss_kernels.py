"""The FDS kernels of csrc/fds.cu and the loss / LDS kernels of csrc/loss_lds.cu, one launch at a time through the C ABI,
against float64 references computed on the GPU or against restatements of the kernels' own fp32 / fp64 operation order.
Outputs are prefilled with NaN (float) or a sentinel (int), so every element must be written and every element a call
must leave alone keeps its bits.  u = 2^-24 (fp32), U64 = 2^-53 (fp64).

  label_flags / bin_rows  bit-exact against bin_index (age: int(fp32(v - lo)) with out-of-range labels folded into an
                          edge bin only when its flag is set; depth: clamp(int(fp32(v * 10))); EDGES5: the first float32
                          edge above the label).  The depth and EDGES5 rules are pinned to torch / np.histogram in
                          tests/test_fds_loss_kernels_cpu.py.
  fds_accumulate          counts bit-exact.  sums / sumsq: both the kernel and the float64 reference (index_add_) add the
                          m rows of a bin (and the accumulator's prior value) in some order, each within (m - 1) U64 of
                          the exact sum of |terms|, so they agree within (m_kernel + m_ref - 2) U64 sum|x| (sum x^2; the
                          squares of fp32 values are exact in fp64) -- for any flush order.  Bins without rows keep their
                          bits.
  fds_finalize            mean bit-exact against the restatement mean = sx / n, the EMA in fp32 as
                          fp32(fp32(a * fp32(mean)) + fp32(f * run)).  nvcc contracts sq - sx * mean into one fma (read
                          off the SASS), and values of num within 4 n U64 sq of 0 become 0 (the rounding bound of the fp64
                          sums, derived in fds_finalize_kernel): var is checked within
                          a (4 n U64 sq + 2 U64 |sx mean|) / (n - 1) + 3u (a |var| + f |run|).  End to end from rows
                          (accumulate + finalize), against the two-pass float64 variance: within 3u var + 8 n U64 Q / (n-1).
  fds_smooth_tables       bit-exact against acc = fp32(acc + fp32(w_j * src[reflect(b + j - h)])) in j order, itself
                          within ks u sum |w src| of float64.
  fds_fill_empty          bit-exact against an fp32 walk over the bins in increasing order (bin b reads the already
                          filled b - 1).
  fds_calibrate_fwd/_bwd  bit-exact against fp32((x - m1) * sqrt(clamp(v2 / v1)) + m2) (separate roundings, IEEE sqrt
                          and division) on the rows the kernel must calibrate; every other row bit-identical to the input,
                          rowbin exact.  Row sums of v1 are chosen far from 1e-10 on either side.
  loss_fwd_bwd            mse / l1 / huber per-element gradients bit-exact against the fp32 restatement
                          fp32(fp32(fp32(g * w) * fp32(1 / n)) * grad_scale); n = 1 calls give one element's loss bit for
                          bit.  Focal: expf / tanhf within 2 ulp, powf within 4 ulp (the CUDA programming guide's table):
                          fb = tanh(beta a) within 4u |fb| + u beta a, fb = 2 sigmoid - 1 within 12u (absolute: it cancels
                          at small a, in the reference as well), and the remaining products and sums within 16u of the sum
                          of their terms.  The loss within u |loss| + (n + 1) U64 sum |l| / n of the float64 mean of the
                          kernel's per-element values.
  lds_histogram / weights / table lookup
                          bit-exact against restatements (trunc toward zero, clamp; scipy's convolve1d order with the
                          int64 truncation on the 'inverse' path; np.float32(1 / x); the serial fp64 sum of hist * w; the
                          fp32 scaling), pinned to oracle/dir_oracle.lds_weights on the CPU.

Every bound is multiplied by 1.001 for second-order terms.  The file reruns itself with DIRB200_SMS=7 (grid-stride loops
iterate many times) and with DIRB200_FDS_SMALL=0 DIRB200_FDS_RPC=1 DIRB200_FDS_BLOCK=256 (the grid-wide counting sort
at every n, one flush per row)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = "cuda"
U = 2.0 ** -24
U64 = 2.0 ** -53
SLACK = 1.001
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F64 = torch.float64
SENT = -7777                       # int sentinel of bins / rowbin outputs
AGE, DEPTH, EDGES5 = 0, 1, 2
ERR_WORKSPACE = -3
CLIPS = {AGE: (0.1, 10.0), DEPTH: (0.2, 5.0), EDGES5: (0.1, 10.0)}


def lib():
    import _lib
    return _lib


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def nan_f32(*shape):
    return torch.full(shape, float("nan"), device=DEV)


def f32(v):
    return float(np.float32(v))


def check(name, got, ref, bound):
    ok = (got.double() - ref).abs() <= bound            # NaN (never written) fails
    if not ok.all():
        i = (~ok).nonzero()[0].tolist()
        raise AssertionError(f"{name}: {int((~ok).sum())} of {ok.numel()} elements outside the bound, first at {i}: "
                             f"got {got[tuple(i)].item()!r}, ref {ref[tuple(i)].item()!r}, bound {bound[tuple(i)].item():.3e}")


def check_bits(name, got, ref):
    got, ref = got.contiguous(), ref.to(got.device).contiguous()
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    view = {torch.float32: torch.int32, torch.float64: torch.int64}.get(got.dtype)
    bad = (got.view(view) != ref.view(view)) if view else (got != ref)
    assert not bad.any(), (f"{name}: {int(bad.sum())} of {bad.numel()} elements differ, first at "
                           f"{bad.nonzero()[0].tolist()}: got {got[tuple(bad.nonzero()[0].tolist())].item()!r}, "
                           f"want {ref[tuple(bad.nonzero()[0].tolist())].item()!r}")


# ------------------------------------------------------------------------------------------ restatements (numpy, CPU)
def bin_index(rule, labels, bucket_num, bucket_start, has_lo=None, has_hi=None):
    """The kernels' row -> table row (-1: untouched), restated in numpy on float32 labels.  has_lo / has_hi default to
    whether the edge values occur among the labels (the age rule's flags)."""
    v = np.asarray(labels, dtype=np.float32).reshape(-1)
    lo, hi = np.float32(bucket_start), np.float32(bucket_num - 1)
    nb = bucket_num - bucket_start
    out = np.full(v.shape, -1, dtype=np.int64)
    nan = np.isnan(v)
    if rule == AGE:
        has_lo = bool((v == lo).any()) if has_lo is None else has_lo
        has_hi = bool((v == hi).any()) if has_hi is None else has_hi
        inr = (v >= lo) & (v <= hi)
        out[inr] = (v[inr] - lo).astype(np.int64)       # fp32 subtraction, truncation
        if has_lo:
            out[v < lo] = 0
        if has_hi:
            out[v > hi] = nb - 1
        return out
    last = bucket_num - 1
    with np.errstate(invalid="ignore"):
        if rule == DEPTH:
            b = np.trunc(v * np.float32(10)).astype(np.float64)          # fp32 product, int() truncation
        else:
            edges = (np.arange(bucket_num + 1, dtype=np.float64) * (5.0 / bucket_num)).astype(np.float32)
            b = (np.searchsorted(edges, v, side="right") - 1).astype(np.float64)   # last edge <= label
            b = np.clip(b, 0, last)
            b[v >= np.float32(5)] = last
        b = np.clip(b, bucket_start, last)
    out[~nan] = b[~nan].astype(np.int64) - bucket_start
    return out


def lds_restated(hist, reweight, window, n_total):
    """(per-bin fp32 table as float64, fp32 scaling) of lds_bins_kernel: val = sqrt(h) or clip(h, 5, 1000); the
    convolve1d in scipy's symmetric order (centre tap, then the pairs from the outermost inwards; zero padding), truncated
    on the 'inverse' path; table = fp32(1 / val) where h > 0; s = serial fp64 sum of h * table (exact products);
    scaling = fp32(n_total) / fp32(s)."""
    h = np.asarray(hist, dtype=np.int64)
    hd = h.astype(np.float64)
    val = np.sqrt(hd) if reweight == "sqrt_inv" else np.clip(hd, 5.0, 1000.0)
    if window is not None and len(window):
        w = np.asarray(window, dtype=np.float64)
        k = len(w) // 2
        pad = np.concatenate([np.zeros(k), val, np.zeros(k)])
        acc = val * w[k]
        for j in range(-k, 0):
            acc = acc + (pad[k + j:k + j + len(val)] + pad[k - j:k - j + len(val)]) * w[k + j]
        val = np.trunc(acc) if reweight == "inverse" else acc
    with np.errstate(divide="ignore"):
        table = np.where(h > 0, (1.0 / val).astype(np.float32).astype(np.float64), 0.0)
    s = np.cumsum(hd * table)[-1]
    return table, np.float32(np.float32(n_total) / np.float32(s))


# --------------------------------------------------------------------------------------------------------- binning
def run_bins(rule, labels, bucket_num, bucket_start, flags=None, tail=5):
    L = lib()
    n = labels.numel()
    if flags is None:
        flags = torch.zeros(2, dtype=torch.int32, device=DEV)
    L.call("dirb200_fds_label_flags", L.ptr(labels), n, bucket_num, bucket_start, rule, L.ptr(flags), L.stream_ptr())
    bins = torch.full((n + tail,), SENT, dtype=torch.int32, device=DEV)
    L.call("dirb200_fds_bin_rows", L.ptr(labels), n, bucket_num, bucket_start, rule, L.ptr(flags), L.ptr(bins),
           L.stream_ptr())
    torch.cuda.synchronize()
    assert (bins[n:] == SENT).all(), "bin_rows wrote past n"
    return bins[:n], flags


def age_labels(g, n, with_lo, with_hi, lo=3, hi=99):
    v = torch.randint(-20, 140, (n,), generator=g, device=DEV).float()
    v[::7] += 0.5                                              # non-integer labels truncate
    v = torch.where((v == lo) | (v == hi), torch.full_like(v, 50.0), v)
    if with_lo:
        v[n // 3] = lo
    if with_hi:
        v[n // 2] = hi
    v[n - 1] = float("nan")
    return v


@pytest.mark.parametrize("n", [17, 100_000])
def test_bin_rows_age_rule_with_and_without_edges(n):
    g = gen(n)
    for with_lo in (False, True):
        for with_hi in (False, True):
            lab = age_labels(g, n, with_lo, with_hi)
            bins, flags = run_bins(AGE, lab, 100, 3)
            assert flags.tolist() == [int(with_lo), int(with_hi)]
            check_bits(f"age bins lo={with_lo} hi={with_hi}", bins,
                       torch.from_numpy(bin_index(AGE, lab.cpu().numpy(), 100, 3)).int())
    # flags are OR-ed, not reset: set flags fold out-of-range labels although this batch lacks the edges
    lab = age_labels(g, n, False, False)
    bins, flags = run_bins(AGE, lab, 100, 3, flags=torch.ones(2, dtype=torch.int32, device=DEV))
    assert flags.tolist() == [1, 1]
    check_bits("age bins, flags preset", bins,
               torch.from_numpy(bin_index(AGE, lab.cpu().numpy(), 100, 3, True, True)).int())


def depth_sweep():
    """every k / 10 for k in [0, 120] as fp32, one ulp either side, NaN, negatives and huge values"""
    k = np.float32(np.arange(0, 121) / 10.0)
    v = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(100)),
                        np.float32([np.nan, -0.05, -3, 1e9, np.inf, -np.inf])])
    return v.astype(np.float32)


def edges_sweep(num):
    e = (np.arange(num + 1) * (5.0 / num)).astype(np.float32)
    v = np.concatenate([e, np.nextafter(e, np.float32(-1)), np.nextafter(e, np.float32(10)),
                        np.float32([np.nan, -1, 5, 7, 2.5, 4.9999])])
    return v.astype(np.float32)


@pytest.mark.parametrize("rule,bucket_num,bucket_start", [(DEPTH, 100, 7), (DEPTH, 100, 0), (EDGES5, 50, 0),
                                                          (EDGES5, 50, 4), (EDGES5, 7, 0), (EDGES5, 7, 2)])
def test_bin_rows_depth_and_edges5_at_every_edge(rule, bucket_num, bucket_start):
    v = depth_sweep() if rule == DEPTH else edges_sweep(bucket_num)
    lab = torch.from_numpy(v).to(DEV)
    flags = torch.full((2,), 5, dtype=torch.int32, device=DEV)
    bins, flags = run_bins(rule, lab, bucket_num, bucket_start, flags=flags)
    assert flags.tolist() == [5, 5], "label_flags touched the flags under a rule without edge folding"
    check_bits("bins", bins, torch.from_numpy(bin_index(rule, v, bucket_num, bucket_start)).int())


def test_bin_rows_and_flags_n_zero_launch_nothing():
    L = lib()
    flags = torch.zeros(2, dtype=torch.int32, device=DEV)
    bins = torch.full((4,), SENT, dtype=torch.int32, device=DEV)
    n0 = L.launch_count()
    L.call("dirb200_fds_label_flags", None, 0, 100, 3, AGE, L.ptr(flags), L.stream_ptr())
    L.call("dirb200_fds_bin_rows", None, 0, 100, 3, AGE, L.ptr(flags), L.ptr(bins), L.stream_ptr())
    torch.cuda.synchronize()
    assert L.launch_count() == n0 and (bins == SENT).all() and (flags == 0).all()


# ------------------------------------------------------------------------------------------------------ accumulate
def acc_ws(n, nb, short=0, fill=0xFF):
    need = lib().raw("dirb200_fds_accumulate_workspace_bytes")(n, nb)
    return torch.full((need - short,), fill, dtype=torch.uint8, device=DEV)


def accumulate(feat, bins, n, d, nb, sums, sumsq, counts, ws=None):
    L = lib()
    ws = acc_ws(n, nb) if ws is None else ws
    return L.raw("dirb200_fds_accumulate")(L.ptr(feat), L.ptr(bins), n, d, nb, L.ptr(sums), L.ptr(sumsq),
                                           L.ptr(counts), L.ptr(ws), ws.numel(), L.stream_ptr())


def acc_reference(feat, bins, nb, d):
    """float64 (count, sum x, sum x^2, sum |x|) per bin of the rows whose bin is in [0, nb)"""
    ok = (bins >= 0) & (bins < nb)
    idx, x = bins[ok].long(), feat[ok].double()
    z = lambda: torch.zeros(nb, d, dtype=F64, device=DEV)
    return (torch.bincount(idx, minlength=nb), z().index_add_(0, idx, x), z().index_add_(0, idx, x * x),
            z().index_add_(0, idx, x.abs()))


def make_bins(layout, n, nb, g):
    if layout == "random":
        b = torch.randint(0, nb, (n,), generator=g, device=DEV)
    elif layout == "hot":                                   # one hot bin, a few rows elsewhere
        b = torch.full((n,), nb // 2, device=DEV, dtype=torch.int64)
        b[::97] = torch.randint(0, nb, (b[::97].numel(),), generator=g, device=DEV)
    elif layout == "every_row":                             # a bin change at every row
        b = torch.arange(n, device=DEV) % nb
    elif layout == "runs":                                  # runs of 129 and 7 rows straddle the chunk edges
        r = torch.arange(n, device=DEV)
        b = torch.where(r % 2000 < 1000, (r // 129) % nb, (r // 7) % nb)
    b = b.int()
    if n > 3:                                               # dropped rows: bin -1 and bin >= nb
        b[1::53] = -1
        b[2::61] = nb
        b[3::67] = nb + 1000
    return b


def run_accumulate_case(n, d, nb, layout, seed, misaligned=False, prior=False, two_calls=False):
    g = gen(seed)
    bins = make_bins(layout, n, nb, g)
    store = torch.randn(n * d + 1, generator=g, device=DEV) * 3 + 1
    off = 1 if misaligned else 0                           # a 4-byte aligned view: the VEC = 1 path
    feat = store[off:off + n * d].view(n, d)
    if prior:                                               # accumulate into non-zero accumulators
        sums0 = torch.randn(nb, d, generator=g, device=DEV, dtype=F64) * 100
        sq0 = torch.rand(nb, d, generator=g, device=DEV, dtype=F64) * 100
        cnt0 = torch.randint(0, 1000, (nb,), generator=g, device=DEV)
    else:
        sums0 = torch.zeros(nb, d, dtype=F64, device=DEV)
        sq0 = torch.zeros(nb, d, dtype=F64, device=DEV)
        cnt0 = torch.zeros(nb, dtype=torch.int64, device=DEV)
    sums, sumsq, counts = sums0.clone(), sq0.clone(), cnt0.clone()
    parts = [(0, n // 2), (n // 2, n)] if two_calls else [(0, n)]
    ws = acc_ws(n, nb)
    for a, b in parts:
        rc = accumulate(feat[a:b], bins[a:b], b - a, d, nb, sums, sumsq, counts, ws=ws)
        assert rc == 0, lib().last_error()
    torch.cuda.synchronize()
    cnt, s, q, A = acc_reference(feat, bins, nb, d)
    check_bits("counts", counts, cnt0 + cnt)
    m = (cnt.double() + (1.0 if prior else 0.0))[:, None]
    k = (2 * m - 2).clamp(min=0) * U64 * SLACK
    check("sums", sums, sums0 + s, k * (A + sums0.abs()))
    check("sumsq", sumsq, sq0 + q, k * (q + sq0))
    empty = cnt == 0
    check_bits("sums of bins without rows", sums[empty], sums0[empty])
    check_bits("sumsq of bins without rows", sumsq[empty], sq0[empty])


# (n, d, nb, layout)
ACC_CASES = [(n, 64, 100, "random") for n in (1, 8191, 8192, 16384, 16385, 65535, 65536)] + [
    (12208, 2048, 97, "random"),          # AgeDB-DIR epoch
    (191509, 2048, 100, "random"),        # IMDB-WIKI-DIR epoch
    (5749, 12000, 50, "random"),          # STS-B-DIR epoch, d = 12 000 (a partial last column slice)
] + [(5000, d, 37, "random") for d in (1, 3, 7, 4, 2052)] + [
    (20000, 16, 1, "random"), (9000, 8, 4096, "every_row"), (9000, 8, 4097, "every_row"),
    (30000, 8, 8192, "every_row"),
    (40000, 64, 100, "hot"), (12000, 64, 100, "every_row"), (70000, 32, 100, "runs"), (5000, 32, 100, "runs"),
]


@pytest.mark.parametrize("n,d,nb,layout", ACC_CASES, ids=[f"n{n}-d{d}-nb{nb}-{l}" for n, d, nb, l in ACC_CASES])
def test_fds_accumulate(n, d, nb, layout):
    run_accumulate_case(n, d, nb, layout, seed=n + d + nb)


def test_fds_accumulate_nyud2_depth_rows():
    """NYUD2-DIR's per-pixel FDS: 138 624 pixel rows of 128 channels (batch 8 at 114 x 152), depth bins clamp(int(d *
    10), 7, 99) -> nb = 93, made by bin_rows itself."""
    g = gen(93)
    n, d = 138624, 128
    depth = torch.rand(n, generator=g, device=DEV) * 9.3 + 0.7
    bins, _ = run_bins(DEPTH, depth, 100, 7)
    feat = torch.relu(torch.randn(n, d, generator=g, device=DEV) + 0.4)
    sums = torch.zeros(93, d, dtype=F64, device=DEV)
    sumsq, counts = torch.zeros_like(sums), torch.zeros(93, dtype=torch.int64, device=DEV)
    assert accumulate(feat, bins, n, d, 93, sums, sumsq, counts) == 0
    torch.cuda.synchronize()
    cnt, s, q, A = acc_reference(feat, bins, 93, d)
    check_bits("counts", counts, cnt)
    k = (2 * cnt.double() - 2).clamp(min=0)[:, None] * U64 * SLACK
    check("sums", sums, s, k * A)
    check("sumsq", sumsq, q, k * q)


@pytest.mark.parametrize("case", ["misaligned", "prior", "two_calls", "misaligned_grid_sort"])
def test_fds_accumulate_edges(case):
    if case == "misaligned":                                # d % 4 == 0 but a 4-byte aligned pointer: the VEC = 1 path
        run_accumulate_case(5000, 64, 50, "random", 1, misaligned=True)
    elif case == "misaligned_grid_sort":
        run_accumulate_case(70000, 20, 50, "runs", 2, misaligned=True)
    elif case == "prior":
        run_accumulate_case(20000, 36, 60, "random", 3, prior=True)
    else:                                                   # two streamed calls into the same accumulators
        run_accumulate_case(30000, 40, 70, "random", 4, two_calls=True, prior=True)


def test_fds_accumulate_workspace_one_byte_short():
    L = lib()
    n, d, nb = 100, 8, 10
    feat = torch.randn(n, d, device=DEV)
    bins = torch.zeros(n, dtype=torch.int32, device=DEV)
    sums = torch.zeros(nb, d, dtype=F64, device=DEV)
    sumsq, counts = torch.zeros_like(sums), torch.zeros(nb, dtype=torch.int64, device=DEV)
    n0 = L.launch_count()
    rc = accumulate(feat, bins, n, d, nb, sums, sumsq, counts, ws=acc_ws(n, nb, short=1))
    torch.cuda.synchronize()
    assert rc == ERR_WORKSPACE and "workspace too small" in L.last_error()
    assert L.launch_count() == n0 and (sums == 0).all() and (counts == 0).all()


# -------------------------------------------------------------------------------------------------------- finalize
def finalize(sums, sumsq, counts, mean, var, tracked, momentum, first):
    L = lib()
    nb, d = mean.shape
    L.call("dirb200_fds_finalize", L.ptr(sums), L.ptr(sumsq), L.ptr(counts), nb, d, L.ptr(mean), L.ptr(var),
           L.ptr(tracked), -1.0 if momentum is None else momentum, int(first), L.stream_ptr())
    torch.cuda.synchronize()


def finalize_factor(counts, tracked, momentum, first):
    """float64 EMA factor per bin and the fp32-rounded (a, f) = (1 - factor, factor)"""
    dn = counts.double()
    if first:
        fac = torch.zeros_like(dn)
    elif momentum is not None:
        fac = torch.full_like(dn, momentum)
    else:
        fac = 1.0 - dn / (tracked + counts.float()).double()      # float32 buffer += n
    return (1.0 - fac).float(), fac.float()


def ema(a, f, cur32, run):
    return (a[:, None] * cur32) + (f[:, None] * run)           # two fp32 products, one fp32 sum


@pytest.mark.parametrize("mode", ["first", "momentum", "tracked"])
def test_fds_finalize_restated(mode):
    g = gen(len(mode))
    nb, d = 40, 300
    counts = torch.randint(1, 3000, (nb,), generator=g, device=DEV)
    counts[[3, 17, 39]] = 0                                  # empty bins: untouched
    counts[[5, 6]] = 1                                       # one row: var exactly 0
    mu = torch.randn(nb, d, generator=g, device=DEV, dtype=F64) * 2
    sd = torch.rand(nb, d, generator=g, device=DEV, dtype=F64)
    mu[:, 7], sd[:, 7] = 1000.0, 1e-3                        # large mean, small variance: the cancellation term
    cn = counts.double()[:, None]
    sums = mu * cn
    sumsq = (sd * sd * (cn - 1).clamp(min=0) + mu * mu * cn)
    sums[5:7], sumsq[5:7] = mu[5:7], mu[5:7] ** 2            # one row: sq == sx^2 exactly
    run_m = torch.randn(nb, d, generator=g, device=DEV)
    run_v = torch.rand(nb, d, generator=g, device=DEV)
    tracked = torch.randint(0, 5000, (nb,), generator=g, device=DEV).float()
    tracked[8] = 2.0 ** 24                                   # tracked past 2^24: fp32(2^24 + n) rounds
    counts[8] = 3
    cn = counts.double()[:, None]
    sums[8], sumsq[8] = mu[8] * 3, mu[8] ** 2 * 3 + 2 * sd[8] ** 2
    momentum = 0.9 if mode == "momentum" else None
    first = mode == "first"
    m, v, t = run_m.clone(), run_v.clone(), tracked.clone()
    finalize(sums, sumsq, counts, m, v, t, momentum, first)

    a, f = finalize_factor(counts, tracked, momentum, first)
    has = counts > 0
    mean = sums / cn
    check_bits("running_mean", m[has], ema(a, f, mean.float(), run_m)[has])
    num = sumsq - sums * mean
    vref = (num / (cn - 1)).clamp(min=0).where(cn > 1, torch.zeros_like(num))
    e64 = ((4 * cn * U64 * sumsq + 2 * U64 * (sums * mean).abs()) / (cn - 1)).where(cn > 1, torch.zeros_like(num))
    ref = a.double()[:, None] * vref + f.double()[:, None] * run_v.double()
    bound = SLACK * (a.double()[:, None] * e64 + 3 * U * (a.double()[:, None] * vref + f.double()[:, None] * run_v.double()))
    check("running_var", v[has], ref[has], bound[has])
    one = counts == 1
    check_bits("running_var of one-row bins", v[one], ema(a, f, torch.zeros_like(run_v), run_v)[one])
    check_bits("running_mean of empty bins", m[~has], run_m[~has])
    check_bits("running_var of empty bins", v[~has], run_v[~has])
    check_bits("num_samples_tracked", t, torch.where(has, tracked + counts.float(), tracked))
    assert float(t[8]) == 2.0 ** 24 + 4


def accumulate_finalize(feat, bins, nb):
    n, d = feat.shape
    sums = torch.zeros(nb, d, dtype=F64, device=DEV)
    sumsq, counts = torch.zeros_like(sums), torch.zeros(nb, dtype=torch.int64, device=DEV)
    assert accumulate(feat, bins, n, d, nb, sums, sumsq, counts) == 0
    m, v = torch.zeros(nb, d, device=DEV), torch.ones(nb, d, device=DEV)    # first update: factor 0 times these
    finalize(sums, sumsq, counts, m, v, torch.zeros(nb, device=DEV), None, True)
    return m, v, counts


@pytest.mark.parametrize("m_rows,nb", [(5000, 1), (5000, 4), (33, 64), (191509, 1)])
def test_fds_finalize_constant_columns_have_zero_variance(m_rows, nb):
    """2048 columns, each constant within a bin (constants of every magnitude, both signs), m_rows > 32 rows per bin:
    torch.var of equal values is exactly 0, and calibrate_mean_var branches on it -- so running_var must be exactly 0
    whatever order the fp64 atomics flushed the sums in, and running_mean exactly the constant."""
    g = gen(m_rows + nb)
    d = 2048
    c = (torch.randn(nb, d, generator=g, device=DEV) * torch.exp2(torch.randint(-20, 20, (nb, d), generator=g,
                                                                                 device=DEV).float()))
    c[c == 0] = 1.0
    bins = torch.arange(nb, device=DEV, dtype=torch.int32).repeat_interleave(m_rows)
    bins = bins[torch.randperm(bins.numel(), generator=g, device=DEV)]
    feat = c[bins.long()]
    m, v, counts = accumulate_finalize(feat, bins, nb)
    assert (counts == m_rows).all()
    pos = int((v != 0).sum())
    assert pos == 0, f"{pos} of {v.numel()} constant columns have a non-zero variance (max {float(v.abs().max()):.3e})"
    check_bits("mean of constant columns", m, c)


@pytest.mark.parametrize("n,d,nb", [(12208, 2048, 97), (70000, 64, 10), (3000, 7, 5)])
def test_fds_accumulate_finalize_end_to_end(n, d, nb):
    """against the two-pass float64 mean / unbiased variance of each bin's rows"""
    g = gen(n)
    bins = torch.randint(0, nb, (n,), generator=g, device=DEV).int()
    feat = torch.relu(torch.randn(n, d, generator=g, device=DEV) + 0.5)
    feat[:, 0] = 1000 + 1e-3 * torch.randn(n, generator=g, device=DEV)    # large mean, small variance
    feat[:, 1] = 0
    m, v, counts = accumulate_finalize(feat, bins, nb)
    x = feat.double()
    cnt = counts.double()[:, None]
    mean = torch.zeros(nb, d, dtype=F64, device=DEV).index_add_(0, bins.long(), x) / cnt
    dev2 = torch.zeros(nb, d, dtype=F64, device=DEV).index_add_(0, bins.long(), (x - mean[bins.long()]) ** 2)
    Q = torch.zeros(nb, d, dtype=F64, device=DEV).index_add_(0, bins.long(), x * x)
    var = dev2 / (cnt - 1)
    check("mean", m, mean, SLACK * (U * mean.abs() + 2 * cnt * U64 * Q.sqrt() / cnt.sqrt()))
    check("var", v, var, SLACK * (3 * U * var + 8 * cnt * U64 * Q / (cnt - 1)))
    assert (v[:, 1] == 0).all()


# ---------------------------------------------------------------------------------------------------- smooth tables
def window(kernel, ks, sigma):
    from oracle import dir_oracle as O
    return O.fds_kernel_window(kernel, ks, sigma) if ks > 1 else np.ones(1, dtype=np.float32)


def reflect(k, nb):
    k = np.where(k < 0, -k, k)
    return np.where(k >= nb, 2 * (nb - 1) - k, k)


@pytest.mark.parametrize("kernel,ks,sigma,nb", [("gaussian", 1, 1, 1), ("gaussian", 1, 1, 100), ("gaussian", 3, 1, 2),
                                                ("gaussian", 5, 2, 3), ("triang", 5, 1, 100), ("laplace", 3, 2, 100),
                                                ("gaussian", 33, 8, 17), ("laplace", 33, 4, 17),
                                                ("triang", 33, 1, 100), ("gaussian", 9, 1, 97)])
def test_fds_smooth_tables_restated(kernel, ks, sigma, nb):
    L = lib()
    d = 300
    w = window(kernel, ks, sigma)
    src = torch.randn(nb, d, generator=gen(ks + nb), device=DEV)
    dst = nan_f32(nb + 1, d)                                 # one row past the table stays NaN
    L.call("dirb200_fds_smooth_tables", L.ptr(src), nb, d, w.ctypes.data_as(L.P), ks, L.ptr(dst), L.stream_ptr())
    torch.cuda.synchronize()
    assert dst[nb].isnan().all()
    h = (ks - 1) // 2
    acc = torch.zeros(nb, d, device=DEV)
    ref64 = torch.zeros(nb, d, dtype=F64, device=DEV)
    mag = torch.zeros_like(ref64)
    for j in range(ks):
        k = torch.from_numpy(reflect(np.arange(nb) + j - h, nb)).to(DEV)
        term = torch.tensor(float(w[j]), device=DEV) * src[k]
        acc = acc + term
        ref64 += float(w[j]) * src[k].double()
        mag += abs(float(w[j])) * src[k].double().abs()
    check("fp32 restatement vs float64", acc, ref64, SLACK * ks * U * mag)
    check_bits("smooth_tables", dst[:nb], acc)


# ------------------------------------------------------------------------------------------------------ fill empty
@pytest.mark.parametrize("nb,empty", [(1, [0]), (2, [0]), (2, [1]), (2, [0, 1]), (10, [0, 1, 4, 5, 6, 9]),
                                      (10, list(range(10))), (50, [0, 1, 2, 20, 21, 47, 48, 49]), (7, [])])
def test_fds_fill_empty_increasing_order(nb, empty):
    L = lib()
    d = 130
    g = gen(nb + len(empty))
    counts = torch.randint(1, 100, (nb,), generator=g, device=DEV)
    counts[empty] = 0
    mean, var = torch.randn(nb, d, generator=g, device=DEV), torch.rand(nb, d, generator=g, device=DEV)
    m, v = mean.clone(), var.clone()
    L.call("dirb200_fds_fill_empty", L.ptr(counts), nb, d, L.ptr(m), L.ptr(v), L.stream_ptr())
    torch.cuda.synchronize()
    rm, rv = mean.clone(), var.clone()
    if nb >= 2:
        for b in range(nb):
            if b in empty:
                for t in (rm, rv):
                    t[b] = t[b + 1] if b == 0 else (t[b - 1] if b == nb - 1 else (t[b - 1] + t[b + 1]) / 2)
    check_bits("mean", m, rm)
    check_bits("var", v, rv)


# ------------------------------------------------------------------------------------------------------- calibrate
def calib_tables(g, rule, nb, d):
    """(m1, v1, m2, v2) with: bin 0 all zero (sum(v1) = 0 -> identity), bin 1 v1 ~ 1e-13 (sum far below 1e-10), under
    the age rule dead channels (v1 = 0) and under the depth / STS-B rules bins 2 / 3 with one bad channel (v1 <= 0,
    v2 < 0) -> those rows untouched; clamps at both ends."""
    m1, m2 = torch.randn(nb, d, generator=g, device=DEV), torch.randn(nb, d, generator=g, device=DEV)
    v1 = torch.rand(nb, d, generator=g, device=DEV) + 0.05
    v2 = torch.rand(nb, d, generator=g, device=DEV) * 4
    v1[0] = 0
    v1[1] = 1e-13 / d
    if rule == AGE:
        v1[:, 1::5] = 0
    else:
        v1[2, d // 2] = 0
        v2[3, d - 1] = -1e-3
    v1[4, 0], v2[5, -1] = 1e-7, 1e-9                        # clamp at clip_max / clip_min
    return m1, v1, m2, v2


def calib_labels(g, rule, b, bucket_num, bucket_start):
    if rule == AGE:
        v = torch.randint(bucket_start, bucket_num, (b,), generator=g, device=DEV).float()
        v[::11] = bucket_num + 20                           # above hi: folded only when hi occurs (it does)
        v[1::13] = bucket_start - 2                          # below lo: lo never occurs -> untouched
        v = torch.where(v == bucket_start, torch.full_like(v, bucket_start + 1.0), v)
        v[b // 2] = bucket_num - 1
    elif rule == DEPTH:
        v = torch.rand(b, generator=g, device=DEV) * 10.5
    else:
        v = torch.round(torch.rand(b, generator=g, device=DEV) * 20) / 4
    if b > 3:
        v[3] = float("nan")
    # bins 0..5 (the special tables) get rows
    special = {AGE: lambda k: bucket_start + k, DEPTH: lambda k: (bucket_start + k) / 10 + 0.05,
               EDGES5: lambda k: (bucket_start + k + 0.5) * 5 / bucket_num}[rule]
    for k in range(6):
        if 10 + k < b:
            v[10 + k] = special(k)
    return v


def calib_restated(rule, x, lab, bucket_num, bucket_start, m1, v1, m2, v2):
    """(expected output, expected rowbin, gradient scale per element)"""
    clip_min, clip_max = CLIPS[rule]
    bins = torch.from_numpy(bin_index(rule, lab.cpu().numpy(), bucket_num, bucket_start)).to(DEV)
    ok = bins >= 0
    b = bins.clamp(min=0)
    tot = v1.double().sum(1)[b]
    ok &= ~(tot < 1e-10)
    if rule != AGE:
        ok &= ~((v1 <= 0) | (v2 < 0)).any(1)[b]
    a = v1[b]
    live = ok[:, None] & ((a != 0) if rule == AGE else torch.ones_like(a, dtype=torch.bool))
    fac = torch.clamp(v2[b] / a, f32(clip_min), f32(clip_max))
    s = torch.sqrt(fac)
    y = torch.where(live, (x - m1[b]) * s + m2[b], x)
    return y, torch.where(ok, bins, torch.full_like(bins, -1)).int(), torch.where(live, s, torch.ones_like(s))


CAL_CASES = [(AGE, 1, 2048), (AGE, 256, 2048), (AGE, 2048, 2048), (AGE, 2049, 2048), (AGE, 300, 1),
             (AGE, 2049, 128), (DEPTH, 138624, 128), (DEPTH, 2048, 128), (DEPTH, 2049, 128), (DEPTH, 256, 1),
             (EDGES5, 128, 12000), (EDGES5, 2049, 12000), (EDGES5, 1, 12000), (EDGES5, 256, 2048)]


@pytest.mark.parametrize("rule,b,d", CAL_CASES, ids=[f"rule{r}-b{b}-d{d}" for r, b, d in CAL_CASES])
def test_fds_calibrate_fwd_bwd_restated(rule, b, d):
    L = lib()
    bucket_num, bucket_start = {AGE: (100, 3), DEPTH: (100, 7), EDGES5: (50, 0)}[rule]
    nb = bucket_num - bucket_start
    clip_min, clip_max = CLIPS[rule]
    g = gen(rule * 1000 + b + d)
    m1, v1, m2, v2 = calib_tables(g, rule, nb, d)
    lab = calib_labels(g, rule, b, bucket_num, bucket_start)
    x0 = torch.randn(b, d, generator=g, device=DEV)
    x = x0.clone()
    rowbin = torch.full((b + 3,), SENT, dtype=torch.int32, device=DEV)
    flags = torch.full((2,), 9, dtype=torch.int32, device=DEV)
    L.call("dirb200_fds_calibrate_fwd", L.ptr(x), L.ptr(lab), b, d, bucket_num, bucket_start, rule, L.ptr(m1), L.ptr(v1),
           L.ptr(m2), L.ptr(v2), clip_min, clip_max, L.ptr(rowbin), L.ptr(flags), L.stream_ptr())
    torch.cuda.synchronize()
    y, rb, s = calib_restated(rule, x0, lab, bucket_num, bucket_start, m1, v1, m2, v2)
    assert (rowbin[b:] == SENT).all()
    check_bits("rowbin", rowbin[:b], rb)
    check_bits("calibrated rows", x, y)
    untouched = rb < 0
    check_bits("untouched rows", x[untouched], x0[untouched])
    if b > 20:
        assert untouched.any() and (~untouched).any()

    gout = torch.randn(b, d, generator=g, device=DEV)
    gin = nan_f32(b, d)
    L.call("dirb200_fds_calibrate_bwd", rule, L.ptr(gout), L.ptr(rowbin), b, d, L.ptr(v1), L.ptr(v2), clip_min, clip_max,
           L.ptr(gin), L.stream_ptr())
    torch.cuda.synchronize()
    check_bits("calibrate bwd", gin, gout * s)
    L.call("dirb200_fds_calibrate_bwd", rule, L.ptr(gout), L.ptr(rowbin), b, d, L.ptr(v1), L.ptr(v2), clip_min, clip_max,
           L.ptr(gout), L.stream_ptr())                   # in place
    torch.cuda.synchronize()
    check_bits("calibrate bwd in place", gout, gin)


# ------------------------------------------------------------------------------------------------------------ loss
KIND = {"mse": 0, "l1": 1, "focal_mse": 2, "focal_l1": 3, "huber": 4}


def loss_call(kind, pred, target, weight, beta, gamma, act, grad_scale, with_grad=True, ws=None):
    L = lib()
    n = pred.numel()
    ws = torch.full((L.raw("dirb200_loss_workspace_bytes")(n),), 0xFF, dtype=torch.uint8, device=DEV) if ws is None else ws
    out = nan_f32(1)
    grad = nan_f32(n) if with_grad else None
    L.call("dirb200_loss_fwd_bwd", KIND[kind], L.ptr(pred), L.ptr(target), L.ptr(weight), n, beta, gamma,
           0 if act == "sigmoid" else 1, grad_scale, L.ptr(out), L.ptr(grad), L.ptr(ws), ws.numel(), L.stream_ptr())
    torch.cuda.synchronize()
    return out, grad


def loss_restated(kind, pred, target, weight, beta, gamma, act):
    """(per-element loss l, per-element gradient g before the 1/n and grad_scale factors, bound on l, bound on g):
    the fp32 restatement for mse / l1 / huber (bounds 0), a float64 evaluation with derived bounds for the focal kinds"""
    d = pred - target                                        # fp32, as the kernel
    a, sg = d.abs(), torch.sign(d)
    w = torch.ones_like(d) if weight is None else weight
    zero = torch.zeros_like(d, dtype=F64)
    bt = torch.tensor(f32(beta), device=DEV)
    if kind == "mse":
        return (d * d) * w, (2 * d) * w, zero, zero
    if kind == "l1":
        return a * w, sg * w, zero, zero
    if kind == "huber":
        small = a < bt
        l = torch.where(small, ((0.5 * a) * a) / bt, a - 0.5 * bt)
        gr = torch.where(small, d / bt, sg)
        return l * w, gr * w, zero, zero
    dd, ad, sd, wd = d.double(), a.double(), sg.double(), w.double()
    b64, gm = f32(beta), f32(gamma)
    if act == "tanh":
        fb = torch.tanh(b64 * ad)
        dfb = b64 * (1 - fb * fb)
        efb = 4 * U * fb.abs() + U * b64 * ad               # tanhf (2 ulp) and the rounded argument
    else:
        s = torch.sigmoid(b64 * ad)
        fb, dfb = 2 * s - 1, 2 * b64 * s * (1 - s)
        efb = 12 * U * s + U * fb.abs()                     # expf (2 ulp), 1 + e, 1 / x; then 2s - 1
    edfb = 4 * b64 * efb + 8 * U * dfb.abs()
    if gm == 1.0:
        f, df, ef, edf = fb, dfb, efb, edfb
    else:
        f = fb.abs() ** gm
        df = gm * fb.abs() ** (gm - 1) * dfb
        ef = 8 * U * f + gm * fb.abs() ** (gm - 1) * efb
        edf = 12 * U * df.abs() + gm * (gm - 1) * fb.abs() ** max(gm - 2, 0) * efb * dfb.abs() + \
            gm * fb.abs() ** (gm - 1) * edfb
    mm = dd * dd if kind == "focal_mse" else ad
    dm = 2 * dd if kind == "focal_mse" else sd
    l = mm * f * wd
    gr = (dm * f + mm * df * sd) * wd
    el = wd * (16 * U * (mm * f).abs() + mm * ef)
    eg = wd * (16 * U * ((dm * f).abs() + (mm * df).abs()) + dm.abs() * ef + mm * edf)
    return l, gr, el, eg


def check_loss(kind, pred, target, weight, beta, gamma, act, grad_scale, out, grad):
    n = pred.numel()
    l, gr, el, eg = loss_restated(kind, pred, target, weight, beta, gamma, act)
    inv_n = torch.tensor(f32(1.0 / np.float32(n)), device=DEV)
    gs = torch.tensor(f32(grad_scale), device=DEV)
    if grad is not None:
        if kind in ("mse", "l1", "huber"):
            check_bits(f"{kind} grad", grad, (gr * inv_n) * gs)
        else:
            scale = float(inv_n) * float(gs)
            check(f"{kind} grad", grad, gr * scale, SLACK * (eg * abs(scale) + 2 * U * (gr * scale).abs()))
    ld = l.double()
    ref = ld.sum() / n
    bound = SLACK * (U * ref.abs() + (n + 1) * U64 * ld.abs().sum() / n + el.sum() / n)
    check(f"{kind} loss", out, ref.view(1), bound.view(1))


LOSS_N = [1, 255, 256, 257, 262144, 262145, 138624, 554496]
LOSS_CFG = [("mse", 1.0, 1.0, "sigmoid"), ("l1", 1.0, 1.0, "sigmoid"), ("huber", 1.1, 1.0, "sigmoid"),
            ("focal_mse", 0.2, 1.0, "sigmoid"), ("focal_mse", 0.2, 2.0, "tanh"), ("focal_l1", 0.2, 1.0, "tanh"),
            ("focal_l1", 0.2, 2.0, "sigmoid")]


@pytest.mark.parametrize("n", LOSS_N)
@pytest.mark.parametrize("kind,beta,gamma,act", LOSS_CFG, ids=[f"{k}-b{b}-g{g}-{a}" for k, b, g, a in LOSS_CFG])
def test_loss_fwd_bwd(kind, beta, gamma, act, n):
    g = gen(n + len(kind))
    pred = torch.randn(n, generator=g, device=DEV) * 3 + 30
    target = torch.randint(0, 60, (n,), generator=g, device=DEV).float()
    if n > 8:
        pred[:4] = target[:4] + torch.tensor([1.1, -1.1, 0.0, 1e-3], device=DEV)   # |d| == beta (huber), d == 0, small d
    weight = torch.rand(n, generator=g, device=DEV) + 0.5
    for w, gscale in ((weight, 0.5), (None, 1.0)):
        out, grad = loss_call(kind, pred, target, w, beta, gamma, act, gscale)
        check_loss(kind, pred, target, w, beta, gamma, act, gscale, out, grad)
    out2, _ = loss_call(kind, pred, target, weight, beta, gamma, act, 0.5, with_grad=False)   # grad_out = NULL
    ws = torch.full((lib().raw("dirb200_loss_workspace_bytes")(n),), 0xFF, dtype=torch.uint8, device=DEV)
    out3, _ = loss_call(kind, pred, target, weight, beta, gamma, act, 0.5, ws=ws)
    out4, _ = loss_call(kind, pred, target, weight, beta, gamma, act, 0.5, ws=ws)             # same dirty workspace
    check_bits("loss without gradient", out2, out3)
    check_bits("loss, second call on one workspace", out4, out3)


@pytest.mark.parametrize("kind", ["mse", "l1", "huber"])
def test_loss_single_element_bit_exact(kind):
    """n = 1: the loss is fp32(l) itself; |d| on both sides of beta and at beta (huber), d == 0.  At |d| == beta the two
    Huber branches round differently for this beta: fp32(fp32(0.5 beta * beta) / beta) != beta - 0.5 beta."""
    beta = f32(3.353080987930298)
    assert f32(f32(f32(0.5 * beta) * beta) / beta) != beta - 0.5 * beta
    ds = [0.0, beta, -beta, np.nextafter(np.float32(beta), np.float32(0)), np.nextafter(np.float32(beta), np.float32(9)),
          0.3, -7.5, 1e-30]
    for dv in ds:
        for wv in (None, 0.7):
            t = torch.tensor([0.0], device=DEV)
            p = t + torch.tensor([float(np.float32(dv))], device=DEV)
            w = None if wv is None else torch.tensor([wv], device=DEV)
            out, grad = loss_call(kind, p, t, w, beta, 1.0, "sigmoid", 1.0)
            l, gr, _, _ = loss_restated(kind, p, t, w, beta, 1.0, "sigmoid")
            check_bits(f"{kind} loss at d={dv}", out, l)
            check_bits(f"{kind} grad at d={dv}", grad, gr)


# ------------------------------------------------------------------------------------------------------------- LDS
def lds_hist(labels, max_target, hist=None):
    L = lib()
    hist = torch.zeros(max_target, dtype=torch.int64, device=DEV) if hist is None else hist
    L.call("dirb200_lds_histogram", L.ptr(labels), labels.numel(), max_target, L.ptr(hist), L.stream_ptr())
    torch.cuda.synchronize()
    return hist


def hist_restated(labels, max_target):
    b = np.clip(np.trunc(labels.cpu().numpy().astype(np.float64)), 0, max_target - 1).astype(np.int64)
    return torch.from_numpy(np.bincount(b, minlength=max_target)).to(DEV)


@pytest.mark.parametrize("max_target", [1, 121, 8192])
def test_lds_histogram(max_target):
    g = gen(max_target)
    n = 300_000
    lab = torch.rand(n, generator=g, device=DEV) * (max_target * 1.2 + 10) - 5    # negatives, past the last bin
    lab[:6] = torch.tensor([-0.9, -0.0, 0.999, max_target - 1, max_target, 1e30], device=DEV)
    prior = torch.randint(0, 1000, (max_target,), generator=g, device=DEV)
    h = lds_hist(lab, max_target, prior.clone())
    check_bits("histogram into a non-zero hist", h, prior + hist_restated(lab, max_target))


LDS_CASES = [("sqrt_inv", 0), ("inverse", 0), ("sqrt_inv", 1), ("inverse", 1), ("sqrt_inv", 5), ("inverse", 5),
             ("sqrt_inv", 33), ("inverse", 33)]


@pytest.mark.parametrize("reweight,ks", LDS_CASES, ids=[f"{r}-ks{k}" for r, k in LDS_CASES])
def test_lds_weights_restated_and_sharded(reweight, ks):
    L = lib()
    from oracle import dir_oracle as O
    mt = 121
    g = gen(ks + len(reweight))
    lab = (torch.randn(20000, generator=g, device=DEV) * 15 + 40).clamp(0, 130).floor()
    lab = lab[(lab < 60) | (lab > 70)]                        # empty bins 60..70
    lab[:5] = torch.tensor([0.0, 120.0, 130.0, 0.5, 119.99], device=DEV)
    n = lab.numel()
    hist = lds_hist(lab, mt)
    win = O.lds_kernel_window("gaussian", ks, 2) if ks > 1 else (np.ones(1) if ks == 1 else None)
    if win is not None:
        win = np.ascontiguousarray(np.maximum(win, win[::-1]))        # the entry point wants it exactly symmetric
    wptr = None if win is None else win.ctypes.data_as(L.P)
    table, scaling = lds_restated(hist.cpu().numpy(), reweight, win, n)
    bins = np.clip(np.trunc(lab.cpu().numpy()), 0, mt - 1).astype(np.int64)
    want = torch.from_numpy((scaling * table[bins].astype(np.float32)).astype(np.float32)).to(DEV)
    scratch = torch.full((2 * mt + 2,), float("nan"), dtype=F64, device=DEV)
    out = nan_f32(n + 1)
    L.call("dirb200_lds_weights", L.ptr(lab), n, mt, L.REWEIGHT[reweight], wptr, 0 if win is None else len(win),
           L.ptr(hist), L.ptr(scratch), L.ptr(out), L.stream_ptr())
    torch.cuda.synchronize()
    assert out[n].isnan()
    check_bits("lds weights", out[:n], want)
    for lo, hi in ((0, 1), (1, n // 3), (n // 3, n)):         # slices of the column with the whole column's histogram
        part = nan_f32(hi - lo)
        L.call("dirb200_lds_weights_sharded", L.ptr(lab[lo:hi]), hi - lo, n, mt, L.REWEIGHT[reweight], wptr,
               0 if win is None else len(win), L.ptr(hist), L.ptr(scratch), L.ptr(part), L.stream_ptr())
        torch.cuda.synchronize()
        check_bits(f"sharded slice [{lo}, {hi})", part, out[lo:hi])


def test_lds_table_lookup_at_every_boundary():
    L = lib()
    k = np.float32(np.arange(0, 101) / 10.0)
    v = np.concatenate([k, np.nextafter(k, np.float32(-1)), np.nextafter(k, np.float32(100)),
                        np.float32([-5, -0.01, 11, 1e9, 1e30])]).astype(np.float32)
    values = torch.from_numpy(v).to(DEV)
    table = torch.randn(101, generator=gen(101), device=DEV)
    for max_bin in (100, 60, 0):
        out = nan_f32(len(v) + 1)
        L.call("dirb200_lds_table_lookup", L.ptr(values), len(v), 10.0, max_bin, L.ptr(table), L.ptr(out), L.stream_ptr())
        torch.cuda.synchronize()
        b = np.clip(np.trunc(v * np.float32(10)), 0, max_bin).astype(np.int64)
        assert out[len(v)].isnan()
        check_bits(f"table lookup (max_bin {max_bin})", out[:len(v)], table[torch.from_numpy(b).to(DEV)])


# --------------------------------------------------------------------------------------------------------- reruns
@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"},
                                 {"DIRB200_FDS_SMALL": "0", "DIRB200_FDS_RPC": "1", "DIRB200_FDS_BLOCK": "256"}],
                         ids=["seven_sms", "grid_sort_one_row_chunks"])
def test_fds_loss_kernels_rerun(env):
    """This file again in a subprocess (the variables are read once per process): with the grids capped at 7 SMs, and
    with the accumulate's single-CTA sort off, one row per chunk (a flush at every row) and 256-thread CTAs."""
    if os.environ.get("DIRB200_FDS_LOSS_RERUN"):
        pytest.skip("already a rerun")
    e = dict(os.environ, DIRB200_FDS_LOSS_RERUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__)],
                       env=e, cwd=ROOT, capture_output=True, text=True, timeout=2400)
    assert r.returncode == 0, r.stdout[-4000:] + r.stderr[-2000:]
