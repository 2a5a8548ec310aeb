"""CPU oracle for the DIR hot path (FDS / LDS / weighted losses / calibration).

TEST INFRASTRUCTURE ONLY.  Nothing in the product path
(`imbalanced-regression_b200/`) may import this module; only `tests/`,
`__graft_entry__.smoke()` and `bench.py`'s cpu_baseline / `--impl reference`
legs do, and only as the checker / the timed CPU baseline.

Each function is an independent numpy restatement of the reference algorithm
(YyzHarry/imbalanced-regression @ a6fdc45) and cites the reference lines it
follows.  The restatement is pinned against the reference itself: the
fixtures in `tests/golden/*.npz` were produced by importing the reference's
own modules (see `tests/golden/make_golden.py`) and
`tests/test_oracle_golden.py` checks this file against them.  The reference
ships no tests / golden vectors of its own (SURVEY.md §4), so this is the
strongest pin available.
"""
from __future__ import annotations

import math
import numpy as np


# --------------------------------------------------------------------------
# kernel windows
# --------------------------------------------------------------------------
def _gaussian_impulse_response(ks: int, sigma: float, dtype) -> np.ndarray:
    """scipy.ndimage.gaussian_filter1d applied to a centred unit impulse of
    length ks, default mode='reflect', truncate=4.0 -- restated without scipy.

    The filter radius is int(4*sigma+0.5); taps that fall outside the ks-long
    signal are folded back by (half-sample symmetric) reflection, which is why
    the FDS / LDS windows are not plain sampled Gaussians.
    (agedb-dir/fds.py:41-44, agedb-dir/utils.py:113-115)
    """
    half = (ks - 1) // 2
    radius = int(4.0 * float(sigma) + 0.5)
    x = np.arange(-radius, radius + 1, dtype=np.float64)
    phi = np.exp(-0.5 / (float(sigma) * float(sigma)) * x ** 2)
    phi = phi / phi.sum()
    sig = np.zeros(ks, dtype=np.float64)
    sig[half] = 1.0
    out = np.zeros(ks, dtype=np.float64)
    period = 2 * ks
    for i in range(ks):
        acc = 0.0
        for j in range(-radius, radius + 1):
            # correlate1d with a symmetric kernel; index i+j reflected
            # ("reflect" == half-sample symmetric: d c b a | a b c d | d c b a)
            k = (i + j) % period
            if k < 0:
                k += period
            if k >= ks:
                k = period - 1 - k
            acc += phi[j + radius] * sig[k]
        out[i] = acc
    return out.astype(dtype)


def fds_kernel_window(kernel: str, ks: int, sigma: float) -> np.ndarray:
    """FDS smoothing window, float32, normalised to sum 1.
    (agedb-dir/fds.py:37-52)"""
    assert kernel in ("gaussian", "triang", "laplace")
    half = (ks - 1) // 2
    if kernel == "gaussian":
        g = _gaussian_impulse_response(ks, sigma, np.float32)
        w = g / sum(g)
    elif kernel == "triang":
        t = triang_window(ks)
        w = t / sum(t)
    else:
        lap = [math.exp(-abs(x) / sigma) / (2.0 * sigma) for x in range(-half, half + 1)]
        w = np.asarray(lap) / sum(lap)
    return np.asarray(w, dtype=np.float32)


def lds_kernel_window(kernel: str, ks: int, sigma: float) -> np.ndarray:
    """LDS window, float64, normalised to max 1.  (agedb-dir/utils.py:110-122)"""
    assert kernel in ("gaussian", "triang", "laplace")
    half = (ks - 1) // 2
    if kernel == "gaussian":
        g = _gaussian_impulse_response(ks, sigma, np.float64)
        w = g / max(g)
    elif kernel == "triang":
        w = triang_window(ks)
    else:
        lap = [math.exp(-abs(x) / sigma) / (2.0 * sigma) for x in range(-half, half + 1)]
        w = np.asarray(lap) / max(lap)
    return np.asarray(w, dtype=np.float64)


def triang_window(m: int) -> np.ndarray:
    """scipy.signal.windows.triang(M) (symmetric) restated."""
    n = np.arange(1, (m + 1) // 2 + 1, dtype=np.float64)
    if m % 2 == 0:
        w = (2 * n - 1.0) / m
        return np.concatenate([w, w[::-1]])
    w = 2 * n / (m + 1.0)
    return np.concatenate([w, w[-2::-1]])


# --------------------------------------------------------------------------
# LDS weights
# --------------------------------------------------------------------------
def lds_histogram(labels, max_target: int = 121) -> np.ndarray:
    """bin = min(max_target-1, int(label)); int64 counts.
    (agedb-dir/datasets.py:60-63)"""
    hist = np.zeros(max_target, dtype=np.int64)
    for v in np.asarray(labels).reshape(-1):
        hist[min(max_target - 1, int(v))] += 1
    return hist


def convolve1d_constant(x: np.ndarray, w: np.ndarray) -> np.ndarray:
    """scipy.ndimage.convolve1d(x, w, mode='constant') for an odd-length
    SYMMETRIC w, restated with scipy's own accumulation order (its symmetric
    fast path: centre tap first, then (x[i-j] + x[i+j]) * w[j] from the outermost
    pair inwards, float64, no fused multiply-add) and its output-dtype rule:
    the result takes the INPUT's dtype, so an integer histogram (the
    'inverse' re-weighting, np.clip of Python ints) is truncated back to
    int64, while the sqrt_inv histogram stays float64.
    (agedb-dir/datasets.py:66-67, 76-77)"""
    x = np.asarray(x)
    xd = x.astype(np.float64)
    w = np.asarray(w, dtype=np.float64)
    h = len(w) // 2
    assert len(w) % 2 == 1 and np.all(np.abs(w - w[::-1]) <= np.finfo(np.float64).eps)
    n = len(xd)
    pad = np.concatenate([np.zeros(h), xd, np.zeros(h)])
    out = np.zeros(n, dtype=np.float64)
    for i in range(n):
        c = i + h
        acc = pad[c] * w[h]
        for j in range(-h, 0):
            acc = acc + (pad[c + j] + pad[c - j]) * w[h + j]
        out[i] = acc
    if np.issubdtype(x.dtype, np.integer):
        return np.trunc(out).astype(np.int64)
    return out


def lds_weights(labels, reweight: str, max_target: int = 121, lds: bool = False,
                lds_kernel: str = "gaussian", lds_ks: int = 5, lds_sigma: float = 2):
    """Per-sample loss weights.  (agedb-dir/datasets.py:55-83)
    Returns (hist int64[max_target], weights float32[N]) or (hist, None)."""
    assert reweight in ("none", "inverse", "sqrt_inv")
    assert reweight != "none" if lds else True
    labels = np.asarray(labels).reshape(-1)
    hist = lds_histogram(labels, max_target)
    if reweight == "none" or labels.size == 0:
        return hist, None
    if reweight == "sqrt_inv":
        val = np.sqrt(hist.astype(np.float64))
    else:
        val = np.clip(hist, 5, 1000)                   # stays int64 (see convolve1d_constant)
    if lds:
        val = convolve1d_constant(val, lds_kernel_window(lds_kernel, lds_ks, lds_sigma))
    bins = np.minimum(max_target - 1, labels.astype(np.int64))
    w = (1.0 / val[bins]).astype(np.float32)          # np.float32(1 / x)  :80
    scaling = np.float32(len(w)) / np.sum(w)           # float32 pairwise sum :81
    return hist, (np.float32(scaling) * w).astype(np.float32)


# --------------------------------------------------------------------------
# FDS
# --------------------------------------------------------------------------
def fds_bin_index(labels, bucket_num: int, bucket_start: int) -> np.ndarray:
    """Row -> FDS table row, reproducing the unique-label loop's three masks
    (agedb-dir/fds.py:91-99, 120-143).  -1 == row not touched.
    Out-of-range labels fold into an edge bin only when the edge value itself
    occurs among the labels.  Contract: integer-valued labels."""
    lab = np.asarray(labels, dtype=np.float32).reshape(-1)
    lo, hi = np.float32(bucket_start), np.float32(bucket_num - 1)
    has_lo = bool((lab == lo).any())
    has_hi = bool((lab == hi).any())
    out = np.full(lab.shape, -1, dtype=np.int32)
    inr = (lab >= lo) & (lab <= hi)
    out[inr] = (lab[inr] - lo).astype(np.int32)
    if has_lo:
        out[lab < lo] = 0
    if has_hi:
        out[lab > hi] = int(bucket_num - 1 - bucket_start)
    return out


def fds_batch_stats(features, labels, bucket_num, bucket_start):
    """Per-bin (count, mean, unbiased var [0 when n==1]) in float64 -> float32.
    (agedb-dir/fds.py:100-102)"""
    f = np.asarray(features, dtype=np.float64)
    bins = fds_bin_index(labels, bucket_num, bucket_start)
    nb = bucket_num - bucket_start
    cnt = np.zeros(nb, dtype=np.int64)
    mean = np.zeros((nb, f.shape[1]), dtype=np.float32)
    var = np.zeros((nb, f.shape[1]), dtype=np.float32)
    for b in range(nb):
        rows = f[bins == b]
        n = rows.shape[0]
        cnt[b] = n
        if n == 0:
            continue
        mean[b] = rows.mean(0)
        var[b] = rows.var(0, ddof=1) if n > 1 else 0.0
    return cnt, mean, var


def fds_stats_from_bins(features, bins, nb):
    """Per-bin (count, mean, unbiased var [0 when n==1]) given the table row of every feature row (-1 = untouched):
    the same quantities as fds_batch_stats / agedb-dir/fds.py:100-102, computed with one stable sort and segmented
    float64 sums so that BASELINE-size inputs (2.46 M rows x 128, 5 749 rows x 12 000) finish in seconds.  Pinned to
    the per-bin loop of fds_batch_stats by tests/test_oracle_golden.py."""
    f = np.asarray(features)
    bins = np.asarray(bins).reshape(-1)
    keep = np.nonzero(bins >= 0)[0]
    order = keep[np.argsort(bins[keep], kind="stable")]
    sb = bins[order]
    cnt = np.bincount(sb, minlength=nb).astype(np.int64)
    mean = np.zeros((nb, f.shape[1]), dtype=np.float32)
    var = np.zeros((nb, f.shape[1]), dtype=np.float32)
    if order.size == 0:
        return cnt, mean, var
    starts = np.concatenate([[0], np.cumsum(cnt)[:-1]])
    present = np.nonzero(cnt)[0]
    # column blocks bound the float64 scratch (rows x 512 x 8 B)
    for c0 in range(0, f.shape[1], 512):
        blk = f[order, c0:c0 + 512].astype(np.float64)
        s1 = np.add.reduceat(blk, starts[present], axis=0)
        m = s1 / cnt[present, None]
        dev = blk - np.repeat(m, cnt[present], axis=0)
        s2 = np.add.reduceat(dev * dev, starts[present], axis=0)
        mean[present, c0:c0 + 512] = m
        v = np.where(cnt[present, None] > 1, s2 / np.maximum(cnt[present, None] - 1, 1), 0.0)
        var[present, c0:c0 + 512] = v
    return cnt, mean, var


class FDSState:
    """Numpy restatement of fds.FDS's buffers and state machine
    (agedb-dir/fds.py:16-35, 54-113), including the by-reference alias of
    `running_*_last_epoch` onto `running_*` (:55-56)."""

    def __init__(self, feature_dim, bucket_num=100, bucket_start=3, start_update=0,
                 start_smooth=1, kernel="gaussian", ks=5, sigma=2, momentum=0.9):
        nb = bucket_num - bucket_start
        self.feature_dim, self.bucket_num, self.bucket_start = feature_dim, bucket_num, bucket_start
        self.window = fds_kernel_window(kernel, ks, sigma)
        self.half_ks = (ks - 1) // 2
        self.momentum, self.start_update, self.start_smooth = momentum, start_update, start_smooth
        self.epoch = int(start_update)
        self.running_mean = np.zeros((nb, feature_dim), np.float32)
        self.running_var = np.ones((nb, feature_dim), np.float32)
        self.running_mean_last_epoch = np.zeros((nb, feature_dim), np.float32)
        self.running_var_last_epoch = np.ones((nb, feature_dim), np.float32)
        self.smoothed_mean_last_epoch = np.zeros((nb, feature_dim), np.float32)
        self.smoothed_var_last_epoch = np.ones((nb, feature_dim), np.float32)
        self.num_samples_tracked = np.zeros(nb, np.float32)

    def update_last_epoch_stats(self, epoch):                     # fds.py:78-82
        if epoch == self.epoch + 1:
            self.epoch += 1
            self.running_mean_last_epoch = self.running_mean      # alias  :55
            self.running_var_last_epoch = self.running_var        # alias  :56
            self.smoothed_mean_last_epoch = smooth_bins(self.running_mean, self.window)
            self.smoothed_var_last_epoch = smooth_bins(self.running_var, self.window)

    def update_running_stats(self, features, labels, epoch):      # fds.py:84-113
        if epoch < self.epoch:
            return
        cnt, mean, var = fds_batch_stats(features, labels, self.bucket_num, self.bucket_start)
        for b in np.nonzero(cnt)[0]:
            n = float(cnt[b])
            self.num_samples_tracked[b] += np.float32(n)
            factor = self.momentum if self.momentum is not None else \
                (1 - n / float(self.num_samples_tracked[b]))
            factor = 0 if epoch == self.start_update else factor
            a = np.float32(1 - factor)
            f = np.float32(factor)
            self.running_mean[b] = a * mean[b] + f * self.running_mean[b]
            self.running_var[b] = a * var[b] + f * self.running_var[b]

    def smooth(self, features, labels, epoch, clip=(0.1, 10.0)):  # fds.py:115-144
        if epoch < self.start_smooth:
            return features
        return fds_calibrate(features, np.asarray(labels).reshape(-1), self.bucket_num,
                             self.bucket_start, self.running_mean_last_epoch,
                             self.running_var_last_epoch, self.smoothed_mean_last_epoch,
                             self.smoothed_var_last_epoch, clip)


def smooth_bins(table: np.ndarray, window: np.ndarray) -> np.ndarray:
    """Reflect-pad by half_ks along the bin axis, then ks-tap correlation.
    (agedb-dir/fds.py:58-67; F.pad mode='reflect' excludes the edge sample.)"""
    t = np.asarray(table, dtype=np.float32)
    nb = t.shape[0]
    ks = len(window)
    h = (ks - 1) // 2
    out = np.zeros_like(t)
    for b in range(nb):
        acc = np.zeros(t.shape[1], dtype=np.float32)
        for j in range(ks):
            k = b + j - h
            if k < 0:
                k = -k
            if k >= nb:
                k = 2 * (nb - 1) - k
            acc = acc + np.float32(window[j]) * t[k]
        out[b] = acc
    return out


def calibrate_mean_var(matrix, m1, v1, m2, v2, clip_min=0.1, clip_max=10.0):
    """(agedb-dir/utils.py:97-107) float32, same operation order."""
    x = np.asarray(matrix, dtype=np.float32)
    m1, v1, m2, v2 = (np.asarray(a, dtype=np.float32) for a in (m1, v1, m2, v2))
    if np.sum(v1, dtype=np.float32) < 1e-10:
        return x
    valid = v1 != 0
    out = x.copy()
    with np.errstate(divide="ignore", invalid="ignore"):
        fac = np.clip(v2[valid] / v1[valid], np.float32(clip_min), np.float32(clip_max))
    out[:, valid] = (x[:, valid] - m1[valid]) * np.sqrt(fac) + m2[valid]
    return out


def fds_calibrate(features, labels, bucket_num, bucket_start, m1, v1, m2, v2, clip=(0.1, 10.0)):
    x = np.array(features, dtype=np.float32, copy=True)
    bins = fds_bin_index(labels, bucket_num, bucket_start)
    for b in np.unique(bins):
        if b < 0:
            continue
        rows = bins == b
        x[rows] = calibrate_mean_var(x[rows], m1[b], v1[b], m2[b], v2[b], clip[0], clip[1])
    return x


def fds_calibrate_scale(labels, bucket_num, bucket_start, v1, v2, clip=(0.1, 10.0)):
    """d(out)/d(in) of fds_calibrate per element (backward oracle)."""
    bins = fds_bin_index(labels, bucket_num, bucket_start)
    d = v1.shape[1]
    s = np.ones((len(bins), d), dtype=np.float32)
    for i, b in enumerate(bins):
        if b < 0 or np.sum(v1[b], dtype=np.float32) < 1e-10:
            continue
        valid = v1[b] != 0
        with np.errstate(divide="ignore", invalid="ignore"):
            fac = np.clip(v2[b][valid] / v1[b][valid], np.float32(clip[0]), np.float32(clip[1]))
        s[i, valid] = np.sqrt(fac)
    return s


# --------------------------------------------------------------------------
# weighted losses  (agedb-dir/loss.py:5-48) -- forward and d/d(inputs)
# --------------------------------------------------------------------------
def _sigmoid(x):
    return 1.0 / (1.0 + np.exp(-x))


def weighted_loss(kind, inputs, targets, weights=None, activate="sigmoid", beta=None, gamma=1.0):
    """Returns (loss float32 scalar, dloss/dinputs float32).  float64 inside."""
    x = np.asarray(inputs, dtype=np.float64)
    t = np.asarray(targets, dtype=np.float64)
    d = x - t
    a = np.abs(d)
    sg = np.sign(d)
    n = d.size
    if kind == "mse":
        l, g = d * d, 2 * d
    elif kind == "l1":
        l, g = a, sg
    elif kind in ("focal_mse", "focal_l1"):
        beta = 0.2 if beta is None else beta
        if activate == "tanh":
            fb = np.tanh(beta * a)
            dfb = beta * (1 - fb * fb)
        else:
            s = _sigmoid(beta * a)
            fb = 2 * s - 1
            dfb = 2 * beta * s * (1 - s)
        f = fb ** gamma
        df = (gamma * np.where(gamma == 1.0, 1.0, fb ** (gamma - 1.0))) * dfb  # d f / d a
        if kind == "focal_mse":
            l = d * d * f
            g = 2 * d * f + d * d * df * sg
        else:
            l = a * f
            g = sg * f + a * df * sg
    elif kind == "huber":
        beta = 1.0 if beta is None else beta
        small = a < beta
        l = np.where(small, 0.5 * a * a / beta, a - 0.5 * beta)
        g = np.where(small, d / beta, sg)
    else:
        raise ValueError(kind)
    if weights is not None:
        w = np.broadcast_to(np.asarray(weights, dtype=np.float64), d.shape)
        l, g = l * w, g * w
    return np.float32(l.mean()), (g / n).astype(np.float32)


# --------------------------------------------------------------------------
# FDS variants of nyud2-dir / sts-b-dir (SURVEY.md §8 rows f-2 / f-3)
# --------------------------------------------------------------------------
def bin_index_depth10(labels, bucket_num, bucket_start):
    """clamp(int(float32(label) * float32(10)), bucket_start, bucket_num - 1) - bucket_start
    (nyud2-dir/models/fds.py:51-53)."""
    lab = np.asarray(labels, dtype=np.float32).reshape(-1)
    b = (lab * np.float32(10)).astype(np.int64)
    return (np.clip(b, bucket_start, bucket_num - 1) - bucket_start).astype(np.int32)


def bin_index_edges5(labels, bucket_num, bucket_start):
    """np.histogram-style buckets over [0, 5] (sts-b-dir/fds.py:51-57): the first float32 edge greater than the
    label, minus one; label == 5 -> last bucket; clamped below by bucket_start."""
    lab = np.asarray(labels, dtype=np.float32).reshape(-1)
    edges = np.linspace(0.0, 5.0, bucket_num + 1).astype(np.float32)
    out = np.empty(lab.shape, dtype=np.int32)
    for i, v in enumerate(lab):
        if v == np.float32(5.0):
            out[i] = bucket_num - 1
        else:
            out[i] = max(int(np.nonzero(edges > v)[0][0]) - 1, bucket_start)
    return out - bucket_start


def calibrate_mean_var_v2(matrix, m1, v1, m2, v2, clip_min, clip_max):
    """nyud2-dir/util.py:151-162 == sts-b-dir/util.py:63-73, AS IT BEHAVES on PyTorch >= 1.2: the mask
    `((v1 > 0.) + (v2 >= 0.)) == 2` adds two bool tensors (a logical OR) and compares with 2, which is never
    true -- so if any channel has v1 <= 0 or v2 < 0 the matrix comes back unchanged; otherwise all channels are
    calibrated.  (The fixtures were produced by running the reference, so they pin exactly this.)"""
    x = np.asarray(matrix, dtype=np.float32)
    m1, v1, m2, v2 = (np.asarray(a, dtype=np.float32) for a in (m1, v1, m2, v2))
    if np.sum(v1, dtype=np.float32) < 1e-10:
        return x
    if (v1 <= 0).any() or (v2 < 0).any():
        return x
    fac = np.clip(v2 / v1, np.float32(clip_min), np.float32(clip_max))
    return (x - m1) * np.sqrt(fac) + m2


class FDSVariantState(FDSState):
    """FDSState with another bucket rule.  variant 'nyud2': rows = pixels of [B,C,H,W] maps, clip (0.2, 5),
    no alias of the last-epoch tables (device hops); variant 'stsb': edge buckets, clip (0.5, 2), empty buckets
    filled from their neighbours after every update (sts-b-dir/fds.py:112-125), alias kept."""

    def __init__(self, variant, feature_dim, bucket_num, bucket_start, **kw):
        super().__init__(feature_dim, bucket_num, bucket_start, **kw)
        self.variant = variant
        self.clip = (0.2, 5.0) if variant == "nyud2" else (0.5, 2.0)
        self.bin_fn = bin_index_depth10 if variant == "nyud2" else bin_index_edges5

    def update_last_epoch_stats(self, epoch):
        was = self.epoch
        super().update_last_epoch_stats(epoch)
        if self.variant == "nyud2" and self.epoch != was:
            self.running_mean_last_epoch = self.running_mean.copy()
            self.running_var_last_epoch = self.running_var.copy()

    def _rows(self, features, labels):
        f = np.asarray(features, dtype=np.float32)
        if f.ndim == 4:
            f = f.transpose(0, 2, 3, 1).reshape(-1, f.shape[1])
        return f, np.asarray(labels, dtype=np.float32).reshape(-1)

    def update_running_stats(self, features, labels, epoch):
        if epoch < self.epoch:
            return
        f, lab = self._rows(features, labels)
        bins = self.bin_fn(lab, self.bucket_num, self.bucket_start)
        nb = self.bucket_num - self.bucket_start
        seen = np.zeros(nb, dtype=bool)
        for b in np.unique(bins):
            rows = f[bins == b].astype(np.float64)
            n = rows.shape[0]
            seen[b] = True
            self.num_samples_tracked[b] += np.float32(n)
            factor = self.momentum if self.momentum is not None else (1 - n / float(self.num_samples_tracked[b]))
            factor = 0 if epoch == self.start_update else factor
            a, fm = np.float32(1 - factor), np.float32(factor)
            mean = rows.mean(0).astype(np.float32)
            var = (rows.var(0, ddof=1) if n > 1 else np.zeros(rows.shape[1])).astype(np.float32)
            self.running_mean[b] = a * mean + fm * self.running_mean[b]
            self.running_var[b] = a * var + fm * self.running_var[b]
        if self.variant == "stsb":
            for b in range(nb):
                if seen[b]:
                    continue
                for t in (self.running_mean, self.running_var):
                    if b == 0:
                        t[0] = t[1]
                    elif b == nb - 1:
                        t[b] = t[b - 1]
                    else:
                        t[b] = (t[b - 1] + t[b + 1]) / np.float32(2.0)

    def smooth(self, features, labels, epoch):
        if epoch < self.start_smooth:
            return np.asarray(features, dtype=np.float32)
        shape = np.asarray(features).shape
        f, lab = self._rows(features, labels)
        bins = self.bin_fn(lab, self.bucket_num, self.bucket_start)
        x = f.copy()
        for b in np.unique(bins):
            rows = bins == b
            x[rows] = calibrate_mean_var_v2(x[rows], self.running_mean_last_epoch[b], self.running_var_last_epoch[b],
                                            self.smoothed_mean_last_epoch[b], self.smoothed_var_last_epoch[b],
                                            *self.clip)
        if len(shape) == 4:
            bsz, c, h, w = shape
            return x.reshape(bsz, h, w, c).transpose(0, 3, 1, 2)
        return x


# --------------------------------------------------------------------------
# evaluation metrics
# --------------------------------------------------------------------------
def shot_metrics(preds, labels, train_labels, many_shot_thr: int = 100, low_shot_thr: int = 20) -> dict:
    """Many / median / low-shot MSE, L1, G-Mean -- follows agedb-dir/train.py:338-391 (+ 'overall', :286-335).

    Group of a test sample = by the number of training samples whose int(label) equals the sample's label value:
    > many_shot_thr -> many, < low_shot_thr -> low, else median (train.py:366-381).  Vectorised instead of the
    reference's loop over np.unique(labels); sums in float64."""
    preds = np.asarray(preds, dtype=np.float32).reshape(-1)
    labels = np.asarray(labels, dtype=np.float32).reshape(-1)
    tl = np.asarray(train_labels).astype(int).reshape(-1)                     # train.py:339
    counts = np.asarray([np.count_nonzero(tl == l) for l in labels])         # len(train_labels[train_labels == l])
    err = (preds - labels).astype(np.float64)                                 # float32 difference, widened
    groups = {"overall": np.ones(labels.shape, bool), "many": counts > many_shot_thr, "low": counts < low_shot_thr}
    groups["median"] = ~groups["many"] & ~groups["low"]
    out = {}
    with np.errstate(divide="ignore", invalid="ignore"):
        for name, m in groups.items():
            n = np.count_nonzero(m)
            e = err[m]
            out[name] = {"mse": np.sum(e * e) / n, "l1": np.sum(np.abs(e)) / n,
                         "gmean": float(np.exp(np.sum(np.log(np.abs(e))) / n)), "count": int(n)}
    return out


# --------------------------------------------------------------------------
# STS-B re-weighting / LDS (SURVEY.md §8 row f-3)
# --------------------------------------------------------------------------
def stsb_lds_weights(scores, reweight: str, lds: bool = False, lds_kernel: str = "gaussian", lds_ks: int = 5,
                     lds_sigma: float = 2, bucket_num: int = 50):
    """Per-sentence-pair loss weights of sts-b-dir/tasks.py:44-73: histogram of the float32 scores over `bucket_num`
    equal bins of [0, 5] (np.histogram edges in the scores' dtype; score == 5 -> last bin), sqrt for 'sqrt_inv',
    optional LDS convolve (zero padded; an integer histogram -- the 'inverse' path -- is truncated back to integers
    by scipy, as in the age datasets), w = float32(1 / value[bin]) rescaled to mean 1.  No clipping of the counts
    here (unlike agedb-dir/datasets.py:66-67).  Returns (hist int64[bucket_num], weights float32[N])."""
    assert reweight in ("inverse", "sqrt_inv")
    s = np.asarray(scores, dtype=np.float32).reshape(-1)
    bins = bin_index_edges5(s, bucket_num, 0).astype(np.int64)
    hist = np.bincount(bins, minlength=bucket_num).astype(np.int64)
    val = np.sqrt(hist.astype(np.float64)) if reweight == "sqrt_inv" else hist
    if lds:
        val = convolve1d_constant(val, lds_kernel_window(lds_kernel, lds_ks, lds_sigma))
    with np.errstate(divide="ignore"):
        w = (1.0 / np.asarray(val)[bins]).astype(np.float32)            # np.float32(1 / x)        tasks.py:69
    scaling = np.float32(len(w)) / np.sum(w)                             # float32 sum             tasks.py:70
    return hist, (np.float32(scaling) * w).astype(np.float32)
