"""GPU parity of the evaluation reductions (dirb200_int_label_histogram / dirb200_shot_metrics through the
train.py mirror) against the reference-generated fixture and the numpy oracle.  Counts and the histogram are
integers (bit-exact); the error sums are fp64 on both sides (1e-6 relative, the float32 difference is shared).

The group edges (training counts 19 / 20 / 21 / 99 / 100 / 101, many == low, labels absent from training, not integer
valued, above every training label and 0, one exact zero error) against the reference's own rows
(tests/golden/shot_edges.npz); the histogram's truncation, NaN and range rules; empty groups; sizes 1 ... 600 003;
train.validate against the reference's validate; two identical calls giving identical bits.  The file reruns itself
with DIRB200_SMS=7."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
from util import golden, assert_close
from oracle import dir_oracle as O

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rows(sd):
    return [[sd[k][m] for m in ("mse", "l1", "gmean")] for k in ("many", "median", "low")]


@pytest.mark.parametrize("tag", ["a", "b"])
def test_shot_metrics_vs_reference_golden(tag):
    import train as T
    g = golden("metrics")
    sd = T.shot_metrics(torch.from_numpy(g[f"{tag}_preds"]).cuda(), torch.from_numpy(g[f"{tag}_labels"]).cuda(),
                        g["train_labels"])
    assert_close(_rows(sd), g[f"{tag}_ref"], rtol=1e-6, atol=1e-12, what=f"shot metrics {tag}")
    assert_close([sd["overall"][m] for m in ("mse", "l1", "gmean")], g[f"{tag}_overall"], rtol=1e-6, atol=1e-12)


def test_shot_metrics_large_random_vs_oracle_and_exact_counts():
    import _lib
    rng = np.random.RandomState(5)
    train = np.clip(np.round(rng.gamma(6.0, 6.5, size=191509)), 0, 140).astype(np.float32)   # IMDB-WIKI-sized column
    labels = np.clip(np.round(rng.gamma(6.0, 6.5, size=50000)), 0, 150).astype(np.float32)
    labels[::501] += 0.5                                   # non-integer label values: training count 0 -> low shot
    preds = (labels + rng.randn(labels.size) * 5).astype(np.float32)
    dev = torch.device("cuda")
    t, l, p = (torch.from_numpy(a).to(dev) for a in (train, labels, preds))
    nbins = 160
    hist = torch.zeros(nbins, dtype=torch.int64, device=dev)
    _lib.call("dirb200_int_label_histogram", _lib.ptr(t), t.numel(), nbins, _lib.ptr(hist), _lib.stream_ptr())
    assert np.array_equal(hist.cpu().numpy(), np.bincount(train.astype(int), minlength=nbins))   # bit-exact
    out = torch.empty(4, 4, dtype=torch.float64, device=dev)
    _lib.call("dirb200_shot_metrics", _lib.ptr(p), _lib.ptr(l), p.numel(), _lib.ptr(hist), nbins, 100, 20,
              _lib.ptr(out), _lib.stream_ptr())
    o = out.cpu().numpy()
    want = O.shot_metrics(preds, labels, train)
    for row, name in enumerate(("overall", "many", "median", "low")):
        assert int(o[row, 0]) == want[name]["count"], name                                       # bit-exact
        assert_close([o[row, 1] / o[row, 0], o[row, 2] / o[row, 0], np.exp(o[row, 3] / o[row, 0])],
                     [want[name][m] for m in ("mse", "l1", "gmean")], rtol=1e-6, atol=1e-12, what=name)
    assert int(o[0, 0]) == labels.size and int(o[1, 0] + o[2, 0] + o[3, 0]) == labels.size


def test_validate_mirror_reports_overall_and_shots():
    import train as T

    class Const(torch.nn.Module):
        def forward(self, x):
            return x[:, :1] * 0 + 30.0

    labels = torch.tensor([[25.], [30.], [41.], [30.]])
    loader = [(torch.zeros(2, 3), labels[:2], None), (torch.zeros(2, 3), labels[2:], None)]
    mse, l1, gm = T.validate(loader, Const().cuda(), train_labels=np.asarray([30] * 150 + [25] * 50 + [41] * 3))
    assert abs(mse - (25 + 0 + 121 + 0) / 4) < 1e-9 and abs(l1 - (5 + 0 + 11 + 0) / 4) < 1e-9 and gm == 0.0


# ------------------------------------------------------------------------------------------ group edges and sizes
def device_sums(preds, labels, train, many=100, low=20):
    """dirb200_int_label_histogram + dirb200_shot_metrics as train.shot_metrics calls them: (out[4][4], hist)."""
    import _lib
    dev = torch.device("cuda")
    p, l, t = (torch.as_tensor(np.asarray(a, np.float32)).reshape(-1).to(dev) for a in (preds, labels, train))
    top = lambda a: float(np.nanmax(a)) if np.asarray(a).size and not np.isnan(a).all() else 0.0
    nbins = int(max(top(train), top(labels), 0.0)) + 2
    hist = torch.zeros(nbins, dtype=torch.int64, device=dev)
    _lib.call("dirb200_int_label_histogram", _lib.ptr(t), t.numel(), nbins, _lib.ptr(hist), _lib.stream_ptr())
    out = torch.full((4, 4), float("nan"), dtype=torch.float64, device=dev)
    _lib.call("dirb200_shot_metrics", _lib.ptr(p), _lib.ptr(l), p.numel(), _lib.ptr(hist), nbins, many, low,
              _lib.ptr(out), _lib.stream_ptr())
    return out.cpu().numpy(), hist.cpu().numpy()


def sums64(preds, labels, train, many=100, low=20):
    """float64 restatement of the per-group (count, sum d^2, sum |d|, sum log|d|) with the training counts looked up
    by int(train_label) (dir_oracle.shot_metrics' rule, vectorised for large inputs); d is the float32 difference."""
    tl = np.asarray(train, np.float32)
    tl = tl[~np.isnan(tl)].astype(np.int64)
    hist = np.bincount(tl[tl >= 0], minlength=1)
    lab = np.asarray(labels, np.float32)
    hit = (lab == np.floor(lab)) & (lab >= 0) & (lab < hist.size)
    count = np.where(hit, hist[np.where(hit, lab, 0).astype(np.int64)], 0)
    d = (np.asarray(preds, np.float32) - lab).astype(np.float64)
    groups = [np.ones(lab.shape, bool), count > many, (count <= many) & (count >= low), count < low]
    with np.errstate(divide="ignore"):
        return np.asarray([[m.sum(), np.sum(d[m] ** 2), np.sum(np.abs(d[m])), np.sum(np.log(np.abs(d[m])))]
                           for m in groups])


def assert_sums(o, want, rtol):
    assert np.array_equal(o[:, 0], want[:, 0]), (o[:, 0], want[:, 0])                      # counts: exact
    for row in range(4):
        c = want[row, 0]
        if c == 0:
            assert np.array_equal(o[row, 1:], [0.0, 0.0, 0.0]), row                        # empty group: exact zeros
            continue
        got = [o[row, 1] / c, o[row, 2] / c, np.exp(o[row, 3] / c)]
        ref = [want[row, 1] / c, want[row, 2] / c, np.exp(want[row, 3] / c)]
        assert_close(got, ref, rtol=rtol, atol=0.0, what=f"row {row}")


@pytest.mark.parametrize("tag", ["edges", "equal", "zero"])
def test_shot_group_edges_vs_reference_golden(tag):
    """Training counts 19 / 20 / 21 / 99 / 100 / 101 at (100, 20), counts 4 / 5 / 6 at many == low == 5, labels with
    a fractional part, absent from training, above every training label and 0, a -0.5 and a 13.6 training label
    (counted by int()), NaN training labels: the reference's own rows (its float32 sums: 1e-6) and the oracle's exact
    group counts."""
    import train as T
    g = golden("shot_edges")
    train, labels, preds = g[f"{tag}_train"], g[f"{tag}_labels"], g[f"{tag}_preds"]
    many, low = (int(v) for v in g[f"{tag}_thr"])
    sd = T.shot_metrics(torch.from_numpy(preds).cuda(), torch.from_numpy(labels).cuda(), train, many, low)
    assert_close(_rows(sd), g[f"{tag}_ref"], rtol=1e-6, atol=0.0, what=f"shot rows {tag}")
    o, _ = device_sums(preds, labels, train, many, low)
    with np.errstate(invalid="ignore"):
        want = O.shot_metrics(preds, labels, train, many, low)
    assert [int(o[r, 0]) for r in range(4)] == [want[k]["count"] for k in ("overall", "many", "median", "low")]
    assert_sums(o, sums64(preds, labels, train, many, low), rtol=1e-12)
    if tag == "zero":                     # the exact hit zeroes the median G-Mean only; many / low keep their bits
        ref = T.shot_metrics(g["edges_preds"], labels, train, many, low)
        assert sd["median"]["gmean"] == 0.0 and sd["overall"]["gmean"] == 0.0
        for k in ("many", "low"):
            assert sd[k] == ref[k], k


def test_int_label_histogram_truncates_skips_nan_and_drops_out_of_range():
    """int(label) toward zero (-0.5 and -0.99 -> bin 0, as C and numpy's astype(int)), NaN skipped, bins < 0 and
    >= nbins dropped; the counts are ADDED to what the histogram holds."""
    import _lib
    nbins = 8
    vals = np.asarray([-0.5, -0.99, -1.0, -1.5, 0.0, 0.999, np.nan, 1.0, 6.999, 7.0, 7.5, 8.0, 11.0, 1e9, -1e9,
                       3.5, np.nan, 2.0], np.float32)
    rng = np.random.RandomState(3)
    for n in (vals.size, 700_001):                        # the second: every thread of the 4 x SMs grid loops
        t = vals if n == vals.size else rng.choice(vals, n)
        dev = torch.device("cuda")
        hist = torch.arange(nbins, dtype=torch.int64, device=dev) * 1000
        tt = torch.from_numpy(t).to(dev)
        _lib.call("dirb200_int_label_histogram", _lib.ptr(tt), tt.numel(), nbins, _lib.ptr(hist), _lib.stream_ptr())
        b = t[~np.isnan(t)].astype(np.int64)
        want = np.bincount(b[(b >= 0) & (b < nbins)], minlength=nbins) + np.arange(nbins) * 1000
        assert np.array_equal(hist.cpu().numpy(), want), n


@pytest.mark.parametrize("case", ["all_many", "all_median", "all_low", "no_training_labels"])
def test_empty_groups_report_zero_count_and_nan(case):
    """The reference raises on an empty group (np.hstack([])); the driver reports count 0 and NaN means, as the
    oracle does, and the other groups as usual."""
    import train as T
    rng = np.random.RandomState(7)
    train = {"all_many": np.full(300, 5.0), "all_median": np.full(50, 5.0), "all_low": np.full(3, 5.0),
             "no_training_labels": np.zeros(0)}[case].astype(np.float32)
    labels = np.full(37, 5.0, np.float32)
    preds = (labels + rng.randn(labels.size)).astype(np.float32)
    with np.errstate(invalid="ignore", divide="ignore"):
        want = O.shot_metrics(preds, labels, train)
        sd = T.shot_metrics(preds, labels, train)
    o, _ = device_sums(preds, labels, train)
    for row, k in enumerate(("overall", "many", "median", "low")):
        assert int(o[row, 0]) == want[k]["count"], k
        for m in ("mse", "l1", "gmean"):
            if want[k]["count"] == 0:
                assert np.isnan(sd[k][m]), (k, m)
            else:
                assert_close(sd[k][m], want[k][m], rtol=1e-12, atol=0.0, what=f"{k} {m}")


@pytest.mark.parametrize("n", [1, 255, 256, 257, 600_003])
def test_shot_metrics_sizes_vs_float64(n):
    """One sample, one CTA's worth +- 1, and 600 003 (every thread of the reducing CTA loops): counts exact, the
    means and G-Mean to 1e-12 of a float64 restatement (both sides sum in fp64, in different orders)."""
    rng = np.random.RandomState(n)
    train = np.clip(np.round(rng.gamma(6.0, 6.5, size=max(n, 20_000))), 0, 140).astype(np.float32)
    labels = np.clip(np.round(rng.gamma(6.0, 6.5, size=n)), 0, 150).astype(np.float32)
    labels[::7] += 0.25
    preds = (labels + rng.randn(n) * 5).astype(np.float32)
    o, _ = device_sums(preds, labels, train)
    assert_sums(o, sums64(preds, labels, train), rtol=1e-12)
    assert int(o[0, 0]) == n


class _Ident(torch.nn.Module):
    def forward(self, x):
        return x[:, :1]


def _reference_validate(batches):
    """agedb-dir/train.py:286-335 restated: per-batch float32 MSE / L1 means into batch-size-weighted AverageMeters,
    G-Mean = scipy.stats.gmean of the float32 |error| of every sample."""
    from scipy.stats import gmean
    from utils import AverageMeter
    mse, l1 = AverageMeter('mse'), AverageMeter('l1')
    errs = []
    for p, t in batches:
        d = p - t
        mse.update(float(np.mean(d * d, dtype=np.float32)), p.shape[0])
        l1.update(float(np.mean(np.abs(d), dtype=np.float32)), p.shape[0])
        errs.append(np.abs(d).reshape(-1))
    return mse.avg, l1.avg, float(gmean(np.concatenate(errs).astype(np.float64)))


def test_validate_matches_the_reference_validate(monkeypatch):
    """train.validate over a loader whose last batch is short (390 = 6 x 64 + 6): overall MSE / L1 within 1e-6 of the
    reference's AverageMeters of per-batch float32 means, G-Mean to 1e-12 of scipy.stats.gmean, and the many /
    median / low rows it computes against the reference's own rows."""
    import train as T
    g = golden("shot_edges")
    preds, labels, train = g["edges_preds"], g["edges_labels"], g["edges_train"]
    batches = [(preds[i:i + 64, None], labels[i:i + 64, None]) for i in range(0, labels.size, 64)]
    assert batches[-1][0].shape[0] == labels.size % 64 != 0
    loader = [(torch.from_numpy(p.copy()), torch.from_numpy(t.copy()), None) for p, t in batches]
    seen = []
    real = T.shot_metrics
    monkeypatch.setattr(T, "shot_metrics", lambda *a, **k: seen.append(real(*a, **k)) or seen[-1])
    mse, l1, gm = T.validate(loader, _Ident().cuda(), train_labels=train)
    want = _reference_validate(batches)
    assert_close([mse, l1], want[:2], rtol=1e-6, atol=0.0, what="overall mse / l1")
    assert_close(gm, want[2], rtol=1e-12, atol=0.0, what="overall gmean")
    assert len(seen) == 1
    assert_close(_rows(seen[0]), g["edges_ref"], rtol=1e-6, atol=0.0, what="validate's shot rows")


@pytest.mark.parametrize("n", [11_022, 600_003])
def test_identical_calls_give_identical_bits(n):
    """The IMDB-WIKI-DIR val / test size and a large one: two calls, the same 16 doubles bit for bit (the sums have a
    fixed order), and so the same metrics out of train.shot_metrics."""
    import train as T
    rng = np.random.RandomState(n + 1)
    train = np.clip(np.round(rng.gamma(6.0, 6.5, size=191_509)), 0, 186).astype(np.float32)
    labels = np.clip(np.round(rng.gamma(6.0, 6.5, size=n)), 0, 186).astype(np.float32)
    preds = (labels + rng.randn(n) * 7).astype(np.float32)
    a, _ = device_sums(preds, labels, train)
    b, _ = device_sums(preds, labels, train)
    assert a.tobytes() == b.tobytes()
    p, l = torch.from_numpy(preds).cuda(), torch.from_numpy(labels).cuda()
    assert T.shot_metrics(p, l, train) == T.shot_metrics(p, l, train)


# ------------------------------------------------------------------------------------------------- few SMs
@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_metrics_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process): the histogram's grid
    shrinks to 28 CTAs, so every thread loops at the sizes above."""
    if os.environ.get("DIRB200_METRICS_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_METRICS_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
