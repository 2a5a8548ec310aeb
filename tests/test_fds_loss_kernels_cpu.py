"""CPU-only companions of tests/test_gpu_fds_loss_kernels.py.

1. The restatements that file checks the kernels against are pinned here to what they restate: the EDGES5 rule to the
   reference's np.histogram edges on float32 labels, the depth rule to torch's fp32 `labels * 10`, and the LDS table /
   scaling restatement to oracle/dir_oracle.lds_weights.
2. Every FDS, loss and LDS entry point refuses bad arguments on the host, with a message, before any CUDA call.  The
   pointers are dummies that must never be dereferenced, so a call that got past its checks would fault on a GPU machine
   and fail without one.

Found by these tests: dirb200_fds_calibrate_bwd accepted an unknown bin_rule and more than 2^31 - 1 rows (its launch's
grid size is 32 bits: b = 2^32 + 1 processed one row and returned success), dirb200_fds_smooth_tables accepted d <= 0,
and dirb200_lds_weights / _sharded took a negative ks (odd and <= 33) as "no smoothing"."""
import ctypes

import numpy as np
import pytest
import torch

from test_gpu_fds_loss_kernels import AGE, DEPTH, EDGES5, bin_index, depth_sweep, edges_sweep, lds_restated

D = ctypes.c_void_p(16)               # stands for a device buffer
D2 = ctypes.c_void_p(32)              # another one (entry points that refuse aliasing)
BIG = (2 ** 31, 2 ** 32 + 1)


def lib():
    import _lib
    return _lib


def refused(name, *args, msg, rc=-1):
    L = lib()
    got = L.raw(name)(*args)
    err = L.last_error()
    assert got == rc and msg in err, (name, args, got, err)


# ----------------------------------------------------------------------------------------- restatements, pinned
@pytest.mark.parametrize("num,start", [(50, 0), (50, 4), (7, 0), (7, 2), (3, 0), (101, 0)])
def test_edges5_restatement_matches_np_histogram_edges(num, start):
    """sts-b-dir/fds.py's _get_bucket_idx: edges of np.histogram over (0, 5) with float32 input; label == 5 -> last;
    otherwise the first edge above the label, minus one, clamped below by bucket_start"""
    _, edges = np.histogram(np.array([], dtype=np.float32), bins=num, range=(0., 5.))
    v = edges_sweep(num)
    v = v[(v >= 0) & (v <= 5)]
    want = np.array([num - 1 if x == np.float32(5) else max(int(np.where(edges > x)[0][0]) - 1, start) for x in v])
    np.testing.assert_array_equal(bin_index(EDGES5, v, num, start), want - start)


@pytest.mark.parametrize("num,start", [(100, 7), (100, 0), (50, 3)])
def test_depth_restatement_matches_torch(num, start):
    v = depth_sweep()
    v = v[np.isfinite(v) & (np.abs(v) < 1e6)]
    want = (torch.from_numpy(v) * 10).long().clamp(start, num - 1) - start
    np.testing.assert_array_equal(bin_index(DEPTH, v, num, start), want.numpy())


@pytest.mark.parametrize("reweight,ks,kernel", [("sqrt_inv", 0, None), ("inverse", 0, None), ("sqrt_inv", 5, "gaussian"),
                                                ("inverse", 5, "gaussian"), ("inverse", 9, "triang"),
                                                ("sqrt_inv", 33, "laplace"), ("inverse", 33, "gaussian")])
def test_lds_restatement_matches_oracle(reweight, ks, kernel):
    """the per-bin table bit for bit; the scaling (a serial fp64 sum over bins in the kernel, a float32 pairwise sum over
    samples in the oracle) within 2^-18"""
    from oracle import dir_oracle as O
    rng = np.random.RandomState(ks)
    labels = np.clip(np.floor(rng.randn(20000) * 15 + 40), 0, 130)
    labels = labels[(labels < 60) | (labels > 70)].astype(np.float32)
    hist, want = O.lds_weights(labels, reweight, lds=ks > 0, lds_kernel=kernel or "gaussian", lds_ks=max(ks, 1),
                               lds_sigma=2)
    win = O.lds_kernel_window(kernel, ks, 2) if ks else None
    table, scaling = lds_restated(hist, reweight, win, labels.size)
    bins = np.minimum(120, labels.astype(np.int64))
    got = (scaling * table[bins].astype(np.float32)).astype(np.float32)
    ratio = got.astype(np.float64) / want
    assert np.all(np.abs(ratio - ratio[0]) <= 2.0 ** -22 * ratio[0]), "per-bin tables differ"
    assert abs(ratio[0] - 1) <= 2.0 ** -18, ratio[0]


# ------------------------------------------------------------------------------------------------ host refusals
def test_label_flags_and_bin_rows_refuse_bad_arguments():
    for rule in (-1, 3):
        refused("dirb200_fds_label_flags", D, 10, 100, 3, rule, D, None, msg="fds_label_flags: unknown bin_rule")
        refused("dirb200_fds_bin_rows", D, 10, 100, 3, rule, D, D, None, msg="fds_bin_rows: unknown bin_rule")
    for args in ((D, -1, 100, 3, AGE, D), (D, 10, 100, 3, AGE, None), (None, 10, 100, 3, AGE, D),
                 (D, 10, 3, 3, AGE, D), (D, 10, 2, 3, AGE, D)):
        refused("dirb200_fds_label_flags", *args, None, msg="fds_label_flags")
    for rule in (AGE, DEPTH, EDGES5):
        for args in ((D, -1, 100, 3, rule, D, D), (D, 10, 100, 3, rule, None, D), (D, 10, 100, 3, rule, D, None),
                     (None, 10, 100, 3, rule, D, D), (D, 10, 3, 3, rule, D, D)):
            refused("dirb200_fds_bin_rows", *args, None, msg="fds_bin_rows")


def acc_args(n=100, d=8, nb=10, feat=D, bins=D, sums=D, sumsq=D, counts=D, ws=D, ws_bytes=None):
    need = lib().raw("dirb200_fds_accumulate_workspace_bytes")(max(n, 0), max(nb, 1))
    return (feat, bins, n, d, nb, sums, sumsq, counts, ws, need if ws_bytes is None else ws_bytes, None)


@pytest.mark.parametrize("kw", [dict(n=-1), dict(d=0), dict(d=-4), dict(nb=0), dict(nb=8193), dict(n=2 ** 31),
                                dict(sums=None), dict(sumsq=None), dict(counts=None), dict(feat=None), dict(bins=None),
                                dict(ws=None)], ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_fds_accumulate_refuses_bad_arguments(kw):
    refused("dirb200_fds_accumulate", *acc_args(**kw), msg="fds_accumulate")


def test_fds_accumulate_refuses_a_short_workspace():
    need = lib().raw("dirb200_fds_accumulate_workspace_bytes")(100, 10)
    refused("dirb200_fds_accumulate", *acc_args(ws_bytes=need - 1), msg="workspace too small", rc=-3)


def test_fds_finalize_and_fill_empty_refuse_bad_arguments():
    base = [D, D, D, 10, 8, D, D, D, 0.9, 0, None]
    for k, v in ((0, None), (1, None), (2, None), (5, None), (6, None), (7, None), (3, 0), (3, -1), (4, 0), (4, -1)):
        a = list(base)
        a[k] = v
        refused("dirb200_fds_finalize", *a, msg="fds_finalize")
    base = [D, 10, 8, D, D, None]
    for k, v in ((0, None), (3, None), (4, None), (1, 0), (1, -1), (2, 0), (2, -1)):
        a = list(base)
        a[k] = v
        refused("dirb200_fds_fill_empty", *a, msg="fds_fill_empty")


def test_fds_smooth_tables_refuses_bad_arguments():
    w = np.ones(33, dtype=np.float32)
    wp = w.ctypes.data_as(ctypes.c_void_p)
    base = [D, 100, 8, wp, 5, D2, None]
    for k, v in ((0, None), (3, None), (5, None), (5, D), (4, 0), (4, 4), (4, 35), (4, -1), (1, 2), (1, 0),
                 (2, 0), (2, -1)):
        a = list(base)
        a[k] = v
        refused("dirb200_fds_smooth_tables", *a, msg="fds_smooth_tables")
    a = list(base)
    a[1], a[4] = 16, 33                                      # 33 taps need 17 bins
    refused("dirb200_fds_smooth_tables", *a, msg="fds_smooth_tables")


def cal_fwd_args(b=100, d=8, bucket_num=100, bucket_start=3, rule=AGE, x=D, labels=D, m1=D, v1=D, m2=D, v2=D,
                 rowbin=D, flags=D):
    return (x, labels, b, d, bucket_num, bucket_start, rule, m1, v1, m2, v2, 0.1, 10.0, rowbin, flags, None)


@pytest.mark.parametrize("kw", [dict(rule=-1), dict(rule=3), dict(b=-1), dict(d=0), dict(d=-1), dict(bucket_num=3),
                                dict(x=None), dict(labels=None), dict(m1=None), dict(v1=None), dict(m2=None),
                                dict(v2=None), dict(rowbin=None), dict(b=3000, flags=None)] + [dict(b=b) for b in BIG],
                         ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_fds_calibrate_fwd_refuses_bad_arguments(kw):
    refused("dirb200_fds_calibrate_fwd", *cal_fwd_args(**kw), msg="fds_calibrate_fwd")


def cal_bwd_args(rule=AGE, gout=D, rowbin=D, b=100, d=8, v1=D, v2=D, gin=D):
    return (rule, gout, rowbin, b, d, v1, v2, 0.1, 10.0, gin, None)


@pytest.mark.parametrize("kw", [dict(rule=-1), dict(rule=3), dict(rule=99), dict(b=-1), dict(d=0), dict(d=-1),
                                dict(gout=None), dict(rowbin=None), dict(v1=None), dict(v2=None), dict(gin=None)] +
                         [dict(b=b) for b in BIG], ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_fds_calibrate_bwd_refuses_bad_arguments(kw):
    refused("dirb200_fds_calibrate_bwd", *cal_bwd_args(**kw), msg="fds_calibrate_bwd")


def loss_args(kind=0, pred=D, target=D, n=100, act=0, out=D, ws=D, ws_bytes=None):
    need = lib().raw("dirb200_loss_workspace_bytes")(max(n, 1))
    return (kind, pred, target, None, n, 1.0, 1.0, act, 1.0, out, D, ws, need if ws_bytes is None else ws_bytes, None)


@pytest.mark.parametrize("kw", [dict(kind=-1), dict(kind=5), dict(act=2), dict(act=-1), dict(n=0), dict(n=-1),
                                dict(pred=None), dict(target=None), dict(out=None), dict(ws=None)],
                         ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_loss_refuses_bad_arguments(kw):
    refused("dirb200_loss_fwd_bwd", *loss_args(**kw), msg="loss")


def test_loss_refuses_a_short_workspace():
    need = lib().raw("dirb200_loss_workspace_bytes")(100)
    refused("dirb200_loss_fwd_bwd", *loss_args(ws_bytes=need - 1), msg="workspace too small", rc=-3)


def test_lds_histogram_and_lookup_refuse_bad_arguments():
    for args in ((D, -1, 121, D), (D, 10, 0, D), (D, 10, 8193, D), (D, 10, 121, None), (None, 10, 121, D)):
        refused("dirb200_lds_histogram", *args, None, msg="lds_histogram")
    for args in ((D, -1, 10.0, 100, D, D), (D, 10, 10.0, -1, D, D), (D, 10, 10.0, 100, None, D),
                 (None, 10, 10.0, 100, D, D), (D, 10, 10.0, 100, D, None)):
        refused("dirb200_lds_table_lookup", *args, None, msg="lds_table_lookup")


def test_lds_weights_refuse_bad_arguments():
    sym = np.array([0.5, 1.0, 0.5])
    asym = np.array([0.5, 1.0, 0.25])
    wp = lambda a: a.ctypes.data_as(ctypes.c_void_p)
    # (labels, n, n_total, max_target, reweight, window, ks, hist, scratch, out)
    base = [D, 100, 100, 121, 1, wp(sym), 3, D, D, D]
    cases = [(4, 0), (4, 3), (1, 0), (1, -1), (2, 99), (3, 0), (3, 8193), (0, None), (7, None), (8, None), (9, None),
             (6, 2), (6, 35), (6, -1), (5, None), (5, wp(asym))]
    for k, v in cases:
        a = list(base)
        a[k] = v
        refused("dirb200_lds_weights_sharded", *a, None, msg="lds_weights")
        if k != 2:
            refused("dirb200_lds_weights", *(a[:2] + a[3:]), None, msg="lds_weights")
