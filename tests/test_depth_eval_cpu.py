"""CPU-only checks of the NYUD2-DIR depth evaluation: the numpy oracle (oracle.depth_oracle.depth_metrics) against the
fixture the reference's own nyud2-dir/util.py Evaluator produced (tests/golden/make_golden_depth_eval.py), and the
argument checks of the C entry point and the Python mirror, which need no device."""
import ctypes

import numpy as np
import pytest
import torch
from util import golden
from oracle import depth_oracle as O

METRICS = ("MSE", "RMSE", "ABS_REL", "LG10", "MAE", "DELTA1", "DELTA2", "DELTA3", "NUM")
SHOTS = ("overall", "many", "medium", "few")


def shot_idx(g):
    return {k: g[f"shot_{k}"].tolist() for k in ("many", "medium", "few")}


def rows(metric_dict, shots=SHOTS):
    return np.asarray([[float(metric_dict[s][m]) for m in METRICS] for s in shots], dtype=np.float64)


def check_rows(got, want, rtol=1e-6, lg10_rtol=1e-6, what=""):
    """NUM and DELTA1-3 equal; MSE / RMSE / ABS_REL / MAE within rtol and LG10 within lg10_rtol relative; the same
    IEEE class (NaN, +inf, -inf, finite) everywhere."""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    assert got.shape == want.shape, (what, got.shape, want.shape)
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, got, want)
    assert np.array_equal(np.isposinf(got), np.isposinf(want)) and np.array_equal(np.isneginf(got),
                                                                                    np.isneginf(want)), (what, got, want)
    exact = [METRICS.index(m) for m in ("NUM", "DELTA1", "DELTA2", "DELTA3")]
    assert np.array_equal(got[:, exact], want[:, exact]), (what, got[:, exact], want[:, exact])
    for m in ("MSE", "RMSE", "ABS_REL", "LG10", "MAE"):
        k = METRICS.index(m)
        fin = np.isfinite(want[:, k])
        tol = lg10_rtol if m == "LG10" else rtol
        err = np.abs(got[fin, k] - want[fin, k]) / np.maximum(np.abs(want[fin, k]), 1e-300)
        assert not (err > tol).any(), (what, m, got[:, k], want[:, k])


@pytest.mark.parametrize("case", ["a", "b", "d"])
def test_oracle_matches_reference_evaluate_shot(case):
    g = golden("depth_eval")
    acc, md = O.depth_metrics(g[f"{case}_output"], g[f"{case}_target"], shot_idx(g))
    check_rows(rows(md), g[f"{case}_ref"], what=case)
    # the counts behind the dict: overall = the sum of the groups and of the pixels in none (exact integers)
    assert acc[0, 0] == g[f"{case}_target"].size
    assert (acc[1:, 0].sum() <= acc[0, 0]) and acc[0, 8] == 0 and acc[0, 9] == 0


def test_oracle_matches_reference_evaluate_with_nan_targets():
    g = golden("depth_eval")
    acc, md = O.depth_metrics(g["c_output"], g["c_target"], shot_idx(g))
    check_rows(rows(md, ("overall",)), g["c_ref"], what="c")
    assert acc[0, 8] == np.isnan(g["c_target"]).sum() > 0
    assert acc[0, 0] + acc[0, 8] == g["c_target"].size


def test_fixture_covers_the_bin_edges_and_delta_ties():
    """Fixture A's targets put k / 1000 on both sides of every fp32 bin edge (0.7 * 10.f is exactly 7, a double
    product would give 6.99999988) and beyond the clamp at 99; the planted ratios are exactly 1.25^k."""
    g = golden("depth_eval")
    t, o = g["a_target"], g["a_output"]
    bins = np.minimum(np.trunc(t * np.float32(10)).astype(np.int64), 99)
    assert set(range(100)) <= set(bins.tolist())
    assert (t * np.float32(10) >= 100).any()
    assert bins[t == np.float32(0.7)][0] == 7 and int(np.float64(np.float32(0.7)) * 10) == 6
    r = np.maximum(o / t, t / o)
    for thr in (1.25, 1.5625, 1.953125):
        assert (r == np.float32(thr)).sum() >= 6


def test_depth_metrics_entry_point_rejects_bad_arguments_without_a_device():
    import _lib
    d = ctypes.c_void_p(16)                  # stands for a device buffer; never dereferenced
    fn = _lib.raw("dirb200_depth_metrics_accumulate")
    ws = _lib.raw("dirb200_depth_metrics_workspace_bytes")(4, 228, 304)
    assert ws >= 64 + 40 * 8

    def refused(*args, msg, rc=-1):
        got = fn(*args)
        err = _lib.last_error()
        assert got == rc and msg in err, (got, err)

    refused(d, 114, 152, d, d, 4, 0, 304, d, 100, d, d, ws, None, msg="bad shape")
    refused(d, 0, 152, d, d, 4, 228, 304, d, 100, d, d, ws, None, msg="bad shape")
    refused(d, 114, 152, d, d, -1, 228, 304, d, 100, d, d, ws, None, msg="bad shape")
    refused(d, 114, 152, d, d, 4, 65536, 65536, d, 100, d, d, ws, None, msg="2^31")
    refused(d, 114, 152, d, d, 4, 228, 304, None, 100, d, d, ws, None, msg="group_of_bin")
    refused(d, 114, 152, d, d, 4, 228, 304, d, 0, d, d, ws, None, msg="group_of_bin")
    refused(None, 114, 152, d, d, 4, 228, 304, d, 100, d, d, ws, None, msg="null")
    refused(d, 114, 152, d, d, 4, 228, 304, d, 100, None, d, ws, None, msg="null")
    refused(d, 114, 152, d, d, 4, 228, 304, d, 100, d, None, ws, None, msg="null")
    refused(d, 114, 152, d, d, 4, 228, 304, d, 100, d, d, ws - 1, None, msg="workspace", rc=-3)


def test_mirror_refuses_cpu_tensors_and_bad_shot_lists():
    import _lib
    from depth_eval import Evaluator, group_table
    with pytest.raises(ValueError):
        group_table({"many": [3, 4], "few": [4]})
    with pytest.raises(ValueError):
        group_table({"many": [100]})
    g = golden("depth_eval")
    table = group_table(shot_idx(g))
    assert (table == 1).sum() == len(g["shot_many"]) and (table == 3).sum() == len(g["shot_few"])
    assert table[46] == 2 and table[47] == 1
    ev = Evaluator(shot_idx(g))
    assert Evaluator.get_bin_idx(np.float32(0.7)) == 7 and Evaluator.get_bin_idx(np.float32(-0.05)) == 0
    assert Evaluator.get_bin_idx(np.float32(-0.1)) == -1 and Evaluator.get_bin_idx(np.float32(12.0)) == 99
    with pytest.raises(_lib.Dirb200Error):
        ev(torch.ones(4), torch.ones(4))
    with pytest.raises(_lib.Dirb200Error):
        ev.add(torch.ones(1, 1, 2, 2), torch.ones(1, 1, 3, 3), torch.ones(1, 1, 3, 3, dtype=torch.bool))
    with pytest.raises(_lib.Dirb200Error):
        Evaluator.evaluate(torch.ones(4), torch.ones(4))
