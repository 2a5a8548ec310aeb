"""CPU checks of the STS-B-DIR training pieces: the float64 restatement of STSShotAverage.get_metric (used as the oracle
of tests/test_gpu_stsb_train.py) against the reference's own util.py (fixture tests/golden/stsb_metrics.npz, made by
tests/golden/make_golden_stsb_metrics.py), and the refusals of the new C entry points (dirb200_grad_norm_multi,
dirb200_adam_step_multi_clipped, dirb200_stsb_shot_metrics) and of optim.Adam's max_grad_norm, all before any CUDA
call.  Every device pointer below is a dummy that must never be dereferenced: a call that got past its checks would
fault on a GPU machine and fail without one."""
import ctypes
import warnings

import numpy as np
import pytest
import torch
from scipy.stats import gmean, pearsonr, spearmanr

from util import golden

D = 16                                 # stands for a device buffer (16-byte aligned)
SHOTS = ('overall', 'many', 'medium', 'few')
# sts-b-dir/util.py:110-113
SHOT_IDX = {'many': [0, 10, 12, 14, 16, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 49],
            'medium': [2, 4, 6, 8, 27, 35, 37]}
CASES = ('edges', 'groups', 'constant', 'pairs', 'random', 'big')


def shot_group(labels):
    """1 many, 2 medium, 3 few: the bin of the float32 np.histogram edges over [0, 5] (5.0 in the last bin, a negative
    label bin -1), looked up in util.py's table; any other bin is few."""
    edges = np.histogram(np.array([], dtype=np.float32), bins=50, range=(0., 5.))[1].astype(np.float32)
    lab = np.asarray(labels, dtype=np.float32)
    b = np.where(lab >= 5.0, 49, np.searchsorted(edges, lab, side='right') - 1)
    g = np.full(lab.shape, 3)
    g[np.isin(b, SHOT_IDX['many'])] = 1
    g[np.isin(b, SHOT_IDX['medium'])] = 2
    return g


def shot_metrics_oracle(pred, label):
    """float64 [4, 6] (rows SHOTS; num_samples, mse, l1, gmean, pearsonr, spearmanr) as util.py:123-172 defines them."""
    x = np.asarray(pred, dtype=np.float32).astype(np.float64) * 5.0
    y = np.asarray(label, dtype=np.float32).astype(np.float64)
    g = shot_group(label)
    out = np.zeros((4, 6))
    for row in range(4):
        sel = np.ones(x.shape, bool) if row == 0 else g == row
        xs, ys = x[sel], y[sel]
        n = xs.size
        out[row, 0] = n
        if n == 0:
            continue
        d = np.abs(xs - ys)
        out[row, 1], out[row, 2] = np.mean(d ** 2), np.mean(d)
        out[row, 3] = gmean(np.where(d == 0.0, 1e-10, d))
        if n > 1:
            with warnings.catch_warnings():
                warnings.simplefilter("ignore")
                out[row, 4], out[row, 5] = pearsonr(xs, ys)[0], spearmanr(xs, ys)[0]
    return out


def assert_metrics(got, want, what):
    """counts exact; NaN where want is NaN; otherwise |got - want| <= 1e-12 max(|want|, 1) (the correlations' error
    scales with 1, not with r, when r is near 0)."""
    got, want = np.asarray(got), np.asarray(want)
    assert np.array_equal(got[:, 0], want[:, 0]), (what, got[:, 0], want[:, 0])
    assert np.array_equal(np.isnan(got), np.isnan(want)), (what, got, want)
    ok = np.isnan(want) | (np.abs(got - want) <= 1e-12 * np.maximum(np.abs(want), 1.0))
    assert ok.all(), (what, got, want, np.abs(got - want))


@pytest.mark.parametrize("case", CASES)
def test_metrics_oracle_matches_the_reference_scorer(case):
    z = golden("stsb_metrics")
    assert_metrics(shot_metrics_oracle(z[f"{case}:pred"], z[f"{case}:label"]), z[f"{case}:want"], case)


def test_fixture_covers_the_edge_cases():
    z = golden("stsb_metrics")
    edges = np.histogram(np.array([], dtype=np.float32), bins=50, range=(0., 5.))[1].astype(np.float32)
    lab = z["edges:label"]
    for e in edges:
        assert e in lab and (e == 0 or np.nextafter(e, np.float32(-1)) in lab) and \
            (e == 5 or np.nextafter(e, np.float32(10)) in lab)
    assert (z["edges:pred"].astype(np.float64) * 5 == lab).sum() >= 5                 # exact zero differences
    assert list(z["groups:want"][:, 0]) == [41, 40, 0, 1]                            # an empty group, a group of one
    assert np.isnan(z["constant:want"][2:, 4:]).all()                                # constant y, constant x
    assert z["big:pred"].size == 51200 and np.unique(z["big:pred"]).size < 51200     # ties


# ------------------------------------------------------------------------------------------------ refusals
def lib():
    import _lib as L
    import optim
    return L, optim


def grad_table(n=3, edits=()):
    t = np.zeros(n, dtype=[('grad', np.uint64), ('numel', np.int64)])
    t['grad'], t['numel'] = D, 8
    for k, i, v in edits:
        t[k][i] = v
    return t


def refused(name, *args, msg, rc=-1):
    L, _ = lib()
    got = L.raw(name)(*args)
    err = L.last_error()
    assert got == rc and msg in err, (name, got, err)


def test_grad_norm_multi_refuses_bad_arguments():
    L, optim = lib()
    assert optim._GRAD_SEGMENT.itemsize == 16
    need = L.raw("dirb200_grad_norm_multi_workspace_bytes")()
    assert need >= 8 * 1024 + 16
    P = lambda t: t.ctypes.data_as(ctypes.c_void_p)
    t = grad_table()
    for a in ((None, 3, 5.0, D, need, D, None), (P(t), 0, 5.0, D, need, D, None), (P(t), -1, 5.0, D, need, D, None),
              (P(t), 3, 0.0, D, need, D, None), (P(t), 3, -1.0, D, need, D, None), (P(t), 3, float('nan'), D, need, D,
                                                                                    None),
              (P(t), 3, 5.0, None, need, D, None), (P(t), 3, 5.0, D, need, None, None)):
        refused("dirb200_grad_norm_multi", *a, msg="bad arguments")
    refused("dirb200_grad_norm_multi", P(t), 3, 5.0, D + 4, need, D, None, msg="8-byte aligned")
    refused("dirb200_grad_norm_multi", P(t), 3, 5.0, D, need - 1, D, None, msg="workspace too small", rc=-3)
    for i in (0, 2):
        bad = grad_table(edits=[('grad', i, 0)])
        refused("dirb200_grad_norm_multi", P(bad), 3, 5.0, D, need, D, None, msg=f"segment {i} has a null pointer")
        bad = grad_table(edits=[('grad', i, D + 2)])
        refused("dirb200_grad_norm_multi", P(bad), 3, 5.0, D, need, D, None, msg=f"segment {i} is not 4-byte aligned")
        bad = grad_table(edits=[('numel', i, -1)])
        refused("dirb200_grad_norm_multi", P(bad), 3, 5.0, D, need, D, None, msg=f"segment {i} has numel")
    bad = grad_table(1500, [('numel', 1499, 4096 * 2 ** 31 + 1)])      # a long table is checked in full first
    refused("dirb200_grad_norm_multi", P(bad), 1500, 5.0, D, need, D, None, msg="segment 1499 has numel")


def test_adam_multi_clipped_refuses_bad_arguments():
    L, optim = lib()
    t = np.zeros(3, dtype=optim._SEGMENT)
    for k in ('param', 'grad', 'exp_avg', 'exp_avg_sq'):
        t[k] = D
    t['numel'], t['bc1'], t['bc2_sqrt'] = 8, 0.1, 0.03
    P = t.ctypes.data_as(ctypes.c_void_p)
    args = (1e-3, 0.9, 0.999, 1e-8, 1e-5)
    refused("dirb200_adam_step_multi_clipped", P, 3, *args, None, None, msg="clip_coef is null")
    refused("dirb200_adam_step_multi_clipped", None, 3, *args, D, None, msg="adam_step_multi_clipped: bad arguments")
    refused("dirb200_adam_step_multi_clipped", P, 0, *args, D, None, msg="adam_step_multi_clipped: bad arguments")
    t['exp_avg'][1] = 0
    refused("dirb200_adam_step_multi_clipped", P, 3, *args, D, None, msg="segment 1 has a null pointer")
    t['exp_avg'][1], t['bc1'][2] = D, 0.0
    refused("dirb200_adam_step_multi_clipped", P, 3, *args, D, None, msg="segment 2 has bias corrections")


def test_stsb_shot_metrics_refuses_bad_arguments():
    L, _ = lib()
    ws = L.raw("dirb200_stsb_shot_metrics_workspace_bytes")
    assert ws(100) == 1600 and ws(0) == 0 and ws(-1) == 0
    for n in (-1, 2 ** 22 + 1, 2 ** 30 + 1):
        refused("dirb200_stsb_shot_metrics", D, D, n, D, 2 ** 40, D, None, msg="out of range")
    for a in ((None, D, 100, D, 1600, D, None), (D, None, 100, D, 1600, D, None), (D, D, 100, None, 1600, D, None),
              (D, D, 100, D, 1600, None, None), (None, None, 0, None, 0, None, None)):
        refused("dirb200_stsb_shot_metrics", *a, msg="null pointer")
    refused("dirb200_stsb_shot_metrics", D, D, 100, D + 8, 1600, D, None, msg="16-byte aligned")
    refused("dirb200_stsb_shot_metrics", D, D, 100, D, 1599, D, None, msg="workspace too small", rc=-3)


def test_optim_adam_refuses_a_bad_max_grad_norm_and_cpu_tensors():
    L, optim = lib()
    p = torch.zeros(4, requires_grad=True)
    for v in (0.0, -5.0, float('nan')):
        with pytest.raises(ValueError):
            optim.Adam([p], 1e-3, max_grad_norm=v)
    p.grad = torch.ones(4)
    opt = optim.Adam([p], 1e-3, max_grad_norm=5.0)
    assert opt.last_grad_norm() is None
    with pytest.raises(L.Dirb200Error, match="CUDA"):
        opt.step()
    assert len(opt.state) == 0 and opt.last_grad_norm() is None
    # the option is the optimizer's, not a group's: state_dict() keeps torch.optim.Adam's layout
    assert 'max_grad_norm' not in opt.state_dict()['param_groups'][0]
    assert set(opt.state_dict()['param_groups'][0]) <= set(torch.optim.Adam([p], 1e-3).state_dict()['param_groups'][0])
