"""Numpy restatement of the NYUD2-DIR test-time evaluation (nyud2-dir/util.py:35-133, Evaluator) -- TEST
INFRASTRUCTURE ONLY: the parity oracle of depth_eval.py / dirb200_depth_metrics_accumulate (nothing in the product path
imports it)."""
from __future__ import annotations

import math

import numpy as np


DEPTH_SHOTS = ("overall", "many", "medium", "few")


def depth_metrics(output, target, shot_idx):
    """Evaluator.evaluate_shot (util.py:53-78, 88-133) restated in numpy: fp32 element terms, float64 sums.

    Returns (acc, metric_dict).  acc float64[4][10]: rows overall / many / medium / few; columns NUM (non-NaN
    targets), sum d^2, sum d, sum d/t, sum |lg10 o - lg10 t|, delta1-3 counts, NaN targets, +-inf targets.  A NaN
    target zeroes its terms (setNanToZero); NaN and inf targets belong to no shot group (the reference's int()
    raises on them, which this function does not).  metric_dict is the reference's dict built from acc."""
    o = np.asarray(output, dtype=np.float32).reshape(-1)
    t = np.asarray(target, dtype=np.float32).reshape(-1)
    nan = np.isnan(t)
    o, t = np.where(nan, np.float32(0), o), np.where(nan, np.float32(0), t)
    ln10 = np.float32(math.log(10))
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        d = np.abs(o - t)
        rel = np.where(nan, np.float32(0), d / t)
        lg = np.where(nan, np.float32(0), np.abs(np.log(o) / ln10 - np.log(t) / ln10))
        yz, zy = o / t, t / o
        r = np.where(yz < zy, zy, yz)                                 # maxOfTwo: NaN keeps o / t
        p = t * np.float32(10)
        bins = np.full(t.shape, -1, dtype=np.int64)
        fin = np.isfinite(t)
        bins[fin] = np.minimum(np.trunc(p[fin]).astype(np.int64), 99)   # min(int(x * np.float32(10)), 99)
    terms = [~nan, d * d, d, rel, lg, r <= np.float32(1.25), r <= np.float32(1.5625), r <= np.float32(1.953125)]
    terms = [np.where(nan, 0, x).astype(np.float64) for x in terms]
    acc = np.zeros((4, 10), dtype=np.float64)
    groups = [np.ones(t.shape, bool)]
    for shot in DEPTH_SHOTS[1:]:
        groups.append(fin & np.isin(bins, np.asarray(list(shot_idx.get(shot, ())), dtype=np.int64)))
    for g, m in enumerate(groups):
        for k, x in enumerate(terms):
            acc[g, k] = np.sum(x[m], dtype=np.float64)
    acc[0, 8] = np.count_nonzero(nan)
    acc[0, 9] = np.count_nonzero(np.isinf(t))
    metric_dict = {}
    for g, shot in enumerate(DEPTH_SHOTS):
        n = acc[g, 0]
        e = {"MSE": 0, "RMSE": 0, "ABS_REL": 0, "LG10": 0, "MAE": 0, "DELTA1": 0, "DELTA2": 0, "DELTA3": 0, "NUM": 0}
        if n > 0:
            with np.errstate(divide="ignore", invalid="ignore"):
                e.update(MSE=acc[g, 1] / n, MAE=acc[g, 2] / n, ABS_REL=acc[g, 3] / n, LG10=acc[g, 4] / n, NUM=int(n))
            for k in range(3):
                e[f"DELTA{k + 1}"] = float(np.float32(acc[g, 5 + k]) / np.float32(n))
        with np.errstate(invalid="ignore"):
            e["RMSE"] = np.sqrt(e["MSE"])
        metric_dict[shot] = e
    return acc, metric_dict
