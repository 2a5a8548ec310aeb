"""Golden fixture for STS-B-DIR's shot metrics (sts-b-dir/util.py:101-172, STSShotAverage.get_metric), produced by
running the REFERENCE's own util.py (numpy, scipy and torch only) on the CPU.

Run in the build container only (needs the reference tree, read-only):

    python tests/golden/make_golden_stsb_metrics.py

Each case feeds the reference scorer fp32 numpy vectors, as models.py:108-111 does, in batches of 128, and records
get_metric(reset=True) with metric=['mse', 'l1', 'gmean', 'pearsonr', 'spearmanr'] (tasks.py:86).  Cases:
  edges      labels on every np.histogram edge over [0, 5] (50 bins), one float32 ulp either side, 0 and 5.0;
             predictions rounded to 0.01 (ties), five exact zero differences
  groups     labels in many bins only, one few label and no medium one: an empty group and a group of one
  constant   the medium group's labels all equal (y constant) and the few group's predictions all equal (x
             constant); the overall group is not constant
  pairs      a few group of two, a medium group of two with tied predictions (NaN)
  random     N = 1000, continuous labels in [0, 5], predictions label / 5 + noise
  big        N = 51 200 (400 validation intervals of 128): labels on the 0.2 grid and continuous, predictions
             rounded to 1e-3 (many ties)

Stored per case: {case}:pred, {case}:label (float32) and {case}:want float64 [4, 6], rows overall / many / medium / few,
columns num_samples, mse, l1, gmean, pearsonr, spearmanr (NaN where the reference gives NaN).
"""
import os
import sys
import warnings

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/sts-b-dir"
SHOTS = ('overall', 'many', 'medium', 'few')
COLS = ('num_samples', 'mse', 'l1', 'gmean', 'pearsonr', 'spearmanr')
F32 = np.float32


def edges_case(rng):
    e = np.histogram(np.array([], dtype=F32), bins=50, range=(0., 5.))[1].astype(F32)
    lab = np.concatenate([e, np.nextafter(e, F32(-1)), np.nextafter(e, F32(10)), [F32(0), F32(5)]])
    lab = lab[(lab >= 0) & (lab <= 5)].astype(F32)
    pred = np.round(rng.uniform(0, 1, lab.size), 2).astype(F32)
    zero_pred = np.array([0.5, 0.0, 1.0, 0.25, 0.75], dtype=F32)     # 5 pred == label exactly
    zero_lab = np.array([2.5, 0.0, 5.0, 1.25, 3.75], dtype=F32)
    return np.concatenate([pred, zero_pred]), np.concatenate([lab, zero_lab])


def groups_case(rng):
    many_bins = [0, 10, 12, 14, 16, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 49]
    lab = np.array([(b + rng.uniform(0.2, 0.8)) * 0.1 for b in rng.choice(many_bins, 40)] + [0.15], dtype=F32)
    return rng.uniform(0, 1, lab.size).astype(F32), lab


def constant_case(rng):
    many = np.array([0.05, 1.05, 1.25, 2.45, 4.95, 3.05], dtype=F32)
    medium = np.full(6, 0.25, dtype=F32)                       # bin 2
    few = np.array([0.15, 0.35, 1.15, 2.15, 3.15, 4.75], dtype=F32)
    lab = np.concatenate([many, medium, few])
    pred = np.concatenate([rng.uniform(0, 1, 12), np.full(6, 0.3)]).astype(F32)
    return pred, lab


def pairs_case(rng):
    lab = np.array([0.05, 1.05, 2.05, 3.05, 0.15, 0.35, 0.25, 0.45], dtype=F32)   # many x4, few x2, medium x2
    pred = np.array([0.1, 0.3, 0.2, 0.7, 0.4, 0.2, 0.6, 0.6], dtype=F32)
    return pred, lab


def random_case(rng):
    lab = rng.uniform(0, 5, 1000).astype(F32)
    return (lab / 5 + rng.normal(0, 0.1, lab.size)).astype(F32), lab


def big_case(rng):
    n = 51200
    lab = np.where(rng.uniform(size=n) < 0.5, np.round(rng.uniform(0, 5, n) * 5) / 5, rng.uniform(0, 5, n))
    lab = lab.astype(F32)
    pred = np.round(lab / 5 + rng.normal(0, 0.15, n), 3).astype(F32)
    return pred, lab


CASES = {'edges': edges_case, 'groups': groups_case, 'constant': constant_case, 'pairs': pairs_case,
         'random': random_case, 'big': big_case}


def main():
    sys.path.insert(0, REF)
    from util import STSShotAverage
    out = {}
    for k, (name, fn) in enumerate(CASES.items()):
        pred, lab = fn(np.random.RandomState(100 + k))
        scorer = STSShotAverage(metric=['mse', 'l1', 'gmean', 'pearsonr', 'spearmanr'])
        for lo in range(0, pred.size, 128):
            scorer(pred[lo:lo + 128], lab[lo:lo + 128])
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")              # scipy warns on the constant groups
            m = scorer.get_metric(reset=True)
        want = np.array([[float(m[s][c]) for c in COLS] for s in SHOTS], dtype=np.float64)
        out[f"{name}:pred"], out[f"{name}:label"], out[f"{name}:want"] = pred, lab, want
        print(name, pred.size, want[:, 0].astype(int).tolist())
    np.savez_compressed(os.path.join(HERE, "stsb_metrics.npz"), **out)


if __name__ == "__main__":
    main()
