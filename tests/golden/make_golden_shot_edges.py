"""Golden fixture for the shot metrics at their group edges, produced by running the REFERENCE's own `shot_metrics`
(agedb-dir/train.py:338-391, lifted with make_golden_metrics.reference_function) on constructed inputs.

Run in the build container only (needs /root/reference, read-only):

    python tests/golden/make_golden_shot_edges.py

Cases (tag: training column / test labels / thresholds):
  edges  training counts 19, 20, 21, 99, 100, 101 and 150 for one label each (labels 10 .. 16); label 0's count of 20
         includes one -0.5 (int(-0.5) == 0); label 13's count of 99 includes one 13.6 and label 20's 25 are all 20.3
         (counts go by int(train_label)); three NaN training labels.  Test labels add 12.5 and 20.3 (not integers:
         count 0), 50 (absent) and 120 (above every training label).  Thresholds (100, 20).
  equal  many == low == 5: training counts 4, 5 and 6 -> low, median, many.
  zero   `edges` with one exact hit (error 0) in the median group only: its G-Mean is 0, the other groups keep theirs.
Only the reference's outputs on these inputs are stored (shot_edges.npz); nothing from the reference is copied.
"""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_metrics import reference_function  # noqa: E402


def edges_case(rng):
    train = np.concatenate([
        np.full(19, 0.0), [-0.5],                                          # label 0: 20 -> median
        np.full(19, 10.0), np.full(20, 11.0), np.full(21, 12.0),           # 19 low, 20 median, 21 median
        np.full(98, 13.0), [13.6], np.full(100, 14.0), np.full(101, 15.0),  # 99 median, 100 median, 101 many
        np.full(150, 16.0), np.full(25, 20.3), [np.nan, np.nan, np.nan],
    ]).astype(np.float32)
    rng.shuffle(train)
    values = np.asarray([0, 10, 11, 12, 13, 14, 15, 16, 20, 12.5, 20.3, 50, 120], np.float32)
    labels = np.repeat(values, rng.randint(3, 90, size=values.size)).astype(np.float32)
    rng.shuffle(labels)
    preds = (labels + rng.randn(labels.size).astype(np.float32) * 4).astype(np.float32)
    return train, labels, preds


def main():
    shot_metrics = reference_function("shot_metrics")
    rng = np.random.RandomState(11)
    cases = {}
    train, labels, preds = edges_case(rng)
    cases["edges"] = (train, labels, preds, (100, 20))
    eq_train = np.concatenate([np.full(4, 30.0), np.full(5, 31.0), np.full(6, 32.0)]).astype(np.float32)
    eq_labels = np.repeat(np.asarray([30, 31, 32], np.float32), [7, 9, 5])
    eq_preds = (eq_labels + rng.randn(eq_labels.size).astype(np.float32) * 3).astype(np.float32)
    cases["equal"] = (eq_train, eq_labels, eq_preds, (5, 5))
    zpreds = preds.copy()
    hit = np.nonzero(labels == 14)[0][0]                                  # count 100: median
    zpreds[hit] = labels[hit]
    cases["zero"] = (train, labels, zpreds, (100, 20))
    out = {}
    for tag, (tr, lab, pr, (many, low)) in cases.items():
        with np.errstate(invalid="ignore", divide="ignore"):
            sd = shot_metrics(pr, lab, tr, many_shot_thr=many, low_shot_thr=low)
        out[f"{tag}_train"], out[f"{tag}_labels"], out[f"{tag}_preds"] = tr, lab, pr
        out[f"{tag}_thr"] = np.asarray([many, low], np.int64)
        out[f"{tag}_ref"] = np.asarray([[sd[g][m] for m in ("mse", "l1", "gmean")] for g in ("many", "median", "low")],
                                       dtype=np.float64)
        print(tag, lab.size, out[f"{tag}_ref"].tolist())
    np.savez_compressed(os.path.join(HERE, "shot_edges.npz"), **out)


if __name__ == "__main__":
    main()
