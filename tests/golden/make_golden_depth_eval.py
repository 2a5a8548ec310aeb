"""Golden fixture for the NYUD2-DIR depth evaluation, produced by running the REFERENCE's own Evaluator.

Run in the build container only (needs /root/reference, read-only):

    python tests/golden/make_golden_depth_eval.py

nyud2-dir/util.py is imported unmodified (it runs on the CPU) and its Evaluator is driven on seeded inputs; only the
inputs, its outputs, the shot_idx lists it carries and the first 32 balanced test masks are stored, as data.

  A  flat targets on the 1 mm grid k / 1000 (k = 1..10500, every bin edge and the clamp at 99) plus planted exact
     delta ratios, streamed in calls of 1, 7, 1000 and the rest, then evaluate_shot();
  B  test.py's loop body at batch 1 on 32 images: synthetic 16-bit mm depths / 1000 (ToTensor(is_test=True)),
     smooth 114 x 152 predictions, F.interpolate(align_corners=True), the balanced test mask; the masked, up-sampled
     vectors and the metric dict are stored;
  C  NaN targets through Evaluator.evaluate (overall only);
  D  zero / negative targets and predictions (inf / NaN results) through evaluate_shot().
Metric dicts are stored as float64[4][9]: rows overall / many / medium / few, columns METRICS.
"""
import importlib.util
import os

import numpy as np
import torch
import torch.nn.functional as F

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/nyud2-dir"
METRICS = ("MSE", "RMSE", "ABS_REL", "LG10", "MAE", "DELTA1", "DELTA2", "DELTA3", "NUM")
SHOTS = ("overall", "many", "medium", "few")


def reference_util():
    spec = importlib.util.spec_from_file_location("nyud2_reference_util", os.path.join(REF, "util.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def as_rows(md, shots=SHOTS):
    return np.asarray([[float(md[s][m]) for m in METRICS] for s in shots], dtype=np.float64)


def flat_a():
    t = (np.arange(1, 10501, dtype=np.float32) / np.float32(1000)).astype(np.float32)
    rng = np.random.RandomState(0)
    o = (t * np.exp(rng.randn(t.size) * 0.25).astype(np.float32)).astype(np.float32)
    # exact ratios at the delta thresholds, both ways round, and one float above each
    planted_t, planted_o = [], []
    for r in (1.25, 1.5625, 1.953125):
        for base in (4.0, 0.5, 2.0):
            planted_t += [base, base * r, base]
            planted_o += [base * r, base, np.nextafter(np.float32(base * r), np.float32(np.inf))]
    t = np.concatenate([t, np.asarray(planted_t, np.float32)])
    o = np.concatenate([o, np.asarray(planted_o, np.float32)])
    perm = rng.permutation(t.size)
    return o[perm], t[perm]


def synthetic_b(n):
    rng = np.random.RandomState(1)
    yy, xx = np.meshgrid(np.arange(228), np.arange(304), indexing="ij")
    depth_mm, preds = [], []
    py, px = np.meshgrid(np.arange(114), np.arange(152), indexing="ij")
    for i in range(n):
        a, b, c = rng.uniform(0.01, 0.05, 3)
        field = 5200 + 4700 * np.sin(a * yy + b * xx + c * i) * np.cos(0.013 * xx - a * yy)
        depth_mm.append(np.clip(np.round(field + rng.randn(228, 304) * 40), 1, 10500).astype(np.uint16))
        p = 5.0 + 4.6 * np.sin(2 * a * py + 2 * b * px + c * i + 0.3) * np.cos(0.026 * px - 2 * a * py)
        preds.append(p.astype(np.float32))
    return np.stack(depth_mm), np.stack(preds)


def main():
    U = reference_util()
    E = U.Evaluator()
    out = {f"shot_{k}": np.asarray(v, dtype=np.int32) for k, v in E.shot_idx.items()}

    # A
    o, t = flat_a()
    E.reset()
    lo = 0
    for k in (1, 7, 1000, t.size - 1008):
        E(torch.from_numpy(o[lo:lo + k]), torch.from_numpy(t[lo:lo + k]))
        lo += k
    out.update(a_output=o, a_target=t, a_chunks=np.asarray([1, 7, 1000, t.size - 1008], np.int64),
               a_ref=as_rows(E.evaluate_shot()))

    # B
    masks = np.load(os.path.join(REF, "data", "test_balanced_mask.npy"), mmap_mode="r")[:32].astype(bool)
    depth_mm, preds = synthetic_b(32)
    E.reset()
    vo, vt = [], []
    for i in range(32):
        depth = torch.from_numpy(depth_mm[i].astype(np.float32))[None, None] / 1000   # ToTensor(is_test=True)
        output = F.interpolate(torch.from_numpy(preds[i])[None, None], size=[depth.size(2), depth.size(3)],
                               mode="bilinear", align_corners=True)
        mask = torch.from_numpy(masks[i])[None, None]
        E(output[mask], depth[mask])
        vo.append(output[mask].numpy())
        vt.append(depth[mask].numpy())
    out.update(b_masks=np.packbits(masks.reshape(-1)), b_mask_shape=np.asarray(masks.shape, np.int64),
               b_output=np.concatenate(vo), b_target=np.concatenate(vt), b_ref=as_rows(E.evaluate_shot()))

    # C
    rng = np.random.RandomState(2)
    t = rng.uniform(0.3, 9.5, 4000).astype(np.float32)
    o = (t + rng.randn(t.size).astype(np.float32) * 0.4).astype(np.float32)
    o = np.abs(o) + np.float32(0.01)
    t[::13] = np.nan
    out.update(c_output=o, c_target=t,
               c_ref=as_rows({"overall": U.Evaluator.evaluate(torch.from_numpy(o), torch.from_numpy(t))},
                             ("overall",)))

    # D
    rng = np.random.RandomState(3)
    t = rng.uniform(0.5, 9.0, 600).astype(np.float32)
    o = (t * rng.uniform(0.7, 1.4, t.size)).astype(np.float32)
    t[5], o[5] = 0, 1.5            # target 0: ABS_REL inf, ratio inf
    t[17], o[17] = 0, 0            # 0 / 0: ABS_REL NaN, LG10 NaN
    t[40], o[40] = 3.0, 0          # prediction 0: LG10 inf
    t[77], o[77] = 5.0, -1.0       # negative prediction: LG10 NaN (medium; the inf above stays in many)
    t[90], o[90] = -0.05, 0.2      # bin 0
    t[91], o[91] = -0.1, 0.2       # bin -1: no group
    t[92], o[92] = -2.5, 0.2       # bin -25: no group
    E.reset()
    E(torch.from_numpy(o), torch.from_numpy(t))
    out.update(d_output=o, d_target=t, d_ref=as_rows(E.evaluate_shot()))

    np.savez_compressed(os.path.join(HERE, "depth_eval.npz"), **out)
    for k in ("a_ref", "b_ref", "c_ref", "d_ref"):
        print(k, out[k], sep="\n")


if __name__ == "__main__":
    main()
