"""NYUD2-DIR test-set evaluation timing: the fused device evaluator (depth_eval.Evaluator.add, one kernel per batch)
against test.py's path on the same data (torch CUDA F.interpolate(align_corners=True), boolean indexing, a .cpu() per
image and the reference's own Evaluator where oracle/_ref holds a copy of nyud2-dir/util.py, the numpy oracle
otherwise).  Synthetic test set of the real size: 654 images, depth 228 x 304, predictions 114 x 152, the balanced
test masks of the fixture repeated.  Prints one JSON line; needs a CUDA device.

    python tools/nyud2_eval_bench.py [--reps 5]
"""
import argparse
import importlib.util
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

HBM_TBPS = 3.35          # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, limit = (q.stdout.strip().partition(",") if q.returncode == 0 else ("?", "", "?"))
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": limit.strip()}


def data(n=654):
    from test_gpu_depth_eval import _real_masks, _synthetic
    pred, depth = _synthetic(n, seed=0)
    depth = torch.nan_to_num(depth, nan=1.0)       # evaluate_shot refuses NaN depths, as the reference does
    return pred, depth, _real_masks(n)


def time_device(pred, depth, mask, shot, batch, reps):
    from depth_eval import Evaluator
    ev = Evaluator(shot)
    for lo in range(0, pred.shape[0], batch):       # warm-up: allocations, module load
        ev.add(pred[lo:lo + batch], depth[lo:lo + batch], mask[lo:lo + batch])
    ev.evaluate_shot()
    e2e = []
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.reset()
        for lo in range(0, pred.shape[0], batch):
            ev.add(pred[lo:lo + batch], depth[lo:lo + batch], mask[lo:lo + batch])
        md = ev.evaluate_shot()
        e2e.append(time.perf_counter() - t0)
    # kernel time alone: the profiler's device durations of depth_metrics_kernel over one pass
    from torch.profiler import ProfilerActivity, profile
    ev.reset()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for lo in range(0, pred.shape[0], batch):
            ev.add(pred[lo:lo + batch], depth[lo:lo + batch], mask[lo:lo + batch])
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if "depth_metrics_kernel" in e.name and e.device_type.name == "CUDA"]
    kernel_ms = sum(e.device_time_total for e in kern) / 1e3 if kern else float("nan")
    return md, sorted(e2e)[len(e2e) // 2] * 1e3, kernel_ms, len(kern)


def reference_evaluator(shot):
    """The reference's Evaluator (copy under oracle/_ref) or, without it, the numpy oracle behind the same calls."""
    from oracle import ref_nyud2
    if ref_nyud2.available():
        spec = importlib.util.spec_from_file_location("nyud2_reference_util", ref_nyud2.UTIL)
        mod = importlib.util.module_from_spec(spec)
        spec.loader.exec_module(mod)
        ev = mod.Evaluator()
        ev.shot_idx = shot
        return ev, "reference nyud2-dir/util.py Evaluator (oracle/_ref)"
    from oracle import depth_oracle as O

    class OracleEvaluator:
        def __init__(self):
            self.o, self.t = [], []

        def __call__(self, output, depth):
            self.o.append(output.squeeze().view(-1).cpu().numpy())
            self.t.append(depth.squeeze().view(-1).cpu().numpy())

        def evaluate_shot(self):
            return O.depth_metrics(np.concatenate(self.o), np.concatenate(self.t), shot)[1]
    return OracleEvaluator(), "numpy oracle (oracle/_ref has no nyud2-dir/util.py)"


def time_reference(pred, depth, mask, shot):
    ev, kind = reference_evaluator(shot)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(pred.shape[0]):                 # test.py:47-54 at batch 1 (getTestingData(args, 1))
        output = F.interpolate(pred[i:i + 1], size=[depth.size(2), depth.size(3)], mode="bilinear",
                               align_corners=True)
        ev(output[mask[i:i + 1]], depth[i:i + 1][mask[i:i + 1]])
    t1 = time.perf_counter()
    md = ev.evaluate_shot()
    t2 = time.perf_counter()
    return md, (t2 - t0) * 1e3, (t1 - t0) * 1e3, kind


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nyud2_eval_bench needs a CUDA device")
    import logging
    logging.disable(logging.INFO)
    from util import golden
    g = golden("depth_eval")
    shot = {k: g[f"shot_{k}"].tolist() for k in ("many", "medium", "few")}
    pred, depth, mask = data()
    n, _, h, w = depth.shape
    ph, pw = pred.shape[2:]
    out = {"tool": "nyud2_eval_bench", **card(), "images": n, "depth_hw": [h, w], "pred_hw": [ph, pw],
           "mask_density": round(float(mask.float().mean()), 4)}
    dense_bytes = n * h * w * (1 + 4) + n * ph * pw * 4       # mask + target + prediction, each read once
    out["bytes_if_every_input_read_once"] = dense_bytes
    for batch in (1, 8):
        md, e2e, kms, launches = time_device(pred, depth, mask, shot, batch, args.reps)
        out[f"device_b{batch}"] = {"end_to_end_ms": round(e2e, 3), "kernel_ms_total": round(kms, 4),
                                   "kernel_launches": launches,
                                   "kernel_us_per_launch": round(1e3 * kms / max(launches, 1), 2),
                                   "dense_bytes_over_kernel_time_TBps": round(dense_bytes / (kms * 1e-3) / 1e12, 3),
                                   "share_of_3.35TBps": round(dense_bytes / (kms * 1e-3) / 1e12 / HBM_TBPS, 3),
                                   "overall_rmse": md["overall"]["RMSE"]}
    md, e2e, loop_ms, kind = time_reference(pred, depth, mask, shot)
    out["reference_style_b1"] = {"end_to_end_ms": round(e2e, 1), "loop_ms": round(loop_ms, 1),
                                 "evaluate_shot_ms": round(e2e - loop_ms, 1), "evaluator": kind,
                                 "overall_rmse": float(md["overall"]["RMSE"])}
    out["speedup_b1"] = round(e2e / out["device_b1"]["end_to_end_ms"], 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
