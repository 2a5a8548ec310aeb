"""Times NYUD2-DIR's input pipeline: the device transform (loaddata.gpu_depth_transform_batch: flip, spline rotation,
crop, depth resize, Lighting, ColorJitter, Normalize, weights) per batch at 8 and 32 with CUDA events; the host side
of the device path per sample (JPEG + PNG decode and Scale(240), loaddata.depthDataset.__getitem__); and the
reference's per-sample chain (nyud2-dir/loaddata.py:108-125 after decode) plus _get_weights on one CPU thread.
Synthetic 640 x 480 inputs, written to a temporary directory.  Prints one JSON line per measurement.

    python tools/nyud2_input_bench.py [--iters 50] [--host-samples 20] [--ref-samples 10]
"""
import argparse
import json
import os
import random
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "imbalanced-regression_b200")]


def card():
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception:
        pl = "unknown"
    return name, pl


def device_times(iters):
    import loaddata
    tab = loaddata.depthDataset._get_bucket_weights(argparse.Namespace(reweight='inverse', lds=True, lds_kernel='gaussian',
                                                                      lds_ks=5, lds_sigma=2, bucket_num=100, bucket_start=7))
    out = {}
    for n in (8, 32):
        g = torch.Generator(device="cuda").manual_seed(n)
        img = torch.randint(0, 256, (n, 240, 320, 3), dtype=torch.uint8, device="cuda", generator=g)
        dep = torch.randint(0, 256, (n, 240, 320), dtype=torch.uint8, device="cuda", generator=g)
        p = loaddata.draw_nyud2_train_params(n, random.Random(n), torch.Generator().manual_seed(n))
        for _ in range(5):
            loaddata.gpu_depth_transform_batch(img, dep, "train", params=p, bucket_weights=tab)
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(iters):
            loaddata.gpu_depth_transform_batch(img, dep, "train", params=p, bucket_weights=tab)
        b.record()
        torch.cuda.synchronize()
        out[n] = a.elapsed_time(b) / iters
        # draws on the host for a batch (part of a training step's input cost)
        t0 = time.perf_counter()
        for _ in range(10):
            loaddata.draw_nyud2_train_params(n)
        out[f"draw{n}"] = (time.perf_counter() - t0) / 10 * 1e3
    return out


def host_times(samples, ref_samples):
    import loaddata
    from oracle import nyu_transform_ref
    d = tempfile.mkdtemp()
    os.makedirs(os.path.join(d, "nyu2_train"))
    r = np.random.RandomState(0)
    yy, xx = np.indices((480, 640))
    lines = []
    for k in range(samples):
        im = np.stack([xx * 255 // 639, yy * 255 // 479, (xx + yy) % 256], -1) + r.randint(0, 40, (480, 640, 3))
        Image.fromarray(np.clip(im, 0, 255).astype(np.uint8)).save(os.path.join(d, "nyu2_train", f"{k}.jpg"), quality=90)
        Image.fromarray(((xx // 3 + yy // 5 + 17 * k) % 256).astype(np.uint8)).save(os.path.join(d, "nyu2_train", f"{k}.png"))
        lines.append(f"data/nyu2_train/{k}.jpg,data/nyu2_train/{k}.png")
    with open(os.path.join(d, "nyu2_train.csv"), "w") as f:
        f.write("\n".join(lines) + "\n")
    args = argparse.Namespace(data_dir=d, reweight='inverse', lds=True, lds_kernel='gaussian', lds_ks=5, lds_sigma=2,
                              bucket_num=100, bucket_start=7)
    ds = loaddata.depthDataset(d, os.path.join(d, "nyu2_train.csv"), args=args)
    ds[0]
    t0 = time.perf_counter()
    for k in range(samples):
        ds[k]
    host = (time.perf_counter() - t0) / samples * 1e3
    res = {"host_decode_scale_ms_per_sample": round(host, 3)}
    if nyu_transform_ref.available():
        torch.set_num_threads(1)
        _, ld = nyu_transform_ref.load()
        ref = ld.getTrainingData(args, 1).dataset          # the reference's dataset with its own Compose
        ref[0]
        t0 = time.perf_counter()
        for k in range(ref_samples):
            ref[k % samples]
        res["reference_chain_and_weights_ms_per_sample"] = round((time.perf_counter() - t0) / ref_samples * 1e3, 3)
    else:
        res["reference_chain_and_weights_ms_per_sample"] = "not measured: oracle/_ref has no copy of the reference"
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--host-samples", type=int, default=20)
    ap.add_argument("--ref-samples", type=int, default=10)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "the device transform is timed on a GPU"
    name, pl = card()
    dev = device_times(a.iters)
    for n in (8, 32):
        print(json.dumps({"metric": "nyud2_device_transform_ms_per_batch", "batch": n, "value": round(dev[n], 4),
                          "host_draws_ms_per_batch": round(dev[f"draw{n}"], 3), "gpu": name, "power_limit": pl}))
    print(json.dumps(dict(metric="nyud2_host_input_ms_per_sample", **host_times(a.host_samples, a.ref_samples),
                          note="one CPU thread for the reference; decode + Scale for the device path")))


if __name__ == "__main__":
    main()
