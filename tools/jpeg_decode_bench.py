"""Device JPEG decode + Pillow bilinear resize (datasets.JpegBatch) against the host path it replaces.

Batches of 256 seeded synthetic JPEGs (Pillow, quality 90, 4:2:0) at 250 x 250, 500 x 500, 800 x 1000 and a mixed-size
batch.  The content is a smooth field plus noise: it sets the entropy density, so the numbers stand for files of that
density only (real AgeDB / IMDB-WIKI files were not used).  Reported per batch:
  * device time of each stage (torch.profiler kernel times, a separate run) and of the whole decode + resize (CUDA
    events), and the whole JpegBatch.cuda() call from host bytes: pinned copy, kernels and the status read;
  * Pillow decode + Resize((224, 224)) on one host thread, the host path of the same images;
  * torchvision.io.decode_jpeg(device='cuda') + resize, with the count of bytes that differ from Pillow's;
  * with --train_step, a ResNet-50 training step of that batch (batch 256, 224 x 224) fed by JpegBatch.cuda(), against
    the same step fed by an already-resized uint8 batch (the --device_transform loop).
The card's name and power limit are printed with the numbers.

    python tools/jpeg_decode_bench.py [--iters 20] [--train_step] [--out results/jpeg_decode_bench.json]
"""
import argparse
import io
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "imbalanced-regression_b200")]

import datasets as D  # noqa: E402

S = 224


def synthetic_jpeg(h, w, seed):
    from PIL import Image
    rng = np.random.RandomState(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    base = 128 + 90 * np.sin(xx / rng.uniform(5, 40) + yy / rng.uniform(5, 40))[..., None] * rng.uniform(0.3, 1, 3)
    arr = np.clip(base + rng.normal(0, 12, size=(h, w, 3)), 0, 255).astype(np.uint8)
    bio = io.BytesIO()
    Image.fromarray(arr).save(bio, "JPEG", quality=90)
    return bio.getvalue()


def batch_items(sizes, seed):
    items = []
    for i, (h, w) in enumerate(sizes):
        raw = synthetic_jpeg(h, w, seed + i)
        rc, desc, iv = D.parse_jpeg(raw)
        assert rc == 0
        items.append(D.EncodedJpeg(raw, desc, iv, S))
    return items


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
    except Exception as e:                                   # noqa: BLE001
        return f"unknown ({e})"


def events_ms(fn, iters):
    fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def stage_ms(fn):
    from torch.profiler import ProfilerActivity, profile
    fn()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA], acc_events=True) as prof:
        fn()
        torch.cuda.synchronize()
    out = {}
    for ev in prof.key_averages():
        for name in ("jpeg_plan", "jpeg_tables", "jpeg_entropy", "jpeg_idct", "jpeg_colour", "resize_plan",
                     "resize_coeff", "resize_kernel"):
            if name in ev.key:
                t = getattr(ev, "device_time_total", None)
                if t is None:
                    t = ev.cuda_time_total
                out[name] = out.get(name, 0.0) + t / 1000.0
    return out


def pillow_ms(batch, count):
    from PIL import Image
    raw = batch.data[:batch.raw_lengths[0]].numpy().tobytes()
    D.host_resize_u8(Image.open(io.BytesIO(raw)).convert("RGB"), S)          # imports and first-call set-up
    t0 = time.perf_counter()
    outs = []
    for j in range(count):
        lo = int(batch.offsets[j])
        raw = batch.data[lo:lo + batch.raw_lengths[j]].numpy().tobytes()
        outs.append(D.host_resize_u8(Image.open(io.BytesIO(raw)).convert("RGB"), S))
    return (time.perf_counter() - t0) * 1000.0 / count, torch.stack(outs)


def nvjpeg(batch, iters, want):
    try:
        import torchvision
        from torchvision.io import decode_jpeg
        from torchvision.transforms.v2 import functional as F
        raws = [batch.data[int(batch.offsets[j]):int(batch.offsets[j + 1])] for j in range(len(batch.jpeg_pos))]

        def run():
            imgs = decode_jpeg(raws, device="cuda")
            return torch.stack([F.resize(im, [S, S], antialias=True) for im in imgs]).permute(0, 2, 3, 1)
        ms = events_ms(run, iters)
        got = run().cpu()
        return {"torchvision": torchvision.__version__, "ms": ms,
                "bytes_differing_from_pillow": int((got[:want.shape[0]] != want).sum()), "bytes_compared": int(want.numel())}
    except Exception as e:                                   # noqa: BLE001
        return {"unavailable": f"{type(e).__name__}: {e}"}


def train_step_ms(batch, iters):
    from resnet import resnet50
    from optim import FusedAdam
    from loss import weighted_l1_loss
    model = resnet50().cuda()
    model.train()
    opt = FusedAdam(model.parameters(), lr=1e-4)
    t = torch.rand(batch.n, 1, device="cuda") * 100
    w = torch.ones_like(t)
    pre = batch.cuda()

    def step(images):
        x = D.gpu_transform_batch(images, train=True)
        loss = weighted_l1_loss(model(x, t, 0), t, w)
        opt.zero_grad()
        loss.backward()
        opt.step()
    res = {}
    for _ in range(2):                                       # alternate the two feeds: the spread shows
        res.setdefault("resized_u8_ms", []).append(events_ms(lambda: step(pre), iters))
        res.setdefault("device_decode_ms", []).append(events_ms(lambda: step(batch.cuda(non_blocking=True)), iters))
    return res


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--iters", type=int, default=20)
    p.add_argument("--pillow_images", type=int, default=64, help="images timed on the host thread per batch")
    p.add_argument("--train_step", action="store_true")
    p.add_argument("--out", default="")
    a = p.parse_args()
    assert torch.cuda.is_available(), "the measurement needs a CUDA device"
    rng = np.random.RandomState(0)
    mixed = [(int(h), int(w)) for h, w in zip(rng.randint(150, 1000, 256), rng.randint(150, 1000, 256))]
    batches = {"250x250": [(250, 250)] * 256, "500x500": [(500, 500)] * 256, "800x1000": [(800, 1000)] * 256,
               "mixed_150-1000": mixed}
    result = {"card": card(), "batch": 256, "out_size": S, "quality": 90, "subsampling": "4:2:0", "batches": {}}
    print(f"card: {result['card']}")
    for k, (name, sizes) in enumerate(batches.items()):
        items = batch_items(sizes, seed=1000 * k)
        batch = D.JpegBatch(items).pin_memory()
        out = batch.cuda()
        pil_ms, want = pillow_ms(batch, min(a.pillow_images, batch.n))
        assert torch.equal(out[:want.shape[0]].cpu(), want), "device result differs from Pillow"
        dev = {k: torch.from_numpy(np.ascontiguousarray(v)).cuda() if isinstance(v, np.ndarray) else v.cuda()
               for k, v in dict(data=batch.data, offsets=batch.offsets, descs=batch.descs, intervals=batch.intervals,
                                hw=batch.hw, rgb_offsets=batch.rgb_offsets).items()}
        import _lib
        m = batch.n
        rgb = torch.empty(int(batch.rgb_offsets[-1]), dtype=torch.uint8, device="cuda")
        status = torch.empty(m, dtype=torch.int32, device="cuda")
        ws = torch.empty(batch.decode_ws, dtype=torch.uint8, device="cuda")
        rws = torch.empty(batch.resize_ws, dtype=torch.uint8, device="cuda")
        res = torch.empty(m, S, S, 3, dtype=torch.uint8, device="cuda")

        def kernels():
            st = _lib.stream_ptr()
            _lib.call("dirb200_jpeg_decode", _lib.ptr(dev["data"]), _lib.ptr(dev["offsets"]), _lib.ptr(dev["descs"]),
                      _lib.ptr(dev["intervals"]), m, _lib.ptr(rgb), _lib.ptr(dev["rgb_offsets"]), _lib.ptr(status),
                      _lib.ptr(ws), ws.numel(), st)
            _lib.call("dirb200_resize_bilinear_u8", _lib.ptr(rgb), _lib.ptr(dev["rgb_offsets"]), _lib.ptr(dev["hw"]), m,
                      S, S, _lib.ptr(res), _lib.ptr(rws), rws.numel(), st)
        row = {"file_mbytes": batch.data.numel() / 1e6, "decode_resize_device_ms": events_ms(kernels, a.iters),
               "stages_ms": stage_ms(kernels),
               "jpegbatch_cuda_from_pinned_ms": events_ms(lambda: batch.cuda(non_blocking=True), a.iters),
               "pillow_one_thread_ms_per_image": pil_ms,
               "pillow_one_thread_ms_per_batch": pil_ms * batch.n,
               "torchvision_nvjpeg": nvjpeg(batch, a.iters, want)}
        if a.train_step and name == "500x500":
            row["train_step"] = train_step_ms(batch, a.iters)
        result["batches"][name] = row
        print(name, json.dumps(row))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(result, f, indent=1)


if __name__ == "__main__":
    main()
