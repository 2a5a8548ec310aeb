"""NYUD2-DIR encoder timing: resnet.E_resnet (the native ResNet-50 runner in multi-scale mode) forward + backward with
seeded gradients on all four block outputs, against the reference's own E_resnet (nyud2-dir/models/modules.py:33-58)
under torch / cuDNN at the same shapes, where __graft_entry__.build() copied it into oracle/_ref (oracle/encoder_ref.py);
the tool says so when that copy is absent.  Shapes: 228 x 304 at batch 8 (nyud2-dir/train.py:26: 32 over 4 GPUs) and
480 x 640 at batch 32.  Conv TFLOP/s are algorithmic FLOPs (computed from the shapes below) over the step time.
Prints one JSON line; needs a CUDA device.

    python tools/nyud2_encoder_bench.py [--steps 20] [--warmup 5]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

SHAPES = [(8, 228, 304), (32, 480, 640)]
LAYERS = (3, 4, 6, 3)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, limit = (q.stdout.strip().partition(",") if q.returncode == 0 else ("?", "", "?"))
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": limit.strip()}


def conv_flops(n, h, w):
    """Algorithmic FLOPs (2 per multiply-add) of the encoder's convolutions: (forward, forward + backward).  The
    backward is a data and a weight gradient per conv (each as many FLOPs as the forward), except the stem's, whose
    input needs no gradient."""
    def conv(hi, wi, cin, cout, k, s, p):
        ho, wo = (hi + 2 * p - k) // s + 1, (wi + 2 * p - k) // s + 1
        return 2.0 * n * ho * wo * cout * cin * k * k, ho, wo
    stem, h, w = conv(h, w, 3, 64, 7, 2, 3)
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    fwd, inplanes = 0.0, 64
    for li, nblocks in enumerate(LAYERS):
        planes = 64 << li
        for b in range(nblocks):
            s = 2 if (b == 0 and li > 0) else 1
            f1, _, _ = conv(h, w, inplanes, planes, 1, 1, 0)
            f2, ho, wo = conv(h, w, planes, planes, 3, s, 1)
            f3, _, _ = conv(ho, wo, planes, planes * 4, 1, 1, 0)
            fwd += f1 + f2 + f3
            if b == 0:
                fwd += conv(h, w, inplanes, planes * 4, 1, s, 0)[0]
            h, w, inplanes = ho, wo, planes * 4
    return stem + fwd, 3 * (stem + fwd) - stem


def time_steps(step, steps, warmup):
    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        step()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def seeded_grads(outs):
    g = torch.Generator(device="cuda").manual_seed(1)
    return [torch.randn(o.shape, generator=g, device="cuda", dtype=torch.float32).to(o.dtype) for o in outs]


def native_arm(n, h, w, steps, warmup):
    from resnet import E_resnet, resnet50
    torch.manual_seed(0)
    E = E_resnet(resnet50()).cuda()
    E.train()
    x = torch.randn(n, 3, h, w, device="cuda")
    grads = seeded_grads(E(x))

    def step():
        torch.autograd.backward(E(x), grads)
    ms = time_steps(step, steps, warmup)
    del E
    return ms


def reference_arm(n, h, w, steps, warmup):
    from oracle import encoder_ref
    if not encoder_ref.available():
        return None
    sys.path.insert(0, encoder_ref.REF_DIR)          # `from models import ...`; models/fds.py imports util.py
    from models import modules, resnet as ref_resnet
    torch.manual_seed(0)
    E = modules.E_resnet(ref_resnet.resnet50()).cuda()
    E.train()
    x = torch.randn(n, 3, h, w, device="cuda")
    grads = seeded_grads(E(x))

    def step():
        torch.autograd.backward(E(x), grads)
    ms = time_steps(step, steps, warmup)
    del E
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "nyud2_encoder_bench needs a CUDA device"
    out = dict(card(), runs=[])
    from oracle import encoder_ref
    if not encoder_ref.available():
        out["reference"] = "absent: oracle/_ref/nyud2-dir/models not installed (run __graft_entry__.build() where " \
                           "the reference checkout exists)"
    for n, h, w in SHAPES:
        _, flops = conv_flops(n, h, w)
        r = dict(batch=n, h=h, w=w, conv_gflop_fwd_bwd=round(flops / 1e9, 1))
        ms = native_arm(n, h, w, a.steps, a.warmup)
        r.update(native_ms=round(ms, 3), native_conv_tflops=round(flops / ms / 1e9, 1))
        torch.cuda.empty_cache()
        ref = reference_arm(n, h, w, a.steps, a.warmup)
        if ref is not None:
            r.update(reference_ms=round(ref, 3), reference_conv_tflops=round(flops / ref / 1e9, 1),
                     reference_backend="torch %s fp32, cuDNN %s, tf32 %s" % (
                         torch.__version__, torch.backends.cudnn.version(), torch.backends.cudnn.allow_tf32))
        torch.cuda.empty_cache()
        out["runs"].append(r)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
