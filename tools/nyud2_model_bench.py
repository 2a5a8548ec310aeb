"""NYUD2-DIR net.model timing (net.model, nyud2-dir/models/net.py:5-22) on one GPU; prints one JSON line with the card's
name and power limit.

  train      one training step of nyud2-dir/train.py:195-204 at 228 x 304 batch 8: model(image, depth, epoch) with FDS
             smoothing active, the LDS-weighted loss torch.mean(((out - depth) ** 2) * weight), .backward() and
             torch.optim.Adam(weight_decay=1e-4)
  eval       model(image) in eval() under no_grad, batch 1 and 8
  head       R's depth head at 8 x 114 x 152 x 128: dirb200_depth_head_fwd / _dgrad / _wgrad, each with its achieved
             bytes/s against 3.35 TB/s (the H100 SXM's data-sheet HBM3 bandwidth), next to the path it replaces (the
             64-channel zero-padded wgmma convolution + a bf16 bias add, forward and backward through autograd)

native = this package; reference = the reference's own net.model under torch fp32 / cuDNN (benchmark on, TF32 on),
where __graft_entry__.build() copied nyud2-dir/models into oracle/_ref (oracle/encoder_ref.py, oracle/net_ref.py);
reported as not measured otherwise.  The arms alternate within one run (--rounds rounds of --steps steps each); each figure is the
median over rounds of the mean step time (CUDA events).

    python tools/nyud2_model_bench.py [--steps 10] [--warmup 3] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

BLOCKS = [256, 512, 1024, 2048]
HBM = 3.35e12


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    f = [s.strip() for s in q.stdout.strip().split(",")] if q.returncode == 0 else ["?", "?", "?"]
    return {"gpu": f[0], "power_limit": f[1], "max_sm_clock": f[2] if len(f) > 2 else "?"}


def args_ns():
    return SimpleNamespace(fds=True, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1,
                           fds_kernel="gaussian", fds_ks=5, fds_sigma=2.0, fds_mmt=0.9)


def seed_tables(fds, dev):
    g = torch.Generator(device=dev).manual_seed(1)
    nb, c = fds.running_mean.shape
    fds.running_mean_last_epoch = 0.3 * torch.randn(nb, c, device=dev, generator=g)
    fds.running_var_last_epoch = 0.5 + torch.rand(nb, c, device=dev, generator=g)
    fds.smoothed_mean_last_epoch = 0.3 * torch.randn(nb, c, device=dev, generator=g)
    fds.smoothed_var_last_epoch = 0.5 + torch.rand(nb, c, device=dev, generator=g)


def native_model():
    import net
    import resnet
    torch.manual_seed(0)
    m = net.model(args_ns(), resnet.E_resnet(resnet.resnet50()), 2048, BLOCKS).cuda()
    seed_tables(m.R.FDS, "cuda")
    return m


def reference_model():
    from oracle import encoder_ref, net_ref
    if not net_ref.available():
        return None
    sys.path.insert(0, encoder_ref.REF_DIR)
    from models import modules, net, resnet
    torch.manual_seed(0)
    m = net.model(args_ns(), modules.E_resnet(resnet.resnet50()), 2048, BLOCKS).cuda()
    seed_tables(m.R.FDS, "cuda")
    return m


def data(n):
    g = torch.Generator(device="cuda").manual_seed(n)
    image = torch.randn(n, 3, 228, 304, device="cuda", generator=g)
    depth = 0.5 + 9.5 * torch.rand(n, 1, 114, 152, device="cuda", generator=g)
    weight = 0.5 + torch.rand(n, 1, 114, 152, device="cuda", generator=g)
    return image, depth, weight


def train_step(m, opt, image, depth, weight):
    def step():
        m.train()
        opt.zero_grad()
        out, _ = m(image, depth, 1)
        loss = torch.mean(((out - depth) ** 2) * weight)
        loss.backward()
        opt.step()
    return step


def eval_step(m, image):
    def step():
        m.eval()
        with torch.no_grad():
            m(image)
    return step


def time_ms(step, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def head_arms(n=8, h=114, w=152, c=128):
    """(name -> step, name -> bytes) of the head kernels and of the padded-conv path they replace."""
    import _lib
    import dense_ops as O
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.relu(torch.randn(n, h, w, c, device="cuda", generator=g)).to(torch.bfloat16)
    wt = torch.randn(1, c, 5, 5, device="cuda", generator=g) * 0.02
    b = torch.randn(1, device="cuda", generator=g)
    dy = torch.randn(n, h, w, 1, device="cuda", generator=g)
    y = torch.empty(n, h, w, 1, device="cuda")
    dx = torch.empty_like(x)
    dw, db = torch.empty_like(wt), torch.empty_like(b)
    nb = _lib.raw("dirb200_depth_head_wgrad_workspace_bytes")(n, h, w, c)
    ws = torch.empty(nb, dtype=torch.uint8, device="cuda")
    st = _lib.stream_ptr()
    xp = x.detach().clone().requires_grad_(True)
    wp = wt.detach().clone().requires_grad_(True)
    bp = b.detach().clone().requires_grad_(True)
    dyb = dy.to(torch.bfloat16)

    def padded_fwd():
        with torch.no_grad():
            O.conv2d_nhwc(xp, wp, 1, 2) + bp.to(torch.bfloat16)

    def padded_fwd_bwd():
        (O.conv2d_nhwc(xp, wp, 1, 2) + bp.to(torch.bfloat16)).backward(dyb)

    def head_fwd_bwd():
        O.depth_head(xp, wp, bp).backward(dy)

    steps = {
        "fwd": lambda: _lib.call("dirb200_depth_head_fwd", _lib.ptr(x), _lib.ptr(wt), _lib.ptr(b), _lib.ptr(y), n, h, w,
                                 c, st),
        "dgrad": lambda: _lib.call("dirb200_depth_head_dgrad", _lib.ptr(dy), _lib.ptr(wt), _lib.ptr(dx), n, h, w, c, st),
        "wgrad": lambda: _lib.call("dirb200_depth_head_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(db),
                                   _lib.ptr(ws), nb, n, h, w, c, st),
        "head_fwd_bwd": head_fwd_bwd,
        "padded_conv_fwd": padded_fwd,
        "padded_conv_fwd_bwd": padded_fwd_bwd,
    }
    px = n * h * w
    nbytes = {"fwd": px * c * 2 + px * 4, "dgrad": px * 4 + px * c * 2, "wgrad": px * c * 2 + px * 4}
    return steps, nbytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "nyud2_model_bench needs a CUDA device"
    torch.backends.cudnn.benchmark = True
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    arms = {}
    models = {"native": native_model()}
    ref = reference_model()
    if ref is not None:
        models["reference"] = ref
    image8, depth8, weight8 = data(8)
    image1, _, _ = data(1)
    for name, m in models.items():
        opt = torch.optim.Adam(m.parameters(), 1e-4, weight_decay=1e-4)
        arms[f"train_b8_{name}"] = train_step(m, opt, image8, depth8, weight8)
        arms[f"eval_b8_{name}"] = eval_step(m, image8)
        arms[f"eval_b1_{name}"] = eval_step(m, image1)
    head_steps, head_bytes = head_arms()
    arms.update({f"head_{k}": v for k, v in head_steps.items()})
    for step in arms.values():
        for _ in range(a.warmup):
            step()
    torch.cuda.synchronize()
    times = {k: [] for k in arms}
    for _ in range(a.rounds):
        for k, step in arms.items():
            times[k].append(time_ms(step, a.steps))
    ms = {k: statistics.median(v) for k, v in times.items()}
    out = dict(card(), bench="nyud2_model", steps=a.steps, rounds=a.rounds)
    for k in ("train_b8", "eval_b8", "eval_b1"):
        out[k + "_ms"] = {arm: round(ms[f"{k}_{arm}"], 3) if f"{k}_{arm}" in ms else "not measured"
                          for arm in ("native", "reference")}
    head = {}
    for k, v in head_steps.items():
        e = {"us": round(1e3 * ms[f"head_{k}"], 2)}
        if k in head_bytes:
            bw = head_bytes[k] / (ms[f"head_{k}"] * 1e-3)
            e.update(bytes=head_bytes[k], GBps=round(bw / 1e9, 1), of_3p35TBps=round(bw / HBM, 3))
        head[k] = e
    out["head_8x114x152x128"] = head
    print(json.dumps(out))


if __name__ == "__main__":
    main()
