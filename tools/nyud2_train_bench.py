"""NYUD2-DIR training-step timing (nyud2_train.py, nyud2-dir/train.py) on one GPU; prints one JSON line with the card's
name and power limit.

  optimizer  one Adam step over net.model's 245 parameters (67,569,473 fp32 values, weight decay 1e-4) under three arms
             alternated within the run: optim.Adam (dirb200_adam_step_multi), torch.optim.Adam (default foreach) and
             torch.optim.Adam(fused=True), each as called (host work included: back-to-back steps are host-bound when
             the host takes longer than the kernels), and optim.Adam's kernel alone (dirb200_adam_step_multi relaunched
             on one prebuilt segment table).  Each with its achieved bytes/s against the 28 B per parameter one fused
             pass needs (read param, grad, exp_avg, exp_avg_sq; write param, exp_avg, exp_avg_sq) and 3.35 TB/s, the
             H100 SXM's data-sheet HBM3 bandwidth
  train      one full training step at 228 x 304, batch 8 and batch 32: zero_grad, model(image, depth, epoch) with FDS
             smoothing active, loss.weighted_mse_loss, backward, and the step of each optimizer arm
  fds        one batch of the epoch-end FDS collection (batch 8): the train-mode forward under no_grad and
             FDSDepth.accumulate_map of its 128-channel feature map

Every figure is the median over --rounds rounds of the mean over --steps calls, timed with CUDA events after --warmup
calls.

    python tools/nyud2_train_bench.py [--steps 10] [--warmup 3] [--rounds 5]
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

import numpy as np  # noqa: E402
import torch  # noqa: E402

HBM = 3.35e12
BYTES_PER_PARAM = 28


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    f = [s.strip() for s in q.stdout.strip().split(",")] if q.returncode == 0 else ["?", "?", "?"]
    return {"gpu": f[0], "power_limit": f[1], "max_sm_clock": f[2] if len(f) > 2 else "?"}


def make_model(dev):
    import net
    import resnet
    args = SimpleNamespace(fds=True, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1,
                           fds_kernel="gaussian", fds_ks=5, fds_sigma=2.0, fds_mmt=0.9)
    torch.manual_seed(0)
    m = net.model(args, resnet.E_resnet(resnet.resnet50()), 2048, [256, 512, 1024, 2048]).to(dev)
    g = torch.Generator(device=dev).manual_seed(1)
    fds = m.R.FDS
    nb, c = fds.running_mean.shape
    fds.running_mean_last_epoch = 0.3 * torch.randn(nb, c, device=dev, generator=g)
    fds.running_var_last_epoch = 0.5 + torch.rand(nb, c, device=dev, generator=g)
    fds.smoothed_mean_last_epoch = 0.3 * torch.randn(nb, c, device=dev, generator=g)
    fds.smoothed_var_last_epoch = 0.5 + torch.rand(nb, c, device=dev, generator=g)
    return m


def batch(n, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(n, 3, 228, 304, device=dev, generator=g)
    depth = 0.5 + 9.5 * torch.rand(n, 1, 114, 152, device=dev, generator=g)
    weight = 0.5 + torch.rand(n, 1, 114, 152, device=dev, generator=g)
    return x, depth, weight


def timed(fn, steps):
    start, stop = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for _ in range(steps):
        fn()
    stop.record()
    stop.synchronize()
    return start.elapsed_time(stop) / steps


def alternate(arms, steps, warmup, rounds):
    """{name: median over rounds of the mean ms per call}, the arms alternated within each round."""
    for fn in arms.values():
        for _ in range(warmup):
            fn()
    torch.cuda.synchronize()
    got = {k: [] for k in arms}
    for _ in range(rounds):
        for k, fn in arms.items():
            got[k].append(timed(fn, steps))
    return {k: statistics.median(v) for k, v in got.items()}


def kernel_only(opt, params):
    """One dirb200_adam_step_multi launch over a segment table built once from opt's state (step 1 corrections)."""
    import _lib
    import optim
    opt.step()                                   # creates the moments
    st = [opt.state[p] for p in params]
    t = np.empty(len(params), dtype=optim._SEGMENT)
    t['param'] = [p.data_ptr() for p in params]
    t['grad'] = [p.grad.data_ptr() for p in params]
    t['exp_avg'] = [s['exp_avg'].data_ptr() for s in st]
    t['exp_avg_sq'] = [s['exp_avg_sq'].data_ptr() for s in st]
    t['numel'] = [p.numel() for p in params]
    t['bc1'], t['bc2_sqrt'] = optim._bias_corrections(0.9, 0.999, 1)
    ptr, n = t.ctypes.data_as(_lib.P), len(params)
    stream = _lib.stream_ptr()

    def fn():
        _lib.call("dirb200_adam_step_multi", ptr, n, 1e-4, 0.9, 0.999, 1e-8, 1e-4, stream)
    fn.table = t                                 # keeps the table alive
    return fn


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("nyud2_train_bench needs a CUDA device")
    import optim
    from loss import weighted_mse_loss
    dev = torch.device("cuda", 0)
    out = {"bench": "nyud2_train", **card(), "steps": a.steps, "warmup": a.warmup, "rounds": a.rounds}

    m = make_model(dev)
    m.train()
    params = list(m.parameters())
    n_params = sum(p.numel() for p in params)
    out.update(tensors=len(params), parameters=n_params)
    opts = {"optim.Adam": optim.Adam(params, 1e-4, weight_decay=1e-4),
            "torch_foreach": torch.optim.Adam(params, 1e-4, weight_decay=1e-4),
            "torch_fused": torch.optim.Adam(params, 1e-4, weight_decay=1e-4, fused=True)}

    # the optimizer step alone, on gradients of one real backward
    x, depth, weight = batch(8, dev)
    out_, _ = m(x, depth, 1)
    weighted_mse_loss(out_, depth, weight).backward()
    arms = {k: o.step for k, o in opts.items()}
    arms["optim.Adam_kernel_only"] = kernel_only(opts["optim.Adam"], params)
    ms = alternate(arms, a.steps, a.warmup, a.rounds)
    need = BYTES_PER_PARAM * n_params
    out["optimizer_step"] = {k: {"ms": round(v, 4), "TB_per_s": round(need / (v * 1e-3) / 1e12, 3),
                                 "share_of_hbm": round(need / (v * 1e-3) / HBM, 3)} for k, v in ms.items()}
    out["optimizer_step_floor_ms"] = round(need / HBM * 1e3, 4)

    # full training steps
    for n in (8, 32):
        x, depth, weight = batch(n, dev, seed=n)

        def step(opt):
            def fn():
                opt.zero_grad()
                o, _ = m(x, depth, 1)
                weighted_mse_loss(o, depth, weight).backward()
                opt.step()
            return fn
        ms = alternate({k: step(o) for k, o in opts.items()}, a.steps, a.warmup, a.rounds)
        out[f"train_step_b{n}_ms"] = {k: round(v, 3) for k, v in ms.items()}
        out[f"peak_mem_b{n}_GB"] = round(torch.cuda.max_memory_allocated() / 1e9, 2)

    # one FDS collection batch
    x, depth, _ = batch(8, dev, seed=3)
    fds = m.R.FDS

    def collect():
        with torch.no_grad():
            _, feature = m(x, depth, 1)
            fds.accumulate_map(feature, depth)
    fds.begin_epoch_stats(torch.empty(0, device=dev))
    out["fds_collect_b8_ms"] = round(alternate({"fds": collect}, a.steps, a.warmup, a.rounds)["fds"], 3)
    fds.abort_epoch_stats()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
