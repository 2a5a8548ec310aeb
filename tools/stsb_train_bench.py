"""STS-B-DIR training pieces on the device, at the reference's sizes (batch 128, d_word 300, d_hid 1500, 2 layers,
frozen embeddings, synthetic sentence lengths <= 40):

- clip + Adam over the model's trainable parameters: optim.Adam(max_grad_norm=5) (one norm launch, then the clipped
  multi-tensor Adam), clip_grad_norm_ + optim.Adam, and clip_grad_norm_ + torch's fused Adam.  Achieved bytes/s count
  4 B of norm read and 28 B of Adam traffic per parameter (read p, g, m, v; write p, m, v);
- a training step (forward, backward, clip / Adam) with the fused clipping and with clip_grad_norm_ + optim.Adam;
- STSShotAverage.get_metric at N = 1 000 and 51 200 (400 validation intervals of 128): the device kernel, with the
  host-to-device copy, against a host computation in the reference's style (a np.histogram edge search per label,
  numpy means, scipy's pearsonr / spearmanr / gmean).

Prints one JSON line with the card name and power limit read in the same run.

    python tools/stsb_train_bench.py [--steps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time
from types import SimpleNamespace

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "imbalanced-regression_b200"), os.path.join(ROOT, "tools")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

from stsb_model_bench import Task, Vocab, batch, card, timed  # noqa: E402

MANY = {0, 10, 12, 14, 16, 18, 20, 22, 24, 26, 28, 30, 32, 34, 36, 38, 40, 42, 44, 46, 48, 49}   # util.py:110-113
MEDIUM = {2, 4, 6, 8, 27, 35, 37}


def host_get_metric(pred, label):
    """The reference's host algorithm: one edge search per label, then numpy / scipy per group."""
    from scipy.stats import gmean, pearsonr, spearmanr
    bins = []
    for v in label.tolist():
        edges = np.histogram(np.array([], dtype=np.float32), bins=50, range=(0., 5.))[1]
        bins.append(49 if v == 5. else int(np.where(edges > v)[0][0]) - 1)
    shot = np.array(['many' if b in MANY else 'medium' if b in MEDIUM else 'few' for b in bins])
    x, y = np.array(pred.tolist()) * 5., np.array(label.tolist())
    out = {}
    for s in ('overall', 'many', 'medium', 'few'):
        sel = np.ones(x.size, bool) if s == 'overall' else shot == s
        xs, ys = x[sel], y[sel]
        d = np.abs(xs - ys)
        out[s] = (np.mean(d ** 2), np.mean(d), gmean(np.where(d == 0., 1e-10, d)), pearsonr(xs, ys)[0],
                  spearmanr(xs, ys)[0])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import optim
    import stsb_data
    from models import build_model
    dev = torch.device("cuda", 0)
    B, T, D, H, V = 128, 40, 300, 1500, 20000
    args = SimpleNamespace(d_word=D, n_layers_highway=0, glove=1, train_words=0, d_hid=H, n_layers_enc=2, dropout=0.2,
                           fds=0, start_smooth=1, cuda=0, loss='mse', huber_beta=0.5)
    torch.manual_seed(0)
    model = build_model(args, Vocab(), torch.randn(V, D), [Task()])
    params = [p for p in model.parameters() if p.requires_grad]
    n = sum(p.numel() for p in params)
    res = {"card": card(), "batch": B, "T": T, "d_word": D, "d_hid": H, "trainable_params": n}

    # clip + Adam alone, on fixed gradients
    g = torch.Generator(device=dev).manual_seed(0)
    for p in params:
        p.grad = torch.randn(p.shape, device=dev, generator=g) * 1e-3
    fused = optim.Adam(params, lr=1e-4, weight_decay=1e-5, max_grad_norm=5.0)
    plain = optim.Adam(params, lr=1e-4, weight_decay=1e-5)
    tfused = torch.optim.Adam(params, lr=1e-4, weight_decay=1e-5, fused=True)
    variants = {
        "fused_clip_adam": fused.step,
        "clip_grad_norm_then_optim_adam": lambda: (torch.nn.utils.clip_grad_norm_(params, 5.0), plain.step()),
        "clip_grad_norm_then_torch_fused_adam": lambda: (torch.nn.utils.clip_grad_norm_(params, 5.0), tfused.step()),
    }
    for name, fn in variants.items():
        ms = timed(fn, a.steps, a.warmup)
        res[f"{name}_ms"] = ms
        res[f"{name}_tb_per_s"] = 32.0 * n / (ms * 1e-3) / 1e12
    s1, s2, label = batch(B, T, V, dev, 0)

    def step(opt, clip):
        def run():
            model.train()
            out = model(Task(), 0, s1, s2, label=label)
            opt.zero_grad()
            out['loss'].backward()
            if clip:
                torch.nn.utils.clip_grad_norm_(params, 5.0)
            opt.step()
        return run

    res["train_step_fused_clip_ms"] = timed(step(fused, False), a.steps, a.warmup)
    res["train_step_clip_grad_norm_ms"] = timed(step(plain, True), a.steps, a.warmup)
    res["train_step_fused_clip_ms_again"] = timed(step(fused, False), a.steps, a.warmup)

    # get_metric: device (host buffer -> device -> kernel -> host) against the reference-style host computation
    rs = np.random.RandomState(0)
    for N in (1000, 51200):
        lab = np.where(rs.uniform(size=N) < 0.5, np.round(rs.uniform(0, 5, N) * 5) / 5, rs.uniform(0, 5, N))
        lab = lab.astype(np.float32)
        pred = (lab / 5 + rs.normal(0, 0.15, N)).astype(np.float32)
        scorer = stsb_data.STSShotAverage(['mse', 'l1', 'gmean', 'pearsonr', 'spearmanr'])
        for lo in range(0, N, 128):
            scorer(pred[lo:lo + 128], lab[lo:lo + 128])
        res[f"get_metric_device_n{N}_ms"] = timed(scorer.get_metric, max(a.steps, 5), a.warmup)
        dp, dl = torch.from_numpy(pred).to(dev), torch.from_numpy(lab).to(dev)
        res[f"shot_metrics_kernels_n{N}_ms"] = timed(lambda: stsb_data.shot_metrics(dp, dl), max(a.steps, 5), a.warmup)
        t0 = time.perf_counter()
        want = host_get_metric(pred, lab)
        res[f"get_metric_host_n{N}_ms"] = (time.perf_counter() - t0) * 1e3
        got = scorer.get_metric()
        res[f"get_metric_n{N}_max_rel_diff"] = max(
            abs(got[s][k] - w) / max(abs(w), 1.0) for s in want
            for k, w in zip(('mse', 'l1', 'gmean', 'pearsonr', 'spearmanr'), want[s]))
    print(json.dumps(res))


if __name__ == "__main__":
    main()
