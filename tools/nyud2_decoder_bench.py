"""NYUD2-DIR decoder D + multi-scale fusion MFF timing (dense_ops.D / MFF, nyud2-dir/models/modules.py:6-31, 61-128):
forward + backward with seeded output gradients on E_resnet-shaped NHWC bf16 block maps, at 228 x 304 batch 8 and
480 x 640 batch 32.

  stored    the modules' default: each up-projection's input up-sampled and stored, then conv1 + conv2 as ONE
            convolution (weights concatenated along Cout)
  unfused   the plain composition: the stored up-sample, then conv1 and conv2 as two conv2d_nhwc calls (16-channel
            convolutions padded to 64 each)
  reference the reference's own D / MFF under torch fp32 / cuDNN with TF32 on (NCHW), where __graft_entry__.build()
            copied them into oracle/_ref (oracle/encoder_ref.py); reported as not measured otherwise

The two native forms alternate within one run (--rounds rounds of --steps steps each); each figure is the median step
time over rounds, with the peak memory allocated during a step.  Prints one JSON line with the card name and power
limit.

    python tools/nyud2_decoder_bench.py [--steps 5] [--warmup 2] [--rounds 3]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

SHAPES = [(8, 228, 304), (32, 480, 640)]
CHANNELS = (256, 512, 1024, 2048)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, limit = (q.stdout.strip().partition(",") if q.returncode == 0 else ("?", "", "?"))
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": limit.strip()}


def unfused_branch_convs(self, x, size):
    """UpProjection.branch_convs as the plain composition: the stored up-sample, then conv1 and conv2 as two
    conv2d_nhwc calls (16-channel convolutions padded to 64 each)."""
    import dense_ops as O
    up = O.upsample_bilinear(x, size)

    def conv(wt):
        c = wt.shape[0]
        if c % 64 == 0:
            return O._ConvFn.apply(up, wt, 1, 2)
        wp = torch.cat([wt, wt.new_zeros(64 - c % 64, *wt.shape[1:])], 0)
        return O.split_channels(O._ConvFn.apply(up, wp, 1, 2), [c])[0]
    return conv(self.conv1.weight), conv(self.conv2.weight)


def blocks(n, h, w, nchw=False):
    from resnet import _feature_maps
    g = torch.Generator(device="cuda").manual_seed(0)
    out = []
    for c, (hh, ww) in zip(CHANNELS, _feature_maps(h, w)[1:]):
        t = torch.relu(torch.randn(n, hh, ww, c, device="cuda", generator=g))
        out.append(t.permute(0, 3, 1, 2).contiguous() if nchw else t.to(torch.bfloat16))
    return out


def time_steps(step, steps):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps, (torch.cuda.max_memory_allocated() - base) / 2 ** 30


def native_step(Dm, Mm, xs):
    def step():
        d = Dm(*xs)
        m = Mm(*xs, (d.shape[1], d.shape[2]))
        torch.autograd.backward([d, m], [torch.ones_like(d), torch.ones_like(m)])
        for mod in (Dm, Mm):
            for p in mod.parameters():
                p.grad = None
    return step


def reference(n, h, w, steps, warmup):
    from oracle import encoder_ref
    if not os.path.exists(os.path.join(encoder_ref.REF_DIR, "models", "modules.py")):
        return {"ref_ms": "not measured (reference modules not installed)"}
    sys.path.insert(0, encoder_ref.REF_DIR)
    from models import modules
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    Dm, Mm = modules.D(2048).cuda().train(), modules.MFF(list(CHANNELS)).cuda().train()
    xs = [x.requires_grad_(False) for x in blocks(n, h, w, nchw=True)]

    def step():
        d = Dm(*xs)
        m = Mm(*xs, [d.size(2), d.size(3)])
        torch.autograd.backward([d, m], [torch.ones_like(d), torch.ones_like(m)])
        for mod in (Dm, Mm):
            for p in mod.parameters():
                p.grad = None
    for _ in range(warmup):
        step()
    ms, gb = time_steps(step, steps)
    return {"ref_ms": round(ms, 2), "ref_peak_gib": round(gb, 2)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-reference", action="store_true")
    a = ap.parse_args()
    import dense_ops as O
    paired = O.UpProjection.branch_convs
    forms = (("stored", paired), ("unfused", unfused_branch_convs))
    out = {"tool": "nyud2_decoder_bench", **card(), "shapes": []}
    for n, h, w in SHAPES:
        torch.manual_seed(0)
        Dm, Mm = O.D(2048).cuda().train(), O.MFF(list(CHANNELS)).cuda().train()
        xs = blocks(n, h, w)
        step = native_step(Dm, Mm, xs)
        res = {"n": n, "h": h, "w": w}

        def use(branch):
            O.UpProjection.branch_convs = branch
        for form, branch in forms:
            use(branch)
            res[f"{form}_ms"], res[f"{form}_peak_gib"] = [], 0.0
            for _ in range(a.warmup):
                step()
        for _ in range(a.rounds):
            for form, branch in forms:
                use(branch)
                ms, gb = time_steps(step, a.steps)
                res[f"{form}_ms"].append(round(ms, 2))
                res[f"{form}_peak_gib"] = round(max(res[f"{form}_peak_gib"], gb), 2)
        use(paired)
        for form, _ in forms:
            res[f"{form}_median_ms"] = statistics.median(res[f"{form}_ms"])
        del Dm, Mm, xs, step
        torch.cuda.empty_cache()
        if not a.no_reference:
            try:
                res.update(reference(n, h, w, a.steps, a.warmup))
            except torch.cuda.OutOfMemoryError:
                res["ref_ms"] = "not measured (out of memory)"
            torch.cuda.empty_cache()
        out["shapes"].append(res)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
