"""ResNet family timing: one training step (FDS smoothing with epoch >= 2 tables, LDS-weighted L1 loss, backward, Adam;
the step of bench.py on one GPU) and one eval forward, at batch 256 x 224^2, for resnet18 / 34 / 50 / 101 / 152 on the
native runner -- against the reference's own ResNet (agedb-dir/resnet.py, fp32 under torch / cuDNN with TF32 on) where
__graft_entry__.build() copied it into oracle/_ref (oracle/ref_step.py); the tool says so when that copy is absent.
Conv TFLOP/s are algorithmic FLOPs (2 per multiply-add over the model's convolutions: 1.814 / 3.663 / 4.087 / 7.799 /
11.51 GMAC per 224^2 image for ResNet-18 / 34 / 50 / 101 / 152) over the measured time; the training step counts the
forward, the data gradient (not the stem's) and the weight gradient of every conv.  Prints the card's name and power
limit and one JSON line; needs a CUDA device.

    python tools/resnet_family_bench.py [--steps 10] [--warmup 3] [--depths 18,34,50,101,152] [--no-reference]
"""
import argparse
import importlib
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

BATCH, HW = 256, 224
DEPTHS = {18: ("BasicBlock", (2, 2, 2, 2)), 34: ("BasicBlock", (3, 4, 6, 3)), 50: ("Bottleneck", (3, 4, 6, 3)),
          101: ("Bottleneck", (3, 4, 23, 3)), 152: ("Bottleneck", (3, 8, 36, 3))}
FDS_ARGS = dict(bucket_num=100, bucket_start=0, start_update=0, start_smooth=1, kernel="gaussian", ks=5, sigma=2,
                momentum=0.9)


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, limit = (q.stdout.strip().partition(",") if q.returncode == 0 else ("?", "", "?"))
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": limit.strip()}


def conv_macs(depth, h=HW, w=HW):
    """(multiply-adds per image of every conv, of the stem alone) for an h x w input."""
    block, layers = DEPTHS[depth]

    def conv(hi, wi, cin, cout, k, s, p):
        ho, wo = (hi + 2 * p - k) // s + 1, (wi + 2 * p - k) // s + 1
        return ho * wo * cout * cin * k * k, ho, wo
    stem, h, w = conv(h, w, 3, 64, 7, 2, 3)
    h, w = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    total, inplanes = 0, 64
    for li, nblocks in enumerate(layers):
        planes = 64 << li
        out = planes * (1 if block == "BasicBlock" else 4)
        for b in range(nblocks):
            s = 2 if (b == 0 and li > 0) else 1
            if block == "BasicBlock":
                f1, ho, wo = conv(h, w, inplanes, planes, 3, s, 1)
                f2, _, _ = conv(ho, wo, planes, planes, 3, 1, 1)
                total += f1 + f2
            else:
                f1, _, _ = conv(h, w, inplanes, planes, 1, 1, 0)
                f2, ho, wo = conv(h, w, planes, planes, 3, s, 1)
                f3, _, _ = conv(ho, wo, planes, out, 1, 1, 0)
                total += f1 + f2 + f3
            if b == 0 and (s != 1 or inplanes != out):
                total += conv(h, w, inplanes, out, 1, s, 0)[0]
            h, w, inplanes = ho, wo, out
    return stem + total, stem


def time_ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(steps):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / steps


def batch(seed=1000):
    """A synthetic batch (x, targets, LDS weights: sqrt_inv + gaussian ks5 sigma2 over a synthetic label column)."""
    from datasets import lds_prepare_weights
    g = torch.Generator().manual_seed(seed)
    labels = torch.randint(0, 100, (12208,), generator=g).float()
    w_all = torch.as_tensor(lds_prepare_weights(labels.numpy(), "sqrt_inv", lds=True, lds_kernel="gaussian", lds_ks=5,
                                                lds_sigma=2)).float()
    idx = torch.randint(0, labels.numel(), (BATCH,), generator=g)
    x = torch.randn(BATCH, 3, HW, HW, generator=g)
    return x.cuda(), labels[idx].reshape(-1, 1).cuda(), w_all.reshape(-1)[idx].reshape(-1, 1).cuda(), labels


def warm_fds(fds, labels, dim, native):
    """FDS in its epoch >= 2 state (train.py:269-281 order) from two synthetic epochs of features."""
    gen = torch.Generator(device="cuda").manual_seed(123)
    lab = labels.cuda()
    for epoch in (0, 1):
        feats = torch.relu(torch.randn(lab.numel(), dim, device="cuda", generator=gen) + 0.5)
        fds.update_last_epoch_stats(epoch)
        if native:
            fds.begin_epoch_stats(lab)
            for i in range(0, lab.numel(), 4096):
                fds.accumulate_batch(feats[i:i + 4096], lab[i:i + 4096])
            fds.finish_epoch_stats(epoch)
        else:
            fds.update_running_stats(feats, lab, epoch)
    fds.update_last_epoch_stats(2)


def native_arm(depth, steps, warmup):
    import resnet
    from loss import weighted_l1_loss
    from optim import FusedAdam
    torch.manual_seed(0)
    model = getattr(resnet, f"resnet{depth}")(fds=True, **FDS_ARGS).cuda()
    x, t, w, labels = batch()
    warm_fds(model.FDS, labels, model.FDS.feature_dim, native=True)
    opt = FusedAdam(model.parameters(), lr=1e-3)

    def train_step():
        model.train()
        out, _ = model(x, t, 2)
        loss = weighted_l1_loss(out, t, w)
        opt.zero_grad()
        loss.backward()
        opt.step()

    def eval_step():
        model.eval()
        with torch.no_grad():
            model(x)
    ms = time_ms(train_step, steps, warmup), time_ms(eval_step, steps, warmup)
    del model, opt
    return ms


def reference_modules():
    """The reference's resnet / loss modules from oracle/_ref/agedb-dir (None when absent), imported under their own
    names with this package's same-named modules put back afterwards."""
    from oracle import ref_step
    if not ref_step.available():
        return None
    names = ("resnet", "fds", "loss", "utils")
    saved_path, saved = list(sys.path), {k: sys.modules.get(k) for k in names}
    try:
        sys.path.insert(0, ref_step.REF_DIR)
        for k in names:
            sys.modules.pop(k, None)
        mods = importlib.import_module("resnet"), importlib.import_module("loss")
    finally:
        sys.path[:] = saved_path
        for k, v in saved.items():
            sys.modules.pop(k, None)
            if v is not None:
                sys.modules[k] = v
    return mods


def reference_arm(mods, depth, steps, warmup):
    ref_resnet, ref_loss = mods
    block, layers = DEPTHS[depth]
    torch.backends.cudnn.allow_tf32 = True
    torch.backends.cuda.matmul.allow_tf32 = True
    torch.backends.cudnn.benchmark = True
    torch.manual_seed(0)
    model = ref_resnet.ResNet(getattr(ref_resnet, block), list(layers), fds=True, **FDS_ARGS).cuda()
    x, t, w, labels = batch()
    warm_fds(model.FDS, labels, model.FDS.feature_dim, native=False)
    opt = torch.optim.Adam(model.parameters(), lr=1e-3)

    def train_step():
        model.train()
        out, _ = model(x, t, 2)
        loss = ref_loss.weighted_l1_loss(out, t, w)
        opt.zero_grad()
        loss.backward()
        opt.step()

    def eval_step():
        model.eval()
        with torch.no_grad():
            model(x)
    ms = time_ms(train_step, steps, warmup), time_ms(eval_step, steps, warmup)
    del model, opt
    return ms


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--depths", default="18,34,50,101,152")
    ap.add_argument("--no-reference", dest="no_reference", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "resnet_family_bench needs a CUDA device"
    out = dict(card(), batch=BATCH, hw=HW, runs=[])
    mods = None if a.no_reference else reference_modules()
    if mods is None and not a.no_reference:
        out["reference"] = "absent: oracle/_ref/agedb-dir not installed (run __graft_entry__.build() where the " \
                           "reference checkout exists)"
    for depth in (int(d) for d in a.depths.split(",")):
        macs, stem = conv_macs(depth)
        fwd = 2.0 * BATCH * macs
        train = 3 * fwd - 2.0 * BATCH * stem                      # no data gradient of the input
        r = dict(model=f"resnet{depth}", gmac_per_image=round(macs / 1e9, 3))
        tr, ev = native_arm(depth, a.steps, a.warmup)
        r.update(native_train_ms=round(tr, 2), native_train_conv_tflops=round(train / tr / 1e9, 1),
                 native_eval_ms=round(ev, 2), native_eval_conv_tflops=round(fwd / ev / 1e9, 1))
        torch.cuda.empty_cache()
        if mods is not None:
            rtr, rev = reference_arm(mods, depth, a.steps, a.warmup)
            r.update(reference_train_ms=round(rtr, 2), reference_train_conv_tflops=round(train / rtr / 1e9, 1),
                     reference_eval_ms=round(rev, 2), reference_eval_conv_tflops=round(fwd / rev / 1e9, 1),
                     train_speedup=round(rtr / tr, 2), eval_speedup=round(rev / ev, 2))
            torch.cuda.empty_cache()
        out["runs"].append(r)
        print(json.dumps(r), file=sys.stderr, flush=True)
    out["reference_backend"] = "torch %s fp32, cuDNN %s, tf32 on" % (torch.__version__, torch.backends.cudnn.version())
    print(json.dumps(out))


if __name__ == "__main__":
    main()
