"""BASELINE config 4 figures (NYUD2-DIR, synthetic 640x480 -> refinement input [32, 128, 240, 320]): the operators of the
refinement module R (nyud2-dir/models/modules.py:128-174) on one GPU -- the 5x5 128->128 convolution (fprop / dgrad /
wgrad), the FDS update over the 2.46 M x 128 pixel features, bilinear up-sampling and the per-pixel LDS-weighted loss
pieces are timed with CUDA events (L2 flushed between repetitions).  One JSON line; not part of bench.py's headline."""
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200")):
    sys.path.insert(0, p)
import torch  # noqa: E402


def timed(fn, reps=5):
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        flush.fill_(1)
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b))
    return sorted(ts)[len(ts) // 2]


def main():
    import _lib, _convlib  # noqa: F401
    import dense_ops as D
    from fds_variants import FDSDepth
    n, h, w, c, k = 32, 240, 320, 128, 5
    dev = "cuda"
    x = torch.randn(n, h, w, c, device=dev).to(torch.bfloat16)
    dy = torch.randn(n, h, w, c, device=dev).to(torch.bfloat16)
    wt = (torch.randn(c, c, k, k, device=dev) / (c * k * k) ** 0.5)
    st = _lib.stream_ptr()
    wf = torch.empty(c, k, k, c, dtype=torch.bfloat16, device=dev)
    wd = torch.empty(c, k, k, c, dtype=torch.bfloat16, device=dev)
    _lib.call("dirb200_conv_prep_weights", _lib.ptr(wt), c, c, k, k, 0, _lib.ptr(wf), _lib.ptr(wd), st)
    y = torch.empty_like(x)
    dx = torch.empty_like(x)
    shape = (n, h, w, c, c, k, k, 1, 2)
    nbytes = _lib.raw("dirb200_conv_wgrad_workspace_bytes")(*shape, 0)
    ws = torch.empty(nbytes, dtype=torch.uint8, device=dev)
    dw = torch.empty(c, c, k, k, dtype=torch.float32, device=dev)
    gflop = 2.0 * n * h * w * c * c * k * k / 1e9
    out = {"workload": "NYUD2-DIR refinement module R at BASELINE config 4 size: [32, 128, 240, 320] bf16 NHWC, 5x5 128->128",
           "conv_gflop": gflop}
    for name, fn in (("fprop", lambda: _lib.call("dirb200_conv_fprop", _lib.ptr(x), _lib.ptr(wf), _lib.ptr(y), *shape, 0, st)),
                     ("dgrad", lambda: _lib.call("dirb200_conv_dgrad", _lib.ptr(dy), _lib.ptr(wd), _lib.ptr(dx), *shape, st)),
                     ("wgrad", lambda: _lib.call("dirb200_conv_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(ws),
                                                 nbytes, *shape, 0, 0, st))):
        ms = timed(fn)
        out[f"conv5x5_{name}_ms"] = round(ms, 3)
        out[f"conv5x5_{name}_tflops"] = round(gflop / ms, 1)
    # bilinear up-sampling of a decoder stage (D.up4: 114x152 -> 228x304 in the reference's geometry; here 120x160 -> 240x320, 64 ch)
    xs = torch.randn(n, 120, 160, 64, device=dev).to(torch.bfloat16)
    up = torch.empty(n, 240, 320, 64, dtype=torch.bfloat16, device=dev)
    ms = timed(lambda: _lib.call("dirb200_upsample_bilinear_fwd", _lib.ptr(xs), n, 120, 160, 64, 240, 320, _lib.ptr(up), st))
    out["upsample_fwd_ms"] = round(ms, 3)
    out["upsample_fwd_gbs"] = round((xs.numel() + up.numel()) * 2 / ms / 1e6, 1)
    gdn = torch.empty_like(xs)
    ms = timed(lambda: _lib.call("dirb200_upsample_bilinear_bwd", _lib.ptr(up), n, 120, 160, 64, 240, 320, _lib.ptr(gdn), st))
    out["upsample_bwd_ms"] = round(ms, 3)
    # FDS over the pixel features of one batch: [n*h*w, 128] fp32, depth bins clamp(int(d*10), 7, 99)
    fds = FDSDepth(feature_dim=c, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1, kernel="gaussian", ks=5,
                   sigma=2, momentum=0.9).to(dev)
    feats = torch.relu(torch.randn(n * h * w, c, device=dev) + 0.5)
    depth = torch.empty(n * h * w, device=dev).uniform_(0.7, 10.0)
    def fds_update():                       # the accumulation itself on the [pixels, 128] rows (what the NHWC layout already is)
        fds.begin_epoch_stats(depth)
        fds.accumulate_batch(feats, depth)
        fds.finish_epoch_stats(0)
    ms = timed(fds_update, reps=3)
    out["fds_update_ms"] = round(ms, 3)
    out["fds_update_gbs"] = round(feats.numel() * 4 / ms / 1e6, 1)
    # the whole refinement module R (conv0-bn0-relu-conv1-bn1-relu-conv2, training mode), forward + backward
    del x, dy, y, dx, ws, feats, depth, up, xs, gdn
    torch.cuda.empty_cache()
    m = D.RefinementR(c).to(dev)
    m.train()
    xin = torch.randn(n, h, w, c, device=dev).to(torch.bfloat16).requires_grad_(True)
    gout = torch.randn(n, h, w, 1, device=dev).to(torch.bfloat16)
    def r_step():
        m.zero_grad(set_to_none=True)
        xin.grad = None
        m(xin).backward(gout)
    ms = timed(r_step, reps=3)
    out["R_module_fwd_bwd_ms"] = round(ms, 2)
    out["R_module_conv_gflop_fwd_bwd"] = round(3 * 2 * gflop + 3 * 2.0 * n * h * w * c * 64 * k * k / 1e9, 1)   # conv2 runs 64 padded outputs
    out["R_module_images_per_s"] = round(n / ms * 1e3, 1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
