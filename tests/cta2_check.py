"""Standalone GPU check + per-layer timing of the conv GEMMs under the kernel's run-time switches (not collected
by pytest; tests/test_gpu_conv_variants.py runs the parity half in subprocesses).

    python tests/cta2_check.py parity                    # defaults: tiled / im2col TMA (plain GEMMs + fused
                                                          # BN-statistics and folded-BN epilogues)
    DIRB200_IM2COL=0 python tests/cta2_check.py parity   # cp.async gather for the 3x3 / strided convs
    DIRB200_ATMA=0   python tests/cta2_check.py parity   # cp.async gather for every conv
    <switches> python tests/cta2_check.py time [substr]  # per-layer fprop/dgrad/wgrad times, batch-256 ResNet-50 shapes
                                                          # (also written to $DIRB200_OUT or the temp dir, conv_layers_<tag>.json)
    <switches> python tests/cta2_check.py one <substr> fprop|dgrad|wgrad   # a few launches of one layer (profiler target)

The switches are read once per process, hence the separate invocations.
"""
import json
import os
import sys
import tempfile
import traceback

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "imbalanced-regression_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import torch  # noqa: E402

PARITY = [
    # n, h, w, cin, cout, k, stride, pad
    (2, 8, 8, 64, 256, 1, 1, 0),        # one tile, the second consumer half entirely out of range
    (2, 8, 8, 128, 128, 3, 2, 1),       # stride-2 dgrad parity classes
    (2, 8, 8, 256, 512, 1, 2, 0),
    (3, 7, 7, 512, 512, 3, 1, 1),       # ragged M (147 rows = 2 m-tiles), 72 k-blocks
    (1, 14, 14, 1024, 256, 1, 1, 0),    # 16 k-blocks > ring depth
    (4, 7, 7, 512, 2048, 1, 1, 0),      # 16 n-tiles
    (5, 9, 11, 64, 128, 3, 2, 1),       # odd sizes
    (16, 56, 56, 64, 256, 1, 1, 0),     # 392 m-tiles x 2 n-tiles over the persistent CTAs
    (16, 28, 28, 128, 128, 3, 1, 1),    # BN=128, 98 m-tiles, 18 k-blocks
    (37, 14, 14, 256, 256, 3, 1, 1),    # ragged last m-tile (57 m-tiles)
    (64, 14, 14, 256, 1024, 1, 1, 0),   # several tiles per cluster, accumulator double buffering
    (75, 14, 14, 256, 256, 3, 1, 1),    # 115 m-tiles of a 3x3: im2col TMA, odd tile count
    (64, 28, 28, 512, 256, 1, 1, 0),    # tiled TMA, 8 k-blocks
    (4, 56, 56, 64, 64, 3, 1, 1),       # layer1 3x3: 64-wide tiles
    (3, 12, 20, 64, 64, 3, 1, 1),
]

# (name, n, h, w, cin, cout, k, stride, pad, count): every distinct non-stem conv of the batch-256 ResNet-50 step
# (SURVEY.md section 8d) and how many times it occurs in the network
LAYERS = [
    ("l1.0.c1 64->64 1x1 56", 256, 56, 56, 64, 64, 1, 1, 0, 1),
    ("l1.c2 64->64 3x3 56", 256, 56, 56, 64, 64, 3, 1, 1, 3),
    ("l1.c3 64->256 1x1 56", 256, 56, 56, 64, 256, 1, 1, 0, 4),
    ("l1.c1 256->64 1x1 56", 256, 56, 56, 256, 64, 1, 1, 0, 2),
    ("l2.0.c1 256->128 1x1 56", 256, 56, 56, 256, 128, 1, 1, 0, 1),
    ("l2.0.c2 128->128 3x3/2 56", 256, 56, 56, 128, 128, 3, 2, 1, 1),
    ("l2.c3 128->512 1x1 28", 256, 28, 28, 128, 512, 1, 1, 0, 4),
    ("l2.ds 256->512 1x1/2 56", 256, 56, 56, 256, 512, 1, 2, 0, 1),
    ("l2.c1 512->128 1x1 28", 256, 28, 28, 512, 128, 1, 1, 0, 3),
    ("l2.c2 128->128 3x3 28", 256, 28, 28, 128, 128, 3, 1, 1, 3),
    ("l3.0.c1 512->256 1x1 28", 256, 28, 28, 512, 256, 1, 1, 0, 1),
    ("l3.c2s 256->256 3x3/2 28", 256, 28, 28, 256, 256, 3, 2, 1, 1),
    ("l3.c3 256->1024 1x1 14", 256, 14, 14, 256, 1024, 1, 1, 0, 6),
    ("l3.ds 512->1024 1x1/2 28", 256, 28, 28, 512, 1024, 1, 2, 0, 1),
    ("l3.c1 1024->256 1x1 14", 256, 14, 14, 1024, 256, 1, 1, 0, 5),
    ("l3.c2 256->256 3x3 14", 256, 14, 14, 256, 256, 3, 1, 1, 5),
    ("l4.0.c1 1024->512 1x1 14", 256, 14, 14, 1024, 512, 1, 1, 0, 1),
    ("l4.0.c2 512->512 3x3/2 14", 256, 14, 14, 512, 512, 3, 2, 1, 1),
    ("l4.c3 512->2048 1x1 7", 256, 7, 7, 512, 2048, 1, 1, 0, 3),
    ("l4.ds 1024->2048 1x1/2 14", 256, 14, 14, 1024, 2048, 1, 2, 0, 1),
    ("l4.c1 2048->512 1x1 7", 256, 7, 7, 2048, 512, 1, 1, 0, 2),
    ("l4.c2 512->512 3x3 7", 256, 7, 7, 512, 512, 3, 1, 1, 2),
]


def parity():
    from test_gpu_conv import run_conv
    import test_gpu_conv_epilogues as E
    # the plain GEMMs, then the fused BatchNorm epilogues (statistics + finalize, folded BN) of
    # tests/test_gpu_conv_epilogues.py on its shapes
    cases = [(run_conv, cfg) for cfg in PARITY]
    cases += [(E.test_fprop_bn_stats_and_finalize, s) for s in E.SHAPES]
    cases += [(E.test_fprop_affine_epilogue, s) for s in E.SHAPES]
    bad = 0
    for fn, cfg in cases:
        try:
            fn(*cfg) if fn is run_conv else fn(cfg)
            torch.cuda.synchronize()
            print("PASS", fn.__name__, cfg, flush=True)
        except Exception as e:  # noqa: BLE001
            bad += 1
            print("FAIL", fn.__name__, cfg, repr(e)[:300], flush=True)
            traceback.print_exc()
            try:
                torch.cuda.synchronize()
            except Exception:  # noqa: BLE001  (sticky CUDA error: nothing more can run in this process)
                print("CUDA context lost; stopping", flush=True)
                break
    print(f"parity: {len(cases) - bad}/{len(cases)} ok (switches: " + " ".join(f"{k}={v}" for k, v in os.environ.items() if k.startswith("DIRB200_")) + ")")
    return bad


def _layer_tensors(n, h, w, cin, cout, k, stride, pad):
    ho, wo = (h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1
    x = torch.randn(n, h, w, cin, device="cuda").to(torch.bfloat16)
    dy = torch.randn(n, ho, wo, cout, device="cuda").to(torch.bfloat16)
    wf = (torch.randn(cout, k, k, cin, device="cuda") / (cin * k * k) ** 0.5).to(torch.bfloat16)
    wd = wf.permute(3, 1, 2, 0).contiguous()
    y = torch.empty(n, ho, wo, cout, dtype=torch.bfloat16, device="cuda")
    dx = torch.empty(n, h, w, cin, dtype=torch.bfloat16, device="cuda")
    dw = torch.zeros(cout, cin, k, k, dtype=torch.float32, device="cuda")
    return ho, wo, x, dy, wf, wd, y, dx, dw


def _call(which, shape, x, dy, wf, wd, y, dx, dw, ws, st):
    import _lib
    if which == "fprop":
        _lib.call("dirb200_conv_fprop", _lib.ptr(x), _lib.ptr(wf), _lib.ptr(y), *shape, 0, st)
    elif which == "dgrad":
        _lib.call("dirb200_conv_dgrad", _lib.ptr(dy), _lib.ptr(wd), _lib.ptr(dx), *shape, st)
    else:
        _lib.call("dirb200_conv_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(ws), ws.numel(), *shape, 0, 0, st)


def time_layers(reps=10, only=None):
    import _lib, _convlib  # noqa: F401
    out = {}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device="cuda")
    total = {"fprop": 0.0, "dgrad": 0.0, "wgrad": 0.0}
    for name, n, h, w, cin, cout, k, stride, pad, count in LAYERS:
        if only and only not in name:
            continue
        ho, wo, x, dy, wf, wd, y, dx, dw = _layer_tensors(n, h, w, cin, cout, k, stride, pad)
        shape = (n, h, w, cin, cout, k, k, stride, pad)
        ws = torch.empty(_lib.raw("dirb200_conv_wgrad_workspace_bytes")(*shape, 0), dtype=torch.uint8, device="cuda")
        st = _lib.stream_ptr()
        res = {}
        for which in ("fprop", "dgrad", "wgrad"):
            ts = []
            for it in range(reps + 2):
                flush.fill_(it & 1)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                _call(which, shape, x, dy, wf, wd, y, dx, dw, ws, st)
                e1.record()
                torch.cuda.synchronize()
                if it >= 2:
                    ts.append(e0.elapsed_time(e1))
            ms = sorted(ts)[len(ts) // 2]
            flops = 2.0 * n * ho * wo * cout * cin * k * k
            res[which] = {"ms": round(ms, 4), "tflops": round(flops / ms / 1e9, 1)}
            total[which] += ms * count
        res["count"] = count
        out[name] = res
        print(f"{name:28s} x{count}  fprop {res['fprop']['ms']:.3f} ms {res['fprop']['tflops']:6.0f}   "
              f"dgrad {res['dgrad']['ms']:.3f} ms {res['dgrad']['tflops']:6.0f}   "
              f"wgrad(+reduce) {res['wgrad']['ms']:.3f} ms {res['wgrad']['tflops']:6.0f} TF/s", flush=True)
    print("per-step totals (count-weighted, without the stem): " + ", ".join(f"{k} {v:.3f} ms" for k, v in total.items())
          + f", all {sum(total.values()):.3f} ms", flush=True)
    out["_total_ms"] = total
    tag = os.environ.get("DIRB200_TAG", "default")
    out_dir = os.environ.get("DIRB200_OUT", tempfile.gettempdir())
    os.makedirs(out_dir, exist_ok=True)
    json.dump(out, open(os.path.join(out_dir, f"conv_layers_{tag}.json"), "w"), indent=1)


def one_layer(sub, which, reps=4):
    """A few launches of one layer / one GEMM form: the target of an `ncu -k regex:igemm` capture."""
    import _lib, _convlib  # noqa: F401
    for name, n, h, w, cin, cout, k, stride, pad, count in LAYERS:
        if sub not in name:
            continue
        ho, wo, x, dy, wf, wd, y, dx, dw = _layer_tensors(n, h, w, cin, cout, k, stride, pad)
        shape = (n, h, w, cin, cout, k, k, stride, pad)
        ws = torch.empty(_lib.raw("dirb200_conv_wgrad_workspace_bytes")(*shape, 0), dtype=torch.uint8, device="cuda")
        for _ in range(reps):
            _call(which, shape, x, dy, wf, wd, y, dx, dw, ws, _lib.stream_ptr())
        torch.cuda.synchronize()
        print("ran", name, which, reps)
        return


if __name__ == "__main__":
    mode = sys.argv[1] if len(sys.argv) > 1 else "parity"
    if mode == "parity":
        sys.exit(1 if parity() else 0)
    if mode == "one":
        one_layer(sys.argv[2], sys.argv[3])
    else:
        time_layers(only=sys.argv[2] if len(sys.argv) > 2 else None)
