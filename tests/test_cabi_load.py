"""CPU-only: the C-ABI library loads and exports every symbol include/dirb200.h
declares; argument validation works without a GPU (no compute calls)."""
import ctypes
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    txt = open(os.path.join(ROOT, "include", "dirb200.h")).read()
    txt = re.sub(r"/\*.*?\*/", "", txt, flags=re.S)
    return sorted(set(re.findall(r"\b(dirb200_[a-z0-9_]+)\s*\(", txt)))


def test_library_exports_every_declared_symbol():
    import _lib
    import _convlib, resnet  # noqa: F401  (register the conv-stack / runner bindings)
    lib = ctypes.CDLL(_lib.LIB_PATH)
    syms = header_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/dirb200.h but not exported"
    # and the Python binding table covers the header
    assert set(syms) <= set(_lib.exported_symbols()), set(syms) - set(_lib.exported_symbols())


def test_version_and_error_channel():
    import _lib
    assert _lib.raw("dirb200_version")() >= 100
    # invalid argument is rejected before any CUDA call
    rc = _lib.raw("dirb200_fds_smooth_tables")(None, 10, 4, None, 5, None, None)
    assert rc == -1 and "null" in _lib.last_error()
    rc = _lib.raw("dirb200_loss_fwd_bwd")(99, None, None, None, 4, 0.0, 1.0, 0, 1.0, None, None, None, 0, None)
    assert rc == -1 and "kind" in _lib.last_error()


def test_no_cpu_fallback():
    import pytest
    import torch
    import _lib
    from loss import weighted_l1_loss
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(_lib.Dirb200Error):
        weighted_l1_loss(torch.zeros(4, 1), torch.zeros(4, 1))


def test_wgrad_split_search_never_leaves_a_straggler_wave():
    """Host-side scheduling of the wgrad split-K GEMM (csrc/conv_igemm.cu: conv_wgrad_splits), observable without a
    GPU through dirb200_conv_wgrad_workspace_bytes = splits * K_total * Cout * 4, with the SM count the library itself
    uses (num_sms(): the device's, capped by DIRB200_SMS; the H100 SXM's 132 when no device is present).  For every conv of the batch-256 ResNet-50: the work items (tiles x splits) must fill the
    persistent CTAs' waves to >= 85 % -- a ceil(2*SMs/tiles) rule leaves a straggler wave of a few items on the 3x3
    layers -- and every split keeps >= 8 k-blocks."""
    import _lib, _convlib  # noqa: F401
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count if torch.cuda.is_available() else 132
    cap = int(os.environ.get("DIRB200_SMS", "0") or 0)
    if 0 < cap < sms:
        sms = cap
    convs = []          # (h, cin, cout, k, stride, pad)
    h, inpl = 56, 64
    for li, nb in enumerate((3, 4, 6, 3)):
        pl = 64 << li
        for b in range(nb):
            s = 2 if (b == 0 and li > 0) else 1
            convs += [(h, inpl, pl, 1, 1, 0), (h, pl, pl, 3, s, 1), (h // s, pl, pl * 4, 1, 1, 0)]
            if b == 0:
                convs.append((h, inpl, pl * 4, 1, s, 0))
            inpl, h = pl * 4, h // s
    assert len(convs) == 52
    worst = 1.0
    for (hh, cin, cout, k, s, p) in convs:
        nbytes = _lib.raw("dirb200_conv_wgrad_workspace_bytes")(256, hh, hh, cin, cout, k, k, s, p, 0)
        splits = nbytes // (k * k * cin * cout * 4)
        assert splits >= 1 and nbytes == splits * k * k * cin * cout * 4
        ho = (hh + 2 * p - k) // s + 1
        kblocks = (256 * ho * ho + 63) // 64
        bn = 128 if cout % 128 == 0 else 64
        tiles = ((k * k * cin // 64 + 1) // 2) * (cout // bn)
        items = tiles * splits
        waves = -(-items // sms)
        fill = items / (waves * sms)
        worst = min(worst, fill)
        assert fill >= 0.85, (hh, cin, cout, k, s, splits, items)
        assert kblocks // splits >= 8
    assert worst >= 0.85


def test_conv_plan_selects_the_intended_gemm_forms():
    """Host-only selection logic of the conv stage (dirb200_conv_plan; no device needed): the batch-256 ResNet-50 shapes
    get the forms DESIGN.md section 4 describes."""
    import ctypes
    import _lib, _convlib  # noqa: F401

    def plan(h, cin, cout, k, s, p, op, stem=0, hw_in=None):
        a = (ctypes.c_int * 7)()
        hh = hw_in or h
        rc = _lib.raw("dirb200_conv_plan")(256, hh, hh, cin, cout, k, k, s, p, stem, op, a)
        assert rc == 0, _lib.last_error()
        return dict(zip(("bn", "pairs", "feed", "patch_rows", "splits", "launches", "bn_moments"), a))

    GATHER, TILED, IM2COL = 0, 1, 2
    # layer1 conv2 (64 -> 64 3x3 at 56x56): im2col TMA, 64-wide tiles in all three passes; its dgrad carries BN moments
    for op in (0, 1, 2):
        q = plan(56, 64, 64, 3, 1, 1, op)
        assert (q["feed"], q["patch_rows"], q["bn"], q["pairs"]) == (IM2COL, 0, 64, 0), q
    assert plan(56, 64, 64, 3, 1, 1, 1)["bn_moments"] == 1
    # 1x1 stride-1 GEMMs: tiled TMA, 128-wide tiles wherever N allows (one m64n128 wgmma per consumer warpgroup)
    assert plan(56, 64, 256, 1, 1, 0, 0) == dict(bn=128, pairs=0, feed=TILED, patch_rows=0, splits=1, launches=1, bn_moments=0)
    q = plan(14, 256, 1024, 1, 1, 0, 0)
    assert (q["bn"], q["pairs"], q["feed"]) == (128, 0, TILED)
    q = plan(7, 2048, 512, 1, 1, 0, 1)                   # dgrad: N = Cin = 2048, carries BN moments
    assert (q["bn"], q["pairs"], q["bn_moments"]) == (128, 0, 1)
    # 3x3 layers: im2col TMA; stride-2 dgrad = 4 TMA-fed parity-class launches, no BN moments
    q = plan(28, 128, 128, 3, 1, 1, 0)
    assert (q["bn"], q["pairs"], q["feed"]) == (128, 0, IM2COL)
    q = plan(14, 256, 256, 3, 1, 1, 0)
    assert (q["bn"], q["pairs"], q["feed"]) == (128, 0, IM2COL)
    q = plan(56, 128, 128, 3, 2, 1, 1)
    assert (q["feed"], q["launches"], q["bn_moments"]) == (IM2COL, 4, 0)
    q = plan(56, 256, 512, 1, 2, 0, 1)                   # 1x1 stride-2 downsample: only the (even, even) class has a tap
    assert q["launches"] == 1
    # wgrad: split-K (checked in detail by the test above)
    assert plan(14, 256, 256, 3, 1, 1, 2)["pairs"] == 0 and plan(14, 256, 256, 3, 1, 1, 2)["splits"] > 1
    # 5x5 (NYUD2 refinement conv) goes through im2col TMA as well; the stem keeps the cp.async gather
    assert plan(240, 128, 128, 5, 1, 2, 0)["feed"] == IM2COL
    assert plan(224, 3, 64, 7, 2, 3, 0, stem=1)["feed"] == GATHER


def test_fused_epilogue_test_aids_refuse_bad_arguments_before_any_cuda_call():
    """The test-aid entry points of the fused conv epilogues validate their arguments on the host: each call below
    is refused with rc -1 and a message, without a device (every pointer is a dummy that must never be dereferenced)."""
    import ctypes
    import _lib, _convlib  # noqa: F401
    d = ctypes.c_void_p(16)                   # stands for a device buffer
    lay = (ctypes.c_int * 4)(128, 1, 64, 1)

    def refused(name, *args, msg):
        rc = _lib.raw(name)(*args)
        err = _lib.last_error()
        assert rc == -1 and msg in err, (name, rc, err)

    s1 = (2, 8, 8, 64, 64, 3, 3, 1, 1)       # n, h, w, cin, cout, kh, kw, stride, pad
    s2 = (2, 8, 8, 64, 64, 3, 3, 2, 1)
    # BN-backward moments on a stride-2 dgrad (its parity-class launches have no fused form)
    refused("dirb200_conv_dgrad_bn_moments", d, d, d, *s2, d, d, d, d, lay, None, msg="stride-1")
    # the folded-BN epilogue without its scale or shift
    refused("dirb200_conv_fprop_affine", d, d, d, *s1, None, d, None, 1, None, msg="scale / shift")
    refused("dirb200_conv_fprop_affine", d, d, d, *s1, d, None, d, 0, None, msg="scale / shift")
    # Cout not a multiple of 64
    bad_cout = (2, 8, 8, 64, 96, 1, 1, 1, 0)
    refused("dirb200_conv_fprop_bn_stats", d, d, d, *bad_cout, 0, d, lay, None, msg="multiple of 64")
    refused("dirb200_conv_fprop_affine", d, d, d, *bad_cout, d, d, None, 1, None, msg="multiple of 64")
    refused("dirb200_conv_dgrad_bn_moments", d, d, d, *(2, 8, 8, 96, 64, 1, 1, 1, 0), d, d, d, d, lay, None,
            msg="multiple of 64")
    # null pointers
    refused("dirb200_conv_fprop_bn_stats", d, d, d, *s1, 0, None, lay, None, msg="null")
    refused("dirb200_conv_fprop_bn_stats", d, d, d, *s1, 0, d, None, None, msg="null")
    refused("dirb200_conv_fprop_affine", None, d, d, *s1, d, d, None, 1, None, msg="null")
    refused("dirb200_conv_dgrad_bn_moments", d, d, d, *s1, None, d, d, d, lay, None, msg="null")
    refused("dirb200_conv_dgrad_bn_moments", d, d, d, *s1, d, d, d, None, lay, None, msg="null")
    refused("dirb200_bn_finalize_layout", None, lay, 128, 64, d, d, 1e-5, 0.1, d, d, d, d, d, d, None, msg="null")
    refused("dirb200_bn_finalize_layout", d, None, 128, 64, d, d, 1e-5, 0.1, d, d, d, d, d, d, None, msg="null")
    refused("dirb200_bn_bwd_coeffs_layout", d, lay, 128, 64, d, d, d, None, d, d, None, msg="null")
    # a layout whose tiles do not cover the channels
    short = (ctypes.c_int * 4)(128, 1, 32, 1)
    refused("dirb200_bn_finalize_layout", d, short, 128, 64, d, d, 1e-5, 0.1, None, None, d, d, d, d, None,
            msg="layout")
    refused("dirb200_bn_bwd_coeffs_layout", d, short, 128, 64, d, d, d, d, d, d, None, msg="layout")
