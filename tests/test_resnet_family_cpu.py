"""CPU-only checks of the ResNet family (resnet18 / 34 / 50 / 101 / 152):

  * the basic-block form of the float32 oracle (tests/resnet_family_ref.py) against the reference's own ResNet-18
    forward + backward (fixture tests/golden/resnet_family.npz, made by tests/golden/make_golden_resnet_family.py);
  * the native modules' state_dict keys, shapes and parameter counts against the reference's for every depth;
  * the host-side conv plans of the ten convolution shapes ResNet-18 / 34 add at batch 256 x 224^2;
  * dirb200_resnet_create_ex refusing a block kind it does not know, before any CUDA call.
"""
import ctypes

import numpy as np
import pytest
import torch

from util import det_param, golden

import resnet_family_ref as RF

# parameters with the 1-output regressor (the shapes' products; ResNet-50 as test_gpu_resnet.py pins it)
PARAMS = {18: 11177025, 34: 21285185, 50: 23510081, 101: 42502209, 152: 58145857}
FDS_ARGS = dict(bucket_num=100, bucket_start=3, start_update=0, start_smooth=1, kernel="gaussian", ks=5, sigma=2,
                momentum=0.9)


def rel(a, b):
    return float(np.linalg.norm(np.asarray(a, np.float64) - np.asarray(b, np.float64)) /
                 (np.linalg.norm(np.asarray(b, np.float64)) + 1e-30))


def test_oracle_basic_block_matches_reference():
    """The oracle's ResNet-18 (train-mode BN, fp32) against the reference's forward and every parameter gradient."""
    g = golden("resnet_family")
    shapes = RF.param_shapes((2, 2, 2, 2), block="basic")
    assert sum(int(np.prod(s)) for _, s in shapes) == PARAMS[18]
    p = {}
    for n, s in shapes:
        if len(s) == 4:
            v = det_param(n, s, (2.0 / (s[0] * s[2] * s[3])) ** 0.5)
        elif n == "linear.weight":
            v = det_param(n, s, 0.05)
        elif n == "linear.bias":
            v = torch.full(s, 0.1)
        elif n.endswith("weight"):
            v = 1.0 + 0.1 * det_param(n, s, 1.0)
        else:
            v = 0.1 * det_param(n, s, 1.0)
        p[n] = v.requires_grad_(True)
    torch.set_num_threads(8)
    x = det_param("input18", (4, 3, 224, 224), 1.0)
    t = torch.tensor([[31.0], [44.0], [5.0], [70.0]])
    w = torch.tensor([[0.5], [1.5], [1.0], [2.0]])
    stats = {}
    pred, enc = RF.forward(p, x, layers=(2, 2, 2, 2), stats=stats, block="basic")
    loss = ((pred - t).abs() * w).mean()
    loss.backward()
    assert rel(enc.detach().numpy(), g["basic/enc"]) <= 1e-5
    assert rel(pred.detach().numpy(), g["basic/pred"]) <= 1e-5
    assert abs(loss.item() - float(g["basic/loss"])) <= 1e-5 * abs(float(g["basic/loss"]))
    assert rel(stats["bn1.running_mean"].numpy(), g["basic/bn1_running_mean"]) <= 1e-5
    assert rel(stats["bn1.running_var"].numpy(), g["basic/bn1_running_var"]) <= 1e-5
    assert {k.split("/", 1)[1] for k in g.files if k.startswith("grad_at/")} == set(p)
    for n, v in p.items():
        gr = v.grad.reshape(-1).double()
        at = g[f"grad_at/{n}"]
        idx = np.arange(gr.numel()) if gr.numel() <= 4096 else \
            np.unique(np.linspace(0, gr.numel() - 1, 64).round().astype(np.int64))
        assert rel(gr[torch.from_numpy(idx)].numpy(), at) <= 1e-5, (n, rel(gr[torch.from_numpy(idx)].numpy(), at))
        assert abs(gr.sum().item() - float(g[f"grad_sum/{n}"])) <= 1e-5 * float(g[f"grad_abs/{n}"]), n
        assert abs(gr.abs().sum().item() - float(g[f"grad_abs/{n}"])) <= 1e-5 * float(g[f"grad_abs/{n}"]), n


def test_oracle_bottleneck_form_is_resnet_ref():
    from oracle import resnet_ref as R
    assert RF.param_shapes() == R.param_shapes()
    assert RF.param_shapes((3, 4, 23, 3))[-2] == ("linear.weight", (1, 2048))


@pytest.mark.parametrize("depth", [18, 34, 50, 101, 152])
def test_native_state_dict_layout_and_parameter_counts(depth):
    """Keys and shapes of the native module equal the reference's (with and without FDS), its named_parameters() the
    oracle's order, and its flat buffers hold exactly the parameters and BN running statistics."""
    import resnet
    g = golden("resnet_family")
    block, layers = RF.DEPTHS[depth]
    for fds in (False, True):
        torch.manual_seed(0)
        m = getattr(resnet, f"resnet{depth}")(fds=fds, **FDS_ARGS)
        sd = m.state_dict()
        assert sum(p.numel() for p in m.parameters()) == PARAMS[depth]
        assert m.flat_parameters().numel() == PARAMS[depth]
        assert [n for n, _ in m.named_parameters()] == [n for n, _ in RF.param_shapes(layers, block)]
        assert [tuple(p.shape) for _, p in m.named_parameters()] == [s for _, s in RF.param_shapes(layers, block)]
        bns = [b for n, b in m.named_buffers() if n.endswith("running_mean") and not n.startswith("FDS")]
        assert m._flat["running"].numel() == 2 * sum(b.numel() for b in bns)
        if fds:
            assert m.FDS.feature_dim == 512 * RF.expansion(block)
        tag = f"resnet{depth}" + ("_fds" if fds else "")
        if depth == 50:
            continue                                   # resnet.npz / test_gpu_resnet.py pin ResNet-50's layout
        assert list(sd.keys()) == list(g[f"keys/{tag}"]), tag
        want = [tuple(int(d) for d in row if d >= 0) for row in g[f"shapes/{tag}"]]
        assert [tuple(v.shape) for v in sd.values()] == want, tag
        assert int(g[f"n_params/{tag}"]) == PARAMS[depth]


def test_native_basic_block_modules_mirror_the_reference():
    import resnet
    m = resnet.resnet18()
    blk = m.layer1[0]
    assert isinstance(blk, resnet.BasicBlock) and resnet.BasicBlock.expansion == 1
    assert blk.downsample is None and blk.conv1.kernel_size == (3, 3) and blk.conv1.stride == (1, 1)
    b2 = m.layer2[0]
    assert b2.conv1.stride == (2, 2) and b2.conv2.stride == (1, 1) and b2.downsample[0].stride == (2, 2)
    assert m.linear.in_features == 512
    # E_resnet wraps every depth with the reference's E_resnet keys (no linear / FDS)
    e = resnet.E_resnet(m)
    assert not any(k.startswith(("linear", "FDS")) for k in e.state_dict())
    assert "layer4.1.bn2.running_var" in e.state_dict()


def test_basic_block_conv_plans_at_batch_256():
    """dirb200_conv_plan for every conv shape ResNet-18 / 34 add at batch 256 x 224^2 (h, cin, cout, k, stride, pad):
    (bn, feed, splits, launches, bn_moments) of fprop / dgrad / wgrad.  Every one is fed by im2col TMA; the 3x3
    stride-2 dgrads run as 4 parity-class launches; every 3x3 stride-1 dgrad carries the BN-backward moments."""
    import _lib, _convlib  # noqa: F401
    IM2COL = 2
    want = {
        (56, 64, 64, 3, 1, 1): [(64, 1, 1, 0), (64, 1, 1, 1), (64, 26, 1, 0)],
        (56, 64, 128, 3, 2, 1): [(128, 1, 1, 0), (64, 1, 4, 0), (128, 26, 1, 0)],
        (56, 64, 128, 1, 2, 0): [(128, 1, 1, 0), (64, 1, 1, 0), (128, 131, 1, 0)],
        (28, 128, 128, 3, 1, 1): [(128, 1, 1, 0), (128, 1, 1, 1), (128, 14, 1, 0)],
        (28, 128, 256, 3, 2, 1): [(128, 1, 1, 0), (128, 1, 4, 0), (128, 7, 1, 0)],
        (28, 128, 256, 1, 2, 0): [(128, 1, 1, 0), (128, 1, 1, 0), (128, 66, 1, 0)],
        (14, 256, 256, 3, 1, 1): [(128, 1, 1, 0), (128, 1, 1, 1), (128, 11, 1, 0)],
        (14, 256, 512, 3, 2, 1): [(128, 1, 1, 0), (128, 1, 4, 0), (128, 7, 1, 0)],
        (14, 256, 512, 1, 2, 0): [(128, 1, 1, 0), (128, 1, 1, 0), (128, 16, 1, 0)],
        (7, 512, 512, 3, 1, 1): [(128, 1, 1, 0), (128, 1, 1, 1), (128, 4, 1, 0)],
    }
    for (h, ci, co, k, s, p), per_op in want.items():
        for op, (bn, splits, launches, moments) in enumerate(per_op):
            a = (ctypes.c_int * 7)()
            rc = _lib.raw("dirb200_conv_plan")(256, h, h, ci, co, k, k, s, p, 0, op, a)
            assert rc == 0, _lib.last_error()
            got = dict(zip(("bn", "pairs", "feed", "patch_rows", "splits", "launches", "bn_moments"), a))
            assert got == dict(bn=bn, pairs=0, feed=IM2COL, patch_rows=0, splits=splits, launches=launches,
                               bn_moments=moments), ((h, ci, co, k, s, p), op, got)


def test_create_ex_refuses_a_bad_block_kind_without_a_device():
    import _lib
    import resnet  # noqa: F401
    arr = (ctypes.c_int * 4)(2, 2, 2, 2)
    for kind in (-1, 2, 7):
        h = ctypes.c_void_p()
        rc = _lib.raw("dirb200_resnet_create_ex")(4, 64, 64, kind, arr, 4, ctypes.byref(h))
        assert rc == -1 and "bad block kind" in _lib.last_error(), (kind, _lib.last_error())
        assert h.value is None
    # the other arguments are still checked as dirb200_resnet_create checks them
    h = ctypes.c_void_p()
    assert _lib.raw("dirb200_resnet_create_ex")(4, 62, 64, 1, arr, 4, ctypes.byref(h)) == -1
    assert "multiples of 4" in _lib.last_error()
