"""CPU-only checks of NYUD2-DIR's multi-scale encoder (nyud2-dir/models/modules.py:33-58): the oracle's block taps
against the reference's own E_resnet (fixture tests/golden/nyud2_encoder.npz, made by
tests/golden/make_golden_nyud2_encoder.py), the native E_resnet's state_dict layout, and the runner's size rules."""
import ctypes

import numpy as np
import pytest
import torch

from util import det_param, golden


def fixture_params():
    """The fixture's deterministic parameters (make_golden_nyud2_encoder.fill_params) by name."""
    from oracle import resnet_ref as R
    p = {}
    for name, shape in R.param_shapes():
        if name.startswith("linear."):
            continue
        if len(shape) == 4:
            cout, _, k, _ = shape
            p[name] = det_param(name, shape, (2.0 / (k * k * cout)) ** 0.5)
        elif name.endswith("weight"):
            p[name] = 1.0 + 0.1 * det_param(name, shape, 1.0)
        else:
            p[name] = 0.1 * det_param(name, shape, 1.0)
    return p


def rel(a, b):
    return float((a - b).double().norm() / (b.double().norm() + 1e-30))


def test_oracle_block_taps_match_reference_at_odd_stage_sizes():
    """resnet_ref.forward_encoding's block taps and encoder_ref.forward_blocks against the reference's E_resnet on a
    2 x 3 x 36 x 44 input (stage maps 9x11, 5x6, 3x3, 2x2), fp32 train-mode BN."""
    from oracle import resnet_ref as R, encoder_ref as E
    g = golden("nyud2_encoder")
    x = torch.from_numpy(g["x"])
    assert tuple(x.shape) == (2, 3, 36, 44)
    p = fixture_params()
    taps = {}
    with torch.no_grad():
        R.forward_encoding(p, x, taps=taps)
        blocks = E.forward_blocks(p, x)
    for s, bi in enumerate(E.last_blocks()):
        want = torch.from_numpy(g[f"block{s + 1}"])
        assert tuple(taps[f"{bi}.6"].shape) == tuple(want.shape)
        # fp32 on the CPU; the oracle's BatchNorm is written out (mean / biased var) where the reference calls
        # nn.BatchNorm2d, so the two differ by fp32 round-off amplified over up to 16 blocks; layer4 normalises
        # over 8 values per channel (2 x 2 x 2), which amplifies most (1.0e-4 measured)
        assert rel(taps[f"{bi}.6"], want) < 5e-4, (s, rel(taps[f"{bi}.6"], want))
        assert torch.equal(blocks[s], taps[f"{bi}.6"]), s


def test_encoder_state_dict_matches_reference_layout():
    """E_resnet(resnet50()).state_dict(): the reference E_resnet's keys and shapes, in order; loading a state_dict
    (e.g. a torchvision-layout ResNet-50 checkpoint) writes through the flat parameter / statistics views."""
    from resnet import E_resnet, resnet50
    g = golden("nyud2_encoder")
    names = [str(n) for n in g["names"]]
    shapes = [tuple(int(d) for d in row if d >= 0) for row in g["shapes"]]
    torch.manual_seed(0)
    m = resnet50()
    E = E_resnet(m)
    sd = E.state_dict()
    assert list(sd.keys()) == names
    assert [tuple(v.shape) for v in sd.values()] == shapes
    # a checkpoint with the full network's extra keys loads non-strictly; the encoder's keys land in the flat views
    src = {k: (torch.randn_like(v) if v.is_floating_point() else v + 3) for k, v in sd.items()}
    missing, unexpected = E.load_state_dict(dict(src, **{"fc.weight": torch.zeros(1000, 2048)}), strict=False)
    assert missing == [] and unexpected == ["fc.weight"]
    flat = m.flat_parameters()
    assert E.conv1.weight.data_ptr() == flat.data_ptr()
    assert torch.equal(E.layer4[2].bn3.bias, src["layer4.2.bn3.bias"])
    assert torch.equal(m._flat["running"][:64], src["bn1.running_mean"])
    assert int(m.bn1.num_batches_tracked) == int(src["bn1.num_batches_tracked"])
    # a device / dtype move keeps every parameter a view of the (new) flat buffer
    E.float()
    assert E.conv1.weight.data_ptr() == m.flat_parameters().data_ptr()
    assert torch.equal(E.layer4[2].bn3.bias, src["layer4.2.bn3.bias"])


@pytest.mark.parametrize("n,h,w,msg", [
    (2, 226, 304, "multiples of 4"), (2, 228, 302, "multiples of 4"), (2, 230, 32, "multiples of 4"),
    (2, 1028, 304, "at most 1024"), (2, 228, 1028, "at most 1024"), (8193, 228, 304, "at most 8192"),
    (8192, 1024, 1024, "below 2^31")])
def test_resnet_create_refuses_bad_sizes_before_any_cuda_call(n, h, w, msg):
    """H and W must be multiples of 4, at most 1024 (9-bit packed stem-output row / column); N at most 8192 (13-bit
    image index); the stem output below 2^31 pixels.  Each call is refused on the host, without a device."""
    import _lib
    import resnet  # noqa: F401  (registers the runner bindings)
    out = ctypes.c_void_p()
    layers = (ctypes.c_int * 4)(3, 4, 6, 3)
    rc = _lib.raw("dirb200_resnet_create")(n, h, w, layers, 4, ctypes.byref(out))
    err = _lib.last_error()
    assert rc == -1 and msg in err and out.value is None, (rc, err)


def test_feature_maps_at_nyud2_sizes():
    """The stage geometry the encoder returns (and ResNet.peek reads): 228 x 304 -> 114x152, 57x76, 29x38, 15x19,
    8x10."""
    from resnet import _feature_maps
    assert _feature_maps(228, 304) == [(114, 152), (57, 76), (29, 38), (15, 19), (8, 10)]
    assert _feature_maps(480, 640) == [(240, 320), (120, 160), (60, 80), (30, 40), (15, 20)]
    assert _feature_maps(224, 224) == [(112, 112), (56, 56), (28, 28), (14, 14), (7, 7)]
