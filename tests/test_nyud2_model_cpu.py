"""CPU-only checks of NYUD2-DIR's assembled depth network net.model (nyud2-dir/models/net.py:5-22): the functional
restatement oracle/net_ref.py against the reference's own net.model (fixture tests/golden/nyud2_model.npz, made by
tests/golden/make_golden_nyud2_model.py), the native model's state_dict layout with and without FDS, and the argument
checks of R's depth-head entry points."""
import numpy as np
import pytest
import torch

from util import det_param, golden

X_SHAPE = (2, 3, 36, 44)
OUT_SHAPE = (2, 1, 18, 22)
BLOCKS = [256, 512, 1024, 2048]


def sample_idx(numel, k):
    return np.linspace(0, numel - 1, min(numel, k)).astype(np.int64)


def make_args(fds=True):
    """The FDS settings of make_golden_nyud2_model.make_args (nyud2-dir/train.py's defaults)."""
    from types import SimpleNamespace
    return SimpleNamespace(fds=fds, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1,
                           fds_kernel="gaussian", fds_ks=5, fds_sigma=2.0, fds_mmt=0.9)


def fds_tables(nb=93, c=128):
    return {"running_mean_last_epoch": 0.3 * det_param("fds.rm", (nb, c), 1.0),
            "running_var_last_epoch": 0.5 + det_param("fds.rv", (nb, c), 1.0).abs(),
            "smoothed_mean_last_epoch": 0.3 * det_param("fds.sm", (nb, c), 1.0),
            "smoothed_var_last_epoch": 0.5 + det_param("fds.sv", (nb, c), 1.0).abs()}


def depth_and_weight():
    g = torch.Generator().manual_seed(11)
    depth = 0.5 + 9.5 * torch.rand(OUT_SHAPE, generator=g)
    weight = 0.5 + torch.rand(OUT_SHAPE, generator=g)
    return depth, weight


def fill_params(named):
    """make_golden_nyud2_encoder.fill_params: the fixture's deterministic parameter values, in place."""
    with torch.no_grad():
        for name, p in named:
            if p.dim() == 4:
                cout, _, k, _ = p.shape
                p.copy_(det_param(name, p.shape, (2.0 / (k * k * cout)) ** 0.5))
            elif name.endswith("weight"):
                p.copy_(1.0 + 0.1 * det_param(name, p.shape, 1.0))
            else:
                p.copy_(0.1 * det_param(name, p.shape, 1.0))


def fixture_model(fds=True):
    """The native net.model (parameters on the CPU) with the fixture's parameter values and FDS tables."""
    import net
    import resnet
    torch.manual_seed(0)
    m = net.model(make_args(fds), resnet.E_resnet(resnet.resnet50()), 2048, BLOCKS)
    fill_params(list(m.named_parameters()))
    if fds:
        with torch.no_grad():
            for k, v in fds_tables().items():
                getattr(m.R.FDS, k).copy_(v)
    return m


def rel(a, b):
    return float((a.detach().double() - b.detach().double()).norm() / (b.detach().double().norm() + 1e-30))


def test_oracle_matches_reference_fixture():
    """oracle/net_ref.forward (fp32, CPU, FDS smoothing active at epoch 1) against the reference's own net.model:
    output, feature and loss within relative L2 5e-4.  Parameter gradients (the fixture's samples, relative L2, and
    the full norm) within 2e-3 for R.conv2, 3e-2 for the rest of R, 0.1 for D / MFF and 0.2 for E: the loss reaches
    them through up to 16 train-mode BatchNorm backwards over 8 to 792 values per channel, and fp32 round-off alone
    moves them that far (evaluating this same restatement in float64 instead of fp32 changes them by up to 5e-4,
    1.1e-2, 6.1e-2 and 9.1e-2)."""
    from oracle import net_ref
    g = golden("nyud2_model")
    p = {n: q.detach().clone().requires_grad_(True) for n, q in fixture_model(True).named_parameters()}
    depth, weight = depth_and_weight()
    x = det_param("x_nyud2_model", X_SHAPE, 1.0)
    out, feature = net_ref.forward(p, x, depth, 1, dict(tables=fds_tables(), start_smooth=1))
    loss = torch.mean(((out - depth) ** 2) * weight)
    assert rel(out, torch.from_numpy(g["out"])) < 5e-4
    f = feature.reshape(-1)
    assert rel(f[sample_idx(f.numel(), 8192)], torch.from_numpy(g["feature"])) < 5e-4
    assert abs(f.double().norm().item() / float(g["feature_norm"]) - 1) < 5e-4
    assert abs(loss.item() / float(g["loss"]) - 1) < 5e-4
    loss.backward()
    bound = lambda n: 2e-3 if n.startswith("R.conv2") else 3e-2 if n.startswith("R.") else 0.2 if n.startswith("E.") \
        else 0.1
    bad = {}
    for n, q in p.items():
        gq = q.grad.reshape(-1)
        e = (rel(gq[sample_idx(gq.numel(), 128)], torch.from_numpy(g[f"g:{n}"])),
             abs(gq.double().norm().item() / max(float(g[f"n:{n}"]), 1e-30) - 1))
        if max(e) >= bound(n):
            bad[n] = e
    assert not bad, bad


@pytest.mark.parametrize("fds", [True, False], ids=["fds", "no_fds"])
def test_state_dict_matches_reference_layout_and_loads(fds):
    """net.model(args, E_resnet(resnet50()), 2048, [256, 512, 1024, 2048]): the reference's state_dict keys and shapes,
    in order (R.FDS.* buffers with args.fds), and a state_dict in that layout loads strictly, values included."""
    import net
    import resnet
    g = golden("nyud2_model")
    tag = "" if fds else "_nofds"
    names = [str(n) for n in g["names" + tag]]
    shapes = [tuple(int(v) for v in row if v >= 0) for row in g["shapes" + tag]]
    m = net.model(make_args(fds), resnet.E_resnet(resnet.resnet50()), 2048, BLOCKS)
    sd = m.state_dict()
    assert list(sd.keys()) == names
    assert [tuple(v.shape) for v in sd.values()] == shapes
    src = {k: (torch.randn_like(v) if v.is_floating_point() else v + 3) for k, v in sd.items()}
    m.load_state_dict(src, strict=True)
    for k, v in m.state_dict().items():
        assert torch.equal(v, src[k]), k
    assert (m.R.FDS is not None) == fds
    assert net.model(None, resnet.E_resnet(resnet.resnet50()), 2048, BLOCKS).R.FDS is None


def test_model_refuses_an_encoder_that_is_not_e_resnet():
    import net
    import resnet
    with pytest.raises(TypeError):
        net.model(None, resnet.resnet50(), 2048, BLOCKS)


# ------------------------------------------------------------------------- depth-head argument checks
D = 16                       # a non-NULL dummy pointer: a refused call must not reach the device
BAD_SHAPES = [((2, 8, 10, 0), "multiple of 8 from 8 to 256"), ((2, 8, 10, 12), "multiple of 8 from 8 to 256"),
              ((2, 8, 10, 264), "multiple of 8 from 8 to 256"), ((2, 8, 10, -8), "multiple of 8 from 8 to 256"),
              ((0, 8, 10, 128), "must be positive"), ((2, 0, 10, 128), "must be positive"),
              ((2, 8, -1, 128), "must be positive"), ((8192, 1024, 1024, 8), "below 2^31"),
              ((64, 512, 512, 128), "below 2^31")]


@pytest.mark.parametrize("shape,msg", BAD_SHAPES, ids=["x".join(map(str, s)) for s, _ in BAD_SHAPES])
def test_depth_head_refuses_bad_shapes_before_any_cuda_call(shape, msg):
    import _lib
    for name, args in (("dirb200_depth_head_fwd", (D, D, D, D)), ("dirb200_depth_head_dgrad", (D, D, D)),
                       ("dirb200_depth_head_wgrad", (D, D, D, D, D, 1 << 40))):
        rc = _lib.raw(name)(*args, *shape, None)
        assert rc == -1 and msg in _lib.last_error(), (name, rc, _lib.last_error())
    assert _lib.raw("dirb200_depth_head_wgrad_workspace_bytes")(*shape) == 0
    assert msg in _lib.last_error()


def test_depth_head_refuses_null_pointers_and_a_short_workspace():
    import _lib
    shape = (2, 8, 10, 128)
    for i in range(4):
        args = [D] * 4
        args[i] = None
        rc = _lib.raw("dirb200_depth_head_fwd")(*args, *shape, None)
        assert rc == -1 and "null pointer" in _lib.last_error()
    for i in range(3):
        args = [D] * 3
        args[i] = None
        rc = _lib.raw("dirb200_depth_head_dgrad")(*args, *shape, None)
        assert rc == -1 and "null pointer" in _lib.last_error()
    need = _lib.raw("dirb200_depth_head_wgrad_workspace_bytes")(*shape)
    assert need == 1 * 1 * 2 * (25 * 128 + 1) * 4             # one 16 x 32 tile per image
    for i in range(5):
        args = [D] * 5
        args[i] = None
        rc = _lib.raw("dirb200_depth_head_wgrad")(*args, need, *shape, None)
        assert rc == -1 and "null pointer" in _lib.last_error()
    rc = _lib.raw("dirb200_depth_head_wgrad")(D, D, D, D, D, need - 1, *shape, None)
    assert rc == -1 and "workspace too small" in _lib.last_error()
