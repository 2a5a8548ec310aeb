"""CPU-only checks of NYUD2-DIR's decoder D and multi-scale fusion MFF (nyud2-dir/models/modules.py:6-31, 61-128): a
functional float restatement of the reference modules against the reference's own outputs and gradients (fixture
tests/golden/nyud2_decoder.npz, made by tests/golden/make_golden_nyud2_decoder.py), the native modules' state_dict
layout, and the null-pointer check of the eval-mode BatchNorm coefficients entry point."""
import numpy as np
import torch
import torch.nn.functional as F

from util import det_param, golden

CHANNELS = (256, 512, 1024, 2048)
SIZES = ((9, 11), (5, 6), (3, 3), (2, 2))
SAMPLE = 512


def sample_idx(numel):
    return np.linspace(0, numel - 1, min(numel, SAMPLE)).astype(np.int64)


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


def fixture_inputs(batch=2):
    return [torch.relu(det_param(f"x_nyud2_decoder_{s + 1}", (batch, c, h, w), 1.0))
            for s, (c, (h, w)) in enumerate(zip(CHANNELS, SIZES))]


# ---- functional restatement (NCHW, any float dtype, train-mode BatchNorm = batch statistics, biased variance)
def bn_train(x, w, b, eps=1e-5):
    mean = x.mean((0, 2, 3), keepdim=True)
    var = ((x - mean) ** 2).mean((0, 2, 3), keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * w.view(1, -1, 1, 1) + b.view(1, -1, 1, 1)


def up_projection(p, pre, x, size):
    x = F.interpolate(x, size=tuple(size), mode="bilinear", align_corners=False)
    a = torch.relu(bn_train(F.conv2d(x, p[pre + "conv1.weight"], padding=2), p[pre + "bn1.weight"], p[pre + "bn1.bias"]))
    b1 = bn_train(F.conv2d(a, p[pre + "conv1_2.weight"], padding=1), p[pre + "bn1_2.weight"], p[pre + "bn1_2.bias"])
    b2 = bn_train(F.conv2d(x, p[pre + "conv2.weight"], padding=2), p[pre + "bn2.weight"], p[pre + "bn2.bias"])
    return torch.relu(b1 + b2)


def decoder_d(p, xs):
    x = torch.relu(bn_train(F.conv2d(xs[3], p["conv.weight"]), p["bn.weight"], p["bn.bias"]))
    x = up_projection(p, "up1.", x, xs[2].shape[2:])
    x = up_projection(p, "up2.", x, xs[1].shape[2:])
    x = up_projection(p, "up3.", x, xs[0].shape[2:])
    return up_projection(p, "up4.", x, (2 * xs[0].shape[2], 2 * xs[0].shape[3]))


def mff(p, xs, size):
    ms = [up_projection(p, f"up{s + 1}.", x, size) for s, x in enumerate(xs)]
    return torch.relu(bn_train(F.conv2d(torch.cat(ms, 1), p["conv.weight"], padding=2), p["bn.weight"], p["bn.bias"]))


def fixture_modules():
    """Native D(2048) / MFF(256 ... 2048) on the CPU (parameters only) with the fixture's values."""
    from dense_ops import D, MFF
    torch.manual_seed(0)
    Dm, Mm = D(2048), MFF(list(CHANNELS))
    fill_params([("D." + n, q) for n, q in Dm.named_parameters()])
    fill_params([("MFF." + n, q) for n, q in Mm.named_parameters()])
    return Dm, Mm


def rel(a, b):
    return float((a.detach().double() - b.detach().double()).norm() / (b.double().norm() + 1e-30))


def test_functional_restatement_matches_reference_fixture():
    """decoder_d / mff above (fp32, CPU) against the reference's own D and MFF: outputs, input gradients and parameter
    gradients (sampled) of <D, gD> + <MFF, gM> within fp32 round-off (relative L2 < 1e-3)."""
    g = golden("nyud2_decoder")
    Dm, Mm = fixture_modules()
    pd = {n: q.detach().clone().requires_grad_(True) for n, q in Dm.named_parameters()}
    pm = {n: q.detach().clone().requires_grad_(True) for n, q in Mm.named_parameters()}
    xs = [x.requires_grad_(True) for x in fixture_inputs()]
    d = decoder_d(pd, xs)
    m = mff(pm, xs, d.shape[2:])
    assert rel(d, torch.from_numpy(g["d_out"].astype(np.float32))) < 1e-3
    assert rel(m, torch.from_numpy(g["m_out"].astype(np.float32))) < 1e-3
    gD = det_param("g_nyud2_decoder_D", tuple(d.shape), 1.0)
    gM = det_param("g_nyud2_decoder_MFF", tuple(m.shape), 1.0)
    ((d * gD).sum() + (m * gM).sum()).backward()
    for s, x in enumerate(xs):
        gx = x.grad.reshape(-1)
        assert rel(gx[sample_idx(gx.numel())], torch.from_numpy(g[f"dx{s + 1}"])) < 1e-3, s
        assert abs(gx.double().norm().item() / float(g[f"dxn{s + 1}"]) - 1) < 1e-4, s
    for tag, p in (("d", pd), ("m", pm)):
        for n, q in p.items():
            gq = q.grad.reshape(-1)
            assert rel(gq[sample_idx(gq.numel())], torch.from_numpy(g[f"{tag}g:{n}"])) < 1e-3, (tag, n)
            assert abs(gq.double().norm().item() / max(float(g[f"{tag}n:{n}"]), 1e-30) - 1) < 1e-4, (tag, n)


def test_decoder_state_dicts_match_reference_layout():
    """D(2048) and MFF([256, 512, 1024, 2048]): the reference modules' state_dict keys and shapes, in order, so a
    reference checkpoint loads strictly."""
    from dense_ops import D, MFF
    g = golden("nyud2_decoder")
    for tag, mod in (("d", D(2048)), ("m", MFF(list(CHANNELS)))):
        names = [str(n) for n in g[f"{tag}_names"]]
        shapes = [tuple(int(x) for x in row if x >= 0) for row in g[f"{tag}_shapes"]]
        sd = mod.state_dict()
        assert list(sd.keys()) == names
        assert [tuple(v.shape) for v in sd.values()] == shapes
        src = {k: (torch.randn_like(v) if v.is_floating_point() else v + 3) for k, v in sd.items()}
        mod.load_state_dict(src, strict=True)
        for k, v in mod.state_dict().items():
            assert torch.equal(v, src[k]), k


def test_bn_eval_coeffs_refuses_null_pointers():
    import _lib
    import _convlib  # noqa: F401
    rc = _lib.raw("dirb200_bn_eval_coeffs")(64, 16, 16, 1e-5, None, 16, 16, 16, None)
    assert rc == -1 and "null pointer" in _lib.last_error()
