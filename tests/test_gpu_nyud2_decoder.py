"""GPU checks of NYUD2-DIR's decoder D and multi-scale fusion MFF (dense_ops.UpProjection / D / MFF,
nyud2-dir/models/modules.py:6-31, 61-128).

- Fixture parity: the native modules against the reference modules' outputs and gradients (fp32 CPU fixture).
- Teacher-forced parity at 228 x 304 (batch 2): each step of every up-projection against float64 on the same bf16
  operands, per element (conv bounds as tests/test_gpu_conv.py's).
- Eval mode: running statistics used and left bit-unchanged (D, MFF, RefinementR).
The file reruns itself with DIRB200_SMS=7 (few CTAs per conv: multi-wave tile walks, other split-K plans)."""
import os
import subprocess
import sys

import pytest
import torch
import torch.nn.functional as F

from util import det_param

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
BF16_U = 2.0 ** -8
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def KAPPA(K):
    """tests/test_gpu_conv.KAPPA: fp32 accumulation error per unit of the abs-conv for a K-long reduction."""
    return (K / 16 + 16) * U


def nchw(t):
    return t.permute(0, 3, 1, 2)


def nhwc(t):
    return t.permute(0, 2, 3, 1).contiguous()


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-30)).item()


# --------------------------------------------------------------------------------------- module construction
CHANNELS = (256, 512, 1024, 2048)


def make_modules(seed=0):
    from dense_ops import D, MFF
    torch.manual_seed(seed)
    Dm, Mm = D(2048), MFF(list(CHANNELS))
    with torch.no_grad():                     # non-trivial BN affine
        for mod in (Dm, Mm):
            for n, p in mod.named_parameters():
                if p.dim() == 1:
                    p.copy_((1.0 if n.endswith("weight") else 0.0) + 0.1 * det_param(n, p.shape, 1.0))
    return Dm.to(DEV), Mm.to(DEV)


def encoder_blocks(n, h, w, seed=0):
    """Non-negative NHWC bf16 maps with the shapes of E_resnet's block outputs at an h x w input."""
    from resnet import _feature_maps
    maps = _feature_maps(h, w)[1:]
    g = torch.Generator(device=DEV).manual_seed(seed)
    return [torch.relu(torch.randn(n, hh, ww, c, device=DEV, generator=g)).to(torch.bfloat16)
            for c, (hh, ww) in zip(CHANNELS, maps)]


# ---------------------------------------------------------------------------------------------- fixture parity
def test_modules_match_reference_fixture():
    """Native D / MFF (bf16 storage, train mode) against the reference modules' fp32 CPU fixture: outputs and every
    gradient of <D, gD> + <MFF, gM>.  Bounds (relative L2): outputs 3e-2; input gradients 0.2 and parameter gradients
    0.3 on the fixture's samples.  The gradients pass through up to four train-mode BatchNorm backwards over 8 to 792
    values per channel (batch 2 on 2 x 2 .. 18 x 22 maps), each of which removes the gradient's projection on the
    batch statistics and so amplifies the bf16 rounding of everything upstream (0.10 to 0.18 measured for the block
    gradients and at most 0.20 for a parameter gradient, on an H100); the per-step precision is pinned by the
    teacher-forced test below."""
    import numpy as np
    from test_nyud2_decoder_cpu import fixture_modules, fixture_inputs, sample_idx
    from util import golden
    g = golden("nyud2_decoder")
    Dm, Mm = fixture_modules()
    Dm, Mm = Dm.to(DEV).train(), Mm.to(DEV).train()
    xs = [nhwc(x).to(DEV).to(torch.bfloat16).requires_grad_(True) for x in fixture_inputs()]
    d = Dm(*xs)
    m = Mm(*xs, (d.shape[1], d.shape[2]))
    d_ref = torch.from_numpy(g["d_out"].astype(np.float32))
    m_ref = torch.from_numpy(g["m_out"].astype(np.float32))
    errs = {"d_out": rel(nchw(d).cpu(), d_ref), "m_out": rel(nchw(m).cpu(), m_ref)}
    gD = nhwc(det_param("g_nyud2_decoder_D", tuple(d_ref.shape), 1.0)).to(DEV).to(torch.bfloat16)
    gM = nhwc(det_param("g_nyud2_decoder_MFF", tuple(m_ref.shape), 1.0)).to(DEV).to(torch.bfloat16)
    torch.autograd.backward([d, m], [gD, gM])
    for s, x in enumerate(xs):
        gx = nchw(x.grad).float().cpu().reshape(-1)
        errs[f"dx{s + 1}"] = rel(gx[sample_idx(gx.numel())], torch.from_numpy(g[f"dx{s + 1}"]))
    perr = {}
    for tag, mod in (("d", Dm), ("m", Mm)):
        for n, q in mod.named_parameters():
            gq = q.grad.float().cpu().reshape(-1)
            perr[f"{tag}:{n}"] = rel(gq[sample_idx(gq.numel())], torch.from_numpy(g[f"{tag}g:{n}"]))
    print({k: f"{v:.2e}" for k, v in errs.items()}, "worst param", max(perr.items(), key=lambda kv: kv[1]))
    assert errs["d_out"] < 3e-2 and errs["m_out"] < 3e-2, errs
    assert all(errs[f"dx{s + 1}"] < 0.2 for s in range(4)), errs
    assert all(v < 0.3 for v in perr.values()), sorted(perr.items(), key=lambda kv: -kv[1])[:5]


# ------------------------------------------------------------------------------------ teacher-forced parity
def _bn64(y, w, b, eps=1e-5):
    mean = y.mean((0, 2, 3), keepdim=True)
    var = ((y - mean) ** 2).mean((0, 2, 3), keepdim=True)
    return (y - mean) / torch.sqrt(var + eps) * w.double().view(1, -1, 1, 1) + b.double().view(1, -1, 1, 1)


def _check(what, got, ref, bound):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} over the bound, worst excess {(err - bound).max():.3e}"


def _conv_bound(ref, A, K):
    return BF16_U * ref.abs() + (1 + BF16_U) * KAPPA(K) * A


def _bn_bound(ref):
    # one bf16 rounding of the output plus fp32 statistics / normalisation round-off (a few ulps of fp32 on O(1) values)
    return BF16_U * ref.abs() + 1e-4 * (1 + ref.abs())


def _up_projection_teacher_forced(up, x, size, g_out):
    """The module's own steps (branch_convs, bn1, conv1_2_nhwc, the join), each on the native operands of that step,
    against float64; the module's forward is their composition to the bit."""
    import dense_ops as O
    import _lib
    c = up.conv1.out_channels
    cin = x.shape[-1]
    x = x.detach().requires_grad_(True)
    for p in up.parameters():
        p.grad = None
    y1, y2 = up.branch_convs(x, size)
    upx = nchw(O.upsample_bilinear(x.detach(), size)).double()
    wqs = [up.conv1.weight.detach().to(torch.bfloat16).double(), up.conv2.weight.detach().to(torch.bfloat16).double()]
    for name, got, wq in (("conv1", y1, wqs[0]), ("conv2", y2, wqs[1])):
        ref = F.conv2d(upx, wq, padding=2)
        A = F.conv2d(upx.abs(), wq.abs(), padding=2)
        _check(name, nchw(got), ref, _conv_bound(ref, A, 25 * cin))
    y1d = y1.detach().requires_grad_(True)
    x1 = O._bn(y1d, up.bn1, True, True)
    x1_ref = torch.relu(_bn64(nchw(y1d.detach()).double(), up.bn1.weight, up.bn1.bias))
    _check("bn1 + relu", nchw(x1), x1_ref, _bn_bound(x1_ref))
    x1d = x1.detach().requires_grad_(True)
    y12 = up.conv1_2_nhwc(x1d)
    wq12 = up.conv1_2.weight.detach().to(torch.bfloat16).double()
    y12_ref = F.conv2d(nchw(x1d.detach()).double(), wq12, padding=1)
    A12 = F.conv2d(nchw(x1d.detach()).double().abs(), wq12.abs(), padding=1)
    _check("conv1_2", nchw(y12), y12_ref, _conv_bound(y12_ref, A12, 9 * O._pad_to_64(c)))
    y12d = y12.detach().requires_grad_(True)
    y2d = y2.detach().requires_grad_(True)
    out = O.bn_add_relu(y12d, up.bn1_2, y2d, up.bn2, True)
    a64 = nchw(y12d.detach()).double().requires_grad_(True)
    b64 = nchw(y2d.detach()).double().requires_grad_(True)
    out_ref = torch.relu(_bn64(a64, up.bn1_2.weight, up.bn1_2.bias) + _bn64(b64, up.bn2.weight, up.bn2.bias))
    _check("bn1_2 + bn2 + relu", nchw(out), out_ref.detach(), _bn_bound(out_ref.detach()))
    with torch.no_grad():
        assert torch.equal(up(x.detach(), size), out)
    # backward of the join, teacher-forced on g_out; the BN backward's sums over all rows make its error scale with
    # the gradient's RMS, so the bound carries a term relative to it
    out.backward(g_out)
    out_ref.backward(nchw(g_out).double())
    for name, got, ref in (("d bran1", y12d.grad, a64.grad), ("d bran2", y2d.grad, b64.grad)):
        rms = ref.pow(2).mean().sqrt()
        _check(name, nchw(got), ref, 2 * BF16_U * ref.abs() + 2e-3 * rms)
    # backward of the paired conv: d y2 is the native gradient of the join, d y1 a seeded one (its chain runs through
    # bn1); dx through dgrad + the up-sampling backward, dw of conv1 / conv2 through the module's parameters
    g1 = torch.randn(y2d.grad.shape, device=DEV, generator=torch.Generator(device=DEV).manual_seed(c)).to(torch.bfloat16)
    torch.autograd.backward([y1, y2], [g1, y2d.grad])
    n, ho, wo, _ = g1.shape
    cp = O._pad_to_64(2 * c)
    splits = _lib.raw("dirb200_conv_wgrad_workspace_bytes")(n, ho, wo, cin, cp, 5, 5, 1, 2, 0) // (25 * cin * cp * 4)
    kp = -(-(n * ho * wo) // splits)
    gys = [nchw(g1).double(), nchw(y2d.grad).double()]
    for name, wt, gy64 in (("conv1 wgrad", up.conv1.weight, gys[0]), ("conv2 wgrad", up.conv2.weight, gys[1])):
        dw_ref = torch.nn.grad.conv2d_weight(upx, wt.shape, gy64, padding=2)
        A_dw = torch.nn.grad.conv2d_weight(upx.abs(), wt.shape, gy64.abs(), padding=2)
        _check(name, wt.grad.double(), dw_ref, KAPPA(kp) * A_dw + splits * U * A_dw)
    dup_ref = torch.nn.grad.conv2d_input(upx.shape, torch.cat(wqs, 0), torch.cat(gys, 1), padding=2)
    xin = nchw(x.detach()).double().requires_grad_(True)
    F.interpolate(xin, size=tuple(size), mode="bilinear", align_corners=False).backward(dup_ref)
    dx_ref = xin.grad
    rms = dx_ref.pow(2).mean().sqrt()
    # d(up) is stored in bf16 before the up-sampling backward sums up to (2 / scale)^2 of its values
    _check("paired conv dx", nchw(x.grad), dx_ref, 4 * BF16_U * dx_ref.abs() + 2e-2 * rms)
    return out.detach()


def test_teacher_forced_layerwise_at_228x304():
    """Every step of every up-projection of D and MFF at 228 x 304, batch 2, on the native operands of that step,
    against float64 (forward and backward)."""
    Dm, Mm = make_modules()
    Dm.train(), Mm.train()
    xs = encoder_blocks(2, 228, 304)
    import dense_ops as O
    x_d0 = O._bn(O.conv2d_nhwc(xs[3], Dm.conv.weight, 1, 0), Dm.bn, True, True)
    g = torch.Generator(device=DEV).manual_seed(5)
    x = x_d0
    sizes = [xs[2].shape[1:3], xs[1].shape[1:3], xs[0].shape[1:3], (2 * xs[0].shape[1], 2 * xs[0].shape[2])]
    for up, size in zip((Dm.up1, Dm.up2, Dm.up3, Dm.up4), sizes):
        size = tuple(int(v) for v in size)
        gout = torch.randn(x.shape[0], *size, up.conv1.out_channels, device=DEV, generator=g).to(torch.bfloat16)
        x = _up_projection_teacher_forced(up, x, size, gout)
    for up, xb in zip((Mm.up1, Mm.up2, Mm.up3, Mm.up4), xs):
        gout = torch.randn(2, 114, 152, 16, device=DEV, generator=g).to(torch.bfloat16)
        _up_projection_teacher_forced(up, xb, (114, 152), gout)


# ------------------------------------------------------------------------------------------------- eval mode
def _stats(mod):
    return {k: v.clone() for k, v in mod.state_dict().items() if "running" in k or "num_batches" in k}


def test_eval_mode_uses_running_statistics_and_leaves_them_unchanged():
    """D, MFF and RefinementR in eval(): the running statistics (set away from the batch statistics) are bit-unchanged
    by a forward and a backward, each image's output does not depend on the rest of the batch (batch statistics
    would), and the gradients are those of the frozen BatchNorm affine maps."""
    from dense_ops import RefinementR
    Dm, Mm = make_modules()
    R = RefinementR(128).to(DEV)
    with torch.no_grad():
        for mod in (Dm, Mm, R):
            for name, buf in mod.named_buffers():
                if name.endswith("running_mean"):
                    buf.copy_(0.2 * det_param(name + ".rm", buf.shape, 1.0))
                elif name.endswith("running_var"):
                    buf.copy_(0.5 + det_param(name + ".rv", buf.shape, 1.0).abs())
    xs = encoder_blocks(2, 228, 304, seed=3)
    for mod, run in ((Dm, lambda xx: Dm(*xx)), (Mm, lambda xx: Mm(*xx, (114, 152))),
                     (R, lambda xx: R(xx[0][..., :128].contiguous()))):
        mod.eval()
        before = _stats(mod)
        with torch.no_grad():
            full = run(xs)
            one = run([x[:1].contiguous() for x in xs])
        torch.cuda.synchronize()
        after = _stats(mod)
        for k in before:
            assert torch.equal(before[k], after[k]), (type(mod).__name__, k)
        assert torch.equal(full[:1], one), type(mod).__name__
    # gradients flow through the frozen BatchNorms (D, MFF: runs, statistics untouched)
    g = torch.Generator(device=DEV).manual_seed(9)
    for mod, run in ((Dm, lambda xx: Dm(*xx)), (Mm, lambda xx: Mm(*xx, (114, 152)))):
        before = _stats(mod)
        xg = [x.clone().requires_grad_(True) for x in xs]
        out = run(xg)
        out.backward(torch.randn(out.shape, device=DEV, generator=g).to(torch.bfloat16))
        torch.cuda.synchronize()
        assert all(torch.equal(before[k], v) for k, v in _stats(mod).items()), type(mod).__name__
        assert all(p.grad is not None and torch.isfinite(p.grad).all() for p in mod.parameters()), type(mod).__name__
        assert xg[3].grad is not None and torch.isfinite(xg[3].grad.float()).all()
    # R's eval output and gradients are those of the reference computation with the running statistics (fp32 with
    # the bf16-rounded conv weights; the bounds of tests/test_gpu_dense_ops.py's train-mode RefinementR test: ReLU
    # masks flip where bf16 activations sit next to zero)
    x = xs[0][..., :128].contiguous().requires_grad_(True)
    got = R(x)
    gout = torch.randn(got.shape, device=DEV, generator=g).to(torch.bfloat16)
    got.backward(gout)
    xr = nchw(x.detach()).float().requires_grad_(True)
    ps = {n: (p.detach().to(torch.bfloat16).float() if p.dim() == 4 else p.detach().clone()).requires_grad_(True)
          for n, p in R.named_parameters()}

    def bn_eval(t, pre):
        bn = getattr(R, pre)
        return F.batch_norm(t, bn.running_mean, bn.running_var, ps[pre + ".weight"], ps[pre + ".bias"], False, 0.0,
                            bn.eps)
    a = torch.relu(bn_eval(F.conv2d(xr, ps["conv0.weight"], padding=2), "bn0"))
    b = torch.relu(bn_eval(F.conv2d(a, ps["conv1.weight"], padding=2), "bn1"))
    ref = F.conv2d(b, ps["conv2.weight"], ps["conv2.bias"], padding=2)
    ref.backward(nchw(gout).float())
    errs = {"out": rel(nchw(got.detach()).float(), ref.detach()), "dx": rel(nchw(x.grad).float(), xr.grad)}
    for n, p in R.named_parameters():
        errs[n] = rel(p.grad, ps[n].grad)
    assert errs["out"] < 2e-2 and errs["dx"] < 5e-2, errs
    assert all(v < 5e-2 for v in errs.values()), errs


@pytest.mark.parametrize("join", [False, True], ids=["bn_relu", "bn_add_bn_relu"])
def test_eval_bn_backward_per_element(join):
    """The eval-mode BatchNorm backward alone (relu(bn(y)) and relu(bn_a(y_a) + bn_b(y_b))) against float64 on the
    same operands, with the ReLU mask of the stored output: dy = bf16(scale * dz) per element (one rounding of an
    fp32 product), dgamma = invstd * sum dz (y - rm) and dbeta = sum dz within fp32 summation error."""
    import dense_ops as O
    g = torch.Generator(device=DEV).manual_seed(11)
    c, rows = 64, 2 * 57 * 76
    bns = [torch.nn.BatchNorm2d(c).to(DEV).eval() for _ in range(2)]
    with torch.no_grad():
        for i, bn in enumerate(bns):
            bn.weight.copy_(1 + 0.2 * torch.randn(c, device=DEV, generator=g))
            bn.bias.copy_(0.2 * torch.randn(c, device=DEV, generator=g))
            bn.running_mean.copy_(0.3 * torch.randn(c, device=DEV, generator=g))
            bn.running_var.copy_(0.5 + torch.rand(c, device=DEV, generator=g))
    ys = [torch.randn(2, 57, 76, c, device=DEV, generator=g).to(torch.bfloat16).requires_grad_(True) for _ in range(2)]
    before = [(bn.running_mean.clone(), bn.running_var.clone()) for bn in bns]
    out = O.bn_add_relu(ys[0], bns[0], ys[1], bns[1], False) if join else O._bn(ys[0], bns[0], True, False)
    gout = torch.randn(out.shape, device=DEV, generator=g).to(torch.bfloat16)
    out.backward(gout)
    torch.cuda.synchronize()
    for bn, (rm, rv) in zip(bns, before):
        assert torch.equal(bn.running_mean, rm) and torch.equal(bn.running_var, rv)
    dz = gout.double() * (out.double() > 0)
    for i in range(2 if join else 1):
        bn = bns[i]
        invstd = 1.0 / torch.sqrt(bn.running_var.double() + bn.eps)
        scale = bn.weight.double() * invstd
        ref_dy = dz * scale
        # scale carries rsqrtf's few-ulp error
        _check(f"dy{i}", ys[i].grad, ref_dy, (BF16_U + 8 * U) * ref_dy.abs())
        y64 = ys[i].detach().double()
        ref_dg = invstd * (dz * (y64 - bn.running_mean.double())).reshape(-1, c).sum(0)
        ref_db = dz.reshape(-1, c).sum(0)
        # fp32 sums of `rows` terms (serial worst case), then invstd * (S1 - rm * S0)
        A_g = invstd * ((dz.abs() * y64.abs()).reshape(-1, c).sum(0) + bn.running_mean.double().abs() * dz.abs().reshape(-1, c).sum(0))
        A_b = dz.abs().reshape(-1, c).sum(0)
        _check(f"dgamma{i}", bn.weight.grad, ref_dg, (rows + 8) * U * A_g)
        _check(f"dbeta{i}", bn.bias.grad, ref_db, rows * U * A_b)


@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_decoder_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process)."""
    if os.environ.get("DIRB200_DECODER_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_DECODER_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
