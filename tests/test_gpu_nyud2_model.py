"""GPU checks of NYUD2-DIR's assembled depth network net.model (nyud2-dir/models/net.py:5-22) and of R's depth head
(dense_ops.depth_head: dirb200_depth_head_fwd / _dgrad / _wgrad, modules.py:145, 169).

- Head: every element against float64 on the same bf16 operands, with bounds from the kernels' fp32 summation order.
- Head determinism: bit-identical repeats; image 0's output does not depend on the batch.
- Wiring: net.model's forward and every parameter gradient equal calling E, D, MFF, cat_channels and R by hand.
- Teacher-forced R at 8 x 114 x 152 against float64 (oracle/net_ref.refinement), FDS smoothing off and on.
- Fixture parity (loose), the FDS feature view, eval mode, a frozen backbone (--retrain_fc), one Adam step.
The file reruns itself with DIRB200_SMS=7."""
import os
import subprocess
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

from util import det_param

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
BF16_U = 2.0 ** -8
TH, TW = 16, 32                     # the head kernels' pixel tile
BLOCKS = [256, 512, 1024, 2048]
torch.backends.cudnn.allow_tf32 = False
torch.backends.cuda.matmul.allow_tf32 = False


def nchw(t):
    return t.permute(0, 3, 1, 2)


def _check(what, got, ref, bound):
    err = (got.double() - ref).abs()
    bad = ~(err <= bound)                                  # NaN (an element never written) fails
    assert not bad.any(), f"{what}: {int(bad.sum())} of {bad.numel()} over the bound, worst excess {(err - bound).max():.3e}"


# ------------------------------------------------------------------------------------------------ the head
def _head_operands(n, h, w, c, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.relu(torch.randn(n, h, w, c, device=DEV, generator=g)).to(torch.bfloat16)
    wt = torch.randn(1, c, 5, 5, device=DEV, generator=g) * (2.0 / (25 * c)) ** 0.5
    b = torch.randn(1, device=DEV, generator=g)
    dy = torch.randn(n, h, w, 1, device=DEV, generator=g)
    return x, wt, b, dy


def _head_native(x, wt, b, dy):
    import _lib
    n, h, w, c = x.shape
    st = _lib.stream_ptr()
    y = torch.full((n, h, w, 1), float("nan"), device=DEV)
    _lib.call("dirb200_depth_head_fwd", _lib.ptr(x), _lib.ptr(wt), _lib.ptr(b), _lib.ptr(y), n, h, w, c, st)
    dx = torch.full_like(x, float("nan"))
    _lib.call("dirb200_depth_head_dgrad", _lib.ptr(dy), _lib.ptr(wt), _lib.ptr(dx), n, h, w, c, st)
    nb = _lib.raw("dirb200_depth_head_wgrad_workspace_bytes")(n, h, w, c)
    ws = torch.full((nb,), 255, dtype=torch.uint8, device=DEV)
    dw = torch.full_like(wt, float("nan"))
    db = torch.full_like(b, float("nan"))
    _lib.call("dirb200_depth_head_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(db), _lib.ptr(ws), nb,
              n, h, w, c, st)
    torch.cuda.synchronize()
    return y, dx, dw, db


HEAD_SHAPES = [(8, 114, 152, 128), (1, 114, 152, 128), (2, 20, 33, 8), (2, 20, 33, 256), (3, 17, 45, 64),
               (2, 3, 2, 128), (1, 1, 1, 8), (4, 49, 97, 24)]


@pytest.mark.parametrize("shape", HEAD_SHAPES, ids=["x".join(map(str, s)) for s in HEAD_SHAPES])
def test_depth_head_per_element_vs_float64(shape):
    """fwd / dgrad / wgrad against float64 on the same operands (bf16 x, fp32 w, b, dy).  Bounds (u = 2^-24):
    fwd: one serial fp32 chain of 25c products plus the bias, (25c + 2) u (sum |w x| + |b|);
    dgrad: one bf16 rounding of a serial 25-term fp32 sum, 2^-8 |ref| + 27 u sum |w dy|;
    dw / db: serial sums over a tile row (32 pixels) and the tile rows (16) -- db: 16 per lane and a 5-level butterfly
    -- then the tiles in order, (50 + tiles) u sum |terms|."""
    n, h, w, c = shape
    x, wt, b, dy = _head_operands(*shape, seed=sum(shape))
    y, dx, dw, db = _head_native(x, wt, b, dy)
    x64, w64, b64, dy64 = nchw(x).double(), wt.double(), b.double(), nchw(dy).double()
    ref = F.conv2d(x64, w64, b64, padding=2)
    A = F.conv2d(x64.abs(), w64.abs(), padding=2) + b64.abs()
    _check("fwd", nchw(y), ref, (25 * c + 2) * U * A)
    ref = torch.nn.grad.conv2d_input(x64.shape, w64, dy64, padding=2)
    A = torch.nn.grad.conv2d_input(x64.shape, w64.abs(), dy64.abs(), padding=2)
    _check("dgrad", nchw(dx), ref, BF16_U * ref.abs() + 27 * U * A)
    tiles = n * -(-h // TH) * -(-w // TW)
    ref = torch.nn.grad.conv2d_weight(x64, w64.shape, dy64, padding=2)
    A = torch.nn.grad.conv2d_weight(x64.abs(), w64.shape, dy64.abs(), padding=2)
    _check("dw", dw, ref, (50 + tiles) * U * A)
    _check("db", db, dy64.sum().view(1), (50 + tiles) * U * dy64.abs().sum().view(1))


def test_depth_head_is_deterministic_and_batch_independent():
    """Repeated calls give the same bits (fwd, dgrad, dw, db); the forward of image 0 alone equals image 0 of the
    batch, every bit."""
    x, wt, b, dy = _head_operands(8, 114, 152, 128, seed=3)
    first = _head_native(x, wt, b, dy)
    for _ in range(2):
        again = _head_native(x, wt, b, dy)
        for a, z in zip(first, again):
            assert torch.equal(a.view(torch.int16) if a.dtype == torch.bfloat16 else a.view(torch.int32),
                               z.view(torch.int16) if z.dtype == torch.bfloat16 else z.view(torch.int32))
    one = _head_native(x[:1].contiguous(), wt, b, dy[:1].contiguous())
    assert torch.equal(one[0].view(torch.int32), first[0][:1].view(torch.int32))
    assert torch.equal(one[1].view(torch.int16), first[1][:1].view(torch.int16))


# --------------------------------------------------------------------------------------------- the model
def make_args(fds=True, start_smooth=1):
    return SimpleNamespace(fds=fds, bucket_num=100, bucket_start=7, start_update=0, start_smooth=start_smooth,
                           fds_kernel="gaussian", fds_ks=5, fds_sigma=2.0, fds_mmt=0.9)


def seed_fds_tables(fds):
    from test_nyud2_model_cpu import fds_tables
    with torch.no_grad():
        for k, v in fds_tables(fds.bucket_num - fds.bucket_start, fds.feature_dim).items():
            setattr(fds, k, v.to(DEV))


def make_model(fds=True, seed=0):
    import net
    import resnet
    torch.manual_seed(seed)
    m = net.model(make_args(fds), resnet.E_resnet(resnet.resnet50()), 2048, BLOCKS)
    with torch.no_grad():                       # non-trivial BN affine in D / MFF / R
        for n, p in m.named_parameters():
            if p.dim() == 1 and not n.startswith("E."):
                p.copy_((1.0 if n.endswith("weight") else 0.0) + 0.1 * det_param(n, p.shape, 1.0))
    m = m.to(DEV)
    if fds:
        seed_fds_tables(m.R.FDS)
    return m


def inputs(n, h, w, seed=0):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(n, 3, h, w, device=DEV, generator=g)
    depth = 0.5 + 9.5 * torch.rand(n, 1, h // 2, w // 2, device=DEV, generator=g)
    weight = 0.5 + torch.rand(n, 1, h // 2, w // 2, device=DEV, generator=g)
    return x, depth, weight


def loss_fn(out, depth, weight):
    return torch.mean(((out - depth) ** 2) * weight)        # nyud2-dir/train.py:200


def _grads(m):
    return {n: (None if p.grad is None else p.grad.detach().clone()) for n, p in m.named_parameters()}


def _zero(m):
    for p in m.parameters():
        p.grad = None


@pytest.mark.parametrize("fds,epoch", [(False, 0), (True, 0), (True, 1)], ids=["no_fds", "fds_off", "fds_smooth"])
def test_model_equals_its_modules_called_by_hand(fds, epoch):
    """net.model(x, depth, epoch) in training mode: output, feature and every parameter gradient bit-identical to
    E, D, MFF, cat_channels and R called by hand (FDS off; on with epoch < start_smooth; on and smoothing)."""
    import dense_ops
    m = make_model(fds)
    m.train()
    x, depth, weight = inputs(2, 228, 304)
    _zero(m)
    res = m(x, depth, epoch)
    out, feature = res if fds else (res, None)
    assert out.dtype == torch.float32 and tuple(out.shape) == (2, 1, 114, 152)
    loss_fn(out, depth, weight).backward()
    g_model = _grads(m)
    _zero(m)
    b1, b2, b3, b4 = m.E(x)
    d = m.D(b1, b2, b3, b4)
    mf = m.MFF(b1, b2, b3, b4, [d.shape[1], d.shape[2]])
    r = m.R(dense_ops.cat_channels([d, mf]), depth, epoch)
    out2, x1 = r if fds else (r, None)
    out2 = nchw(out2)
    assert torch.equal(out.view(torch.int32), out2.view(torch.int32))
    if fds:
        assert feature.shape == (2, 128, 114, 152) and feature.dtype == torch.bfloat16
        assert torch.equal(feature, nchw(x1))
    loss_fn(out2, depth, weight).backward()
    g_hand = _grads(m)
    for n in g_model:
        assert g_model[n] is not None and torch.equal(g_model[n].view(torch.int32), g_hand[n].view(torch.int32)), n


@pytest.mark.parametrize("epoch", [0, 1], ids=["fds_off", "fds_smooth"])
def test_refinement_teacher_forced_at_8x114x152(epoch):
    """R at 8 x 114 x 152 x 128 on the concatenated native D / MFF output, against oracle/net_ref.refinement in
    float64 with the native bf16 storage points forced: the convolution + BatchNorm + ReLU steps (relative L2 2e-2:
    bf16 conv outputs normalised), FDS smoothing and the depth head per element, R's module forward equal to the
    composition of its steps bit for bit, the returned feature the unsmoothed x1; then the head's gradients per
    element from the native incoming gradient and the smoothed map."""
    import dense_ops as O
    from oracle import net_ref
    m = make_model(True)
    m.train()
    x, depth, weight = inputs(8, 228, 304, seed=4)
    with torch.no_grad():
        b = m.E(x)
        d = m.D(*b)
        xin = O.cat_channels([d, m.MFF(*b, [d.shape[1], d.shape[2]])])
    R = m.R
    x0 = O._bn(O.conv2d_nhwc(xin, R.conv0.weight, 1, 2), R.bn0, True, True)
    x1 = O._bn(O.conv2d_nhwc(x0, R.conv1.weight, 1, 2), R.bn1, True, True)
    x1_s = x1
    if epoch >= R.FDS.start_smooth:
        from fds import FDS
        n, h, w, c = x1.shape
        x1_s = FDS.smooth(R.FDS, x1.float().view(-1, c), depth.reshape(-1).float(), epoch).view(n, h, w, c).to(torch.bfloat16)
    x1_s = x1_s.detach().requires_grad_(True)
    x2 = O.depth_head(x1_s, R.conv2.weight, R.conv2.bias)
    with torch.no_grad():
        out, feature = R(xin, depth, epoch)
    assert torch.equal(out, x2.detach()) and torch.equal(feature, x1)
    p = {k: v.detach().double() for k, v in R.named_parameters()}
    p.update({k: v.detach().to(torch.bfloat16).double() for k, v in R.named_parameters() if v.dim() == 4
              and k != "conv2.weight"})
    fds = dict(tables={k: getattr(R.FDS, k).double() for k in ("running_mean_last_epoch", "running_var_last_epoch",
                                                             "smoothed_mean_last_epoch", "smoothed_var_last_epoch")},
               start_smooth=R.FDS.start_smooth)
    force = {"x0": nchw(x0.detach()).double(), "x1": nchw(x1.detach()).double()}
    if epoch >= 1:
        force["x1_s"] = nchw(x1_s.detach()).double()
    ref_x2, _ = net_ref.refinement(p, nchw(xin).double(), depth.double(), epoch, fds, force=force)
    # the conv + BatchNorm + ReLU steps, each from the native input of that step
    ref_x0 = torch.relu(net_ref.bn_train(F.conv2d(nchw(xin).double(), p["conv0.weight"], padding=2), p["bn0.weight"],
                                         p["bn0.bias"]))
    ref_x1 = torch.relu(net_ref.bn_train(F.conv2d(force["x0"], p["conv1.weight"], padding=2), p["bn1.weight"],
                                         p["bn1.bias"]))
    rel = lambda a, r: ((a.double() - r).norm() / r.norm()).item()
    assert rel(nchw(x0), ref_x0) < 2e-2 and rel(nchw(x1), ref_x1) < 2e-2, (rel(nchw(x0), ref_x0), rel(nchw(x1), ref_x1))
    if epoch >= 1:
        ref_s = net_ref.fds_smooth(force["x1"], depth.double(), fds["tables"])
        # fp32 re-colouring (a few ulps) and one bf16 rounding
        _check("fds smooth", nchw(x1_s.detach()), ref_s, BF16_U * ref_s.abs() + 1e-5 * (1 + ref_s.abs()))
    c = x1.shape[-1]
    x1s64 = nchw(x1_s.detach()).double()
    A = F.conv2d(x1s64.abs(), p["conv2.weight"].abs(), padding=2) + p["conv2.bias"].abs()
    _check("head", nchw(x2.detach()), ref_x2, (25 * c + 2) * U * A)
    # backward of the head, teacher-forced on the native incoming gradient of the LDS-weighted loss
    loss_fn(nchw(x2), depth, weight).backward()
    dy = (2.0 * (nchw(x2.detach()).double() - depth.double()) * weight.double() / x2.numel())
    tiles = 8 * -(-114 // TH) * -(-152 // TW)
    ref_dw = torch.nn.grad.conv2d_weight(x1s64, (1, c, 5, 5), dy, padding=2)
    A_dw = torch.nn.grad.conv2d_weight(x1s64.abs(), (1, c, 5, 5), dy.abs(), padding=2)
    # dy itself is formed by torch in fp32 (a few ulps)
    _check("dw", R.conv2.weight.grad, ref_dw, (50 + tiles + 8) * U * A_dw)
    _check("db", R.conv2.bias.grad, dy.sum().view(1), (50 + tiles + 8) * U * dy.abs().sum().view(1))
    ref_dx = torch.nn.grad.conv2d_input(x1s64.shape, p["conv2.weight"], dy, padding=2)
    A_dx = torch.nn.grad.conv2d_input(x1s64.shape, p["conv2.weight"].abs(), dy.abs(), padding=2)
    _check("dx", nchw(x1_s.grad), ref_dx, BF16_U * ref_dx.abs() + 35 * U * A_dx)


def test_model_against_reference_fixture():
    """The native model on the fixture's input against the reference's own net.model (fp32 CPU), FDS smoothing
    active: a deliberately loose sanity check -- relative L2 below 1.0 on the output and the feature (an unrelated map
    of the same norm is at about 1.4) and the loss within 25 %.  At this size the network is ill-conditioned: its deep
    maps are 2 x 2 and 3 x 3 at batch 2, so train-mode BatchNorms normalise over 8 to 18 values and amplify upstream
    rounding (DESIGN.md §2).  Evaluating the fp32 restatement in float64 instead already moves the output by 5e-4
    relative (about 8000 times fp32's unit round-off), so bf16 storage (2^-9) moves it by O(1): 0.77 (output), 0.86
    (feature) and 10 % (loss) measured on an H100.  The per-step precision is pinned by the teacher-forced tests of
    the encoder, the decoder and R (above)."""
    from test_nyud2_model_cpu import fixture_model, depth_and_weight, sample_idx
    from util import golden
    g = golden("nyud2_model")
    m = fixture_model(True).to(DEV)
    seed_fds_tables(m.R.FDS)
    m.train()
    x = det_param("x_nyud2_model", (2, 3, 36, 44), 1.0).to(DEV)
    depth, weight = depth_and_weight()
    out, feature = m(x, depth.to(DEV), 1)
    rel = lambda a, b: float((a.double() - b.double()).norm() / b.double().norm())
    e_out = rel(out.detach().cpu(), torch.from_numpy(g["out"]))
    f = feature.detach().float().cpu().reshape(-1)
    e_f = rel(f[sample_idx(f.numel(), 8192)], torch.from_numpy(g["feature"]))
    loss = loss_fn(out, depth.to(DEV), weight.to(DEV)).item()
    print(f"fixture: out {e_out:.2e} feature {e_f:.2e} loss {loss:.4f} vs {float(g['loss']):.4f}")
    assert e_out < 1.0 and e_f < 1.0 and abs(loss / float(g["loss"]) - 1) < 0.25


def test_fds_update_from_the_feature_view():
    """R.FDS.update_running_stats(feature, depth, epoch) on the returned [N, 128, h, w] view of the NHWC bf16 map gives
    the same tables, every bit, as the same values passed as a contiguous fp32 NCHW tensor."""
    from fds_variants import FDSDepth
    m = make_model(True)
    m.train()
    x, depth, _ = inputs(2, 228, 304, seed=5)
    with torch.no_grad():
        _, feature = m(x, depth, 0)
    assert not feature.is_contiguous() and feature.stride(1) == 1
    a, b = FDSDepth(128).to(DEV), FDSDepth(128).to(DEV)
    a.update_running_stats(feature, depth, 0)
    b.update_running_stats(feature.float().contiguous(), depth, 0)
    for k, v in a.state_dict().items():
        assert torch.equal(v, b.state_dict()[k]), k


def _buffers(m):
    return {k: v.clone() for k, v in m.state_dict().items() if v.is_floating_point() is False or "running" in k
            or "num_batches" in k}


def test_eval_mode():
    """eval(): running statistics (E's folded-BN forward, D / MFF / R) bit-unchanged by a forward and a backward; the
    output alone is returned, fp32 [N, 1, H/2, W/2], and each image's output does not depend on the batch;
    depth_eval.test on a small synthetic loader equals Evaluator.add on the outputs computed by hand."""
    import depth_eval
    m = make_model(True)
    m.train()
    x, depth, weight = inputs(3, 228, 304, seed=6)
    with torch.no_grad():
        m(x, depth, 1)                                    # running statistics away from their initial values
    m.eval()
    before = _buffers(m)
    out = m(x)
    assert isinstance(out, torch.Tensor) and out.dtype == torch.float32 and tuple(out.shape) == (3, 1, 114, 152)
    loss_fn(out, depth, weight).backward()
    torch.cuda.synchronize()
    after = _buffers(m)
    for k in before:
        assert torch.equal(before[k], after[k]), k
    with torch.no_grad():
        assert torch.equal(m(x[:1]), out[:1].detach())
    g = torch.Generator().manual_seed(7)
    batches = [dict(image=x[i:i + 2].cpu(), depth=(0.5 + 9.5 * torch.rand(len(x[i:i + 2]), 1, 228, 304, generator=g)),
                    mask=torch.rand(len(x[i:i + 2]), 1, 228, 304, generator=g) > 0.3) for i in (0, 2)]
    shot_idx = dict(many=list(range(0, 30)), medium=list(range(30, 60)), few=list(range(60, 100)))
    rmse, metrics = depth_eval.test(batches, m, shot_idx)
    ev = depth_eval.Evaluator(shot_idx)
    with torch.no_grad():
        for bt in batches:
            ev.add(m(bt["image"].to(DEV)), bt["depth"].to(DEV), bt["mask"].to(DEV))
    assert metrics == ev.evaluate_shot() and rmse == metrics["overall"]["RMSE"]


def test_frozen_backbone_trains_only_R():
    """--retrain_fc (nyud2-dir/train.py:128-142): every parameter whose name has no 'R' frozen; after loss, backward and
    an Adam step over the rest, only R's parameters have gradients and changed, and E's flat gradient buffer is
    untouched (the encoder runner's backward does not run)."""
    m = make_model(True)
    m.train()
    for name, p in m.named_parameters():
        if "R" not in name:
            p.requires_grad = False
    assert {n.split(".")[0] for n, p in m.named_parameters() if p.requires_grad} == {"R"}
    opt = torch.optim.Adam([p for p in m.parameters() if p.requires_grad], 1e-4, weight_decay=1e-4)
    x, depth, weight = inputs(2, 228, 304, seed=8)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    out, _ = m(x, depth, 1)
    flat = m.E._resnet.flat_grads().clone()
    opt.zero_grad()
    loss_fn(out, depth, weight).backward()
    opt.step()
    torch.cuda.synchronize()
    assert torch.equal(m.E._resnet.flat_grads(), flat)
    for n, p in m.named_parameters():
        if n.startswith("R."):
            assert p.grad is not None and not torch.equal(p.detach(), before[n]), n
        else:
            assert torch.equal(p.detach(), before[n]), n
            assert n.startswith("E.") or p.grad is None, n


def test_one_training_step_with_adam():
    """Loss, backward and torch.optim.Adam(weight_decay=1e-4) at 228 x 304 batch 2 with FDS smoothing active: every
    parameter finite and changed."""
    m = make_model(True)
    m.train()
    opt = torch.optim.Adam(m.parameters(), 1e-4, weight_decay=1e-4)
    x, depth, weight = inputs(2, 228, 304, seed=9)
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt.zero_grad()
    out, feature = m(x, depth, 1)
    loss = loss_fn(out, depth, weight)
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    for n, p in m.named_parameters():
        assert torch.isfinite(p).all() and not torch.equal(p.detach(), before[n]), n


@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_model_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process)."""
    if os.environ.get("DIRB200_MODEL_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_MODEL_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
