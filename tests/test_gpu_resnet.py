"""GPU parity of the whole native ResNet-50 path (runner + regressor + loss +
optimizer) against the torch fp32 oracle (oracle/resnet_ref.py, itself pinned
to the reference).  The conv stack stores bf16, so it is compared with the
oracle's quant=True mode (same storage points, straight-through rounding):
tolerances are a few bf16 ulps of the tensor scale, stated per check."""
import numpy as np
import pytest
import torch

from util import det_param

pytestmark = pytest.mark.gpu
DEV = "cuda"
import os
_TF32 = os.environ.get("DIRB200_TEST_TF32") == "1"      # diagnosis only: the round-1 setting of the oracle convolutions
torch.backends.cudnn.allow_tf32 = _TF32          # the oracle's convolutions are true fp32
torch.backends.cuda.matmul.allow_tf32 = _TF32


def make_model(fds=False, layers=(3, 4, 6, 3), **kw):
    from resnet import ResNet, Bottleneck
    args = dict(fds=fds, bucket_num=100, bucket_start=3, start_update=0, start_smooth=1, kernel="gaussian",
                ks=9, sigma=1, momentum=0.9)
    args.update(kw)
    torch.manual_seed(0)
    m = ResNet(Bottleneck, list(layers), **args)
    with torch.no_grad():                       # non-trivial BN affine so its gradients are exercised
        for n, p in m.named_parameters():
            if p.dim() == 1 and ("bn" in n or "downsample.1" in n):
                p.copy_((1.0 if n.endswith("weight") else 0.0) + 0.1 * det_param(n, p.shape, 1.0))
    return m.to(DEV)


def oracle_params(m):
    return {n: p.detach().clone().requires_grad_(True) for n, p in m.named_parameters() if not n.startswith("FDS")}


def rel(a, b):
    return ((a - b).norm() / (b.norm() + 1e-12)).item()


def cos(a, b):
    return torch.nn.functional.cosine_similarity(a.reshape(1, -1).double(), b.reshape(1, -1).double()).item()


def test_state_dict_keys_match_reference_layout():
    from oracle import resnet_ref as R
    m = make_model(fds=True)
    names = [n for n, _ in m.named_parameters()]
    assert names == [n for n, _ in R.param_shapes()]
    assert [tuple(p.shape) for _, p in m.named_parameters()] == [s for _, s in R.param_shapes()]
    sd = m.state_dict()
    for k in ("bn1.running_mean", "bn1.running_var", "bn1.num_batches_tracked", "layer1.0.downsample.1.running_var",
              "layer4.2.bn3.num_batches_tracked", "FDS.running_mean", "FDS.smoothed_var_last_epoch", "linear.bias"):
        assert k in sd, k
    assert sum(p.numel() for p in m.parameters()) == 23510081
    assert sum(b.numel() for n, b in m.named_buffers() if not n.startswith("FDS")) == 53173
    # parameters tile one flat buffer; loading a state_dict keeps that
    m2 = make_model(fds=True)
    m2.load_state_dict(sd)
    assert torch.equal(m2.flat_parameters(), m.flat_parameters())
    assert m2.conv1.weight.data_ptr() == m2.flat_parameters().data_ptr()


def _fb(layers, n, hw):
    from oracle import resnet_ref as R
    import loss as L
    m = make_model(layers=layers)
    m.train()
    p = oracle_params(m)
    x = det_param(f"x{n}", (n, 3, hw, hw), 1.0).to(DEV)
    t = (torch.arange(n, dtype=torch.float32, device=DEV).reshape(n, 1) * 5 + 10)
    w = torch.linspace(0.5, 1.5, n, device=DEV).reshape(n, 1)
    pred = m(x, t, 0)
    loss = L.weighted_l1_loss(pred, t, w)
    loss.backward()
    stats = {}
    rpred, renc = R.forward(p, x, layers=layers, stats=stats, quant=True)
    rloss = ((rpred - t).abs() * w).mean()
    rloss.backward()
    enc = m._run_forward(x, training=True)          # encoding (second pass, same batch statistics)
    return m, p, stats, enc, renc.detach(), loss.item(), rloss.item()


def test_forward_backward_vs_oracle_shallow():
    """End-to-end fwd+bwd parity on a 6-block bottleneck net ([2,2,1,1]: identity blocks, stride-1 and stride-2
    downsample blocks, stem, pools, regressor, loss).  A train-mode-BN ResNet at initialisation amplifies any
    perturbation by ~1.15x per layer (measured with tests/debug_layers.py: 1e-4 after the first conv -> 0.3 after
    all 16 blocks of ResNet-50 purely from bf16 round-off flips), so tight end-to-end tolerances are only
    meaningful on a shallow stack; the full depth is covered layer by layer below."""
    from oracle import resnet_ref as R
    layers = (2, 2, 1, 1)
    m, p, stats, enc, renc, loss, rloss = _fb(layers, 16, 64)
    assert rel(enc, renc) < 4e-2 and cos(enc, renc) > 0.999, rel(enc, renc)
    assert abs(loss - rloss) < 2e-2 * abs(rloss) + 1e-3
    rm = 0.9 * stats["bn1.running_mean"] + stats["bn1.running_mean"]      # two training forwards
    assert rel(m.bn1.running_mean, rm) < 1e-3
    assert int(m.bn1.num_batches_tracked) == 2
    named = dict(m.named_parameters())
    for name, rp in p.items():
        g, rg = named[name].grad, rp.grad
        assert g is not None and torch.isfinite(g).all(), name
        # 2 % forward round-off drift flips ~1.5 % of the ReLU masks => ~20-35 % gradient noise (see the
        # teacher-forced test below for the tight comparison)
        assert cos(g, rg) > 0.9 and rel(g, rg) < 0.5, (name, cos(g, rg), rel(g, rg))
    flat_ref = torch.cat([p[nm].grad.reshape(-1) for nm, _ in R.param_shapes(layers)])
    assert rel(m.flat_grads(), flat_ref) < 0.4, rel(m.flat_grads(), flat_ref)


@pytest.mark.parametrize("n,hw", [(16, 64), (4, 224), (256, 224)], ids=["b16_64", "b4_224", "benchmark_b256_224"])
def test_resnet50_layerwise_forward_teacher_forced(n, hw):
    """Every conv / BN+ReLU / residual stage of the full ResNet-50, each checked against the oracle op applied to
    the runner's OWN input of that stage (so errors cannot compound): relative L2 error <= 4e-3 (a bf16 ulp)."""
    from oracle import resnet_ref as R
    import torch.nn.functional as F
    m = make_model()
    m.train()
    p = {k: v.detach() for k, v in m.named_parameters()}
    x = det_param(f"x{n}", (min(n, 16), 3, hw, hw), 1.0).to(DEV)
    if n > 16:     # the benchmark batch: 16 generated images tiled with per-image gains (cheap to build, all distinct)
        x = (x.repeat(n // 16, 1, 1, 1) * torch.linspace(0.5, 1.5, n, device=DEV).reshape(n, 1, 1, 1)).contiguous()
    m._run_forward(x, training=True)
    shape = tuple(x.shape)
    pk = lambda b, w: m.peek(shape, b, w)
    q = lambda t: t.to(torch.bfloat16).float()
    tol = 4e-3

    def check(name, got, ref):
        e = rel(got, ref)
        assert e <= tol, (name, e)

    with torch.no_grad():
        check("stem.y", pk(-1, 0), R._conv(q(x), p["conv1.weight"], 2, 3, True))
        # relu(bn1(.)) is fused into the max pool and never stored: checked through the pooled tensor
        check("stem.pool", pk(-1, 6), F.max_pool2d(q(F.relu(R._bn(pk(-1, 0), p, "bn1.", None, True))), 3, 2, 1))
        bi = 0
        for li, nblocks in enumerate((3, 4, 6, 3)):
            for b in range(nblocks):
                stride = 2 if (b == 0 and li > 0) else 1
                pre = f"layer{li + 1}.{b}."
                xin = pk(-1, 6) if bi == 0 else pk(bi - 1, 6)
                check(pre + "conv1", pk(bi, 0), R._conv(xin, p[pre + "conv1.weight"], 1, 0, True))
                check(pre + "bn1", pk(bi, 1), q(F.relu(R._bn(pk(bi, 0), p, pre + "bn1.", None, True))))
                check(pre + "conv2", pk(bi, 2), R._conv(pk(bi, 1), p[pre + "conv2.weight"], stride, 1, True))
                check(pre + "bn2", pk(bi, 3), q(F.relu(R._bn(pk(bi, 2), p, pre + "bn2.", None, True))))
                check(pre + "conv3", pk(bi, 4), R._conv(pk(bi, 3), p[pre + "conv3.weight"], 1, 0, True))
                o = R._bn(pk(bi, 4), p, pre + "bn3.", None, True)
                if pre + "downsample.0.weight" in p:
                    check(pre + "ds", pk(bi, 5), R._conv(xin, p[pre + "downsample.0.weight"], stride, 0, True))
                    idn = R._bn(pk(bi, 5), p, pre + "downsample.1.", None, True)
                else:
                    idn = xin
                check(pre + "out", pk(bi, 6), q(F.relu(o + idn)))
                bi += 1
        enc = m._run_forward(x, training=True)
        check("avgpool", enc, pk(15, 6).mean(dim=(2, 3)))


TAPS = [("stem.y", -1, 0), ("stem.pool", -1, 6)]      # the stem's activation is not materialised by the runner


@pytest.mark.parametrize("layers,n,hw", [((3, 4, 6, 3), 16, 64), ((3, 4, 6, 3), 4, 224), ((2, 2, 1, 1), 16, 64),
                                         ((3, 4, 6, 3), 256, 224)],
                         ids=["r50_b16_64", "r50_b4_224", "shallow_b16_64", "r50_benchmark_b256_224"])
def test_backward_vs_oracle_teacher_forced(layers, n, hw):
    """Backward parity at full depth: the oracle's forward is teacher-forced to the runner's stored activations
    (same ReLU masks, same BN inputs), its backward is torch autograd in fp32 with bf16 rounding at the points where
    the runner stores bf16 gradients.  Every parameter gradient must then agree to bf16-level error."""
    from oracle import resnet_ref as R
    import loss as L
    m = make_model(layers=layers)
    m.train()
    p = oracle_params(m)
    x = det_param(f"x{n}", (min(n, 16), 3, hw, hw), 1.0).to(DEV)
    if n > 16:     # the benchmark batch (BASELINE config 3 shape): tiled + per-image gains, see the forward test
        x = (x.repeat(n // 16, 1, 1, 1) * torch.linspace(0.5, 1.5, n, device=DEV).reshape(n, 1, 1, 1)).contiguous()
    t = (torch.arange(n, dtype=torch.float32, device=DEV).reshape(n, 1) * 5 + 10) % 101
    w = torch.linspace(0.5, 1.5, n, device=DEV).reshape(n, 1)
    pred = m(x, t, 0)
    L.weighted_l1_loss(pred, t, w).backward()
    force = {}
    names = list(TAPS) + [(f"{b}.{k}", b, k) for b in range(sum(layers)) for k in range(7)]
    for name, b, k in names:
        try:
            force[name] = m.peek(x.shape, b, k, copy=n <= 16)   # big batch: zero-copy bf16 views of the runner's buffers
        except Exception:
            pass                                   # blocks without a downsample branch
    assert len(force) == 2 + 6 * sum(layers) + 4
    rpred, renc = R.forward(p, x, layers=layers, quant=True, force=force)
    ((rpred - t).abs() * w).mean().backward()
    assert rel(pred.detach(), rpred.detach()) < 2e-3
    named = dict(m.named_parameters())
    worst = ("", 1.0, 0.0)
    for name, rp in p.items():
        g, rg = named[name].grad, rp.grad
        c, e = cos(g, rg), rel(g, rg)
        if e > worst[2]:
            worst = (name, c, e)
    print('worst parameter gradient:', worst)
    # bf16 round-off of the stored gradients is itself amplified ~1.1x per layer on the way back to the stem: the worst
    # parameter is always the stem's bn1.bias (a plain sum of the most-amplified gradient tensor); the bound leaves room
    # for that amplification and for the fp32 cuDNN reference's non-deterministic backward algorithms
    assert worst[2] < 0.15 and worst[1] > 0.99, worst
    flat_ref = torch.cat([p[nm].grad.reshape(-1) for nm, _ in R.param_shapes(layers)])
    assert rel(m.flat_grads(), flat_ref) < 3e-2, rel(m.flat_grads(), flat_ref)


def test_resnet50_end_to_end_sanity():
    """Full depth, batch 4 at 224^2 (BASELINE config 1 shape): outputs and gradients stay aligned with the oracle
    within what the chaotic amplification allows (see the shallow test's note)."""
    m, p, stats, enc, renc, loss, rloss = _fb((3, 4, 6, 3), 4, 224)
    assert cos(enc, renc) > 0.9 and np.isfinite(loss)
    assert torch.isfinite(m.flat_grads()).all()
    named = dict(m.named_parameters())
    assert cos(named["linear.weight"].grad, p["linear.weight"].grad) > 0.9
    assert rel(named["linear.bias"].grad, p["linear.bias"].grad) < 1e-3


def test_eval_mode_and_no_grad_paths():
    m = make_model(fds=True)
    x = det_param("xe", (8, 3, 64, 64), 1.0).to(DEV)
    t = torch.full((8, 1), 30.0, device=DEV)
    m.train()
    with torch.no_grad():
        out, feat = m(x, t, 0)                       # collection-pass shape: (pred, encoding)
    assert out.shape == (8, 1) and feat.shape == (8, 2048)
    m.eval()
    y1 = m(x)
    y2 = m(x)
    assert y1.shape == (8, 1) and torch.equal(y1, y2)  # eval: running statistics, deterministic
    assert int(m.bn1.num_batches_tracked) == 1


@pytest.mark.parametrize("n,hw", [(16, 64), (4, 224)], ids=["b16_64", "b4_224"])
def test_eval_forward_folded_bn_layerwise_vs_oracle(n, hw):
    """Inference path (agedb-dir/train.py:286-335: model.eval(), BatchNorm on the running statistics): every
    conv + folded BN [+ ReLU] launch and the conv3 + BN + shortcut + ReLU tail of each block against fp32 torch ops
    applied to the runner's OWN input of that stage (teacher-forced), then the prediction end to end against the
    oracle network in eval mode."""
    import torch.nn.functional as F
    m = make_model()
    m.train()
    with torch.no_grad():               # two training forwards: non-trivial running statistics
        for k in range(2):
            m(det_param(f"xw{k}", (n, 3, hw, hw), 1.0).to(DEV) * (1.0 + 0.5 * k))
    m.eval()
    sd = {k: v.detach().float() for k, v in m.state_dict().items()}
    x = det_param("xev", (n, 3, hw, hw), 1.0).to(DEV)
    with torch.no_grad():
        pred = m(x)
    shape = tuple(x.shape)
    pk = lambda b, w: m.peek(shape, b, w)
    q = lambda t: t.to(torch.bfloat16).float()

    def fold(pre):
        sc = sd[pre + "weight"] * torch.rsqrt(sd[pre + "running_var"] + 1e-5)
        return sc[None, :, None, None], (sd[pre + "bias"] - sd[pre + "running_mean"] * sc)[None, :, None, None]

    def conv(t, w, stride, pad):        # fp32 accumulation over bf16 operands, NOT rounded (the BN is applied first)
        return F.conv2d(q(t), q(w), stride=stride, padding=pad)

    tol = 4e-3
    def check(name, got, ref):
        e = rel(got, ref)
        assert e <= tol, (name, e)

    # DIRB200_FOLDED_EVAL=0: conv -> bf16 raw output -> separate BN-apply pass, so the buffers hold other stages:
    # peek(b, 5) is the RAW downsample output, and the block tail adds the two BN outputs in fp32 before one rounding
    folded = os.environ.get("DIRB200_FOLDED_EVAL", "1")[:1] != "0"
    stored = (lambda t: t) if folded else q     # the unfused path stores the conv output in bf16 before the BN
    with torch.no_grad():
        sc, sh = fold("bn1.")
        check("stem.pool", pk(-1, 6), F.max_pool2d(q(F.relu(pk(-1, 0) * sc + sh)), 3, 2, 1))
        bi = 0
        for li, nblocks in enumerate((3, 4, 6, 3)):
            for b in range(nblocks):
                stride = 2 if (b == 0 and li > 0) else 1
                pre = f"layer{li + 1}.{b}."
                xin = pk(-1, 6) if bi == 0 else pk(bi - 1, 6)
                sc, sh = fold(pre + "bn1.")
                check(pre + "conv1+bn1", pk(bi, 1), q(F.relu(stored(conv(xin, sd[pre + "conv1.weight"], 1, 0)) * sc + sh)))
                sc, sh = fold(pre + "bn2.")
                check(pre + "conv2+bn2", pk(bi, 3),
                      q(F.relu(stored(conv(pk(bi, 1), sd[pre + "conv2.weight"], stride, 1)) * sc + sh)))
                if pre + "downsample.0.weight" in sd:
                    sc, sh = fold(pre + "downsample.1.")
                    if folded:
                        check(pre + "ds", pk(bi, 5), q(conv(xin, sd[pre + "downsample.0.weight"], stride, 0) * sc + sh))
                        idn = pk(bi, 5)
                    else:
                        check(pre + "ds raw", pk(bi, 5), q(conv(xin, sd[pre + "downsample.0.weight"], stride, 0)))
                        idn = pk(bi, 5) * sc + sh
                else:
                    idn = xin
                sc, sh = fold(pre + "bn3.")
                y3 = conv(pk(bi, 3), sd[pre + "conv3.weight"], 1, 0)
                if folded:
                    # the epilogue rounds the BN output to bf16 before the shortcut is added (staging tile), then
                    # rounds again
                    check(pre + "out", pk(bi, 6), q(F.relu(q(y3 * sc + sh) + idn)))
                else:
                    check(pre + "out", pk(bi, 6), q(F.relu(q(y3) * sc + sh + idn)))
                bi += 1
        # end to end: torch's own eval-mode network on the same parameters and running statistics (fp32)
        def bn(t, pre):
            s, h = fold(pre)
            return t * s + h
        t = F.max_pool2d(F.relu(bn(F.conv2d(x, sd["conv1.weight"], stride=2, padding=3), "bn1.")), 3, 2, 1)
        for li, nblocks in enumerate((3, 4, 6, 3)):
            for b in range(nblocks):
                stride = 2 if (b == 0 and li > 0) else 1
                pre = f"layer{li + 1}.{b}."
                o = F.relu(bn(F.conv2d(t, sd[pre + "conv1.weight"]), pre + "bn1."))
                o = F.relu(bn(F.conv2d(o, sd[pre + "conv2.weight"], stride=stride, padding=1), pre + "bn2."))
                o = bn(F.conv2d(o, sd[pre + "conv3.weight"]), pre + "bn3.")
                if pre + "downsample.0.weight" in sd:
                    t = bn(F.conv2d(t, sd[pre + "downsample.0.weight"], stride=stride), pre + "downsample.1.")
                t = F.relu(o + t)
        ref_enc = t.mean(dim=(2, 3))
        ref_pred = ref_enc @ sd["linear.weight"].t() + sd["linear.bias"]
        # 53 bf16-stored layers end to end (every stage is pinned to 4e-3 above): the 2048-d encoding to 4 %, the scalar
        # prediction (a near-cancelling dot product of it) as a sanity bound only
        enc = pk(15, 6).mean(dim=(2, 3))
        assert rel(enc, ref_enc) < 4e-2 and cos(enc, ref_enc) > 0.999, (rel(enc, ref_enc), cos(enc, ref_enc))
        assert (pred - ref_pred).abs().max().item() < 0.05 * ref_enc.abs().mean().item() * sd["linear.weight"].abs().sum().item() + 1e-3


def test_train_step_fused_adam_matches_torch_adam():
    """3 steps of (forward, weighted L1, backward, Adam) with our fused optimizer vs torch.optim.Adam driven by
    the same gradients: parameters stay equal to fp32 rounding."""
    import loss as L
    from optim import FusedAdam
    m = make_model()
    m.train()
    opt = FusedAdam(m.parameters(), lr=1e-3)
    shadow = [p.detach().clone().requires_grad_(True) for p in m.parameters()]
    ref_opt = torch.optim.Adam(shadow, lr=1e-3)
    x = det_param("xa", (8, 3, 64, 64), 1.0).to(DEV)
    t = torch.linspace(5, 80, 8, device=DEV).reshape(8, 1)
    losses = []
    for step in range(3):
        pred = m(x, t, 0)
        loss = L.weighted_l1_loss(pred, t, None)
        opt.zero_grad()
        loss.backward()
        for s, p in zip(shadow, m.parameters()):
            s.grad = p.grad.detach().clone()
        opt.step()
        ref_opt.step()
        losses.append(loss.item())
        for s, p in zip(shadow, m.parameters()):
            assert torch.allclose(s, p, rtol=1e-5, atol=1e-7)
    assert all(np.isfinite(losses))


def test_fds_model_training_step_smooth_active():
    """epoch >= start_smooth with non-trivial FDS tables: forward returns (pred, smoothed encoding) and the
    backward reaches the backbone through the calibration."""
    import loss as L
    m = make_model(fds=True, bucket_num=100, bucket_start=0, ks=5, sigma=2)
    m.train()
    torch.manual_seed(1)
    nb = 100
    m.FDS.running_mean_last_epoch = torch.randn(nb, 2048, device=DEV) * 0.1 + 0.5
    m.FDS.running_var_last_epoch = torch.rand(nb, 2048, device=DEV) + 0.5
    m.FDS.smoothed_mean_last_epoch = torch.randn(nb, 2048, device=DEV) * 0.1 + 0.5
    m.FDS.smoothed_var_last_epoch = torch.rand(nb, 2048, device=DEV) + 0.5
    x = det_param("xf", (8, 3, 64, 64), 1.0).to(DEV)
    t = torch.tensor([[3.], [17.], [17.], [40.], [99.], [120.], [0.], [55.]], device=DEV)
    pred, enc = m(x, t, 2)
    raw = m._run_forward(x, training=True)
    assert not torch.allclose(enc, raw)              # encoding returned is the smoothed one (in-place alias)
    L.weighted_l1_loss(pred, t, torch.ones_like(t)).backward()
    assert m.conv1.weight.grad.abs().sum() > 0 and torch.isfinite(m.flat_grads()).all()


@pytest.mark.parametrize("clip", [None, 0.05], ids=["plain", "max_grad_norm"])
def test_fused_sgd_matches_torch_sgd(clip):
    """dirb200_sgd_step (agedb-dir/train.py:164: SGD, momentum 0.9, weight decay 1e-4) over the flat buffers against
    torch.optim.SGD driven by the same gradients, 4 steps; with max_grad_norm also dirb200_grad_clip_coef against
    torch.nn.utils.clip_grad_norm_ (sts-b-dir/trainer.py:147-149)."""
    from optim import FusedSGD
    m = make_model(layers=(1, 1, 1, 1))
    m.train()
    params = list(m.parameters())
    opt = FusedSGD(params, lr=0.05, momentum=0.9, weight_decay=1e-4, max_grad_norm=clip)
    shadow = [p.detach().clone().requires_grad_(True) for p in params]
    ref_opt = torch.optim.SGD(shadow, lr=0.05, momentum=0.9, weight_decay=1e-4)
    g = torch.Generator(device=DEV).manual_seed(11)
    flat = m.flat_grads()
    for step in range(4):
        flat.copy_(torch.randn(flat.numel(), generator=g, device=DEV) * (1e-3 * (step + 1)))
        for s, p in zip(shadow, params):
            s.grad = p.grad.detach().clone()
        if clip:
            want_norm = torch.nn.utils.clip_grad_norm_(shadow, clip)
        opt.step()
        ref_opt.step()
        if clip:
            assert abs(float(opt.last_grad_norm()) - float(want_norm)) <= 1e-5 * float(want_norm)
        for s, p in zip(shadow, params):
            assert torch.allclose(s, p, rtol=2e-6, atol=1e-8), (step, (s - p).abs().max().item())


def test_fused_adam_with_grad_clip_matches_torch():
    from optim import FusedAdam
    m = make_model(layers=(1, 1, 1, 1))
    m.train()
    params = list(m.parameters())
    opt = FusedAdam(params, lr=1e-3, max_grad_norm=1.0)
    shadow = [p.detach().clone().requires_grad_(True) for p in params]
    ref_opt = torch.optim.Adam(shadow, lr=1e-3)
    g = torch.Generator(device=DEV).manual_seed(12)
    flat = m.flat_grads()
    for step in range(3):
        flat.copy_(torch.randn(flat.numel(), generator=g, device=DEV) * 0.01)
        for s, p in zip(shadow, params):
            s.grad = p.grad.detach().clone()
        torch.nn.utils.clip_grad_norm_(shadow, 1.0)
        opt.step()
        ref_opt.step()
        for s, p in zip(shadow, params):
            assert torch.allclose(s, p, rtol=1e-5, atol=1e-7)
