"""GPU parity of NYUD2-DIR's multi-scale encoder (resnet.E_resnet, nyud2-dir/models/modules.py:33-58) on the native
ResNet-50 runner at sizes that are multiples of 4 but not of 32: the fixture size 36 x 44, the NYUD2 crop 228 x 304
(stage maps 114x152, 57x76, 29x38, 15x19, 8x10: an odd max-pool output, stride-2 convolutions on odd maps, the full
parity-class dgrad of the odd-map downsample) and 480 x 640.  The oracle is oracle/resnet_ref in quant mode (bf16
storage points), teacher-forced to the runner's stored activations, with the bounds of tests/test_gpu_resnet.py."""
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
torch.backends.cudnn.allow_tf32 = False           # the oracle's convolutions are true fp32
torch.backends.cuda.matmul.allow_tf32 = False
LAYERS = (3, 4, 6, 3)
LAST = (2, 6, 12, 15)                              # block index of the last block of layer1..4
SIZES = [(2, 36, 44), (2, 228, 304), (8, 228, 304), (2, 480, 640)]
SIZE_IDS = ["b2_36x44", "b2_228x304", "b8_228x304", "b2_480x640"]


def make_encoder():
    from resnet import E_resnet, resnet50
    torch.manual_seed(0)
    m = resnet50()
    with torch.no_grad():                       # non-trivial BN affine so its gradients are exercised
        for n, p in m.named_parameters():
            if p.dim() == 1 and ("bn" in n or "downsample.1" in n):
                p.copy_((1.0 if n.endswith("weight") else 0.0) + 0.1 * det_param(n, p.shape, 1.0))
    m = m.to(DEV)
    E = E_resnet(m)
    E.train()
    return m, E


def make_input(n, h, w):
    return det_param(f"x_enc{n}_{h}_{w}", (n, 3, h, w), 1.0).to(DEV)


def rel(a, b):
    return ((a.double() - b.double()).norm() / (b.double().norm() + 1e-12)).item()


def cos(a, b):
    return F.cosine_similarity(a.reshape(1, -1).double(), b.reshape(1, -1).double()).item()


def nchw(t):
    return t.permute(0, 3, 1, 2)


@pytest.mark.parametrize("n,h,w", SIZES, ids=SIZE_IDS)
def test_encoder_layerwise_forward_teacher_forced(n, h, w):
    """Every conv / BN+ReLU / residual stage against the oracle op on the runner's own input of that stage (relative
    L2 <= 4e-3, a bf16 ulp); the four returned tensors are the runner's block outputs bit for bit."""
    from oracle import resnet_ref as R
    m, E = make_encoder()
    p = {k: v.detach() for k, v in m.named_parameters()}
    x = make_input(n, h, w)
    with torch.no_grad():
        outs = E(x)
    shape = tuple(x.shape)
    pk = lambda b, k: m.peek(shape, b, k)
    q = lambda t: t.to(torch.bfloat16).float()
    chans = (256, 512, 1024, 2048)
    for s, bi in enumerate(LAST):
        assert outs[s].dtype == torch.bfloat16 and outs[s].shape[0] == n and outs[s].shape[3] == chans[s]
        assert torch.equal(nchw(outs[s]), m.peek(shape, bi, 6, copy=False)), s
    tol = 4e-3

    def check(name, got, ref):
        e = rel(got, ref)
        assert e <= tol, (name, e)

    with torch.no_grad():
        check("stem.y", pk(-1, 0), R._conv(q(x), p["conv1.weight"], 2, 3, True))
        check("stem.pool", pk(-1, 6), F.max_pool2d(q(F.relu(R._bn(pk(-1, 0), p, "bn1.", None, True))), 3, 2, 1))
        bi = 0
        for li, nblocks in enumerate(LAYERS):
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


def test_encoder_eval_forward_folded_bn_vs_oracle():
    """Inference at the reference's test shape (batch 1, 228 x 304; nyud2-dir/test.py): every folded conv + BN
    [+ ReLU] launch and block tail against fp32 torch ops on the runner's own input (4e-3), and the four outputs
    against torch's eval-mode network end to end."""
    m, E = make_encoder()
    with torch.no_grad():                       # two training forwards: non-trivial running statistics
        for k in range(2):
            E(make_input(2, 228, 304) * (1.0 + 0.5 * k))
    E.eval()
    sd = {k: v.detach().float() for k, v in E.state_dict().items()}
    x = make_input(1, 228, 304)
    with torch.no_grad():
        outs = E(x)
    shape = tuple(x.shape)
    pk = lambda b, k: m.peek(shape, b, k)
    q = lambda t: t.to(torch.bfloat16).float()

    def fold(pre):
        sc = sd[pre + "weight"] * torch.rsqrt(sd[pre + "running_var"] + 1e-5)
        return sc[None, :, None, None], (sd[pre + "bias"] - sd[pre + "running_mean"] * sc)[None, :, None, None]

    def conv(t, w, stride, pad):
        return F.conv2d(q(t), q(w), stride=stride, padding=pad)

    tol = 4e-3
    with torch.no_grad():
        for s, bi in enumerate(LAST):
            assert torch.equal(nchw(outs[s]), m.peek(shape, bi, 6, copy=False)), s
        sc, sh = fold("bn1.")
        assert rel(pk(-1, 6), F.max_pool2d(q(F.relu(pk(-1, 0) * sc + sh)), 3, 2, 1)) <= tol
        bi = 0
        for li, nblocks in enumerate(LAYERS):
            for b in range(nblocks):
                stride = 2 if (b == 0 and li > 0) else 1
                pre = f"layer{li + 1}.{b}."
                xin = pk(-1, 6) if bi == 0 else pk(bi - 1, 6)
                sc, sh = fold(pre + "bn1.")
                assert rel(pk(bi, 1), q(F.relu(conv(xin, sd[pre + "conv1.weight"], 1, 0) * sc + sh))) <= tol, pre
                sc, sh = fold(pre + "bn2.")
                assert rel(pk(bi, 3), q(F.relu(conv(pk(bi, 1), sd[pre + "conv2.weight"], stride, 1) * sc + sh))) <= tol, pre
                if pre + "downsample.0.weight" in sd:
                    sc, sh = fold(pre + "downsample.1.")
                    assert rel(pk(bi, 5), q(conv(xin, sd[pre + "downsample.0.weight"], stride, 0) * sc + sh)) <= tol, pre
                    idn = pk(bi, 5)
                else:
                    idn = xin
                sc, sh = fold(pre + "bn3.")
                y3 = conv(pk(bi, 3), sd[pre + "conv3.weight"], 1, 0)
                assert rel(pk(bi, 6), q(F.relu(q(y3 * sc + sh) + idn))) <= tol, pre
                bi += 1

        def bn(t, pre):
            s_, h_ = fold(pre)
            return t * s_ + h_
        t = F.max_pool2d(F.relu(bn(F.conv2d(x, sd["conv1.weight"], stride=2, padding=3), "bn1.")), 3, 2, 1)
        ref = []
        for li, nblocks in enumerate(LAYERS):
            for b in range(nblocks):
                stride = 2 if (b == 0 and li > 0) else 1
                pre = f"layer{li + 1}.{b}."
                o = F.relu(bn(F.conv2d(t, sd[pre + "conv1.weight"]), pre + "bn1."))
                o = F.relu(bn(F.conv2d(o, sd[pre + "conv2.weight"], stride=stride, padding=1), pre + "bn2."))
                o = bn(F.conv2d(o, sd[pre + "conv3.weight"]), pre + "bn3.")
                if pre + "downsample.0.weight" in sd:
                    t = bn(F.conv2d(t, sd[pre + "downsample.0.weight"], stride=stride), pre + "downsample.1.")
                t = F.relu(o + t)
            ref.append(t)
        # up to 53 bf16-stored layers end to end (every stage is pinned to 4e-3 above); unlike the pooled encoding of
        # the ResNet eval test, nothing averages the round-off out of a block output (layer4 measured 5.4e-2 / 0.9985
        # on an H100), so this is a sanity bound
        for s in range(4):
            got = nchw(outs[s]).float()
            assert rel(got, ref[s]) < 1e-1 and cos(got, ref[s]) > 0.995, (s, rel(got, ref[s]), cos(got, ref[s]))


def block_grads(outs, which, tag):
    """Seeded bf16 NHWC gradients for the outputs selected by `which` (None for the others)."""
    return [det_param(f"d{tag}_{s}", tuple(o.shape), 1.0).to(DEV).to(torch.bfloat16) if s in which else None
            for s, o in enumerate(outs)]


def oracle_backward(m, x, d, names=None):
    """Oracle parameter gradients of sum_s <x_block_s, d_s>, teacher-forced to the runner's stored activations."""
    from oracle import resnet_ref as R, encoder_ref as ER
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters() if not k.startswith("linear")}
    force = {"stem.y": m.peek(x.shape, -1, 0, copy=False), "stem.pool": m.peek(x.shape, -1, 6, copy=False)}
    for b in range(sum(LAYERS)):
        for k in range(7):
            try:
                force[f"{b}.{k}"] = m.peek(x.shape, b, k, copy=False)
            except Exception:
                pass                                   # blocks without a downsample branch
    assert len(force) == 2 + 6 * sum(LAYERS) + 4
    blocks = ER.forward_blocks(p, x, quant=True, force=force)
    loss = sum((b * nchw(g).float()).sum() for b, g in zip(blocks, d) if g is not None)
    loss.backward()
    return p


CASES = {"all": (0, 1, 2, 3), "x_block4": (3,), "x_block1": (0,)}


@pytest.mark.parametrize("case", list(CASES))
@pytest.mark.parametrize("n,h,w", SIZES, ids=SIZE_IDS)
def test_encoder_backward_vs_oracle_teacher_forced(n, h, w, case):
    """Seeded bf16 gradients on all four outputs, on x_block4 only and on x_block1 only: every parameter gradient
    against the teacher-forced oracle (flat rel < 3e-2, worst parameter rel < 0.15 with cos > 0.99).  Parameters that
    no gradient reaches keep their previous gradient values exactly."""
    from oracle import resnet_ref as R
    m, E = make_encoder()
    x = make_input(n, h, w)
    m._ensure_grads()
    before = det_param("g_before", (m.flat_grads().numel(),), 1e-3).to(DEV)
    m.flat_grads().copy_(before)
    outs = E(x)
    d = block_grads(outs, CASES[case], f"{n}_{h}_{w}")
    torch.autograd.backward([o for o, g in zip(outs, d) if g is not None], [g for g in d if g is not None])
    torch.cuda.synchronize()
    p = oracle_backward(m, x, d)
    named = dict(m.named_parameters())
    top = max(CASES[case]) + 1                       # deepest layer group a gradient reaches
    worst = ("", 1.0, 0.0)
    got_all, ref_all = [], []
    for name, _ in R.param_shapes():
        if name.startswith("linear"):
            continue
        g = named[name].grad - before[_offset(m, name):_offset(m, name) + named[name].numel()].view_as(named[name])
        group = int(name[5]) if name.startswith("layer") else 0
        if group > top:
            # no gradient reaches this group: its gradients are bit-identical to their previous values
            assert torch.equal(named[name].grad.reshape(-1),
                               before[_offset(m, name):_offset(m, name) + named[name].numel()]), name
            continue
        rg = p[name].grad
        c, e = cos(g, rg), rel(g, rg)
        if e > worst[2]:
            worst = (name, c, e)
        got_all.append(g.reshape(-1))
        ref_all.append(rg.reshape(-1))
        if name == "layer2.0.downsample.0.weight":
            # at 228 x 304 the layer2 downsample runs on the odd 57 x 76 map: the full parity-class dgrad, not the
            # compact one; its input gradient feeds layer1, whose gradients are checked here too
            assert c > 0.99 and e < 0.15, (name, c, e)
    print("worst parameter gradient:", worst)
    assert worst[2] < 0.15 and worst[1] > 0.99, worst
    flat, flat_ref = torch.cat(got_all), torch.cat(ref_all)
    assert rel(flat, flat_ref) < 3e-2, rel(flat, flat_ref)


def _offset(m, name):
    off = 0
    for k, v in m.named_parameters():
        if k == name:
            return off
        off += v.numel()
    raise KeyError(name)


def test_encoder_feeds_dense_ops_head():
    """E -> a dense_ops head (1x1 conv 2048 -> 64 + BN + ReLU on x_block4, bilinear up-sampling to x_block1's size,
    plus a 1x1 conv 256 -> 64 on x_block1), a weighted loss and .backward(): every E parameter gradient against the
    same head in fp32 torch on the teacher-forced oracle."""
    import dense_ops as D
    from oracle import resnet_ref as R, encoder_ref as ER
    m, E = make_encoder()
    x = make_input(2, 228, 304)
    wa = (det_param("head_wa", (64, 2048, 1, 1), (2.0 / 64) ** 0.5)).to(DEV).requires_grad_(True)
    wb = (det_param("head_wb", (64, 256, 1, 1), (2.0 / 64) ** 0.5)).to(DEV).requires_grad_(True)
    gamma = torch.ones(64, device=DEV, requires_grad=True)
    beta = torch.zeros(64, device=DEV, requires_grad=True)
    b1, _, _, b4 = E(x)
    lw = det_param("head_lw", (2, b1.shape[1], b1.shape[2], 64), 1.0).to(DEV)
    hb = D.upsample_bilinear(D.batch_norm_train(D.conv2d_nhwc(b4, wa), gamma, beta, relu=True), b1.shape[1:3])
    out = hb.float() + D.conv2d_nhwc(b1, wb).float()
    (out * lw).mean().backward()
    torch.cuda.synchronize()

    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters() if not k.startswith("linear")}
    force = {"stem.y": m.peek(x.shape, -1, 0, copy=False), "stem.pool": m.peek(x.shape, -1, 6, copy=False)}
    for bi in range(sum(LAYERS)):
        for k in range(7):
            try:
                force[f"{bi}.{k}"] = m.peek(x.shape, bi, k, copy=False)
            except Exception:
                pass
    r1, _, _, r4 = ER.forward_blocks(p, x, quant=True, force=force)
    t = F.relu(F.batch_norm(F.conv2d(r4, wa.detach()), None, None, gamma.detach(), beta.detach(), training=True))
    t = F.interpolate(t, size=tuple(r1.shape[2:]), mode="bilinear", align_corners=False)
    rout = t + F.conv2d(r1, wb.detach())
    (rout * nchw(lw)).mean().backward()
    named = dict(m.named_parameters())
    got, ref = [], []
    worst = ("", 1.0, 0.0)
    for name, _ in R.param_shapes():
        if name.startswith("linear"):
            continue
        g, rg = named[name].grad, p[name].grad
        c, e = cos(g, rg), rel(g, rg)
        if e > worst[2]:
            worst = (name, c, e)
        got.append(g.reshape(-1))
        ref.append(rg.reshape(-1))
    print("worst parameter gradient:", worst)
    # the head itself stores bf16 activations and gradients where the fp32 head does not: the same bounds as the
    # teacher-forced backward hold
    assert worst[2] < 0.15 and worst[1] > 0.99, worst
    assert rel(torch.cat(got), torch.cat(ref)) < 3e-2


def test_encoder_graph_replay_is_bit_identical():
    """Three identical training steps (eager, capture, replay of the forward and of every backward stage) give
    bit-identical outputs and parameter gradients; so does a second replay with only x_block1's gradient, against
    its own eager run."""
    m, E = make_encoder()
    x = make_input(2, 228, 304)

    def step(which):
        m.flat_grads().zero_()
        outs = E(x)
        d = block_grads(outs, which, "replay")
        torch.autograd.backward([o for o, g in zip(outs, d) if g is not None], [g for g in d if g is not None])
        torch.cuda.synchronize()
        return [o.detach().clone() for o in outs], m.flat_grads().clone()

    for which in ((0, 1, 2, 3), (0,)):
        runs = [step(which) for _ in range(3)]
        for outs, grads in runs[1:]:
            assert all(torch.equal(a, b) for a, b in zip(outs, runs[0][0]))
            assert torch.equal(grads, runs[0][1]), which


def test_encoder_and_regressor_backward_do_not_mix():
    """A multi-scale backward stage cannot continue a regressor backward (or the reverse): the runner refuses."""
    import _lib
    m, E = make_encoder()
    x = make_input(2, 36, 44)
    m._ensure_grads()
    outs = m._run_forward_blocks(x, training=True)
    net = m._net(tuple(x.shape))
    d4 = torch.zeros_like(outs[3])
    P = lambda t: _lib.ptr(t)
    _lib.call("dirb200_resnet_backward_blocks_stage", net, 4, P(d4), P(m.flat_parameters()), P(m.flat_grads()),
              _lib.stream_ptr())
    rc = _lib.raw("dirb200_resnet_backward_stage")(net, 3, None, P(m.flat_parameters()), P(m.flat_grads()),
                                                  _lib.stream_ptr())
    assert rc == -1 and "multi-scale" in _lib.last_error()
    torch.cuda.synchronize()


@pytest.mark.parametrize("env", [{"DIRB200_GRAPH": "0"}, {"DIRB200_SMS": "7"}], ids=["graph_off", "sms7"])
def test_encoder_file_under_runner_switch(env):
    """This file once more with eager launches, and with 7 SMs (few CTAs per conv / reduction), in a subprocess (the
    switches are read once per process)."""
    if os.environ.get("DIRB200_ENCODER_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_ENCODER_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not under_runner_switch"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
