"""The basic-block ResNets (resnet18 / resnet34) on the native runner, and one ResNet-101 step, on the GPU.

  * training forward in place, element by element, against float64 (the checks and bounds of
    test_gpu_runner_forward.py, with a basic block's conv2 as the tail conv that meets the shortcut): ResNet-18 at
    4 x 64^2 and 256 x 224^2, a (1, 1, 1, 1) basic net, ResNet-34 at 8 x 224^2;
  * the folded-BN eval forward, per element (test_gpu_runner_forward.check_affine);
  * the backward, teacher-forced against the float32 oracle (tests/resnet_family_ref.py), with the flat-gradient
    bounds of test_gpu_resnet.py;
  * every basic-block conv shape at batch 256 through test_gpu_conv.run_conv (fprop, dgrad, wgrad);
  * multi-scale mode: E_resnet(resnet18()) at 228 x 304 with gradients on all four / on one block output;
  * CUDA-graph replay bit-identical to DIRB200_GRAPH=0;
  * train.train() with FDS over a basic-block net (the FDS refresh order of test_gpu_train_loop.py, 512-d feature);
  * one ResNet-101 step, teacher-forced against the oracle (test_gpu_resnet.py's check at depth 101).
The whole file runs once more in a subprocess with DIRB200_SMS=7."""
import ctypes
import os
import subprocess
import sys

import pytest
import torch

import test_gpu_resnet as TR
import test_gpu_train_loop as TL
from oracle import dir_oracle as O
from test_gpu_conv import run_conv
from test_gpu_nyud2_encoder import block_grads, make_input, nchw
from test_gpu_runner_forward import (BF, WORST, block_input, check_act, check_affine, check_conv,
                                     check_encoding, check_pool, check_stats, coeffs, fma32, folded_eval, lib,
                                     peek_bf16, peek_u8, randomize_bn, raw_y, row_chunks, zbits)
from test_gpu_layer_kernels import unpack_mask
from test_gpu_runner_kernels import peek_conv
from util import det_param

import resnet_family_ref as RF

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def basic_table(layers, H, W):
    """Every conv of a basic-block runner in build order, in test_gpu_runner_kernels.conv_table's tuple form: (block,
    conv, weight name, BN prefix, cin, cout, k, stride, pad, input h, input w, stem); conv 0 / 1 / 3 = conv1 / conv2 /
    downsample."""
    out = [(-1, 0, "conv1.weight", "bn1.", 3, 64, 7, 2, 3, H, W, 1)]
    h, w = (H // 2 - 1) // 2 + 1, (W // 2 - 1) // 2 + 1
    inpl, bi = 64, 0
    for li, nb in enumerate(layers):
        pl = 64 << li
        for b in range(nb):
            s = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            ho, wo = (h - 1) // s + 1, (w - 1) // s + 1
            out += [(bi, 0, pre + "conv1.weight", pre + "bn1.", inpl, pl, 3, s, 1, h, w, 0),
                    (bi, 1, pre + "conv2.weight", pre + "bn2.", pl, pl, 3, 1, 1, ho, wo, 0)]
            if b == 0 and (s != 1 or inpl != pl):
                out.append((bi, 3, pre + "downsample.0.weight", pre + "downsample.1.", inpl, pl, 1, s, 0, h, w, 0))
            inpl, h, w, bi = pl, ho, wo, bi + 1
    return out


def make_basic(layers, fds=False, **kw):
    """ResNet(BasicBlock, layers) with test_gpu_resnet.make_model's seeded, non-trivial BN affine."""
    from resnet import ResNet, BasicBlock
    args = dict(fds=fds, bucket_num=100, bucket_start=3, start_update=0, start_smooth=1, kernel="gaussian", ks=9,
                sigma=1, momentum=0.9)
    args.update(kw)
    torch.manual_seed(0)
    m = ResNet(BasicBlock, list(layers), **args)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if p.dim() == 1 and ("bn" in n or "downsample.1" in n):
                p.copy_((1.0 if n.endswith("weight") else 0.0) + 0.1 * det_param(n, p.shape, 1.0))
    return m.to(DEV)


def by_block(table):
    d = {}
    for cv in table:
        d.setdefault(cv[0], {})[cv[1]] = cv
    return d


def check_basic_block_out(L, net, block, pk2, pkd, has_ds, with_mask, tag):
    """out = bf16(relu(fl32(y2 s2 + h2) + shortcut)) bit for bit (conv2 is the tail), and its mask bits = (out > 0)."""
    y2 = peek_bf16(L, net, block, 2)
    out = peek_bf16(L, net, block, 6)
    c = y2.shape[1]
    assert out.shape == y2.shape and c % 8 == 0
    s2, h2 = coeffs(pk2, c)
    if has_ds:
        yd = peek_bf16(L, net, block, 5)
        sd, hd = coeffs(pkd, c)
    else:
        xin = block_input(L, net, block)          # layer1.0 included: the max-pool output
        assert xin.shape == out.shape
    mask = peek_u8(L, net, block) if with_mask else None
    for q in row_chunks(out.shape[0], c):
        short = fma32(yd[q], sd, hd).double() if has_ds else xin[q].double()
        ref = torch.relu((fma32(y2[q], s2, h2).double() + short).float()).to(BF)
        bad = zbits(out[q]) != zbits(ref)
        assert not bad.any(), f"{tag} block {block} output: {int(bad.sum())} outputs differ"
        if with_mask:
            bad = unpack_mask(mask[q], c) != (out[q].float() > 0)
            assert not bad.any(), f"{tag} block {block} mask: {int(bad.sum())} bits differ"


def check_peek_refusals(L, net):
    """A basic block has no conv3 (peek 4, peek_conv 2) and does not materialise relu(bn2) (peek 3)."""
    ptr, rows, ch = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_int()
    assert L.raw("dirb200_resnet_peek")(net, 0, 4, ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch)) == -1
    assert "no conv3" in L.last_error(), L.last_error()
    assert L.raw("dirb200_resnet_peek")(net, 0, 3, ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch)) == -1
    assert "not materialised" in L.last_error(), L.last_error()
    from test_gpu_runner_kernels import ConvPeek
    pk = ConvPeek()
    assert L.raw("dirb200_resnet_peek_conv")(net, 0, 2, ctypes.byref(pk)) == -1
    assert "no conv3" in L.last_error(), L.last_error()


# ------------------------------------------------------------------------------------------------ forward in place
CASES = [((2, 2, 2, 2), 4, 64, 64), ((2, 2, 2, 2), 256, 224, 224), ((1, 1, 1, 1), 16, 64, 64), ((3, 4, 6, 3), 8, 224, 224)]
IDS = ["r18_b4_64", "r18_b256_224", "basic1111_b16_64", "r34_b8_224"]


def setup(layers, n, h, w):
    L = lib()
    torch.manual_seed(0)
    from resnet import ResNet, BasicBlock
    m = ResNet(BasicBlock, list(layers)).to(DEV).train()
    net = m._net((n, 3, h, w))
    assert L.raw("dirb200_resnet_feature_dim")(net) == 512
    return L, m, net, basic_table(layers, h, w)


@pytest.mark.parametrize("layers,n,h,w", CASES, ids=IDS)
def test_training_forward_in_place(layers, n, h, w):
    L, m, net, table = setup(layers, n, h, w)
    bufs = dict(m.named_buffers())
    g = torch.Generator(device=DEV).manual_seed(n + h + w + 3 * len(layers))
    blk = by_block(table)
    for it in range(3):                     # eager, graph capture, graph replay
        tag = f"forward {it + 1}"
        randomize_bn(m, table, g, running=(it == 0))
        x = torch.randn(n, 3, h, w, generator=g, device=DEV)
        rm0 = {cv[3]: bufs[cv[3] + "running_mean"].double().clone() for cv in table}
        rv0 = {cv[3]: bufs[cv[3] + "running_var"].double().clone() for cv in table}
        nbt0 = {cv[3]: int(bufs[cv[3] + "num_batches_tracked"]) for cv in table}
        enc = m._run_forward(x, training=True)
        torch.cuda.synchronize()
        assert enc.shape == (n, 512)
        for cv in table:
            pk = check_conv(L, net, x, cv, n, tag)
            check_stats(L, net, m, cv, pk, raw_y(L, net, cv), n, rm0[cv[3]], rv0[cv[3]], tag)
            assert int(bufs[cv[3] + "num_batches_tracked"]) == nbt0[cv[3]] + 1, cv[3]
            if cv[11]:
                check_pool(L, net, pk, n, h // 2, w // 2, tag)
            elif cv[1] == 0:
                check_act(L, net, cv[0], 0, pk, tag)
        for bi, convs in sorted(blk.items()):
            if bi >= 0:
                check_basic_block_out(L, net, bi, peek_conv(L, net, bi, 1),
                                      peek_conv(L, net, bi, 3) if 3 in convs else None, 3 in convs, True, tag)
        check_encoding(L, net, enc, n, sum(layers) - 1, tag)
    check_peek_refusals(L, net)
    print(f"\nbasic training forward {IDS[CASES.index((layers, n, h, w))]}: worst error / bound so far: " +
          ", ".join(f"{k} {v:.3f}" for k, v in WORST.items()))


@pytest.mark.parametrize("layers,n,h,w", CASES, ids=IDS)
def test_eval_forward_in_place(layers, n, h, w):
    L, m, net, table = setup(layers, n, h, w)
    g = torch.Generator(device=DEV).manual_seed(7 * n + h + w + 1)
    blk = by_block(table)
    m._run_forward(torch.randn(n, 3, h, w, generator=g, device=DEV), training=True)
    randomize_bn(m, table, g, running=True)
    x = torch.randn(n, 3, h, w, generator=g, device=DEV)
    enc = m._run_forward(x, training=False)
    torch.cuda.synchronize()
    tag = "eval folded" if folded_eval() else "eval unfolded"
    pk = check_conv(L, net, x, table[0], n, tag)
    check_pool(L, net, pk, n, h // 2, w // 2, tag)
    for bi, convs in sorted(blk.items()):
        if bi < 0:
            continue
        has_ds = 3 in convs
        if folded_eval():
            # conv1 -> BN -> ReLU, the downsample -> BN, and conv2 -> BN -> (+ shortcut) -> ReLU: one launch each
            check_affine(L, net, x, n, convs[0], None, peek_bf16(L, net, bi, 1), True, tag)
            if has_ds:
                check_affine(L, net, x, n, convs[3], None, peek_bf16(L, net, bi, 5), False, tag)
            short = peek_bf16(L, net, bi, 5) if has_ds else block_input(L, net, bi)
            check_affine(L, net, x, n, convs[1], short, peek_bf16(L, net, bi, 6), True, tag)
        else:
            pks = {c: check_conv(L, net, x, cv, n, tag) for c, cv in convs.items()}
            check_act(L, net, bi, 0, pks[0], tag)
            check_basic_block_out(L, net, bi, pks[1], pks.get(3), has_ds, False, tag)
    check_encoding(L, net, enc, n, sum(layers) - 1, tag)


# ------------------------------------------------------------------------------------------------ backward
def basic_force(m, x, layers):
    """The runner's stored activations under the oracle's tap names (conv1 raw / act, conv2 raw, downsample, output)."""
    force = {"stem.y": m.peek(x.shape, -1, 0, copy=False), "stem.pool": m.peek(x.shape, -1, 6, copy=False)}
    nds = 0
    for b in range(sum(layers)):
        for k in (0, 1, 2, 6):
            force[f"{b}.{k}"] = m.peek(x.shape, b, k, copy=False)
        try:
            force[f"{b}.5"] = m.peek(x.shape, b, 5, copy=False)
            nds += 1
        except Exception:
            pass                                   # identity blocks
    assert nds == 3, nds                           # layer2.0, layer3.0, layer4.0 (layer1.0 is an identity block)
    return force


@pytest.mark.parametrize("layers,n,hw", [((2, 2, 2, 2), 16, 64), ((1, 1, 1, 1), 16, 64), ((3, 4, 6, 3), 8, 224),
                                         ((2, 2, 2, 2), 256, 224)],
                         ids=["r18_b16_64", "basic1111_b16_64", "r34_b8_224", "r18_b256_224"])
def test_backward_vs_oracle_teacher_forced(layers, n, hw):
    """Every parameter gradient of a regressor step against the oracle teacher-forced to the runner's stored
    activations (test_gpu_resnet.test_backward_vs_oracle_teacher_forced's bounds: worst parameter rel < 0.15 with
    cos > 0.99, flat rel < 3e-2)."""
    import loss as L
    m = make_basic(layers)
    m.train()
    p = TR.oracle_params(m)
    x = det_param(f"x{n}", (min(n, 16), 3, hw, hw), 1.0).to(DEV)
    if n > 16:
        x = (x.repeat(n // 16, 1, 1, 1) * torch.linspace(0.5, 1.5, n, device=DEV).reshape(n, 1, 1, 1)).contiguous()
    t = (torch.arange(n, dtype=torch.float32, device=DEV).reshape(n, 1) * 5 + 10) % 101
    w = torch.linspace(0.5, 1.5, n, device=DEV).reshape(n, 1)
    pred = m(x, t, 0)
    L.weighted_l1_loss(pred, t, w).backward()
    force = basic_force(m, x, layers)
    rpred, _ = RF.forward(p, x, layers=layers, quant=True, force=force, block="basic")
    ((rpred - t).abs() * w).mean().backward()
    assert TR.rel(pred.detach(), rpred.detach()) < 2e-3
    named = dict(m.named_parameters())
    worst = ("", 1.0, 0.0)
    for name, rp in p.items():
        g, rg = named[name].grad, rp.grad
        c, e = TR.cos(g, rg), TR.rel(g, rg)
        if e > worst[2]:
            worst = (name, c, e)
    print("worst parameter gradient:", worst)
    assert worst[2] < 0.15 and worst[1] > 0.99, worst
    flat_ref = torch.cat([p[nm].grad.reshape(-1) for nm, _ in RF.param_shapes(layers, "basic")])
    assert TR.rel(m.flat_grads(), flat_ref) < 3e-2, TR.rel(m.flat_grads(), flat_ref)


def test_resnet101_step_teacher_forced():
    """Depth: one ResNet-101 step at 8 x 224^2, teacher-forced against the oracle with the same bounds."""
    TR.test_backward_vs_oracle_teacher_forced((3, 4, 23, 3), 8, 224)


# ------------------------------------------------------------------------------------------------ conv shapes
@pytest.mark.parametrize("cfg", [
    (56, 64, 64, 3, 1, 1), (56, 64, 128, 3, 2, 1), (56, 64, 128, 1, 2, 0), (28, 128, 128, 3, 1, 1),
    (28, 128, 256, 3, 2, 1), (28, 128, 256, 1, 2, 0), (14, 256, 256, 3, 1, 1), (14, 256, 512, 3, 2, 1),
    (14, 256, 512, 1, 2, 0), (7, 512, 512, 3, 1, 1)],
    ids=lambda c: "h{}_{}to{}_k{}s{}".format(*c[:5]))
def test_basic_block_conv_shapes_at_batch_256(cfg):
    h, ci, co, k, s, p = cfg
    run_conv(256, h, h, ci, co, k, s, p, seed=5, device_rng=True)


# ------------------------------------------------------------------------------------------------ multi-scale
@pytest.mark.parametrize("case", [(0, 1, 2, 3), (0,)], ids=["all", "x_block1"])
def test_encoder_resnet18_backward_vs_oracle(case):
    """E_resnet(resnet18()) at 2 x 228 x 304: the four block outputs (64 / 128 / 256 / 512 channels) equal the runner's
    stored block outputs, and with seeded gradients on all four / on x_block1 only every parameter gradient a gradient
    reaches agrees with the teacher-forced oracle; the others keep their previous values bit for bit."""
    from resnet import E_resnet
    layers = (2, 2, 2, 2)
    m = make_basic(layers)
    E = E_resnet(m)
    E.train()
    x = make_input(2, 228, 304)
    m._ensure_grads()
    before = det_param("g_before18", (m.flat_grads().numel(),), 1e-3).to(DEV)
    m.flat_grads().copy_(before)
    outs = E(x)
    assert [o.shape[-1] for o in outs] == [64, 128, 256, 512]
    for s, o in enumerate(outs):
        assert torch.equal(nchw(o), m.peek(x.shape, 2 * s + 1, 6, copy=False)), s
    d = block_grads(outs, case, "r18")
    torch.autograd.backward([o for o, g in zip(outs, d) if g is not None], [g for g in d if g is not None])
    torch.cuda.synchronize()
    p = {k: v.detach().clone().requires_grad_(True) for k, v in m.named_parameters() if not k.startswith("linear")}
    ro = []
    RF.forward_encoding(p, x, layers=layers, quant=True, force=basic_force(m, x, layers), block="basic", outs=ro)
    sum((b * nchw(g).float()).sum() for b, g in zip(ro, d) if g is not None).backward()
    top = max(case) + 1
    off, worst, got_all, ref_all = 0, ("", 1.0, 0.0), [], []
    for name, v in m.named_parameters():
        k = v.numel()
        if name.startswith("linear"):
            continue
        prev = before[off:off + k]
        group = int(name[5]) if name.startswith("layer") else 0
        if group > top:
            assert torch.equal(v.grad.reshape(-1), prev), name
        else:
            g, rg = v.grad.reshape(-1) - prev, p[name].grad.reshape(-1)
            c, e = TR.cos(g, rg), TR.rel(g, rg)
            if e > worst[2]:
                worst = (name, c, e)
            got_all.append(g)
            ref_all.append(rg)
        off += k
    print("worst parameter gradient:", worst)
    assert worst[2] < 0.15 and worst[1] > 0.99, worst
    assert TR.rel(torch.cat(got_all), torch.cat(ref_all)) < 3e-2


# ------------------------------------------------------------------------------------------------ graph replay
STEP = """
import sys, torch
sys.path[:0] = [{tests!r}, {root!r}, {pkg!r}]
from test_gpu_resnet_family import graph_step
torch.save(graph_step(4), sys.argv[1])
"""


def graph_step(steps):
    """`steps` identical training steps of a ResNet-18 regressor (batch 16, 112^2) with FDS smoothing: per step the
    prediction, the encoding, every parameter gradient and the BN running statistics."""
    import loss as L
    m = make_basic((2, 2, 2, 2), fds=True)
    m.train()
    x = det_param("x_graph", (16, 3, 112, 112), 1.0).to(DEV)
    t = torch.arange(16, dtype=torch.float32, device=DEV).reshape(16, 1) * 6 + 4
    w = torch.linspace(0.5, 1.5, 16, device=DEV).reshape(16, 1)
    out = []
    for _ in range(steps):
        m.flat_grads().zero_()
        running = m._flat["running"].clone()
        pred, enc = m(x, t, 0)
        L.weighted_l1_loss(pred, t, w).backward()
        torch.cuda.synchronize()
        out.append([pred.detach().cpu(), enc.detach().cpu(), m.flat_grads().cpu(), (m._flat["running"] - running).cpu()])
    return out


def test_graph_replay_matches_eager_launches(tmp_path):
    """Four steps in this process (eager, capture, two replays) are bit-identical, step by step, to the same four steps
    in a DIRB200_GRAPH=0 process (the running statistics move on from step to step, so step i meets step i)."""
    f = tmp_path / "eager.pt"
    code = STEP.format(tests=os.path.join(ROOT, "tests"), root=ROOT, pkg=os.path.join(ROOT, "imbalanced-regression_b200"))
    r = subprocess.run([sys.executable, "-c", code, str(f)], env=dict(os.environ, DIRB200_GRAPH="0"), cwd=ROOT,
                       capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    eager = torch.load(f)
    for i, (got, want) in enumerate(zip(graph_step(4), eager)):
        for k, (a, b) in enumerate(zip(got, want)):
            assert torch.equal(a, b), (i, k)


# ------------------------------------------------------------------------------------------------ train.train()
_TL_SETUP = TL._setup


def basic_setup(bucket_num, bucket_start, start_update, start_smooth, momentum=0.9, **kw):
    """test_gpu_train_loop._setup's arguments, data and loader, with its net, optimizer and oracle FDS replaced by a
    ResNet(BasicBlock, [1, 1, 1, 1]) of the same FDS settings and a 512-d oracle FDS."""
    from resnet import ResNet, BasicBlock
    from parallel import DataParallel
    from optim import FusedAdam
    train, args, _, _, loader, _, _ = _TL_SETUP(bucket_num, bucket_start, start_update, start_smooth,
                                                momentum=momentum, **kw)
    torch.manual_seed(0)
    net = ResNet(BasicBlock, [1, 1, 1, 1], fds=True, bucket_num=bucket_num, bucket_start=bucket_start,
                 start_update=start_update, start_smooth=start_smooth, kernel="gaussian", ks=5, sigma=2,
                 momentum=momentum).cuda()
    assert net.FDS.feature_dim == 512
    model = DataParallel(net)
    opt = FusedAdam([p for p in model.parameters()], lr=args.lr)
    ref = O.FDSState(512, bucket_num, bucket_start, start_update=start_update, start_smooth=start_smooth,
                     kernel="gaussian", ks=5, sigma=2, momentum=momentum)
    return train, args, net, model, loader, opt, ref


def test_train_loop_fds_refresh_basic_block(monkeypatch):
    """Three epochs of train.train() with FDS + LDS on a basic-block net: the collection features and all FDS buffers
    against the oracle in the reference's refresh order (test_gpu_train_loop's check, 512-d feature)."""
    monkeypatch.setattr(TL, "_setup", basic_setup)
    TL.test_train_loop_fds_refresh_matches_reference_order((100, 3, 0, 1))


# ------------------------------------------------------------------------------------------------ rerun
def test_whole_file_rerun_sms7():
    """This file again in a fresh process with the grids capped at 7 SMs (the switch is read once per process)."""
    if os.environ.get("DIRB200_SMS"):
        pytest.skip("already a rerun")
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-x", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not rerun"], env=dict(os.environ, DIRB200_SMS="7"), cwd=ROOT, capture_output=True,
                       text=True, timeout=3000)
    assert r.returncode == 0, r.stdout[-5000:] + r.stderr[-2000:]
