"""Plain-PyTorch fp32 restatement of the reference's basic-block ResNet (agedb-dir/resnet.py:14-38 BasicBlock, :73-153
ResNet) next to oracle/resnet_ref.py's bottleneck form, as pure functions over a state_dict -- TEST INFRASTRUCTURE ONLY.

It reuses resnet_ref's conv and bf16 storage points, so that the two forms round at the same places the native runner
stores bf16, and runs its train-mode BN through torch's batch_norm, as the reference does.  Tap names are
resnet_ref's: "{bi}.0" .. "{bi}.2" are conv1 raw / act and conv2 raw, "{bi}.5" the downsample and "{bi}.6" the block
output; a basic block has no "{bi}.3" (relu(bn2) is not stored) and no "{bi}.4".  block="bottleneck" hands over to
resnet_ref unchanged.  Pinned against the reference by tests/test_resnet_family_cpu.py (fixture
tests/golden/resnet_family.npz, made by tests/golden/make_golden_resnet_family.py).
"""
import torch
import torch.nn.functional as F

from oracle import resnet_ref as R
from oracle.resnet_ref import _conv, _q, _rb

DEPTHS = {18: ("basic", (2, 2, 2, 2)), 34: ("basic", (3, 4, 6, 3)), 50: ("bottleneck", (3, 4, 6, 3)),
          101: ("bottleneck", (3, 4, 23, 3)), 152: ("bottleneck", (3, 8, 36, 3))}


def expansion(block):
    return 1 if block == "basic" else 4


def param_shapes(layers=R.LAYERS, block="bottleneck"):
    """(name, shape) in the reference's named_parameters() order (without FDS)."""
    if block == "bottleneck":
        out = R.param_shapes(layers)
        return out[:-2] + [("linear.weight", (1, 512 * 4)), ("linear.bias", (1,))]
    assert block == "basic", block
    out = [("conv1.weight", (64, 3, 7, 7)), ("bn1.weight", (64,)), ("bn1.bias", (64,))]
    inplanes = 64
    for li, nblocks in enumerate(layers):
        planes = 64 << li
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            out += [(pre + "conv1.weight", (planes, inplanes, 3, 3)), (pre + "bn1.weight", (planes,)), (pre + "bn1.bias", (planes,)),
                    (pre + "conv2.weight", (planes, planes, 3, 3)), (pre + "bn2.weight", (planes,)), (pre + "bn2.bias", (planes,))]
            if b == 0 and (stride != 1 or inplanes != planes):
                out += [(pre + "downsample.0.weight", (planes, inplanes, 1, 1)),
                        (pre + "downsample.1.weight", (planes,)), (pre + "downsample.1.bias", (planes,))]
            inplanes = planes
    return out + [("linear.weight", (1, 512)), ("linear.bias", (1,))]


def _bn(x, p, pre, stats, quant):
    """Training-mode BatchNorm through torch's own batch_norm (batch statistics, biased variance, eps 1e-5): the
    reference's nn.BatchNorm2d arithmetic, so that no ReLU downstream flips on fp32 round-off against it; `stats`
    receives the running statistics one momentum-0.1 update from (0, 1) gives."""
    rm = torch.zeros(x.shape[1], dtype=x.dtype, device=x.device)
    rv = torch.ones_like(rm)
    y = F.batch_norm(x, rm, rv, p[pre + "weight"], p[pre + "bias"], training=True, momentum=0.1, eps=1e-5)
    if stats is not None:
        stats[pre + "running_mean"] = rm
        stats[pre + "running_var"] = rv
    return y


def forward_encoding(p, x, layers=R.LAYERS, stats=None, quant=False, taps=None, force=None, block="bottleneck",
                     outs=None):
    """x [B,3,H,W] -> encoding [B, 512 * expansion]; train-mode BN (resnet_ref.forward_encoding's contract).  `outs`
    (basic blocks): a list that receives the output of every layer group, with its autograd history (E_resnet)."""
    if block == "bottleneck":
        return R.forward_encoding(p, x, layers=layers, stats=stats, quant=quant, taps=taps, force=force)
    assert block == "basic", block

    def tap(name, t):
        if force is not None and name in force:
            t = t + (force[name] - t).detach()
        if taps is not None:
            taps[name] = t.detach()
        return t
    x = _q(x, quant)
    x = tap("stem.y", _conv(x, p["conv1.weight"], 2, 3, quant))
    x = tap("stem.a", _q(F.relu(_bn(x, p, "bn1.", stats, quant)), quant))
    x = tap("stem.pool", F.max_pool2d(_rb(x, quant), 3, 2, 1))
    bi = 0
    for li, nblocks in enumerate(layers):
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            idn = _rb(x, quant)
            o = tap(f"{bi}.0", _conv(x, p[pre + "conv1.weight"], stride, 1, quant))
            o = tap(f"{bi}.1", _q(F.relu(_bn(o, p, pre + "bn1.", stats, quant)), quant))
            o = tap(f"{bi}.2", _conv(o, p[pre + "conv2.weight"], 1, 1, quant))
            o = _bn(o, p, pre + "bn2.", stats, quant)
            if pre + "downsample.0.weight" in p:
                idn = tap(f"{bi}.5", _conv(x, p[pre + "downsample.0.weight"], stride, 0, quant))
                idn = _bn(idn, p, pre + "downsample.1.", stats, quant)
            x = tap(f"{bi}.6", _q(F.relu(o + idn), quant))
            bi += 1
        if outs is not None:
            outs.append(x)
    return _rb(x, quant).mean(dim=(2, 3))          # AvgPool2d over the last map + view


def forward(p, x, **kw):
    enc = forward_encoding(p, x, **kw)
    return enc @ p["linear.weight"].t() + p["linear.bias"], enc
