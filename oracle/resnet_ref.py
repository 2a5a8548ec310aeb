"""Plain-PyTorch fp32 restatement of the reference ResNet-50 regressor
(agedb-dir/resnet.py:41-70 Bottleneck, :73-153 ResNet) as pure functions over a
state_dict -- TEST INFRASTRUCTURE ONLY (the checker for the bf16 wgmma conv
stack; see oracle/dir_oracle.py for the rules).

Pinned against the reference itself by tests/test_oracle_golden.py::test_resnet_ref
(fixture tests/golden/resnet.npz, made by tests/golden/make_golden.py).
Written independently with torch.nn.functional; no reference code is imported.
"""
import torch
import torch.nn.functional as F

LAYERS = (3, 4, 6, 3)


def param_shapes(layers=LAYERS):
    """(name, shape) in the reference's named_parameters() order (without FDS)."""
    out = [("conv1.weight", (64, 3, 7, 7)), ("bn1.weight", (64,)), ("bn1.bias", (64,))]
    inplanes = 64
    for li, nblocks in enumerate(layers):
        planes = 64 << li
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            out += [(pre + "conv1.weight", (planes, inplanes, 1, 1)), (pre + "bn1.weight", (planes,)), (pre + "bn1.bias", (planes,)),
                    (pre + "conv2.weight", (planes, planes, 3, 3)), (pre + "bn2.weight", (planes,)), (pre + "bn2.bias", (planes,)),
                    (pre + "conv3.weight", (planes * 4, planes, 1, 1)), (pre + "bn3.weight", (planes * 4,)), (pre + "bn3.bias", (planes * 4,))]
            if b == 0 and (stride != 1 or inplanes != planes * 4):
                out += [(pre + "downsample.0.weight", (planes * 4, inplanes, 1, 1)),
                        (pre + "downsample.1.weight", (planes * 4,)), (pre + "downsample.1.bias", (planes * 4,))]
            inplanes = planes * 4
    out += [("linear.weight", (1, 2048)), ("linear.bias", (1,))]
    return out


def _bn(x, p, pre, stats, quant):
    # training-mode batch norm (batch statistics, biased variance, eps 1e-5)
    mean = x.mean(dim=(0, 2, 3))
    var = x.var(dim=(0, 2, 3), unbiased=False)
    if stats is not None:
        n = x.numel() / x.shape[1]
        stats[pre + "running_mean"] = 0.1 * mean.detach()
        stats[pre + "running_var"] = 0.9 + 0.1 * var.detach() * n / (n - 1)
    y = (x - mean[None, :, None, None]) * torch.rsqrt(var + 1e-5)[None, :, None, None]
    return y * p[pre + "weight"][None, :, None, None] + p[pre + "bias"][None, :, None, None]


def _q(x, quant):
    """bf16 round trip of a stored activation (what the native path keeps in HBM);
    straight-through in the backward."""
    if not quant:
        return x
    return x + (x.to(torch.bfloat16).float() - x).detach()


class _RoundBoth(torch.autograd.Function):
    """bf16 rounding of the value in the forward AND of the gradient in the
    backward: the points where the native path stores a gradient tensor as bf16
    (conv output grads dy, conv input grads from dgrad, the identity-branch dz,
    the avg-pool / max-pool input grads)."""

    @staticmethod
    def forward(ctx, x):
        return x.to(torch.bfloat16).float()

    @staticmethod
    def backward(ctx, g):
        return g.to(torch.bfloat16).float()


def _rb(x, quant):
    return _RoundBoth.apply(x) if quant else x


def _conv(x, w, stride, pad, quant):
    if quant:
        w = w + (w.to(torch.bfloat16).float() - w).detach()
    return _rb(F.conv2d(_rb(x, quant), w, stride=stride, padding=pad), quant)


def forward_encoding(p, x, layers=LAYERS, stats=None, quant=False, taps=None, force=None):
    """x [B,3,H,W] -> encoding [B,2048]; train-mode BN.  quant=True mimics the
    bf16 storage points of the native path (weights, conv outputs, activations)
    with straight-through rounding, so tolerances can be tight."""
    def tap(name, t):
        # `force`: teacher forcing -- substitute the value of a stored activation (keeping the gradient path), so
        # that a backward comparison is not polluted by forward round-off flips of ReLU masks
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
    inplanes = 64
    for li, nblocks in enumerate(layers):
        planes = 64 << li
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            idn = _rb(x, quant)
            o = tap(f"{bi}.0", _conv(x, p[pre + "conv1.weight"], 1, 0, quant))
            o = tap(f"{bi}.1", _q(F.relu(_bn(o, p, pre + "bn1.", stats, quant)), quant))
            o = tap(f"{bi}.2", _conv(o, p[pre + "conv2.weight"], stride, 1, quant))
            o = tap(f"{bi}.3", _q(F.relu(_bn(o, p, pre + "bn2.", stats, quant)), quant))
            o = tap(f"{bi}.4", _conv(o, p[pre + "conv3.weight"], 1, 0, quant))
            o = _bn(o, p, pre + "bn3.", stats, quant)
            if pre + "downsample.0.weight" in p:
                idn = tap(f"{bi}.5", _conv(x, p[pre + "downsample.0.weight"], stride, 0, quant))
                idn = _bn(idn, p, pre + "downsample.1.", stats, quant)
            x = tap(f"{bi}.6", _q(F.relu(o + idn), quant))
            bi += 1
            inplanes = planes * 4
    return _rb(x, quant).mean(dim=(2, 3))          # AvgPool2d(7) on the 7x7 map + view


def forward(p, x, **kw):
    enc = forward_encoding(p, x, **kw)
    return enc @ p["linear.weight"].t() + p["linear.bias"], enc
