"""resnet.py -- drop-in mirror of agedb-dir/resnet.py (= imdb-wiki-dir/resnet.py).

`resnet50(fds=..., bucket_num=..., ...)` returns a module with the reference's
attribute tree (conv1, bn1, layer1..4.{i}.{conv,bn}{1-3}, downsample.{0,1},
linear, FDS), hence the reference's state_dict keys and shapes, the same
`forward(x, targets=None, epoch=None)` contract (resnet.py:127-153) and the
same initialisation (resnet.py:103-109).  `resnet18` / `resnet34` build the
same over `BasicBlock` (resnet.py:14-38; conv1 / conv2 3x3, 512-d feature),
`resnet101` / `resnet152` over deeper `Bottleneck` stacks
(nyud2-dir/models/resnet.py:153-205).

`E_resnet(resnet50())` is NYUD2-DIR's multi-scale encoder
(nyud2-dir/models/modules.py:33-58): the same backbone without avgpool / fc,
returning the four layer-group outputs as NHWC bf16 tensors.

The arithmetic does not go through torch.nn: the conv/BN/ReLU/pool stack runs
in libdirb200's native runner (wgmma implicit-GEMM convolutions + fused
HBM-bound layers, NHWC bf16 with fp32 accumulation), the 2048->1 regressor
and FDS.smooth in their own kernels.  All parameters are views into ONE flat
fp32 buffer (and their .grad into one flat gradient buffer), which is what the
runner, the fused optimizer (optim.py) and the gradient all-reduce consume.
"""
import ctypes
import logging
import math
from ctypes import c_int, c_int64, c_void_p, c_float

import torch
import torch.nn as nn

import _lib
import _convlib  # noqa: F401  (registers conv entry points)
from fds import FDS

print = logging.info

P = c_void_p
_lib.register({
    "dirb200_resnet_create": (c_int, [c_int, c_int, c_int, P, c_int, P]),
    "dirb200_resnet_create_ex": (c_int, [c_int, c_int, c_int, c_int, P, c_int, P]),
    "dirb200_resnet_destroy": (None, [P]),
    "dirb200_resnet_param_count": (c_int64, [P]),
    "dirb200_resnet_running_count": (c_int64, [P]),
    "dirb200_resnet_feature_dim": (c_int64, [P]),
    "dirb200_resnet_device_bytes": (c_int64, [P]),
    "dirb200_resnet_forward": (c_int, [P, P, P, P, c_int, P, P]),
    "dirb200_resnet_backward": (c_int, [P, P, P, P, P]),
    "dirb200_resnet_num_stages": (c_int, [P]),
    "dirb200_resnet_backward_stage": (c_int, [P, c_int, P, P, P, P]),
    "dirb200_resnet_stage_param_range": (c_int, [P, c_int, P, P]),
    "dirb200_resnet_set_profiling": (c_int, [P, c_int]),
    "dirb200_resnet_read_profile": (c_int, [P, P, P]),
    "dirb200_resnet_peek": (c_int, [P, c_int, c_int, P, P, P]),
    "dirb200_resnet_peek_conv": (c_int, [P, c_int, c_int, P]),
    "dirb200_resnet_peek_bn_stats": (c_int, [P, c_int, c_int, P, P]),
    "dirb200_resnet_peek_bn_coef": (c_int, [P, c_int, c_int, P]),
    "dirb200_resnet_set_backward_tap": (c_int, [P, c_int]),
    "dirb200_resnet_peek_backward": (c_int, [P, c_int, P, P, P]),
    "dirb200_resnet_forward_blocks": (c_int, [P, P, P, P, c_int, P, P]),
    "dirb200_resnet_backward_blocks_stage": (c_int, [P, c_int, P, P, P, P]),
    "dirb200_linear1_fwd": (c_int, [P, P, P, c_int64, c_int, P, P]),
    "dirb200_linear1_bwd": (c_int, [P, P, P, c_int64, c_int, P, P, P, P]),
    "dirb200_adam_step": (c_int, [P, P, P, P, c_int64, c_float, c_float, c_float, c_float, c_float, c_int64,
                                  c_float, P, P]),
    "dirb200_adam_step_multi": (c_int, [P, c_int, c_float, c_float, c_float, c_float, c_float, P]),
    "dirb200_sgd_step": (c_int, [P, P, P, c_int64, c_float, c_float, c_float, c_int, c_float, P, P]),
    "dirb200_grad_clip_workspace_bytes": (ctypes.c_size_t, []),
    "dirb200_grad_clip_coef": (c_int, [P, c_int64, c_float, c_float, P, ctypes.c_size_t, P, P]),
    "dirb200_adam_step_multi_clipped": (c_int, [P, c_int, c_float, c_float, c_float, c_float, c_float, P, P]),
    "dirb200_grad_norm_multi_workspace_bytes": (ctypes.c_size_t, []),
    "dirb200_grad_norm_multi": (c_int, [P, c_int, c_float, P, ctypes.c_size_t, P, P]),
})


# ------------------------------------------------------------------ holders
class _Conv(nn.Module):
    """Parameter holder with nn.Conv2d's attribute names (weight only, bias=False)."""

    def __init__(self, cin, cout, k, stride, padding):
        super().__init__()
        self.in_channels, self.out_channels = cin, cout
        self.kernel_size, self.stride, self.padding = (k, k), (stride, stride), (padding, padding)
        self.weight = nn.Parameter(torch.empty(cout, cin, k, k))


class _BN(nn.Module):
    """Parameter / buffer holder with nn.BatchNorm2d's names."""

    def __init__(self, c):
        super().__init__()
        self.num_features = c
        self.weight = nn.Parameter(torch.empty(c))
        self.bias = nn.Parameter(torch.empty(c))
        self.register_buffer('running_mean', torch.zeros(c))
        self.register_buffer('running_var', torch.ones(c))
        self.register_buffer('num_batches_tracked', torch.tensor(0, dtype=torch.long))


class _Linear(nn.Module):
    def __init__(self, cin, cout):
        super().__init__()
        assert cout == 1
        self.in_features, self.out_features = cin, cout
        self.weight = nn.Parameter(torch.empty(cout, cin))
        self.bias = nn.Parameter(torch.empty(cout))
        bound = 1 / math.sqrt(cin)                      # nn.Linear's default init
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        nn.init.uniform_(self.bias, -bound, bound)

    def forward(self, x):
        return _Linear1Fn.apply(x, self.weight, self.bias)


class BasicBlock(nn.Module):
    expansion = 1
    kind = 1              # DIRB200_RESNET_BASIC

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super(BasicBlock, self).__init__()
        self.conv1 = _Conv(inplanes, planes, 3, stride, 1)
        self.bn1 = _BN(planes)
        self.conv2 = _Conv(planes, planes, 3, 1, 1)
        self.bn2 = _BN(planes)
        self.downsample = downsample
        self.stride = stride


class Bottleneck(nn.Module):
    expansion = 4
    kind = 0              # DIRB200_RESNET_BOTTLENECK

    def __init__(self, inplanes, planes, stride=1, downsample=None):
        super(Bottleneck, self).__init__()
        self.conv1 = _Conv(inplanes, planes, 1, 1, 0)
        self.bn1 = _BN(planes)
        self.conv2 = _Conv(planes, planes, 3, stride, 1)
        self.bn2 = _BN(planes)
        self.conv3 = _Conv(planes, planes * 4, 1, 1, 0)
        self.bn3 = _BN(planes * 4)
        self.downsample = downsample
        self.stride = stride


# ------------------------------------------------------------ autograd glue
class _Linear1Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        _lib.require_cuda(x, weight, bias)
        x = x.contiguous()
        n, d = x.shape
        pred = torch.empty(n, 1, dtype=torch.float32, device=x.device)
        _lib.call("dirb200_linear1_fwd", _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), n, d, _lib.ptr(pred),
                  _lib.stream_ptr())
        ctx.save_for_backward(x, weight)
        return pred

    @staticmethod
    def backward(ctx, g):
        x, weight = ctx.saved_tensors
        g = g.contiguous()
        n, d = x.shape
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        dw = torch.empty_like(weight)
        db = torch.empty(1, dtype=torch.float32, device=x.device)
        _lib.call("dirb200_linear1_bwd", _lib.ptr(g), _lib.ptr(x), _lib.ptr(weight), n, d, _lib.ptr(dx),
                  _lib.ptr(dw), _lib.ptr(db), _lib.stream_ptr())
        return dx, dw, db


class _BackboneFn(torch.autograd.Function):
    """x -> encoding through the native runner; the backward accumulates the
    parameter gradients straight into the flat gradient buffer."""

    @staticmethod
    def forward(ctx, x, anchor, model):
        ctx.model = model
        ctx.shape = tuple(x.shape)
        return model._run_forward(x, training=True)

    @staticmethod
    def backward(ctx, g):
        ctx.model._run_backward(ctx.shape, g)
        return None, None, None


class _EncoderFn(torch.autograd.Function):
    """x -> the four layer-group outputs through the native runner; the backward takes a gradient for any subset of
    them (an unused output costs nothing) and accumulates the parameter gradients into the flat gradient buffer."""

    @staticmethod
    def forward(ctx, x, anchor, model):
        ctx.set_materialize_grads(False)
        ctx.model = model
        ctx.shape = tuple(x.shape)
        return model._run_forward_blocks(x, training=True)

    @staticmethod
    def backward(ctx, *grads):
        ctx.model._run_backward(ctx.shape, grads, blocks=True)
        return None, None, None


def _feature_maps(h, w, num_stages=4):
    """(h, w) of the stem output, the max-pool output and the output of layer groups 2..num_stages for an h x w input
    (layer1 keeps the max-pool map)."""
    half = lambda a: (a - 1) // 2 + 1          # 3x3 / pad 1 and 1x1 / pad 0 filters at stride 2
    maps = [(h // 2, w // 2)]
    maps.append((half(maps[0][0]), half(maps[0][1])))
    for _ in range(num_stages - 1):
        maps.append((half(maps[-1][0]), half(maps[-1][1])))
    return maps


class ResNet(nn.Module):

    # FDS defaults as fds.FDS's, for constructions that do not use FDS (E_resnet(resnet50()))
    def __init__(self, block, layers, fds=False, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1,
                 kernel='gaussian', ks=5, sigma=2, momentum=0.9, dropout=None):
        self.inplanes = 64
        super(ResNet, self).__init__()
        assert block in (BasicBlock, Bottleneck), "the native runner implements BasicBlock and Bottleneck ResNets"
        self._block = block
        self._layers = list(layers)
        self.conv1 = _Conv(3, 64, 7, 2, 3)
        self.bn1 = _BN(64)
        self.layer1 = self._make_layer(block, 64, layers[0])
        self.layer2 = self._make_layer(block, 128, layers[1], stride=2)
        self.layer3 = self._make_layer(block, 256, layers[2], stride=2)
        self.layer4 = self._make_layer(block, 512, layers[3], stride=2)
        self.linear = _Linear(512 * block.expansion, 1)

        if fds:
            self.FDS = FDS(
                feature_dim=512 * block.expansion, bucket_num=bucket_num, bucket_start=bucket_start,
                start_update=start_update, start_smooth=start_smooth, kernel=kernel, ks=ks, sigma=sigma,
                momentum=momentum
            )
        self.fds = fds
        self.start_smooth = start_smooth

        self.use_dropout = True if dropout else False
        if self.use_dropout:
            print(f'Using dropout: {dropout}')
            self.dropout = nn.Dropout(p=dropout)

        for m in self.modules():                      # resnet.py:103-109
            if isinstance(m, _Conv):
                n = m.kernel_size[0] * m.kernel_size[1] * m.out_channels
                m.weight.data.normal_(0, math.sqrt(2. / n))
            elif isinstance(m, _BN):
                m.weight.data.fill_(1)
                m.bias.data.zero_()

        self._nets = {}
        self._grad_bucket_hook = None          # callable(lo, hi) on the flat gradient, see _run_backward
        self._anchor = torch.zeros(1, requires_grad=True)
        self._flat = None
        self._flatten()

    def _make_layer(self, block, planes, blocks, stride=1):
        downsample = None
        if stride != 1 or self.inplanes != planes * block.expansion:
            downsample = nn.Sequential(_Conv(self.inplanes, planes * block.expansion, 1, stride, 0),
                                       _BN(planes * block.expansion))
        layers = [block(self.inplanes, planes, stride, downsample)]
        self.inplanes = planes * block.expansion
        for _ in range(1, blocks):
            layers.append(block(self.inplanes, planes))
        return nn.Sequential(*layers)

    # ----------------------------------------------------------- flat storage
    def _backbone_modules(self):
        """conv/bn holders in the runner's (= named_parameters) order."""
        mods = [self.conv1, self.bn1]
        for layer in (self.layer1, self.layer2, self.layer3, self.layer4):
            for blk in layer:
                mods += [blk.conv1, blk.bn1, blk.conv2, blk.bn2]
                if isinstance(blk, Bottleneck):
                    mods += [blk.conv3, blk.bn3]
                if blk.downsample is not None:
                    mods += [blk.downsample[0], blk.downsample[1]]
        return mods

    def _flat_param_list(self):
        ps = []
        for m in self._backbone_modules():
            ps.append(m.weight)
            if isinstance(m, _BN):
                ps.append(m.bias)
        return ps + [self.linear.weight, self.linear.bias]

    def _flatten(self):
        """(Re)build the flat parameter / BN-statistics buffers on the parameters'
        current device and re-point every Parameter / buffer at a view of them."""
        ps = self._flat_param_list()
        dev = ps[0].device
        total = sum(p.numel() for p in ps)
        flat = torch.empty(total, dtype=torch.float32, device=dev)
        off = 0
        for p in ps:
            n = p.numel()
            flat[off:off + n].copy_(p.data.reshape(-1))
            p.data = flat[off:off + n].view(p.shape)
            off += n
        bns = [m for m in self._backbone_modules() if isinstance(m, _BN)]
        running = torch.empty(sum(2 * b.num_features for b in bns), dtype=torch.float32, device=dev)
        nbt = torch.empty(len(bns), dtype=torch.long, device=dev)
        off = 0
        for i, b in enumerate(bns):
            c = b.num_features
            running[off:off + c].copy_(b.running_mean)
            running[off + c:off + 2 * c].copy_(b.running_var)
            b.running_mean = running[off:off + c]
            b.running_var = running[off + c:off + 2 * c]
            nbt[i] = b.num_batches_tracked
            b.num_batches_tracked = nbt[i]
            off += 2 * c
        self._flat = dict(params=flat, running=running, nbt=nbt, grads=None, backbone=total - self.linear.weight.numel() - 1)
        self._anchor = torch.zeros(1, requires_grad=True, device=dev)
        self._grad_views = None

    def _apply(self, fn, *args, **kwargs):
        out = super()._apply(fn, *args, **kwargs)
        if self._flat is not None:
            self._free_nets()
            self._flatten()
        return out

    def flat_parameters(self):
        return self._flat["params"]

    def flat_grads(self):
        self._ensure_grads()
        return self._flat["grads"]

    def _ensure_grads(self):
        ps = self._flat_param_list()
        f = self._flat
        if f["grads"] is None or f["grads"].device != f["params"].device:
            f["grads"] = torch.zeros_like(f["params"])
            views, off = [], 0
            for p in ps:
                views.append(f["grads"][off:off + p.numel()].view(p.shape))
                off += p.numel()
            self._grad_views = views
        if all(p.grad is None for p in ps):
            f["grads"].zero_()
            for p, v in zip(ps, self._grad_views):
                p.grad = v
            return
        for p, v in zip(ps, self._grad_views):
            if p.grad is None:
                v.zero_()
                p.grad = v
            elif p.grad.data_ptr() != v.data_ptr():
                v.copy_(p.grad)
                p.grad = v

    # ------------------------------------------------------------ native nets
    MAX_NETS = 4      # distinct input shapes kept alive (train batch, train tail, val/test batch, val/test tail)

    def _net(self, shape):
        """Native runner for input `shape` (created on first use).  The cache is LRU: a new shape evicts only the
        least recently used runner -- a normal epoch alternates between four shapes and must not rebuild any."""
        net = self._nets.pop(shape, None)
        if net is None:
            while len(self._nets) >= self.MAX_NETS:
                _, old = next(iter(self._nets.items()))
                self._nets.pop(next(iter(self._nets)))
                _lib.raw("dirb200_resnet_destroy")(old)
            n, c, h, w = shape
            assert c == 3, "expected NCHW input with 3 channels"
            handle = c_void_p()
            arr = (c_int * 4)(*self._layers)
            _lib.call("dirb200_resnet_create_ex", n, h, w, self._block.kind, arr, 4, ctypes.byref(handle))
            assert _lib.raw("dirb200_resnet_param_count")(handle) == self._flat["backbone"], "parameter layout mismatch"
            assert _lib.raw("dirb200_resnet_running_count")(handle) == self._flat["running"].numel()
            net = handle
        self._nets[shape] = net          # most recently used last
        return net

    def _free_nets(self):
        for h in self._nets.values():
            _lib.raw("dirb200_resnet_destroy")(h)
        self._nets = {}

    def __del__(self):
        try:
            self._free_nets()
        except Exception:
            pass

    def _run_forward(self, x, training):
        _lib.require_cuda(x, self._flat["params"])
        x = x.detach().to(torch.float32).contiguous()
        net = self._net(tuple(x.shape))
        enc = torch.empty(x.shape[0], 512 * self._block.expansion, dtype=torch.float32, device=x.device)
        _lib.call("dirb200_resnet_forward", net, _lib.ptr(x), _lib.ptr(self._flat["params"]),
                  _lib.ptr(self._flat["running"]), int(training), _lib.ptr(enc), _lib.stream_ptr())
        if training:
            self._flat["nbt"] += 1
        return enc

    def _run_forward_blocks(self, x, training):
        """x fp32 NCHW [n, 3, h, w] -> the outputs of layer1..4, NHWC bf16 [n, h_s, w_s, (64 << s) * expansion]."""
        _lib.require_cuda(x, self._flat["params"])
        x = x.detach().to(torch.float32).contiguous()
        n, _, h, w = x.shape
        net = self._net(tuple(x.shape))
        maps = _feature_maps(h, w, len(self._layers))[1:]
        outs = [torch.empty(n, hs, ws, 64 * self._block.expansion << s, dtype=torch.bfloat16, device=x.device)
                for s, (hs, ws) in enumerate(maps)]
        ptrs = (c_void_p * len(outs))(*[o.data_ptr() for o in outs])
        _lib.call("dirb200_resnet_forward_blocks", net, _lib.ptr(x), _lib.ptr(self._flat["params"]),
                  _lib.ptr(self._flat["running"]), int(training), ptrs, _lib.stream_ptr())
        if training:
            self._flat["nbt"] += 1
        return tuple(outs)

    def _run_backward(self, shape, g, blocks=False):
        """g: the encoding's gradient, or (blocks=True) one gradient (or None) per layer-group output."""
        if shape not in self._nets:
            raise _lib.Dirb200Error(f"backward for input shape {shape}: its runner (and the activations of the forward "
                                    "pass) was evicted -- more than MAX_NETS shapes ran between forward and backward")
        self._ensure_grads()
        if blocks:
            g = [None if t is None else t.detach().to(torch.bfloat16).contiguous() for t in g]
        else:
            g = g.detach().to(torch.float32).contiguous()
        net = self._net(shape)
        hook = self._grad_bucket_hook
        if hook is None and not blocks:
            _lib.call("dirb200_resnet_backward", net, _lib.ptr(g), _lib.ptr(self._flat["params"]),
                      _lib.ptr(self._flat["grads"]), _lib.stream_ptr())
            return
        # stage by stage (layer4 ... layer1, stem); after each layer group its slice of the flat gradient is final and
        # is handed to the hook (parallel.DataParallel: an asynchronous NCCL all-reduce that overlaps the rest)
        for stage in range(_lib.raw("dirb200_resnet_num_stages")(net), -1, -1):
            if blocks:
                _lib.call("dirb200_resnet_backward_blocks_stage", net, stage, _lib.ptr(g[stage - 1] if stage else None),
                          _lib.ptr(self._flat["params"]), _lib.ptr(self._flat["grads"]), _lib.stream_ptr())
            else:
                _lib.call("dirb200_resnet_backward_stage", net, stage, _lib.ptr(g), _lib.ptr(self._flat["params"]),
                          _lib.ptr(self._flat["grads"]), _lib.stream_ptr())
            if stage >= 1 and hook is not None:
                lo, hi = c_int64(), c_int64()
                _lib.call("dirb200_resnet_stage_param_range", net, stage, ctypes.byref(lo), ctypes.byref(hi))
                hook(lo.value, hi.value)

    PROFILE_KINDS = ("prep", "conv_fprop", "conv_dgrad", "conv_wgrad", "wgrad_reduce", "bn_stats", "bn_apply",
                     "bn_bwd_reduce", "bn_bwd_apply", "pool")

    def set_profiling(self, shape, enabled):
        _lib.call("dirb200_resnet_set_profiling", self._net(tuple(shape)), int(enabled))

    def read_profile(self, shape):
        """{kernel class: (milliseconds, launch groups)} recorded since the last read (synchronises)."""
        from ctypes import c_double
        ms = (c_double * 10)()
        cnt = (c_int64 * 10)()
        _lib.call("dirb200_resnet_read_profile", self._net(tuple(shape)), ms, cnt)
        return {k: (ms[i], cnt[i]) for i, k in enumerate(self.PROFILE_KINDS)}

    def peek(self, shape, block, which, copy=True):
        """Test aid: an internal NHWC bf16 activation of the runner for input `shape`, as an fp32 NCHW copy
        (copy=False: a zero-copy bf16 view with NCHW shape / channels-last strides, valid until the next forward)."""
        ptr, rows, ch = c_void_p(), c_int64(), c_int()
        _lib.call("dirb200_resnet_peek", self._net(tuple(shape)), block, which, ctypes.byref(ptr), ctypes.byref(rows),
                  ctypes.byref(ch))

        class _Arr:
            __cuda_array_interface__ = dict(shape=(rows.value * ch.value,), typestr="<u2", data=(ptr.value, False),
                                            version=2)
        flat = torch.as_tensor(_Arr(), device=self._flat["params"].device).view(torch.bfloat16)
        n = shape[0]
        # the net's maps have strictly decreasing pixel counts: the count identifies the map
        h, w = next(m for m in _feature_maps(shape[2], shape[3], len(self._layers)) if m[0] * m[1] * n == rows.value)
        if not copy:
            return flat.view(n, h, w, ch.value).permute(0, 3, 1, 2)
        return flat.float().view(n, h, w, ch.value).permute(0, 3, 1, 2).contiguous()

    # ---------------------------------------------------------------- forward
    def forward(self, x, targets=None, epoch=None):
        if self.training and torch.is_grad_enabled():
            # every .grad must be its view of the flat gradient buffer BEFORE autograd accumulates into it (the fused
            # optimizers and the all-reduce work on the flat buffer); with a frozen backbone (--retrain_fc) the
            # runner's backward, which used to attach them, never runs
            lw = self.linear.weight
            if self._grad_views is None or lw.grad is None or lw.grad.data_ptr() != self._grad_views[-2].data_ptr():
                self._ensure_grads()
        need_bwd = self.training and torch.is_grad_enabled() and \
            any(p.requires_grad for p in self._flat_param_list()[:-2])
        if need_bwd:
            encoding = _BackboneFn.apply(x, self._anchor, self)
        else:
            encoding = self._run_forward(x, training=self.training)

        encoding_s = encoding

        if self.training and self.fds:
            if epoch >= self.start_smooth:
                encoding_s = self.FDS.smooth(encoding_s, targets, epoch)   # in place, as the reference

        if self.use_dropout:
            encoding_s = self.dropout(encoding_s)
        x = self.linear(encoding_s)

        if self.training and self.fds:
            return x, encoding
        else:
            return x


def resnet18(**kwargs):
    return ResNet(BasicBlock, [2, 2, 2, 2], **kwargs)


def resnet34(**kwargs):
    return ResNet(BasicBlock, [3, 4, 6, 3], **kwargs)


def resnet50(**kwargs):
    return ResNet(Bottleneck, [3, 4, 6, 3], **kwargs)


def resnet101(**kwargs):
    return ResNet(Bottleneck, [3, 4, 23, 3], **kwargs)


def resnet152(**kwargs):
    return ResNet(Bottleneck, [3, 8, 36, 3], **kwargs)


class E_resnet(nn.Module):
    """NYUD2-DIR's encoder (nyud2-dir/models/modules.py:33-58): `original_model`'s stem and layer1..4 without avgpool /
    linear.  It shares the native ResNet's holders, flat parameter / gradient / running-statistics buffers and runner
    cache, so its state_dict has the reference E_resnet's keys and loads a torchvision-layout checkpoint of the same
    depth (resnet18 ... resnet152).

    forward(x): x fp32 NCHW [B, 3, H, W] (H, W multiples of 4) -> (x_block1, x_block2, x_block3, x_block4), NHWC bf16
    [B, h_s, w_s, C_s] with C_s = 256, 512, 1024, 2048 over Bottleneck (resnet50 / 101 / 152) and 64, 128, 256, 512 over
    BasicBlock (resnet18 / 34) (the layout dense_ops consumes).  In training mode with
    gradients enabled they carry autograd history into the backbone parameters; x receives no gradient."""

    def __init__(self, original_model, num_features=2048):
        super(E_resnet, self).__init__()
        assert isinstance(original_model, ResNet), "E_resnet wraps the native resnet.ResNet"
        object.__setattr__(self, "_resnet", original_model)      # not a submodule: no linear / FDS keys
        self.conv1 = original_model.conv1
        self.bn1 = original_model.bn1
        self.layer1 = original_model.layer1
        self.layer2 = original_model.layer2
        self.layer3 = original_model.layer3
        self.layer4 = original_model.layer4

    def _apply(self, fn, *args, **kwargs):
        # device / dtype moves go through the owning ResNet, which rebuilds its flat buffers and views (ResNet._apply)
        self._resnet._apply(fn, *args, **kwargs)
        return self

    def forward(self, x):
        m = self._resnet
        if self.training and torch.is_grad_enabled():
            lw = m.linear.weight
            if m._grad_views is None or lw.grad is None or lw.grad.data_ptr() != m._grad_views[-2].data_ptr():
                m._ensure_grads()
            if any(p.requires_grad for p in m._flat_param_list()[:-2]):
                return _EncoderFn.apply(x, m._anchor, m)
        return m._run_forward_blocks(x, training=self.training)
