"""dense_ops.py -- the operators of the NYUD2-DIR decoder / feature-fusion / refinement modules
(nyud2-dir/models/modules.py:6-174) on the native path, as autograd functions over NHWC bf16 tensors:

  conv2d_nhwc(x, weight, stride, padding)   nn.Conv2d(..., bias=False) with 1x1 / 3x3 / 5x5 filters (modules.py:11-20, 63,
                                            107, 134-141): wgmma implicit GEMM, forward + data / weight gradients
  upsample_bilinear(x, size)                F.upsample(x, size=size, mode='bilinear') (modules.py:24)
  cat_channels(tensors)                     torch.cat(tensors, 1) (modules.py:120)
  batch_norm_train(x, weight, bias, ...)    nn.BatchNorm2d in training mode [+ ReLU] (modules.py:13-21, 65, 109, 137-141)

Activations are channels-last bf16 ([N, H, W, C], C a multiple of 64 for the convolutions, of 8 elsewhere); weights stay
the reference's fp32 [Cout, Cin, KH, KW] parameters (state_dict compatible).  Convolutions with fewer than 64 output
channels (the 16-channel MFF branches, the final 1-channel depth conv) are run with the output channels zero-padded to 64.
No CPU path."""
import torch

import _lib
import _convlib  # noqa: F401  (registers the conv entry points)


def _shape(x, weight, stride, padding):
    n, h, w, cin = x.shape
    cout, cin_w, kh, kw = weight.shape
    assert cin == cin_w and kh == kw, (x.shape, weight.shape)
    return (n, h, w, cin, cout, kh, kw, stride, padding)


class _ConvFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, stride, padding):
        _lib.require_cuda(x, weight)
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and weight.dtype == torch.float32
        shape = _shape(x, weight, stride, padding)
        n, h, w, cin, cout, k, _, s, p = shape
        ho, wo = (h + 2 * p - k) // s + 1, (w + 2 * p - k) // s + 1
        st = _lib.stream_ptr()
        wf = torch.empty(cout, k, k, cin, dtype=torch.bfloat16, device=x.device)
        wd = torch.empty(cin, k, k, cout, dtype=torch.bfloat16, device=x.device)
        _lib.call("dirb200_conv_prep_weights", _lib.ptr(weight.contiguous()), cout, cin, k, k, 0, _lib.ptr(wf), _lib.ptr(wd), st)
        y = torch.empty(n, ho, wo, cout, dtype=torch.bfloat16, device=x.device)
        _lib.call("dirb200_conv_fprop", _lib.ptr(x), _lib.ptr(wf), _lib.ptr(y), *shape, 0, st)
        ctx.save_for_backward(x, wd)
        ctx.shape = shape
        return y

    @staticmethod
    def backward(ctx, dy):
        x, wd = ctx.saved_tensors
        shape = ctx.shape
        n, h, w, cin, cout, k, _, s, p = shape
        dy = dy.contiguous()
        st = _lib.stream_ptr()
        dx = dw = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _lib.call("dirb200_conv_dgrad", _lib.ptr(dy), _lib.ptr(wd), _lib.ptr(dx), *shape, st)
        if ctx.needs_input_grad[1]:
            nbytes = _lib.raw("dirb200_conv_wgrad_workspace_bytes")(*shape, 0)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            dw = torch.empty(cout, cin, k, k, dtype=torch.float32, device=x.device)
            _lib.call("dirb200_conv_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(ws), nbytes, *shape, 0, 0, st)
        return dx, dw, None, None


def conv2d_nhwc(x, weight, stride=1, padding=0):
    """x bf16 [N, H, W, Cin] (Cin a multiple of 64), weight fp32 [Cout, Cin, K, K] -> bf16 [N, Ho, Wo, Cout]."""
    cout = weight.shape[0]
    if cout % 64 != 0:                       # narrow heads: zero-padded output channels, sliced off again
        pad = 64 - cout % 64
        wp = torch.cat([weight, weight.new_zeros(pad, *weight.shape[1:])], 0)
        return _ConvFn.apply(x, wp, stride, padding)[..., :cout]
    return _ConvFn.apply(x, weight, stride, padding)


class _UpsampleFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, ho, wo):
        _lib.require_cuda(x)
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.shape[3] % 8 == 0
        n, h, w, c = x.shape
        out = torch.empty(n, ho, wo, c, dtype=torch.bfloat16, device=x.device)
        _lib.call("dirb200_upsample_bilinear_fwd", _lib.ptr(x), n, h, w, c, ho, wo, _lib.ptr(out), _lib.stream_ptr())
        ctx.dims = (n, h, w, c, ho, wo)
        return out

    @staticmethod
    def backward(ctx, dy):
        n, h, w, c, ho, wo = ctx.dims
        dy = dy.contiguous()
        dx = torch.empty(n, h, w, c, dtype=torch.bfloat16, device=dy.device)
        _lib.call("dirb200_upsample_bilinear_bwd", _lib.ptr(dy), n, h, w, c, ho, wo, _lib.ptr(dx), _lib.stream_ptr())
        return dx, None, None


def upsample_bilinear(x, size):
    """F.upsample(x, size=size, mode='bilinear') (align_corners=False) on an NHWC bf16 tensor."""
    return _UpsampleFn.apply(x, int(size[0]), int(size[1]))


class _CatFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, *xs):
        n, h, w = xs[0].shape[:3]
        chans = [int(t.shape[3]) for t in xs]
        total = sum(chans)
        out = torch.empty(n, h, w, total, dtype=torch.bfloat16, device=xs[0].device)
        off = 0
        for t, c in zip(xs, chans):
            assert t.dtype == torch.bfloat16 and t.is_contiguous() and tuple(t.shape[:3]) == (n, h, w)
            _lib.call("dirb200_copy_channels", _lib.ptr(t), c, 0, _lib.ptr(out), total, off, c, n * h * w, _lib.stream_ptr())
            off += c
        ctx.chans = chans
        return out

    @staticmethod
    def backward(ctx, dy):
        dy = dy.contiguous()
        n, h, w, total = dy.shape
        outs, off = [], 0
        for c in ctx.chans:
            g = torch.empty(n, h, w, c, dtype=torch.bfloat16, device=dy.device)
            _lib.call("dirb200_copy_channels", _lib.ptr(dy), total, off, _lib.ptr(g), c, 0, c, n * h * w, _lib.stream_ptr())
            outs.append(g)
            off += c
        return tuple(outs)


def cat_channels(tensors):
    """torch.cat(tensors, 1) for NHWC bf16 tensors (channel counts multiples of 8)."""
    return _CatFn.apply(*tensors)


class _BNTrainFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias, running_mean, running_var, momentum, eps, relu):
        _lib.require_cuda(x, weight, bias)
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.shape[-1] % 8 == 0
        c = x.shape[-1]
        rows = x.numel() // c
        dev = x.device
        out = torch.empty_like(x)
        save = torch.empty(4, c, dtype=torch.float32, device=dev)          # mean, invstd, scale, shift
        ws = torch.empty(_lib.raw("dirb200_bn_workspace_bytes")(c), dtype=torch.uint8, device=dev)
        _lib.call("dirb200_bn_train_fwd", _lib.ptr(x), rows, c, _lib.ptr(weight), _lib.ptr(bias), eps, momentum,
                  _lib.ptr(running_mean), _lib.ptr(running_var), 1 if relu else 0, _lib.ptr(out), _lib.ptr(save[0]),
                  _lib.ptr(save[1]), _lib.ptr(save[2]), _lib.ptr(ws), _lib.stream_ptr())
        ctx.save_for_backward(x, weight, save)
        ctx.relu = relu
        return out

    @staticmethod
    def backward(ctx, g):
        x, weight, save = ctx.saved_tensors
        c = x.shape[-1]
        rows = x.numel() // c
        g = g.contiguous()
        dx = torch.empty_like(x)
        dgamma = torch.zeros(c, dtype=torch.float32, device=x.device)
        dbeta = torch.zeros(c, dtype=torch.float32, device=x.device)
        ws = torch.empty(_lib.raw("dirb200_bn_workspace_bytes")(c), dtype=torch.uint8, device=x.device)
        _lib.call("dirb200_bn_train_bwd", _lib.ptr(g), _lib.ptr(x), rows, c, _lib.ptr(weight), _lib.ptr(save[0]),
                  _lib.ptr(save[1]), _lib.ptr(save[2]), 1 if ctx.relu else 0, _lib.ptr(dgamma), _lib.ptr(dbeta), _lib.ptr(dx),
                  _lib.ptr(ws), _lib.stream_ptr())
        return dx, dgamma, dbeta, None, None, None, None, None


def batch_norm_train(x, weight, bias, running_mean=None, running_var=None, momentum=0.1, eps=1e-5, relu=False):
    """nn.BatchNorm2d(training) [+ ReLU] on an NHWC bf16 tensor (channels 8, 16, 32, ..., 2048: the BN kernels split a
    CTA's 256 threads into channel groups of 8, so e.g. 24 channels are refused); running statistics updated in place
    like torch's."""
    return _BNTrainFn.apply(x, weight, bias, running_mean, running_var, momentum, eps, relu)


class RefinementR(torch.nn.Module):
    """nyud2-dir/models/modules.py:128-174 (module R): conv0 5x5 -> bn0 -> relu -> conv1 5x5 -> bn1 -> relu ->
    [FDS.smooth on the 128-channel map] -> conv2 5x5 (1 channel, bias); parameter names / shapes as the reference's.
    Input / feature maps are NHWC bf16; returns (depth [N, H, W, 1] bf16, features [N, H, W, C]) in training with FDS."""

    def __init__(self, num_features=128, fds=None):
        super().__init__()
        nn = torch.nn
        self.conv0 = nn.Conv2d(num_features, num_features, 5, 1, 2, bias=False)
        self.bn0 = nn.BatchNorm2d(num_features)
        self.conv1 = nn.Conv2d(num_features, num_features, 5, 1, 2, bias=False)
        self.bn1 = nn.BatchNorm2d(num_features)
        self.conv2 = nn.Conv2d(num_features, 1, 5, 1, 2, bias=True)
        self.FDS = fds

    def _bn(self, x, bn, relu):
        return batch_norm_train(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps, relu)

    def forward(self, x, depth=None, epoch=None):
        x0 = self._bn(conv2d_nhwc(x, self.conv0.weight, 1, 2), self.bn0, True)
        x1 = self._bn(conv2d_nhwc(x0, self.conv1.weight, 1, 2), self.bn1, True)
        x1_s = x1
        if self.training and self.FDS is not None and epoch is not None and epoch >= self.FDS.start_smooth:
            from fds import FDS as _FDS          # the [rows, C] form (the NHWC map already is one row per pixel)
            n, h, w, c = x1.shape
            rows = _FDS.smooth(self.FDS, x1.float().view(-1, c), depth.reshape(-1).float(), epoch)
            x1_s = rows.view(n, h, w, c).to(torch.bfloat16)
        x2 = conv2d_nhwc(x1_s, self.conv2.weight, 1, 2) + self.conv2.bias.to(torch.bfloat16)
        if self.training and self.FDS is not None:
            return x2, x1
        return x2
