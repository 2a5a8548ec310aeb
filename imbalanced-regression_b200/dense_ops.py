"""dense_ops.py -- the operators of the NYUD2-DIR decoder / feature-fusion / refinement modules
(nyud2-dir/models/modules.py:6-174) on the native path, as autograd functions over NHWC bf16 tensors:

  conv2d_nhwc(x, weight, stride, padding)   nn.Conv2d(..., bias=False) with 1x1 / 3x3 / 5x5 filters (modules.py:11-20, 63,
                                            107, 134-141): wgmma implicit GEMM, forward + data / weight gradients
  upsample_bilinear(x, size)                F.upsample(x, size=size, mode='bilinear') (modules.py:24)
  cat_channels(tensors)                     torch.cat(tensors, 1) (modules.py:120)
  batch_norm_train(x, weight, bias, ...)    nn.BatchNorm2d in training mode [+ ReLU] (modules.py:13-21, 65, 109, 137-141)
  depth_head(x, weight, bias)               R's 1-channel 5x5 conv2 with bias (modules.py:145, 169): its own memory-bound
                                            kernels, fp32 output

and the modules UpProjection (_UpProjection, modules.py:6-31), D (modules.py:61-94), MFF (modules.py:96-128) and
RefinementR.  In eval() every BatchNorm normalises with its running statistics and leaves them untouched; gradients
flow through it as through the frozen affine map.

Activations are channels-last bf16 ([N, H, W, C], C a multiple of 64 for the convolutions, of 8 elsewhere); weights stay
the reference's fp32 [Cout, Cin, KH, KW] parameters (state_dict compatible).  Convolutions with fewer than 64 output
channels (the 16-channel MFF branches) are run with the output channels zero-padded to 64; the 1-channel depth head has
kernels of its own (depth_head).  No CPU path."""
import ctypes

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


class _SplitFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, y, *sizes):
        n, h, w, total = y.shape
        assert y.dtype == torch.bfloat16 and y.is_contiguous() and sum(sizes) <= total
        outs, off = [], 0
        for c in sizes:
            t = torch.empty(n, h, w, c, dtype=torch.bfloat16, device=y.device)
            _lib.call("dirb200_copy_channels", _lib.ptr(y), total, off, _lib.ptr(t), c, 0, c, n * h * w, _lib.stream_ptr())
            outs.append(t)
            off += c
        ctx.dims = (n, h, w, total)
        ctx.sizes = sizes
        return tuple(outs)

    @staticmethod
    def backward(ctx, *grads):
        n, h, w, total = ctx.dims
        dev = next(g for g in grads if g is not None).device
        covered = sum(ctx.sizes) == total and all(g is not None for g in grads)
        dy = (torch.empty if covered else torch.zeros)(n, h, w, total, dtype=torch.bfloat16, device=dev)
        off = 0
        for g, c in zip(grads, ctx.sizes):
            if g is not None:
                g = g.contiguous()
                _lib.call("dirb200_copy_channels", _lib.ptr(g), c, 0, _lib.ptr(dy), total, off, c, n * h * w,
                          _lib.stream_ptr())
            off += c
        return (dy,) + (None,) * len(ctx.sizes)


class _DepthHeadFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, weight, bias):
        _lib.require_cuda(x, weight, bias)
        assert x.dtype == torch.bfloat16 and x.is_contiguous() and x.dim() == 4
        n, h, w, c = x.shape
        assert tuple(weight.shape) == (1, c, 5, 5) and weight.dtype == torch.float32, (x.shape, weight.shape)
        assert bias.numel() == 1 and bias.dtype == torch.float32
        weight, bias = weight.contiguous(), bias.contiguous()
        y = torch.empty(n, h, w, 1, dtype=torch.float32, device=x.device)
        _lib.call("dirb200_depth_head_fwd", _lib.ptr(x), _lib.ptr(weight), _lib.ptr(bias), _lib.ptr(y), n, h, w, c,
                  _lib.stream_ptr())
        ctx.save_for_backward(x, weight)
        return y

    @staticmethod
    def backward(ctx, dy):
        x, weight = ctx.saved_tensors
        n, h, w, c = x.shape
        dy = dy.to(torch.float32).contiguous()
        st = _lib.stream_ptr()
        dx = dw = db = None
        if ctx.needs_input_grad[0]:
            dx = torch.empty_like(x)
            _lib.call("dirb200_depth_head_dgrad", _lib.ptr(dy), _lib.ptr(weight), _lib.ptr(dx), n, h, w, c, st)
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            nbytes = _lib.raw("dirb200_depth_head_wgrad_workspace_bytes")(n, h, w, c)
            ws = torch.empty(nbytes, dtype=torch.uint8, device=x.device)
            dw = torch.empty(1, c, 5, 5, dtype=torch.float32, device=x.device)
            db = torch.empty(1, dtype=torch.float32, device=x.device)
            _lib.call("dirb200_depth_head_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(db), _lib.ptr(ws),
                      nbytes, n, h, w, c, st)
        return dx, dw, db


def depth_head(x, weight, bias):
    """conv2d(x, weight, bias, stride 1, padding 2) with one output channel (R.conv2, modules.py:145, 169) for x bf16
    [N, H, W, C] (C a multiple of 8 from 8 to 256), weight fp32 [1, C, 5, 5], bias fp32 [1] -> fp32 [N, H, W, 1]."""
    return _DepthHeadFn.apply(x, weight, bias)


def split_channels(y, sizes):
    """The channel ranges [0, s0), [s0, s0 + s1), ... of an NHWC bf16 tensor as contiguous tensors (channels past the
    last range are dropped; their gradient is zero)."""
    return _SplitFn.apply(y, *[int(c) for c in sizes])


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


def _bn_workspace(c, dev):
    return torch.empty(_lib.raw("dirb200_bn_workspace_bytes")(c), dtype=torch.uint8, device=dev)


def _eval_coeffs(gamma, beta, rm, rv, eps, dev):
    """scale, shift [2][c] of an eval-mode BatchNorm from its running statistics (read only)."""
    c = gamma.numel()
    ss = torch.empty(2, c, dtype=torch.float32, device=dev)
    _lib.call("dirb200_bn_eval_coeffs", c, _lib.ptr(gamma), _lib.ptr(beta), eps, _lib.ptr(rm), _lib.ptr(rv),
              _lib.ptr(ss[0]), _lib.ptr(ss[1]), _lib.stream_ptr())
    return ss


class _BNEvalFn(torch.autograd.Function):
    """out = [relu](bn_a(y) [+ bn_b(res_y)]) with eval-mode BatchNorms: scale = gamma * invstd, shift = beta - rm *
    scale from the running statistics, which are only read.  The backward is that of the frozen affine maps: dz = g
    masked by the ReLU, dy = scale * dz, dgamma = invstd * (sum dz y - rm sum dz), dbeta = sum dz (one reduction, one
    apply pass for both inputs, as in training)."""
    @staticmethod
    def forward(ctx, y, res_y, ga, ba, gb, bb, rma, rva, rmb, rvb, eps_a, eps_b, relu):
        _lib.require_cuda(y, res_y)
        assert y.dtype == torch.bfloat16 and y.is_contiguous()
        assert res_y is None or (relu and res_y.shape == y.shape and res_y.is_contiguous())
        c = y.shape[-1]
        rows = y.numel() // c
        dev, st = y.device, _lib.stream_ptr()
        ss = _eval_coeffs(ga, ba, rma, rva, eps_a, dev)
        ss_b = None if res_y is None else _eval_coeffs(gb, bb, rmb, rvb, eps_b, dev)
        out = torch.empty_like(y)
        # the residual form's ReLU depends on both inputs: its mask is kept for the backward
        mask = torch.empty(rows, c // 8, dtype=torch.uint8, device=dev) if res_y is not None else None
        _lib.call("dirb200_layer_bn_apply", _lib.ptr(y), _lib.ptr(ss[0]), _lib.ptr(ss[1]), None, _lib.ptr(res_y),
                  None if ss_b is None else _lib.ptr(ss_b[0]), None if ss_b is None else _lib.ptr(ss_b[1]),
                  1 if relu else 0, rows, c, _lib.ptr(out), _lib.ptr(mask), st)
        ctx.save_for_backward(y, res_y, ga, gb, rma, rva, rmb, rvb, ss, ss_b, mask)
        ctx.eps = (eps_a, eps_b)
        ctx.relu = relu
        return out

    @staticmethod
    def backward(ctx, g):
        y, res_y, ga, gb, rma, rva, rmb, rvb, ss, ss_b, mask = ctx.saved_tensors
        c = y.shape[-1]
        rows = y.numel() // c
        dev, st = y.device, _lib.stream_ptr()
        g = g.contiguous()
        two = res_y is not None
        sc, sh = (ss[0], ss[1]) if (ctx.relu and not two) else (None, None)    # mask re-derived from y
        ws = _bn_workspace(c, dev)
        nblk = ctypes.c_int(0)
        _lib.call("dirb200_layer_bn_bwd_reduce", _lib.ptr(g), None, None, _lib.ptr(y), _lib.ptr(res_y), _lib.ptr(sc),
                  _lib.ptr(sh), _lib.ptr(mask), rows, c, 0, 0, None, _lib.ptr(ws), ctypes.byref(nblk), st)
        dgb = torch.zeros(4, c, dtype=torch.float32, device=dev)          # dgamma_a, dbeta_a, dgamma_b, dbeta_b
        coef = torch.zeros(2, 3, c, dtype=torch.float32, device=dev)      # dy = A dz + B y + C with A = scale
        scratch = torch.empty(3, c, dtype=torch.float32, device=dev)
        ones, zeros = torch.ones(c, device=dev), torch.zeros(c, device=dev)
        for i, (gamma, rm, rv, eps, s_) in enumerate(((ga, rma, rva, ctx.eps[0], ss), (gb, rmb, rvb, ctx.eps[1], ss_b))):
            if s_ is None:
                break
            inv = _eval_coeffs(ones, zeros, rm, rv, eps, dev)             # [0] = invstd of the running variance
            _lib.call("dirb200_layer_bn_bwd_coeffs", _lib.ptr(ws), nblk.value, 3 if two else 2, 1 + i, rows, c,
                      _lib.ptr(rm), _lib.ptr(inv[0]), _lib.ptr(gamma), _lib.ptr(dgb[2 * i]), _lib.ptr(dgb[2 * i + 1]),
                      _lib.ptr(scratch), st)
            coef[i, 0].copy_(s_[0])
        dy = torch.empty_like(y)
        dy2 = torch.empty_like(res_y) if two else None
        _lib.call("dirb200_layer_bn_bwd_apply", _lib.ptr(g), None, _lib.ptr(y), _lib.ptr(coef[0]), _lib.ptr(res_y),
                  _lib.ptr(coef[1]) if two else None, _lib.ptr(sc), _lib.ptr(sh), _lib.ptr(mask), rows, c, 0, 0,
                  _lib.ptr(dy), _lib.ptr(dy2), None, st)
        return (dy, dy2, dgb[0], dgb[1], dgb[2] if two else None, dgb[3] if two else None) + (None,) * 7


def _bn(x, bn, relu, training):
    """bn [+ ReLU]: batch statistics (running statistics updated) in training, the running statistics in eval
    (differentiable in both)."""
    if training:
        return batch_norm_train(x, bn.weight, bn.bias, bn.running_mean, bn.running_var, bn.momentum, bn.eps, relu)
    return _BNEvalFn.apply(x, None, bn.weight, bn.bias, None, None, bn.running_mean, bn.running_var, None, None, bn.eps,
                           bn.eps, relu)


class _BNAddReluFn(torch.autograd.Function):
    """relu(bn_a(y_a) + bn_b(y_b)), both BatchNorms in training mode: one apply pass with the second BN as its
    residual operand, one backward reduction (sum dz, sum dz y_a, sum dz y_b) and one apply pass for both gradients."""
    @staticmethod
    def forward(ctx, y_a, y_b, ga, ba, gb, bb, rma, rva, rmb, rvb, momentum, eps):
        _lib.require_cuda(y_a, y_b)
        assert y_a.shape == y_b.shape and y_a.is_contiguous() and y_b.is_contiguous()
        assert y_a.dtype == torch.bfloat16 and y_b.dtype == torch.bfloat16
        c = y_a.shape[-1]
        rows = y_a.numel() // c
        dev, st = y_a.device, _lib.stream_ptr()
        ws = _bn_workspace(c, dev)
        save = torch.empty(2, 4, c, dtype=torch.float32, device=dev)     # [a, b] x (mean, invstd, scale, shift)
        nblk = ctypes.c_int(0)
        for i, (y, g, b, rm, rv) in enumerate(((y_a, ga, ba, rma, rva), (y_b, gb, bb, rmb, rvb))):
            _lib.call("dirb200_layer_bn_stats", _lib.ptr(y), rows, c, _lib.ptr(ws), ctypes.byref(nblk), st)
            layout = (ctypes.c_int * 4)(nblk.value, 1, c, 1)
            _lib.call("dirb200_bn_finalize_layout", _lib.ptr(ws), layout, rows, c, _lib.ptr(g), _lib.ptr(b), eps,
                      momentum, _lib.ptr(rm), _lib.ptr(rv), _lib.ptr(save[i, 0]), _lib.ptr(save[i, 1]),
                      _lib.ptr(save[i, 2]), _lib.ptr(save[i, 3]), st)
        out = torch.empty_like(y_a)
        mask = torch.empty(rows, c // 8, dtype=torch.uint8, device=dev)
        _lib.call("dirb200_layer_bn_apply", _lib.ptr(y_a), _lib.ptr(save[0, 2]), _lib.ptr(save[0, 3]), None,
                  _lib.ptr(y_b), _lib.ptr(save[1, 2]), _lib.ptr(save[1, 3]), 1, rows, c, _lib.ptr(out), _lib.ptr(mask), st)
        ctx.save_for_backward(y_a, y_b, ga, gb, save, mask)
        return out

    @staticmethod
    def backward(ctx, g):
        y_a, y_b, ga, gb, save, mask = ctx.saved_tensors
        c = y_a.shape[-1]
        rows = y_a.numel() // c
        dev, st = y_a.device, _lib.stream_ptr()
        g = g.contiguous()
        ws = _bn_workspace(c, dev)
        nblk = ctypes.c_int(0)
        _lib.call("dirb200_layer_bn_bwd_reduce", _lib.ptr(g), None, None, _lib.ptr(y_a), _lib.ptr(y_b), None, None,
                  _lib.ptr(mask), rows, c, 0, 0, None, _lib.ptr(ws), ctypes.byref(nblk), st)
        dgb = torch.zeros(4, c, dtype=torch.float32, device=dev)          # dgamma_a, dbeta_a, dgamma_b, dbeta_b
        coef = torch.empty(2, 3, c, dtype=torch.float32, device=dev)
        for i, gamma in enumerate((ga, gb)):
            _lib.call("dirb200_layer_bn_bwd_coeffs", _lib.ptr(ws), nblk.value, 3, 1 + i, rows, c, _lib.ptr(save[i, 0]),
                      _lib.ptr(save[i, 1]), _lib.ptr(gamma), _lib.ptr(dgb[2 * i]), _lib.ptr(dgb[2 * i + 1]),
                      _lib.ptr(coef[i]), st)
        dya, dyb = torch.empty_like(y_a), torch.empty_like(y_b)
        _lib.call("dirb200_layer_bn_bwd_apply", _lib.ptr(g), None, _lib.ptr(y_a), _lib.ptr(coef[0]), _lib.ptr(y_b),
                  _lib.ptr(coef[1]), None, None, _lib.ptr(mask), rows, c, 0, 0, _lib.ptr(dya), _lib.ptr(dyb), None, st)
        return dya, dyb, dgb[0], dgb[1], dgb[2], dgb[3], None, None, None, None, None, None


def bn_add_relu(y_a, bn_a, y_b, bn_b, training):
    """relu(bn_a(y_a) + bn_b(y_b)) (modules.py:26-29): the join of an up-projection's two branches."""
    if training:
        return _BNAddReluFn.apply(y_a, y_b, bn_a.weight, bn_a.bias, bn_b.weight, bn_b.bias, bn_a.running_mean,
                                  bn_a.running_var, bn_b.running_mean, bn_b.running_var, bn_a.momentum, bn_a.eps)
    return _BNEvalFn.apply(y_a, y_b, bn_a.weight, bn_a.bias, bn_b.weight, bn_b.bias, bn_a.running_mean,
                           bn_a.running_var, bn_b.running_mean, bn_b.running_var, bn_a.eps, bn_b.eps, True)


def batch_norm_train(x, weight, bias, running_mean=None, running_var=None, momentum=0.1, eps=1e-5, relu=False):
    """nn.BatchNorm2d(training) [+ ReLU] on an NHWC bf16 tensor (channels 8, 16, 32, ..., 2048: the BN kernels split a
    CTA's 256 threads into channel groups of 8, so e.g. 24 channels are refused); running statistics updated in place
    like torch's."""
    return _BNTrainFn.apply(x, weight, bias, running_mean, running_var, momentum, eps, relu)


class RefinementR(torch.nn.Module):
    """nyud2-dir/models/modules.py:128-174 (module R): conv0 5x5 -> bn0 -> relu -> conv1 5x5 -> bn1 -> relu ->
    [FDS.smooth on the 128-channel map] -> conv2 5x5 (1 channel, bias); parameter names / shapes as the reference's.
    Input / feature maps are NHWC bf16; the depth is fp32 [N, H, W, 1] (depth_head); returns (depth, features
    [N, H, W, C] bf16, unsmoothed) in training with FDS."""

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
        return _bn(x, bn, relu, self.training)

    def forward(self, x, depth=None, epoch=None):
        x0 = self._bn(conv2d_nhwc(x, self.conv0.weight, 1, 2), self.bn0, True)
        x1 = self._bn(conv2d_nhwc(x0, self.conv1.weight, 1, 2), self.bn1, True)
        x1_s = x1
        if self.training and self.FDS is not None and epoch is not None and epoch >= self.FDS.start_smooth:
            from fds import FDS as _FDS          # the [rows, C] form (the NHWC map already is one row per pixel)
            n, h, w, c = x1.shape
            rows = _FDS.smooth(self.FDS, x1.float().view(-1, c), depth.reshape(-1).float(), epoch)
            x1_s = rows.view(n, h, w, c).to(torch.bfloat16)
        x2 = depth_head(x1_s, self.conv2.weight, self.conv2.bias)
        if self.training and self.FDS is not None:
            return x2, x1
        return x2


def _pad_to_64(c):
    return -(-c // 64) * 64


class UpProjection(torch.nn.Module):
    """nyud2-dir/models/modules.py:6-31 (_UpProjection): x = F.upsample(x, size); out = relu(bn1_2(conv1_2(relu(bn1(
    conv1(x))))) + bn2(conv2(x))).  Parameter names / shapes (state_dict keys) as the reference's.

    conv1 and conv2 read the same up-sampled x: they run as ONE convolution with their weights concatenated along Cout,
    and the result is split by channel (branch_convs).  With Cout = 16 (MFF) conv1_2 (16 -> 16, 3x3) runs with its
    input channels zero-padded to 64 (conv1_2_nhwc)."""

    def __init__(self, num_input_features, num_output_features):
        super().__init__()
        nn = torch.nn
        self.conv1 = nn.Conv2d(num_input_features, num_output_features, kernel_size=5, stride=1, padding=2, bias=False)
        self.bn1 = nn.BatchNorm2d(num_output_features)
        self.relu = nn.ReLU(inplace=True)
        self.conv1_2 = nn.Conv2d(num_output_features, num_output_features, kernel_size=3, stride=1, padding=1,
                                 bias=False)
        self.bn1_2 = nn.BatchNorm2d(num_output_features)
        self.conv2 = nn.Conv2d(num_input_features, num_output_features, kernel_size=5, stride=1, padding=2, bias=False)
        self.bn2 = nn.BatchNorm2d(num_output_features)

    def branch_convs(self, x, size):
        """(conv1(up), conv2(up)) for up = F.upsample(x, size): one paired convolution, split by channel."""
        c = self.conv1.out_channels
        w = torch.cat([self.conv1.weight, self.conv2.weight], 0)
        if w.shape[0] % 64 != 0:                      # zero-padded output channels, dropped by the split
            w = torch.cat([w, w.new_zeros(64 - w.shape[0] % 64, *w.shape[1:])], 0)
        y = _ConvFn.apply(upsample_bilinear(x, size), w, 1, 2)
        return split_channels(y, [c, c])

    def conv1_2_nhwc(self, x1):
        """conv1_2(x1); below 64 channels with input and output channels zero-padded to 64."""
        c = self.conv1_2.out_channels
        w = self.conv1_2.weight
        cp = _pad_to_64(c)
        if cp == c:
            return _ConvFn.apply(x1, w, 1, 1)
        n, ho, wo, _ = x1.shape
        xp = cat_channels([x1, x1.new_zeros(n, ho, wo, cp - c)])
        wp = torch.cat([w, w.new_zeros(c, cp - c, 3, 3)], 1)
        wp = torch.cat([wp, wp.new_zeros(cp - c, cp, 3, 3)], 0)
        return split_channels(_ConvFn.apply(xp, wp, 1, 1), [c])[0]

    def forward(self, x, size):
        """x: NHWC bf16 [N, H, W, Cin]; size (Ho, Wo) -> NHWC bf16 [N, Ho, Wo, Cout]."""
        y1, y2 = self.branch_convs(x, size)
        x1 = _bn(y1, self.bn1, True, self.training)
        return bn_add_relu(self.conv1_2_nhwc(x1), self.bn1_2, y2, self.bn2, self.training)


def _hw(t):
    return int(t.shape[1]), int(t.shape[2])


class D(torch.nn.Module):
    """nyud2-dir/models/modules.py:61-94: 1x1 conv + BN + ReLU on x_block4, then four up-projections to the sizes of
    x_block3, x_block2, x_block1 and twice x_block1.  Takes resnet.E_resnet's NHWC bf16 block outputs."""

    def __init__(self, num_features=2048):
        super().__init__()
        nn = torch.nn
        self.conv = nn.Conv2d(num_features, num_features // 2, kernel_size=1, stride=1, bias=False)
        num_features = num_features // 2
        self.bn = nn.BatchNorm2d(num_features)
        self.up1 = UpProjection(num_features, num_features // 2)
        num_features = num_features // 2
        self.up2 = UpProjection(num_features, num_features // 2)
        num_features = num_features // 2
        self.up3 = UpProjection(num_features, num_features // 2)
        num_features = num_features // 2
        self.up4 = UpProjection(num_features, num_features // 2)

    def forward(self, x_block1, x_block2, x_block3, x_block4):
        x_d0 = _bn(conv2d_nhwc(x_block4, self.conv.weight, 1, 0), self.bn, True, self.training)
        x_d1 = self.up1(x_d0, _hw(x_block3))
        x_d2 = self.up2(x_d1, _hw(x_block2))
        x_d3 = self.up3(x_d2, _hw(x_block1))
        h1, w1 = _hw(x_block1)
        return self.up4(x_d3, (2 * h1, 2 * w1))


class MFF(torch.nn.Module):
    """nyud2-dir/models/modules.py:96-128: each block output up-projected to `size` with 16 channels, concatenated,
    then 5x5 conv + BN + ReLU.  Takes resnet.E_resnet's NHWC bf16 block outputs."""

    def __init__(self, block_channel, num_features=64):
        super().__init__()
        nn = torch.nn
        self.up1 = UpProjection(block_channel[0], 16)
        self.up2 = UpProjection(block_channel[1], 16)
        self.up3 = UpProjection(block_channel[2], 16)
        self.up4 = UpProjection(block_channel[3], 16)
        self.conv = nn.Conv2d(num_features, num_features, kernel_size=5, stride=1, padding=2, bias=False)
        self.bn = nn.BatchNorm2d(num_features)

    def forward(self, x_block1, x_block2, x_block3, x_block4, size):
        xs = [up(x, size) for up, x in zip((self.up1, self.up2, self.up3, self.up4),
                                          (x_block1, x_block2, x_block3, x_block4))]
        x = conv2d_nhwc(cat_channels(xs), self.conv.weight, 1, 2)
        return _bn(x, self.bn, True, self.training)
