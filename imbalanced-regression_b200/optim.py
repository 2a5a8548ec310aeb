"""Fused optimizers over the model's flat parameter / gradient buffers
(SURVEY.md §8 f-1): ONE kernel per step instead of torch.optim's 161-tensor
foreach chain.  Semantics follow torch.optim.Adam / torch.optim.SGD as used at
agedb-dir/train.py:163-164 (Adam: no weight decay; SGD: momentum, weight decay).

FusedAdam / FusedSGD work on any set of parameters that tile one contiguous flat
fp32 buffer with their .grad tiling another (resnet.ResNet guarantees both);
otherwise they raise -- there is no per-tensor fallback.  Adam takes any list of
CUDA fp32 tensors (net.model's 245 parameters, nyud2-dir/train.py:146): one
multi-tensor launch per parameter group.
"""
import math

import numpy as np
import torch

import _lib
import resnet  # noqa: F401  (registers dirb200_adam_step / dirb200_sgd_step)


def _flat_span(tensors):
    """(data_ptr, numel) if the tensors tile one contiguous fp32 region in order, else None."""
    base = tensors[0].data_ptr()
    off = 0
    for t in tensors:
        if t.dtype != torch.float32 or not t.is_contiguous() or t.data_ptr() != base + 4 * off:
            return None
        off += t.numel()
    return base, off


class _FlatOptimizer(torch.optim.Optimizer):
    def _span(self, group):
        ps = [p for p in group['params'] if p.requires_grad]
        if not ps:
            return None
        if any(p.grad is None for p in ps):
            raise _lib.Dirb200Error("fused optimizer: a parameter has no .grad (call backward first)")
        sp, sg = _flat_span(ps), _flat_span([p.grad for p in ps])
        if sp is None or sg is None or sp[1] != sg[1]:
            raise _lib.Dirb200Error("fused optimizer needs parameters (and grads) that tile one flat fp32 buffer; "
                                    "pass model.parameters() of a dirb200 resnet in order")
        return ps, sp[0], sg[0], sp[1]

    def _clip_coef(self, group, ps, g_ptr, n):
        """Device scalar min(1, max_norm / ||grad||) of torch.nn.utils.clip_grad_norm_ (sts-b-dir/trainer.py:147-149)
        when the group has `max_grad_norm`; the step kernel multiplies the gradients by it as it reads them."""
        mx = group.get('max_grad_norm')
        if not mx:
            return None
        st = self.state[ps[0]]
        if 'clip_ws' not in st:
            st['clip_ws'] = torch.zeros(_lib.raw("dirb200_grad_clip_workspace_bytes")(), dtype=torch.uint8,
                                        device=ps[0].device)
            st['clip_out'] = torch.zeros(2, dtype=torch.float32, device=ps[0].device)
        _lib.call("dirb200_grad_clip_coef", g_ptr, n, float(group['grad_scale']), float(mx), _lib.ptr(st['clip_ws']),
                  st['clip_ws'].numel(), _lib.ptr(st['clip_out']), _lib.stream_ptr())
        return st['clip_out']

    def last_grad_norm(self):
        """Norm seen by the most recent clipped step (device tensor, no sync) or None."""
        for group in self.param_groups:
            ps = [p for p in group['params'] if p.requires_grad]
            if ps and 'clip_out' in self.state[ps[0]]:
                return self.state[ps[0]]['clip_out'][1]
        return None

    def zero_grad(self, set_to_none=False):
        """Keeps the flat gradient views attached and zeroes them (one memset per group)."""
        for group in self.param_groups:
            ps = [p for p in group['params'] if p.grad is not None]
            if not ps:
                continue
            span = _flat_span([p.grad for p in ps])
            if span is not None:
                flat = torch.as_strided(ps[0].grad, (span[1],), (1,))
                flat.zero_()
            else:
                for p in ps:
                    p.grad.zero_()


class FusedAdam(_FlatOptimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, grad_scale=1.0,
                 max_grad_norm=None):
        super().__init__(params, dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay, grad_scale=grad_scale,
                                      max_grad_norm=max_grad_norm))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            span = self._span(group)
            if span is None:
                continue
            ps, p_ptr, g_ptr, n = span
            st = self.state[ps[0]]
            if 'exp_avg' not in st or st['exp_avg'].numel() != n:
                st['step'] = 0
                st['exp_avg'] = torch.zeros(n, dtype=torch.float32, device=ps[0].device)
                st['exp_avg_sq'] = torch.zeros(n, dtype=torch.float32, device=ps[0].device)
            st['step'] += 1
            b1, b2 = group['betas']
            clip = self._clip_coef(group, ps, g_ptr, n)
            _lib.call("dirb200_adam_step", p_ptr, g_ptr, _lib.ptr(st['exp_avg']), _lib.ptr(st['exp_avg_sq']), n,
                      float(group['lr']), float(b1), float(b2), float(group['eps']), float(group['weight_decay']),
                      int(st['step']), float(group['grad_scale']), _lib.ptr(clip), _lib.stream_ptr())


class FusedSGD(_FlatOptimizer):
    def __init__(self, params, lr, momentum=0, weight_decay=0, grad_scale=1.0, max_grad_norm=None):
        super().__init__(params, dict(lr=lr, momentum=momentum, weight_decay=weight_decay, grad_scale=grad_scale,
                                      max_grad_norm=max_grad_norm))

    @torch.no_grad()
    def step(self, closure=None):
        for group in self.param_groups:
            span = self._span(group)
            if span is None:
                continue
            ps, p_ptr, g_ptr, n = span
            st = self.state[ps[0]]
            first = 'momentum_buffer' not in st or st['momentum_buffer'].numel() != n
            if first:
                st['momentum_buffer'] = torch.zeros(n, dtype=torch.float32, device=ps[0].device)
            clip = self._clip_coef(group, ps, g_ptr, n)
            _lib.call("dirb200_sgd_step", p_ptr, g_ptr, _lib.ptr(st['momentum_buffer']), n, float(group['lr']),
                      float(group['momentum']), float(group['weight_decay']), int(first), float(group['grad_scale']),
                      _lib.ptr(clip), _lib.stream_ptr())


# dirb200_adam_segment (include/dirb200.h): four device pointers, numel, and the tensor's bias corrections
_SEGMENT = np.dtype([('param', np.uint64), ('grad', np.uint64), ('exp_avg', np.uint64), ('exp_avg_sq', np.uint64),
                     ('numel', np.int64), ('bc1', np.float32), ('bc2_sqrt', np.float32)])


def _bias_corrections(beta1, beta2, step):
    """(1 - beta1^t, sqrt(1 - beta2^t)) in double precision from the fp32 betas, as dirb200_adam_step forms them; the
    segment table rounds each to float."""
    b1, b2 = float(np.float32(beta1)), float(np.float32(beta2))
    return 1.0 - math.pow(b1, step), math.sqrt(1.0 - math.pow(b2, step))


class Adam(torch.optim.Optimizer):
    """Drop-in for torch.optim.Adam(params, lr, betas, eps, weight_decay) with coupled L2 weight decay, as
    nyud2-dir/train.py:146 uses it, on any list of CUDA fp32 tensors: one dirb200_adam_step_multi launch per parameter
    group (one per 512 tensors).  As in torch, a parameter whose .grad is None is skipped and its step count does not
    advance; state is kept per parameter ('step' a CPU fp32 scalar tensor, 'exp_avg', 'exp_avg_sq'), so state_dict()
    has torch's layout and loads into torch.optim.Adam and back.  amsgrad and maximize are refused."""

    def __init__(self, params, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, weight_decay=0, amsgrad=False, *,
                 maximize=False):
        if amsgrad:
            raise ValueError("optim.Adam has no amsgrad variant")
        if maximize:
            raise ValueError("optim.Adam has no maximize variant")
        if not 0.0 <= lr:
            raise ValueError(f"Invalid learning rate: {lr}")
        if not 0.0 <= eps:
            raise ValueError(f"Invalid epsilon value: {eps}")
        if not 0.0 <= betas[0] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 0: {betas[0]}")
        if not 0.0 <= betas[1] < 1.0:
            raise ValueError(f"Invalid beta parameter at index 1: {betas[1]}")
        if not 0.0 <= weight_decay:
            raise ValueError(f"Invalid weight_decay value: {weight_decay}")
        super().__init__(params, dict(lr=lr, betas=tuple(betas), eps=eps, weight_decay=weight_decay, amsgrad=False,
                                      maximize=False))

    @staticmethod
    def _refuse(ps, gs, states):
        """Every parameter, gradient and moment must be a dense contiguous CUDA fp32 tensor of the parameter's size, all
        on one device (checked before the first CUDA call)."""
        dev = ps[0].get_device()
        for p, g, st in zip(ps, gs, states):
            ts = (p, g, st['exp_avg'], st['exp_avg_sq']) if st else (p, g)
            n = p.numel()
            for name, t in zip(('param', 'grad', 'exp_avg', 'exp_avg_sq'), ts):
                if not t.is_cuda:
                    _lib.require_cuda(t)
                if t.get_device() != dev:
                    raise _lib.Dirb200Error(f"optim.Adam: a parameter group spans cuda:{dev} and {t.device}")
                if t.dtype is not torch.float32 or t.layout is not torch.strided or not t.is_contiguous() \
                        or t.numel() != n:
                    raise _lib.Dirb200Error(f"optim.Adam: {name} must be a dense contiguous fp32 tensor of the "
                                            f"parameter's {n} elements (got {t.dtype}, {tuple(t.shape)})")
        return dev

    @torch.no_grad()
    def step(self, closure=None):
        loss = None
        if closure is not None:
            with torch.enable_grad():
                loss = closure()
        for group in self.param_groups:
            if group.get('amsgrad') or group.get('maximize') or group.get('decoupled_weight_decay'):
                raise ValueError("optim.Adam: amsgrad, maximize and decoupled weight decay are not supported")
            ps = [p for p in group['params'] if p.grad is not None]
            if not ps:
                continue
            gs = [p.grad for p in ps]
            states = [self.state.get(p) for p in ps]
            dev = self._refuse(ps, gs, states)
            for k, p in enumerate(ps):
                if not states[k]:
                    st = states[k] = self.state[p]
                    st['step'] = torch.tensor(0.0, dtype=torch.float32)
                    st['exp_avg'] = torch.zeros_like(p, memory_format=torch.preserve_format)
                    st['exp_avg_sq'] = torch.zeros_like(p, memory_format=torch.preserve_format)
            steps = [st['step'] for st in states]
            torch._foreach_add_(steps, 1)
            live = [k for k, p in enumerate(ps) if p.numel() > 0]
            if not live:
                continue
            b1, b2 = group['betas']
            table = np.empty(len(live), dtype=_SEGMENT)
            table['param'] = [ps[k].data_ptr() for k in live]
            table['grad'] = [gs[k].data_ptr() for k in live]
            table['exp_avg'] = [states[k]['exp_avg'].data_ptr() for k in live]
            table['exp_avg_sq'] = [states[k]['exp_avg_sq'].data_ptr() for k in live]
            table['numel'] = [ps[k].numel() for k in live]
            bcs = {}
            for k, t in enumerate(torch.stack([steps[k] for k in live]).tolist()):
                if t not in bcs:
                    bcs[t] = _bias_corrections(b1, b2, int(t))
                table['bc1'][k], table['bc2_sqrt'][k] = bcs[t]
            args = (table.ctypes.data_as(_lib.P), len(live), float(group['lr']), float(b1), float(b2),
                    float(group['eps']), float(group['weight_decay']))
            if dev == torch.cuda.current_device():
                _lib.call("dirb200_adam_step_multi", *args, _lib.stream_ptr())
            else:
                with torch.cuda.device(dev):
                    _lib.call("dirb200_adam_step_multi", *args, _lib.stream_ptr())
        return loss
