"""Bidirectional multi-layer LSTM on libdirb200 (sts-b-dir/models.py:40-43: nn.LSTM(d_word, d_hid, n_layers_enc,
bidirectional=True, batch_first=True) run packed by AllenNLP's masked seq2seq wrapper).

`LSTM` has torch.nn.LSTM's parameter names, shapes, gate order (i, f, g, o) and default initialisation, held as fp32
master tensors, so torch.optim, optim.Adam and state_dict() treat it as an nn.LSTM.  Its forward works on the padded
time-major bf16 layout of csrc/lstm.cu (rows = sequences, each with its own length): per layer, one 1x1 conv_fprop
computes the input projection of every step and both directions, then one launch per step runs the recurrence of both
directions.  The reverse direction starts at each row's own last token, and positions at or beyond a row's length
give zero output, as pack_padded_sequence / pad_packed_sequence do.  There is no dropout between layers.

The whole stack is one autograd Function.  Its backward runs the recurrent backward steps, then per layer one 1x1
conv_wgrad for W_ih, one per direction for W_hh, a column sum for the biases and one conv_dgrad for the layer input.
When neither the input nor any parameter needs a gradient, the forward keeps no backward buffers.
"""
import math

import torch
import torch.nn as nn

import _lib
import _convlib  # noqa: F401  (binds the conv entry points)


def pad64(n):
    return (n + 63) // 64 * 64


def _conv_args(T, M, cin, cout):
    # a [T * M, cin] x [cout, cin]^T GEMM as a 1x1 convolution over an n=1, h=T, w=M "image"
    return (1, T, M, cin, cout, 1, 1, 1, 0)


class _StackFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, mod, x, lens, *params):
        T, M, _ = x.shape
        H, Hp = mod.hidden_size, mod.hidden_p
        G2 = 8 * Hp
        save = any(ctx.needs_input_grad)
        st = _lib.stream_ptr()
        layers = []
        inp = x
        for k in range(mod.num_layers):
            w = params[8 * k: 8 * k + 8]
            din, blocks = (mod.input_size, 1) if k == 0 else (2 * H, 2)
            Dp = inp.shape[2]
            dev = x.device
            wih = torch.empty(G2, Dp, dtype=torch.bfloat16, device=dev)
            wihT = torch.empty(Dp, G2, dtype=torch.bfloat16, device=dev)
            whh = torch.empty(2, 4 * Hp, Hp, dtype=torch.bfloat16, device=dev)
            whhT = torch.empty(2, Hp, 4 * Hp, dtype=torch.bfloat16, device=dev)
            bias = torch.empty(2, 4 * Hp, dtype=torch.float32, device=dev)
            _lib.call("dirb200_lstm_prep_weights", *[_lib.ptr(t) for t in w], H, din, blocks, Hp, Dp,
                      _lib.ptr(wih), _lib.ptr(wihT), _lib.ptr(whh), _lib.ptr(whhT), _lib.ptr(bias), st)
            xproj = torch.empty(T, M, G2, dtype=torch.bfloat16, device=dev)
            _lib.call("dirb200_conv_fprop", _lib.ptr(inp), _lib.ptr(wih), _lib.ptr(xproj), *_conv_args(T, M, Dp, G2),
                      0, st)
            S = T + 1 if save else 2
            h = torch.empty(2, S, M, Hp, dtype=torch.bfloat16, device=dev)
            c = torch.empty(2, S, M, Hp, dtype=torch.float32, device=dev)
            gates = torch.empty(2, T, M, 4 * Hp, dtype=torch.float32, device=dev) if save else None
            y = torch.empty(T, M, 2 * Hp, dtype=torch.bfloat16, device=dev)
            _lib.call("dirb200_lstm_layer_fwd", _lib.ptr(xproj), _lib.ptr(whh), _lib.ptr(bias), _lib.ptr(lens), T, M,
                      Hp, int(save), _lib.ptr(h), _lib.ptr(c), _lib.ptr(gates), _lib.ptr(y), st)
            if save:
                layers.append((inp, din, blocks, wihT, whhT, h, c, gates))
            inp = y
        ctx.mod, ctx.layers, ctx.lens = mod, layers, lens
        return inp

    @staticmethod
    def backward(ctx, gy):
        mod, lens = ctx.mod, ctx.lens
        H, Hp = mod.hidden_size, mod.hidden_p
        G2 = 8 * Hp
        T, M, _ = gy.shape
        dev = gy.device
        st = _lib.stream_ptr()
        dy = gy.contiguous()
        grads = [None] * (8 * mod.num_layers)
        dx = None
        for k in reversed(range(mod.num_layers)):
            inp, din, blocks, wihT, whhT, h, c, gates = ctx.layers[k]
            Dp = inp.shape[2]
            dg = torch.empty(2, T, M, 4 * Hp, dtype=torch.bfloat16, device=dev)
            dgt = torch.empty(T, M, G2, dtype=torch.bfloat16, device=dev)
            dc = torch.empty(2, 2, M, Hp, dtype=torch.float32, device=dev)
            _lib.call("dirb200_lstm_layer_bwd", _lib.ptr(whhT), _lib.ptr(dy), _lib.ptr(gates), _lib.ptr(c),
                      _lib.ptr(lens), T, M, Hp, _lib.ptr(dc), _lib.ptr(dg), _lib.ptr(dgt), st)
            if any(ctx.needs_input_grad[3 + 8 * k: 11 + 8 * k]):
                dwih = torch.empty(G2, Dp, dtype=torch.float32, device=dev)
                _wgrad(inp, dgt, dwih, T, M, Dp, G2, st)
                dwhh = torch.empty(2, 4 * Hp, Hp, dtype=torch.float32, device=dev)
                for d in range(2):
                    _wgrad(h[d], dg[d], dwhh[d], T, M, Hp, 4 * Hp, st)
                db = torch.empty(G2, dtype=torch.float32, device=dev)
                _lib.call("dirb200_col_sum_bf16", _lib.ptr(dgt), T * M, G2, _lib.ptr(db), st)
                g = [torch.empty_like(p) for p in mod.layer_params(k)]
                _lib.call("dirb200_lstm_scatter_grads", _lib.ptr(dwih), _lib.ptr(dwhh), _lib.ptr(db), H, din, blocks,
                          Hp, Dp, *[_lib.ptr(t) for t in g], st)
                grads[8 * k: 8 * k + 8] = g
            if k > 0 or ctx.needs_input_grad[1]:
                dx = torch.empty(T, M, Dp, dtype=torch.bfloat16, device=dev)
                _lib.call("dirb200_conv_dgrad", _lib.ptr(dgt), _lib.ptr(wihT), _lib.ptr(dx),
                          *_conv_args(T, M, Dp, G2), st)
                dy = dx
        ctx.layers = None
        return (None, dx if ctx.needs_input_grad[1] else None, None, *grads)


def _wgrad(x, dy, dw, T, M, cin, cout, st):
    """dw[cout, cin] = dy[T*M, cout]^T . x[T*M, cin]; rows of x / dy beyond T*M are not read."""
    args = _conv_args(T, M, cin, cout)
    nbytes = int(_lib.raw("dirb200_conv_wgrad_workspace_bytes")(*args, 0))
    ws = torch.empty(max(nbytes, 16), dtype=torch.uint8, device=x.device)
    _lib.call("dirb200_conv_wgrad", _lib.ptr(x), _lib.ptr(dy), _lib.ptr(dw), _lib.ptr(ws), ws.numel(), *args, 0, 0, st)


class LSTM(nn.Module):
    """torch.nn.LSTM(input_size, hidden_size, num_layers, bidirectional=True) -- parameters only in torch's layout; the
    compute is forward_padded()."""

    def __init__(self, input_size, hidden_size, num_layers=1, bias=True, batch_first=True, dropout=0.,
                 bidirectional=True):
        super().__init__()
        if not (bidirectional and bias and dropout == 0):
            raise ValueError("rnn.LSTM: only the bidirectional LSTM with biases and no inter-layer dropout is built")
        self.input_size, self.hidden_size, self.num_layers = input_size, hidden_size, num_layers
        self.batch_first, self.bidirectional = batch_first, True
        self.hidden_p, self.input_p = pad64(hidden_size), pad64(input_size)
        for k in range(num_layers):
            din = input_size if k == 0 else 2 * hidden_size
            for sfx in ("", "_reverse"):
                self.register_parameter(f"weight_ih_l{k}{sfx}", nn.Parameter(torch.empty(4 * hidden_size, din)))
                self.register_parameter(f"weight_hh_l{k}{sfx}", nn.Parameter(torch.empty(4 * hidden_size, hidden_size)))
                self.register_parameter(f"bias_ih_l{k}{sfx}", nn.Parameter(torch.empty(4 * hidden_size)))
                self.register_parameter(f"bias_hh_l{k}{sfx}", nn.Parameter(torch.empty(4 * hidden_size)))
        self.reset_parameters()

    def reset_parameters(self):
        # torch.nn.RNNBase.reset_parameters: every parameter ~ U(-1/sqrt(H), 1/sqrt(H)), in registration order
        stdv = 1.0 / math.sqrt(self.hidden_size)
        for w in self.parameters():
            nn.init.uniform_(w, -stdv, stdv)

    def layer_params(self, k):
        return [getattr(self, f"{n}_l{k}{sfx}") for sfx in ("", "_reverse")
                for n in ("weight_ih", "weight_hh", "bias_ih", "bias_hh")]

    def get_output_dim(self):
        return 2 * self.hidden_size

    def forward_padded(self, x, lens):
        """x bf16 [T, M, input_p] time-major, zero at t >= lens[m] and in the padding columns; lens int32 [M] on the
        device, each in [1, T] (not checked here).  Returns the last layer's output, bf16 [T, M, 2 hidden_p]: direction
        d's units at columns [d hidden_p, d hidden_p + hidden_size), zeros elsewhere and at t >= lens[m]."""
        _lib.require_cuda(x, lens)
        if x.dtype != torch.bfloat16 or x.dim() != 3 or x.shape[2] != self.input_p or not x.is_contiguous():
            raise ValueError(f"rnn.LSTM: x must be contiguous bf16 [T, M, {self.input_p}], got {x.dtype} "
                             f"{tuple(x.shape)}")
        if lens.dtype != torch.int32 or lens.shape != (x.shape[1],):
            raise ValueError("rnn.LSTM: lens must be int32 [M]")
        params = [p for k in range(self.num_layers) for p in self.layer_params(k)]
        return _StackFn.apply(self, x, lens, *params)
