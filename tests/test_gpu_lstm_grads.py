"""Every gradient of rnn.LSTM's backward (imbalanced-regression_b200/rnn.py, _StackFn.backward) per element against
float64, on the H100.

The backward of one layer k is: dirb200_lstm_layer_bwd (the recurrent steps; tests/test_gpu_stsb_model.py checks it
step by step) gives the gate gradients dg (step order, per direction) and dgt (time order); then
- W_ih grad  = dgt^T . inp                      one 1x1 conv_wgrad, K = T M pixels
- W_hh grad  = sum_s dg[d, s]^T . h[d, s]       one conv_wgrad per direction over h slots 0 .. T-1 (slot s is step s's
                                                 input state, so step s's dg pairs with slot s)
- bias grads = column sums of dgt               dirb200_col_sum_bf16, the same vector for b_ih and b_hh
- dx         = dgt . W_ih (bf16)                one 1x1 conv_dgrad; it is the dy of layer k - 1
and dirb200_lstm_scatter_grads moves the padded, gate-interleaved fp32 results to torch's layout.

The test keeps the buffers the forward saved (out.grad_fn.layers), recomputes dg / dgt from the top layer down with
dirb200_lstm_layer_bwd (deterministic, so the same bits the module saw, provided the module handed each layer the right
dy), and builds float64 references from those bf16 tensors, mapped to torch's layout by the gate permutation and the
input-column map.  u = 2^-24, KAPPA(K) = (K / 16 + 16) u (tests/test_gpu_conv.py), A = the same product of absolute
values:
- W_ih, W_hh: fp32 wgrad, split-K over `splits` partials (dirb200_conv_wgrad_workspace_bytes): within
  (KAPPA(pixels per split) + splits u) A, as conv wgrad in tests/test_gpu_conv.py.
- biases: each thread of col_sum_kernel adds ceil(rows / 8) exact bf16 values in order, then the 8 phase sums are
  added: each addition rounds once relative to a partial sum <= sum |x|, so
  |db - ref| <= (ceil(rows / 8) + 8) u sum |x|.  b_ih and b_hh get the same bits.
- dx: bf16 conv_dgrad output, K = 8 Hp: within 2^-8 |ref| + (1 + 2^-8) KAPPA(8 Hp) A; exactly zero at t >= len (dgt is
  zero there) and in the padded input columns (W_ih is zero there).
- Layer 0's input gradient equals the test's own chain of conv_dgrad outputs bit for bit, which pins the hand-off of
  each layer's dx as the dy of the layer below.
The file reruns itself with DIRB200_SMS=7 (other split-K factors at the small shapes)."""
import os
import subprocess
import sys

import pytest
import torch

from test_gpu_conv import KAPPA, U, check_elementwise
from test_gpu_stsb_model import gate_perm, lens_for, pad64, _same_bits

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = "cuda"


def _wgrad_bound(T, M, cin, cout, A):
    """(KAPPA(pixels per split) + splits u) A for the 1x1 conv_wgrad rnn._wgrad launches."""
    import _lib, _convlib  # noqa: F401
    args = (1, T, M, cin, cout, 1, 1, 1, 0)
    splits = int(_lib.raw("dirb200_conv_wgrad_workspace_bytes")(*args, 0)) // (cin * cout * 4)
    assert splits >= 1
    per_split = -(-(-(-(T * M) // 64)) // splits) * 64
    return (KAPPA(per_split) + splits * U) * A


def _inv_perm(H, Hp):
    """torch gate row (i, f, g, o blocks of H) -> interleaved column of one direction"""
    perm = gate_perm(H, Hp)
    n = torch.arange(4 * Hp)
    inv = torch.empty(4 * H, dtype=torch.long)
    inv[perm[perm >= 0]] = n[perm >= 0]
    return inv.to(DEV)


def _in_cols(din, blocks, Dp):
    """torch input index -> padded input column, and the padded columns no input maps to"""
    real, bp = din // blocks, Dp // blocks
    ic = torch.arange(din)
    jcol = (ic // real) * bp + ic % real
    pad = torch.ones(Dp, dtype=torch.bool)
    pad[jcol] = False
    return jcol.to(DEV), pad.to(DEV)


@pytest.mark.parametrize("din,H,layers,T,M", [(300, 1500, 2, 40, 256), (24, 20, 2, 9, 10), (40, 64, 1, 7, 65)],
                         ids=["stsb", "small", "h64"])
def test_lstm_grads_per_element(din, H, layers, T, M):
    import _lib, _convlib  # noqa: F401
    import rnn
    torch.manual_seed(21)
    lstm = rnn.LSTM(din, H, layers, bidirectional=True, batch_first=True).to(DEV)
    Hp, Dp0 = lstm.hidden_p, lstm.input_p
    G2 = 8 * Hp
    lens = lens_for(M, T, 22).to(DEV)
    mask = torch.arange(T, device=DEV)[:, None] < lens.long()[None, :]          # [T, M]: t < len
    g = torch.Generator(device=DEV).manual_seed(23)
    x = torch.zeros(T, M, Dp0, device=DEV)
    x[..., :din] = torch.randn(T, M, din, device=DEV, generator=g)
    x = (x * mask[..., None]).bfloat16().requires_grad_(True)
    out = lstm.forward_padded(x, lens)
    saved = [tuple(t.detach().clone() if torch.is_tensor(t) else t for t in L) for L in out.grad_fn.layers]
    assert len(saved) == layers
    gy = torch.randn(T, M, 2, Hp, device=DEV, generator=g)
    gy[..., H:] = 0
    gy = (gy * mask[..., None, None]).bfloat16().view(T, M, 2 * Hp)
    out.backward(gy)
    torch.cuda.synchronize()

    inv = _inv_perm(H, Hp)
    nan = float("nan")
    dy = gy
    for k in reversed(range(layers)):
        inp, din_k, blocks, wihT, whhT, h, c, gates = saved[k]
        Dp = inp.shape[2]
        dc = torch.full((2, 2, M, Hp), nan, device=DEV)
        dg = torch.full((2, T, M, 4 * Hp), nan, dtype=torch.bfloat16, device=DEV)
        dgt = torch.full((T, M, G2), nan, dtype=torch.bfloat16, device=DEV)
        _lib.call("dirb200_lstm_layer_bwd", _lib.ptr(whhT), _lib.ptr(dy), _lib.ptr(gates), _lib.ptr(c),
                  _lib.ptr(lens), T, M, Hp, _lib.ptr(dc), _lib.ptr(dg), _lib.ptr(dgt), None)
        torch.cuda.synchronize()
        D = dgt.view(T * M, G2).double()
        X = inp.view(T * M, Dp).double()
        jcol, padcol = _in_cols(din_k, blocks, Dp)
        ref = D.t() @ X
        A = D.abs().t() @ X.abs()
        bound = _wgrad_bound(T, M, Dp, G2, A)
        del X
        dbref = D.sum(0)
        dbabs = D.abs().sum(0)
        p = lstm.layer_params(k)               # (w_ih, w_hh, b_ih, b_hh) forward, then reverse
        for d in range(2):
            rows = d * 4 * Hp + inv
            w_ih, w_hh, b_ih, b_hh = p[4 * d: 4 * d + 4]
            sel = (rows[:, None], jcol[None, :])
            check_elementwise(f"l{k} d{d} weight_ih", w_ih.grad, ref[sel], A[sel], bound[sel])
            check_elementwise(f"l{k} d{d} bias_ih", b_ih.grad, dbref[rows], dbabs[rows],
                              (-(-(T * M) // 8) + 8) * U * dbabs[rows])
            assert _same_bits(b_ih.grad, b_hh.grad), (k, d)
            Hd = h[d, :T].reshape(T * M, Hp).double()
            Dd = dg[d].view(T * M, 4 * Hp).double()
            rh = Dd.t() @ Hd
            Ah = Dd.abs().t() @ Hd.abs()
            bh = _wgrad_bound(T, M, Hp, 4 * Hp, Ah)
            sel = (inv[:, None], torch.arange(H, device=DEV)[None, :])
            check_elementwise(f"l{k} d{d} weight_hh", w_hh.grad, rh[sel], Ah[sel], bh[sel])
            del Hd, Dd, rh, Ah, bh
        del ref, A, bound
        # the layer's input gradient: the test's own conv_dgrad of dgt, then handed down as the next layer's dy
        dx = torch.full((T, M, Dp), nan, dtype=torch.bfloat16, device=DEV)
        _lib.call("dirb200_conv_dgrad", _lib.ptr(dgt), _lib.ptr(wihT), _lib.ptr(dx), *rnn._conv_args(T, M, Dp, G2),
                  None)
        torch.cuda.synchronize()
        W = wihT.double()
        rx = D @ W.t()
        Ax = D.abs() @ W.abs().t()
        check_elementwise(f"l{k} dx", dx.view(T * M, Dp), rx, Ax,
                          2.0 ** -8 * rx.abs() + (1 + 2.0 ** -8) * KAPPA(G2) * Ax)
        del D, W, rx, Ax
        assert torch.all(dx[~mask] == 0) and torch.all(dx[..., padcol] == 0), k
        dy = dx
    assert _same_bits(x.grad, dy)


@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_lstm_grads_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process)."""
    if os.environ.get("DIRB200_LSTM_GRADS_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_LSTM_GRADS_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
