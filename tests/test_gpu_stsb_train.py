"""GPU checks of gradient-norm clipping in the multi-tensor Adam (dirb200_grad_norm_multi,
dirb200_adam_step_multi_clipped, optim.Adam(max_grad_norm)) and of STS-B-DIR's shot metrics
(dirb200_stsb_shot_metrics, stsb_data.STSShotAverage).

Bounds (u = 2^-24):
- Norm.  Each thread squares at most 16 elements of a chunk in an fp32 fma chain: all terms are non-negative, so that
  partial is within 16 u of its exact value (relative).  The partials are added in fp64 (error below 2^-53 per add,
  negligible here); the square root halves the relative error of the sum, to 8 u, and rounding the fp64 root to fp32
  adds up to u.  So |norm - ||g||| <= (8 u + u + 2^-40) ||g|| <= 10 u ||g||.  The coefficient is then fp32 max_norm / (norm + 1e-6) clamped to 1, checked bit for bit from
  the kernel's own norm.
- optim.Adam(max_grad_norm) against clip_grad_norm_ + torch.optim.Adam: torch's fp32 norm and ours differ by about
  1e-6 relative, so the clip coefficients do too.  Adam's step m / (sqrt(v) + eps) is invariant to a common scale of
  the gradients except through eps, so the parameters differ by far less than lr 1e-6 per step; FusedAdam's bound
  (rtol 1e-5, atol 1e-7) holds with room.
- Shot metrics: counts exact, the rest within 1e-12 max(|want|, 1) of the reference scorer (fixture) and of the
  float64 oracle (tests/test_stsb_train_cpu.py); all sums are fp64 in a fixed order.
The file reruns itself with DIRB200_SMS=7."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from util import golden
from test_stsb_train_cpu import CASES, assert_metrics, shot_metrics_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
LR, B1, B2, EPS, WD = 1e-3, 0.9, 0.999, 1e-8, 1e-5          # sts-b-dir/trainer.py:21 (Adam, weight decay 1e-5)
RTOL, ATOL = 1e-5, 1e-7


def L():
    import _lib
    import resnet  # noqa: F401  (binds the optimizer entry points)
    return _lib


def optim():
    import optim as o
    return o


def norm_call(grads, max_norm=5.0, ws=None):
    """dirb200_grad_norm_multi over a list of CUDA fp32 tensors -> (out [coef, norm] NaN-prefilled, workspace)."""
    lib, o = L(), optim()
    t = np.empty(len(grads), dtype=o._GRAD_SEGMENT)
    t['grad'] = [g.data_ptr() if g.numel() else 0 for g in grads]
    t['numel'] = [g.numel() for g in grads]
    if ws is None:
        ws = torch.zeros(lib.raw("dirb200_grad_norm_multi_workspace_bytes")(), dtype=torch.uint8, device=DEV)
    out = torch.full((2,), float('nan'), device=DEV)
    lib.call("dirb200_grad_norm_multi", t.ctypes.data_as(lib.P), len(grads), max_norm, lib.ptr(ws), ws.numel(),
             lib.ptr(out), lib.stream_ptr())
    torch.cuda.synchronize()
    return out, ws


def norm64(grads):
    return float(np.sqrt(sum(float((g.double() ** 2).sum()) for g in grads)))


def coef32(max_norm, norm):
    c = np.float32(max_norm) / (np.float32(norm) + np.float32(1e-6))
    return np.float32(min(c, np.float32(1.0)))


def grad_lists():
    """name -> list of tensors: more than 512 (three launches' worth with empties), views at 4-byte offsets, one big."""
    rs = np.random.RandomState(0)
    g = torch.Generator(device=DEV).manual_seed(0)
    flat = torch.randn(3_000_000, device=DEV, generator=g)
    sizes = rs.randint(0, 3000, 1300)
    sizes[::7] = 0                                            # empty tensors interleaved
    views, at = [], 1                                         # 4-byte offset
    for n in sizes:
        views.append(flat[at:at + int(n)])
        at += int(n)
    big = [torch.randn((1 << 22) + 3, device=DEV, generator=g) * 1e-3]
    mixed = [torch.randn(s, device=DEV, generator=g) * 10 ** float(e) for s, e in
             ((5, 1), (4096, -2), (4097, 0), (1, 3), (0, 0), (123457, -4))]
    return {"1300-views-with-empties": views, "one-big": big, "mixed-scales": mixed,
            "only-empties": [flat[:0], flat[5:5]]}


@pytest.mark.parametrize("name", ["1300-views-with-empties", "one-big", "mixed-scales", "only-empties"])
def test_grad_norm_against_float64_and_bit_identical_on_repeat(name):
    grads = grad_lists()[name]
    out, ws = norm_call(grads)
    want = norm64(grads)
    norm = float(out[1])
    assert abs(norm - want) <= 10 * U * want + 1e-30, (norm, want)
    assert out[0].item() == float(coef32(5.0, out[1].item()))
    again, _ = norm_call(grads, ws=ws)                        # the same workspace, reset by the kernel's ticket
    assert torch.equal(out, again)
    if name == "only-empties":
        assert norm == 0.0 and out[0].item() == 1.0


def test_grad_norm_non_finite_propagates_as_torch():
    g = torch.randn(10000, device=DEV)
    g[17] = float('inf')
    out, _ = norm_call([g])
    assert out[1].item() == float('inf') and out[0].item() == 0.0
    g[18] = float('nan')
    out, _ = norm_call([g])
    assert np.isnan(out[1].item()) and np.isnan(out[0].item())


def adam_tables(segs, step):
    o = optim()
    t = np.empty(len(segs), dtype=o._SEGMENT)
    for k, name in enumerate(('param', 'grad', 'exp_avg', 'exp_avg_sq')):
        t[name] = [s[k].data_ptr() for s in segs]
    t['numel'] = [s[0].numel() for s in segs]
    t['bc1'], t['bc2_sqrt'] = o._bias_corrections(B1, B2, step)
    return t


@pytest.mark.parametrize("offset", [0, 1])
def test_clipped_adam_with_coefficient_one_is_bit_identical(offset):
    lib = L()
    sizes = [int(s) for s in np.random.RandomState(1).randint(1, 3000, 1100)] + [(1 << 20) + 5]
    total = offset + sum(sizes)
    g = torch.Generator(device=DEV).manual_seed(3)
    bufs = [torch.randn(total, device=DEV, generator=g), torch.randn(total, device=DEV, generator=g) * 0.1,
            torch.randn(total, device=DEV, generator=g) * 0.01, torch.rand(total, device=DEV, generator=g) * 1e-3]
    other = [b.clone() for b in bufs]

    def segs(bs):
        out, at = [], offset
        for n in sizes:
            out.append(tuple(b[at:at + n] for b in bs))
            at += n
        return out

    ta, tb = adam_tables(segs(bufs), 3), adam_tables(segs(other), 3)
    one = torch.ones(1, device=DEV)
    lib.call("dirb200_adam_step_multi", ta.ctypes.data_as(lib.P), len(ta), LR, B1, B2, EPS, WD, lib.stream_ptr())
    lib.call("dirb200_adam_step_multi_clipped", tb.ctypes.data_as(lib.P), len(tb), LR, B1, B2, EPS, WD, lib.ptr(one),
             lib.stream_ptr())
    torch.cuda.synchronize()
    for x, y in zip(bufs, other):
        assert torch.equal(x, y)


def test_clipped_adam_scales_the_gradient_as_it_reads_it():
    """A coefficient c gives the bits of the unclipped step on c * g (one fp32 product per element)."""
    lib = L()
    g = torch.Generator(device=DEV).manual_seed(4)
    n = 100003
    bufs = [torch.randn(n, device=DEV, generator=g), torch.randn(n, device=DEV, generator=g),
            torch.randn(n, device=DEV, generator=g) * 0.01, torch.rand(n, device=DEV, generator=g) * 1e-3]
    ref = [b.clone() for b in bufs]
    c = torch.tensor([0.3712], device=DEV)
    ref[1] = ref[1] * c
    grad_before = bufs[1].clone()
    ta, tb = adam_tables([tuple(bufs)], 2), adam_tables([tuple(ref)], 2)
    lib.call("dirb200_adam_step_multi_clipped", ta.ctypes.data_as(lib.P), 1, LR, B1, B2, EPS, WD, lib.ptr(c),
             lib.stream_ptr())
    lib.call("dirb200_adam_step_multi", tb.ctypes.data_as(lib.P), 1, LR, B1, B2, EPS, WD, lib.stream_ptr())
    torch.cuda.synchronize()
    for k in (0, 2, 3):
        assert torch.equal(bufs[k], ref[k])
    assert torch.equal(bufs[1], grad_before)                  # the gradient is not rewritten


# ---------------------------------------------------------------------- optim.Adam(max_grad_norm) vs torch
def stsb_params():
    """The STS-B model's parameters at the reference's sizes (d_word 300, d_hid 1500, 2 layers, frozen embeddings)
    that require grad, and a detached copy for torch."""
    from test_gpu_stsb_model import _build
    model, _ = _build(V=1000, d_word=300, d_hid=1500, train_words=0, fds=1)
    ps = [p for p in model.parameters() if p.requires_grad]
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]
    return ps, shadow


def set_grads(ps, shadow, step, target_norm):
    g = torch.Generator(device=DEV).manual_seed(500 + step)
    gs = [torch.randn(p.shape, device=DEV, generator=g) for p in ps]
    scale = target_norm / norm64(gs)
    for p, s, gr in zip(ps, shadow, gs):
        p.grad, s.grad = gr * scale, gr * scale


def test_optim_adam_max_grad_norm_matches_clip_grad_norm_and_torch_adam():
    ps, shadow = stsb_params()
    mine = optim().Adam(ps, LR, weight_decay=WD, max_grad_norm=5.0)
    ref = torch.optim.Adam(shadow, LR, weight_decay=WD)
    for step, target in enumerate((20.0, 3.0, 5.5, 0.7, 50.0)):        # above and below the threshold
        set_grads(ps, shadow, step, target)
        before = [p.grad.clone() for p in ps[:3]]
        mine.step()
        want_norm = torch.nn.utils.clip_grad_norm_(shadow, 5.0)
        ref.step()
        got_norm = mine.last_grad_norm().item()
        assert abs(got_norm - want_norm.item()) <= 1e-5 * want_norm.item(), (step, got_norm, want_norm.item())
        assert abs(got_norm - target) <= 10 * U * target + 1e-6 * target
        for p, b in zip(ps[:3], before):
            assert torch.equal(p.grad, b)                                # .grad is not rewritten
        for k, (p, s) in enumerate(zip(ps, shadow)):
            assert torch.allclose(p, s, rtol=RTOL, atol=ATOL), (step, k, (p - s).abs().max().item())
    for p, s in zip(ps, shadow):
        for k in ('exp_avg', 'exp_avg_sq'):
            assert torch.allclose(mine.state[p][k], ref.state[s][k], rtol=RTOL, atol=ATOL)


def test_optim_adam_max_grad_norm_state_dict_round_trip_with_torch():
    o = optim()
    g = torch.Generator(device=DEV).manual_seed(9)
    shapes = [(64, 3, 7), (64,), (1,), (4097,), (600, 700)]
    ps = [torch.randn(s, device=DEV, generator=g).requires_grad_(True) for s in shapes]
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]
    mine = o.Adam([{'params': ps[:2]}, {'params': ps[2:], 'lr': 5e-3}], LR, weight_decay=WD, max_grad_norm=5.0)
    for step in range(2):
        set_grads(ps, shadow, step, 12.0)
        mine.step()
    with torch.no_grad():
        for p, s in zip(ps, shadow):
            s.copy_(p)
    ref = torch.optim.Adam([{'params': shadow[:2]}, {'params': shadow[2:], 'lr': 5e-3}], LR, weight_decay=WD)
    ref.load_state_dict(copy.deepcopy(mine.state_dict()))
    mine2 = o.Adam([{'params': ps[:2]}, {'params': ps[2:]}], LR, weight_decay=WD, max_grad_norm=5.0)
    mine2.load_state_dict(copy.deepcopy(ref.state_dict()))
    for step in range(2, 4):
        set_grads(ps, shadow, step, 12.0 if step == 2 else 2.0)
        mine2.step()
        torch.nn.utils.clip_grad_norm_(shadow, 5.0)
        ref.step()
        for p, s in zip(ps, shadow):
            assert torch.allclose(p, s, rtol=RTOL, atol=ATOL)
    assert mine2.state[ps[0]]['step'].item() == 4


def test_optim_adam_refused_step_changes_nothing_and_last_norm_is_kept():
    """A group refused after a valid one leaves every group's state and step count as they were; a norm returned by
    last_grad_norm() keeps its value through later steps."""
    o = optim()
    p = torch.randn(4097, device=DEV).requires_grad_(True)
    q = torch.zeros(3, requires_grad=True)                     # a CPU parameter in the second group
    p.grad, q.grad = torch.randn(4097, device=DEV), torch.ones(3)
    before = p.detach().clone()
    opt = o.Adam([{'params': [p]}, {'params': [q]}], LR, weight_decay=WD, max_grad_norm=5.0)
    with pytest.raises(L().Dirb200Error, match="CUDA"):
        opt.step()
    assert len(opt.state) == 0 and torch.equal(p.detach(), before) and opt.last_grad_norm() is None
    opt = o.Adam([p], LR, weight_decay=WD, max_grad_norm=5.0)
    p.grad = torch.full((4097,), 0.5, device=DEV)
    opt.step()
    first = opt.last_grad_norm()
    want = first.item()
    p.grad = torch.full((4097,), 0.01, device=DEV)
    opt.step()
    assert first.item() == want and opt.last_grad_norm().item() != want
    assert abs(want - 0.5 * 4097 ** 0.5) <= 10 * U * want


# ---------------------------------------------------------------------------------------------- shot metrics
def kernel_metrics(pred, label):
    import stsb_data
    return stsb_data.shot_metrics(torch.from_numpy(np.ascontiguousarray(pred, dtype=np.float32)).to(DEV),
                                  torch.from_numpy(np.ascontiguousarray(label, dtype=np.float32)).to(DEV))


@pytest.mark.parametrize("case", CASES)
def test_shot_metrics_against_the_reference_fixture(case):
    z = golden("stsb_metrics")
    got = kernel_metrics(z[f"{case}:pred"], z[f"{case}:label"])
    assert_metrics(got, z[f"{case}:want"], case)
    assert np.array_equal(got, kernel_metrics(z[f"{case}:pred"], z[f"{case}:label"]), equal_nan=True)


@pytest.mark.parametrize("n,seed", [(0, 0), (1, 1), (2, 2), (257, 3), (5000, 4), (20000, 5)])
def test_shot_metrics_against_float64_oracle_on_random_inputs(n, seed):
    rs = np.random.RandomState(seed)
    label = np.where(rs.uniform(size=n) < 0.3, np.round(rs.uniform(0, 5, n) * 5) / 5, rs.uniform(0, 5, n))
    label = label.astype(np.float32)
    label[:n // 50] = 5.0
    pred = np.round(label / 5 + rs.normal(0, 0.2, n), 2).astype(np.float32)
    assert_metrics(kernel_metrics(pred, label), shot_metrics_oracle(pred, label), f"n={n}")


def test_sts_shot_average_interface():
    import stsb_data
    z = golden("stsb_metrics")
    pred, label = z["random:pred"], z["random:label"]
    scorer = stsb_data.STSShotAverage(metric=['mse', 'l1', 'gmean', 'pearsonr', 'spearmanr'])
    for lo in range(0, pred.size, 128):
        scorer(pred[lo:lo + 128], label[lo:lo + 128])
    m = scorer.get_metric()
    want = z["random:want"]
    for row, shot in enumerate(stsb_data.SHOTS):
        assert list(m[shot]) == ['mse', 'l1', 'gmean', 'pearsonr', 'spearmanr', 'num_samples']
        assert m[shot]['num_samples'] == int(want[row, 0])
        for col, k in enumerate(stsb_data.METRICS[1:], start=1):
            assert abs(m[shot][k] - want[row, col]) <= 1e-12 * max(abs(want[row, col]), 1.0), (shot, k)
    assert scorer.get_metric(reset=True, type='overall') == m['overall']
    assert scorer.get_metric(type='overall')['num_samples'] == 0                  # reset empties it
    scorer(pred[:10], label[:10])
    only = stsb_data.STSShotAverage(metric=['mse'])
    only(pred[:10], label[:10])
    assert set(only.get_metric()['many']) == {'mse', 'num_samples'}
    assert scorer.get_metric()['overall']['mse'] == only.get_metric()['overall']['mse']


# ------------------------------------------------------------------------------------------------- few SMs
@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_stsb_train_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process)."""
    if os.environ.get("DIRB200_STSB_TRAIN_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_STSB_TRAIN_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
