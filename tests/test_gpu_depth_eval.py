"""GPU parity of the NYUD2-DIR depth evaluation (dirb200_depth_metrics_accumulate through depth_eval.py).

The flat path is checked against the fixture of the reference's own Evaluator (tests/golden/make_golden_depth_eval.py):
counts and DELTA exact, MSE / MAE / ABS_REL within 1e-6 (the reference sums in fp32), LG10 within 1e-5 (per-element
logf may differ by an ulp between torch CPU and CUDA).  The fused up-sample + mask form is checked against what
test.py does on the GPU -- torch CUDA F.interpolate(align_corners=True), boolean indexing -- reduced by the numpy
oracle: every count exact (so the in-register interpolation is ATen's to the bit), sums within 1e-12, LG10 1e-6.
The file is also meant to run with DIRB200_SMS=7 (few CTAs, many partials per finishing CTA)."""
import logging

import numpy as np
import pytest
import torch
import torch.nn.functional as F
from util import golden
from oracle import depth_oracle as O
from test_depth_eval_cpu import check_rows, rows, shot_idx

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda")
COUNT_COLS = [0, 5, 6, 7, 8, 9]
SUM_COLS = [1, 2, 3]


def _ev(g):
    from depth_eval import Evaluator
    return Evaluator(shot_idx(g))


def _cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


@pytest.mark.parametrize("case", ["a", "d"])
def test_flat_path_matches_reference_evaluate_shot(case):
    g = golden("depth_eval")
    ev = _ev(g)
    o, t = _cuda(g[f"{case}_output"]), _cuda(g[f"{case}_target"])
    chunks = g["a_chunks"].tolist() if case == "a" else [t.numel()]
    lo = 0
    for k in chunks:
        ev(o[lo:lo + k], t[lo:lo + k])
        lo += k
    check_rows(rows(ev.evaluate_shot()), g[f"{case}_ref"], lg10_rtol=1e-5, what=case)


def test_flat_evaluate_matches_reference_with_nan_targets():
    from depth_eval import Evaluator
    g = golden("depth_eval")
    md = Evaluator.evaluate(_cuda(g["c_output"]), _cuda(g["c_target"]))
    check_rows(rows({"overall": md}, ("overall",)), g["c_ref"], lg10_rtol=1e-5, what="c")


def test_stored_test_time_vectors_match_reference():
    g = golden("depth_eval")
    ev = _ev(g)
    ev(_cuda(g["b_output"]), _cuda(g["b_target"]))
    check_rows(rows(ev.evaluate_shot()), g["b_ref"], lg10_rtol=1e-5, what="b")


def _real_masks(n):
    g = golden("depth_eval")
    shape = tuple(g["b_mask_shape"].tolist())
    m = np.unpackbits(g["b_masks"])[: int(np.prod(shape))].reshape(shape).astype(bool)
    return torch.from_numpy(m[np.arange(n) % shape[0]]).to(DEV)[:, None]


def _synthetic(n, seed):
    """NYUD2 test-set-shaped data: 16-bit mm depths / 1000 at 228 x 304 (a few NaN holes), smooth positive
    predictions at 114 x 152."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    yy = torch.arange(228, device=DEV, dtype=torch.float32)[:, None]
    xx = torch.arange(304, device=DEV, dtype=torch.float32)[None, :]
    a = torch.rand(n, 1, 1, device=DEV, generator=gen) * 0.04 + 0.01
    b = torch.rand(n, 1, 1, device=DEV, generator=gen) * 0.04 + 0.01
    mm = 5200 + 4700 * torch.sin(a * yy + b * xx) * torch.cos(0.013 * xx - a * yy)
    mm = (mm + torch.randn(n, 228, 304, device=DEV, generator=gen) * 40).round().clamp(1, 10500)
    depth = (mm.to(torch.int32).to(torch.float32) / 1000)[:, None].contiguous()
    depth.view(-1)[::997] = float("nan")
    py, px = yy[:114], xx[:, :152]
    pred = 5.0 + 4.6 * torch.sin(2 * a * py + 2 * b * px + 0.3) * torch.cos(0.026 * px - 2 * a * py)
    return pred[:, None].contiguous(), depth


def _reference_style(pred, depth, mask, shot):
    """test.py:52-54 on the GPU (torch CUDA interpolate, boolean indexing) reduced by the numpy oracle."""
    up = F.interpolate(pred, size=[depth.size(2), depth.size(3)], mode="bilinear", align_corners=True)
    return O.depth_metrics(up[mask].cpu().numpy(), depth[mask].cpu().numpy(), shot)[0]


def _fused(ev, pred, depth, mask, batch):
    ev.reset()
    for lo in range(0, pred.shape[0], batch):
        ev.add(pred[lo:lo + batch], depth[lo:lo + batch], mask[lo:lo + batch])
    return ev.counts_and_sums().cpu().numpy()


def _check_acc(got, want, what):
    assert np.array_equal(got[:, COUNT_COLS], want[:, COUNT_COLS]), (what, got[:, COUNT_COLS], want[:, COUNT_COLS])
    assert np.allclose(got[:, SUM_COLS], want[:, SUM_COLS], rtol=1e-12, atol=0), (what, got, want)
    assert np.allclose(got[:, 4], want[:, 4], rtol=1e-6, atol=0), (what, got[:, 4], want[:, 4])


@pytest.mark.parametrize("n,mask_kind", [(32, "real"), (654, "real"), (654, "ones")])
def test_fused_add_matches_torch_interpolate_and_indexing(n, mask_kind):
    g = golden("depth_eval")
    pred, depth = _synthetic(n, seed=n)
    mask = _real_masks(n) if mask_kind == "real" else torch.ones_like(depth, dtype=torch.bool)
    want = _reference_style(pred, depth, mask, shot_idx(g))
    assert want[0, 8] > 0 and all(want[k, 0] > 0 for k in range(4))
    ev = _ev(g)
    for batch in (1, 8):
        _check_acc(_fused(ev, pred, depth, mask, batch), want, f"{n} {mask_kind} batch {batch}")


def test_fused_add_same_size_copies_and_handles_odd_shapes():
    """Equal sizes copy the prediction (ATen's shortcut; inf / NaN predictions pass through), and a 1-row / 1-column
    output uses scale 0; mask None selects every pixel."""
    g = golden("depth_eval")
    ev = _ev(g)
    gen = torch.Generator(device=DEV).manual_seed(3)
    for (ph, pw, h, w) in ((17, 23, 17, 23), (5, 7, 1, 9), (5, 7, 13, 1), (3, 2, 40, 61)):
        pred = torch.rand(3, 1, ph, pw, device=DEV, generator=gen) * 9 + 0.2
        pred.view(-1)[::11] = float("inf")
        depth = torch.rand(3, 1, h, w, device=DEV, generator=gen) * 9 + 0.2
        mask = torch.rand(3, 1, h, w, device=DEV, generator=gen) < 0.5
        for m in (mask, None):
            ev.reset()
            ev.add(pred, depth, m)
            got = ev.counts_and_sums().cpu().numpy()
            want = _reference_style(pred, depth, m if m is not None else torch.ones_like(mask), shot_idx(g))
            assert np.array_equal(np.isnan(got), np.isnan(want)), (ph, pw, h, w)
            fin = np.isfinite(want)
            assert np.array_equal(got[~fin], want[~fin], equal_nan=True) and np.array_equal(got[:, COUNT_COLS], want[:, COUNT_COLS])
            assert np.allclose(got[fin], want[fin], rtol=1e-6, atol=0), (ph, pw, h, w, got, want)


def test_two_identical_evaluations_are_bit_identical():
    g = golden("depth_eval")
    pred, depth = _synthetic(654, seed=11)
    mask = torch.ones_like(depth, dtype=torch.bool)
    ev = _ev(g)
    a = _fused(ev, pred, depth, mask, 8)
    b = _fused(ev, pred, depth, mask, 8)
    assert a.tobytes() == b.tobytes()
    ev.reset()
    ev(pred.reshape(-1), pred.reshape(-1) * 1.1)
    ev(pred.reshape(-1), pred.reshape(-1) * 1.1)
    c = ev.counts_and_sums().cpu().numpy().copy()
    ev.reset()
    ev(pred.reshape(-1), pred.reshape(-1) * 1.1)
    ev(pred.reshape(-1), pred.reshape(-1) * 1.1)
    assert c.tobytes() == ev.counts_and_sums().cpu().numpy().tobytes()


def test_evaluate_shot_raises_on_nan_or_inf_targets_and_evaluate_does_not():
    from depth_eval import Evaluator
    g = golden("depth_eval")
    o = torch.full((4,), 2.0, device=DEV)
    for bad, exc in ((float("nan"), ValueError), (float("inf"), OverflowError), (float("-inf"), OverflowError)):
        t = torch.tensor([1.0, 2.0, bad, 3.0], device=DEV)
        ev = _ev(g)
        ev(o, t)
        with pytest.raises(exc):
            ev.evaluate_shot()
        with pytest.raises(exc):
            Evaluator.get_bin_idx(np.float32(bad))
        md = Evaluator.evaluate(o, t)
        assert md["NUM"] == (3 if bad != bad else 4)
    ev = _ev(g)
    md = ev.evaluate_shot()                          # nothing accumulated: every group all 0, as the reference
    assert all(md[s][m] == 0 for s in md for m in md[s])


class _TinyDepthNet(torch.nn.Module):
    """A deterministic stand-in for the NYUD2 model: 3-channel 228 x 304 input -> positive 1-channel 114 x 152 map."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(0)
        self.conv = torch.nn.Conv2d(3, 1, 3, padding=1)
        with torch.no_grad():
            self.conv.weight.copy_(torch.randn(1, 3, 3, 3, generator=g) * 0.2)
            self.conv.bias.fill_(0.1)

    def forward(self, x):
        return F.softplus(F.avg_pool2d(self.conv(x), 2)) * 4 + 0.3


def test_test_loop_matches_reference_style_loop(caplog):
    import depth_eval
    g = golden("depth_eval")
    shot = shot_idx(g)
    model = _TinyDepthNet().to(DEV)
    gen = torch.Generator().manual_seed(5)
    masks = _real_masks(12).cpu()
    _, depth = _synthetic(12, seed=5)
    depth = depth.cpu()
    loader = [{"image": torch.rand(b, 3, 228, 304, generator=gen), "depth": depth[lo:lo + b].clone(),
               "mask": masks[lo:lo + b].clone()} for lo, b in ((0, 1), (1, 3), (4, 8))]
    for s in loader:
        s["depth"][torch.isnan(s["depth"])] = 1.0        # evaluate_shot refuses NaN depths, as the reference does
    with caplog.at_level(logging.INFO):
        rmse, md = depth_eval.test(loader, model, shot)
    assert "***** TEST RESULTS *****" in caplog.text and " * Few: RMSE" in caplog.text
    outs, tgts = [], []
    with torch.no_grad():
        for s in loader:
            d = s["depth"].to(DEV)
            out = F.interpolate(model(s["image"].to(DEV)), size=[d.size(2), d.size(3)], mode="bilinear",
                                align_corners=True)
            m = s["mask"].to(DEV)
            outs.append(out[m].cpu().numpy())
            tgts.append(d[m].cpu().numpy())
    _, want = O.depth_metrics(np.concatenate(outs), np.concatenate(tgts), shot)
    check_rows(rows(md), rows(want), rtol=1e-12, lg10_rtol=1e-6, what="test()")
    assert rmse == md["overall"]["RMSE"] and md["overall"]["NUM"] == int(sum(x.size for x in tgts))


def test_one_launch_per_add():
    import _lib
    g = golden("depth_eval")
    pred, depth = _synthetic(16, seed=2)
    mask = _real_masks(16)
    ev = _ev(g)
    ev.add(pred[:1], depth[:1], mask[:1])             # allocations happen here
    before = _lib.launch_count()
    for lo in range(0, 16, 4):
        ev.add(pred[lo:lo + 4], depth[lo:lo + 4], mask[lo:lo + 4])
    assert _lib.launch_count() - before == 4
