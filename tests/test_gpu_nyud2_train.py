"""GPU checks of the multi-tensor Adam (dirb200_adam_step_multi, optim.Adam) and of the NYUD2-DIR training driver
(nyud2_train.py, nyud2-dir/train.py) with its test.py entry point (depth_eval.main).

- Kernel: one segment over a flat buffer, and awkward tensor lists (odd sizes, views at 4-byte offsets, more tensors
  than one launch takes), against dirb200_adam_step over the flat buffer: exp_avg and exp_avg_sq the same bits, the
  parameter within the rounding of step_size * m / denom (the multi-tensor kernel writes p -= step_size * q as one fma;
  the flat kernel's compiler fuses it for some float4 lanes and not for others).
- optim.Adam against torch.optim.Adam(weight_decay=1e-4) to FusedAdam's bound (rtol 1e-5, atol 1e-7): 5 steps, grad=None
  skipped, an lr change and two groups, state_dict both ways; 3 steps on net.model with shared gradients.
- The driver end to end on a synthetic NYUD2 directory: checkpoints and their keys, the FDS refresh in the reference's
  order, --resume, --retrain_fc --pretrained, --backbone_weights, and depth_eval.main reproducing the stored metrics.
The file reruns itself with DIRB200_SMS=7."""
import copy
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from util import golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LR, B1, B2, EPS = 1e-3, 0.9, 0.999, 1e-8
RTOL, ATOL = 1e-5, 1e-7                       # FusedAdam's bound (test_train_step_fused_adam_matches_torch_adam)


def optim():
    import optim as o
    return o


def _lib():
    import _lib as L
    import resnet  # noqa: F401  (binds dirb200_adam_step)
    return L


def flat_state(n, seed):
    """p, g, m, v fp32 [n]: m, v as after a few steps (v > 0)."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    p = torch.randn(n, device=DEV, generator=g)
    gr = torch.randn(n, device=DEV, generator=g) * 0.1
    m = torch.randn(n, device=DEV, generator=g) * 0.01
    v = torch.rand(n, device=DEV, generator=g) * 1e-3
    return [p, gr, m, v]


def flat_step(bufs, step, wd):
    L = _lib()
    p, g, m, v = bufs
    L.call("dirb200_adam_step", L.ptr(p), L.ptr(g), L.ptr(m), L.ptr(v), p.numel(), LR, B1, B2, EPS, wd, step, 1.0,
           None, L.stream_ptr())


def same_as_flat(flat, multi, step, what):
    """m, v bit for bit; p within |fma(-s, q, p) - (p - fl(s q))| <= ulp(p) + ulp(s q), |q| = |m / denom| < 16 here."""
    s = LR / (1.0 - np.float32(B1) ** step)
    for x, y, name in zip(flat, multi, "pgmv"):
        if name == "p":
            tol = torch.abs(x) * 2.0 ** -23 + float(np.spacing(np.float32(16 * s)))
            bad = ~((x - y).abs() <= tol)
            assert not bad.any(), (what, name, int(bad.sum()), (x - y).abs().max().item())
        else:
            assert torch.equal(x, y), (what, name)


def multi_step(segs, step, wd):
    """segs: [(p, g, m, v)] views; one dirb200_adam_step_multi call."""
    L, o = _lib(), optim()
    t = np.empty(len(segs), dtype=o._SEGMENT)
    for k, name in enumerate(('param', 'grad', 'exp_avg', 'exp_avg_sq')):
        t[name] = [s[k].data_ptr() for s in segs]
    t['numel'] = [s[0].numel() for s in segs]
    t['bc1'], t['bc2_sqrt'] = o._bias_corrections(B1, B2, step)
    L.call("dirb200_adam_step_multi", t.ctypes.data_as(L.P), len(segs), LR, B1, B2, EPS, wd, L.stream_ptr())


@pytest.mark.parametrize("wd", [0.0, 1e-4])
@pytest.mark.parametrize("step", [1, 7])
def test_one_segment_equals_flat_step(step, wd):
    n = (1 << 20) + 4099
    a = flat_state(n, seed=step)
    b = [t.clone() for t in a]
    flat_step(a, step, wd)
    multi_step([tuple(b)], step, wd)
    torch.cuda.synchronize()
    same_as_flat(a, b, step, "one segment")


def tile(bufs, sizes, offset):
    """Views of consecutive `sizes` into each flat buffer, starting at element `offset`."""
    segs, at = [], offset
    for n in sizes:
        segs.append(tuple(t[at:at + n] for t in bufs))
        at += n
    return segs, at


LISTS = {
    "odd-sizes-aligned": ([1, 3, 5, 4097, (1 << 20) + 1], 0),
    "odd-sizes-at-4B-offset": ([1, 3, 5, 4097, (1 << 20) + 1, 8, 4096], 1),
    "at-8B-offset": ([4096, 12, 8193], 2),
    "1100-tensors-3-launches": (list(np.random.RandomState(0).randint(1, 3000, 1100)), 3),
}


@pytest.mark.parametrize("name", list(LISTS))
def test_tensor_lists_equal_flat_step(name):
    sizes, offset = LISTS[name]
    total = offset + int(sum(sizes))
    a = flat_state(total, seed=len(sizes))
    b = [t.clone() for t in a]
    flat_step(a, 3, 1e-4)
    segs, end = tile(b, [int(s) for s in sizes], offset)
    assert end == total
    multi_step(segs, 3, 1e-4)
    torch.cuda.synchronize()
    same_as_flat([x[offset:] for x in a], [y[offset:] for y in b], 3, name)
    for y, x0 in zip(b, flat_state(total, seed=len(sizes))):       # nothing before the first view is touched
        assert torch.equal(y[:offset], x0[:offset])


# ------------------------------------------------------------------------------------------ optim.Adam vs torch
SHAPES = [(64, 3, 7, 7), (64,), (1,), (3,), (5, 5), (4097,), (128, 128, 5, 5)]


def make_params(seed=0, views=True):
    """A list of CUDA fp32 leaf tensors; with `views`, some are views into one flat buffer at 4-byte offsets."""
    g = torch.Generator(device=DEV).manual_seed(seed)
    ps = [torch.randn(s, device=DEV, generator=g).requires_grad_(True) for s in SHAPES]
    if views:
        flat = torch.randn(1 + 3 + 5 + 4097, device=DEV, generator=g)
        for lo, n in ((1, 3), (4, 5), (9, 4097)):
            v = flat[lo:lo + n].detach()
            v.requires_grad_(True)
            ps.append(v)
    return ps


def set_grads(ps, shadow, seed, skip=()):
    g = torch.Generator(device=DEV).manual_seed(1000 + seed)
    for k, (p, s) in enumerate(zip(ps, shadow)):
        if k in skip:
            p.grad = s.grad = None
            continue
        gr = torch.randn(p.shape, device=DEV, generator=g) * 0.1
        p.grad, s.grad = gr.clone(), gr.clone()


def assert_close(ps, shadow):
    for k, (p, s) in enumerate(zip(ps, shadow)):
        assert torch.allclose(p, s, rtol=RTOL, atol=ATOL), (k, (p - s).abs().max().item())


def test_matches_torch_adam_over_5_steps():
    ps = make_params()
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]
    mine, ref = optim().Adam(ps, LR, weight_decay=1e-4), torch.optim.Adam(shadow, LR, weight_decay=1e-4)
    for step in range(5):
        set_grads(ps, shadow, step)
        mine.step()
        ref.step()
        assert_close(ps, shadow)
    for p, s in zip(ps, shadow):
        for k in ('exp_avg', 'exp_avg_sq'):
            assert torch.allclose(mine.state[p][k], ref.state[s][k], rtol=RTOL, atol=ATOL)
        assert mine.state[p]['step'].item() == 5 and mine.state[p]['step'].device.type == 'cpu'


def test_grad_none_is_skipped_and_its_step_does_not_advance():
    ps = make_params(1)
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]
    mine, ref = optim().Adam(ps, LR, weight_decay=1e-4), torch.optim.Adam(shadow, LR, weight_decay=1e-4)
    before = ps[2].detach().clone()
    set_grads(ps, shadow, 0, skip=(2,))
    mine.step()
    ref.step()
    assert ps[2] not in mine.state and torch.equal(ps[2].detach(), before)
    set_grads(ps, shadow, 1, skip=(0,))
    mine.step()
    ref.step()
    assert mine.state[ps[0]]['step'].item() == 1 and mine.state[ps[2]]['step'].item() == 1
    assert mine.state[ps[1]]['step'].item() == 2
    set_grads(ps, shadow, 2)
    mine.step()
    ref.step()
    assert_close(ps, shadow)


def test_lr_change_and_two_groups():
    ps = make_params(2)
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]

    def groups(t):
        return [{'params': t[:4]}, {'params': t[4:], 'lr': 5e-3, 'weight_decay': 0.0}]

    mine, ref = optim().Adam(groups(ps), LR, weight_decay=1e-4), torch.optim.Adam(groups(shadow), LR, weight_decay=1e-4)
    for step in range(4):
        if step == 2:
            for opt in (mine, ref):
                for gr in opt.param_groups:
                    gr['lr'] *= 0.1
        set_grads(ps, shadow, step)
        mine.step()
        ref.step()
        assert_close(ps, shadow)
    assert mine.param_groups[0]['lr'] == pytest.approx(LR * 0.1) and mine.param_groups[1]['lr'] == pytest.approx(5e-4)


def test_state_dict_round_trip_with_torch_adam():
    o = optim()
    ps = make_params(3)
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]
    mine = o.Adam(ps, LR, weight_decay=1e-4)
    for step in range(2):
        set_grads(ps, shadow, step)
        mine.step()
    with torch.no_grad():
        for p, s in zip(ps, shadow):
            s.copy_(p)
    ref = torch.optim.Adam(shadow, LR, weight_decay=1e-4)
    ref.load_state_dict(copy.deepcopy(mine.state_dict()))    # ours -> torch (a copy: load_state_dict keeps tensors)
    for step in range(2, 4):
        set_grads(ps, shadow, step)
        mine.step()
        ref.step()
        assert_close(ps, shadow)
    # torch -> ours: a fresh optim.Adam continues where torch's is
    ps2 = [s.detach().clone().requires_grad_(True) for s in shadow]
    mine2 = o.Adam(ps2, LR, weight_decay=1e-4)
    mine2.load_state_dict(copy.deepcopy(ref.state_dict()))
    assert set(mine2.state_dict()['state'][0]) == set(ref.state_dict()['state'][0]) == {'step', 'exp_avg', 'exp_avg_sq'}
    for step in range(4, 6):
        set_grads(ps2, shadow, step)
        mine2.step()
        ref.step()
        assert_close(ps2, shadow)


def test_net_model_three_steps_match_torch_adam():
    """net.model's 245 parameters (E's views into the ResNet's flat buffer, D / MFF / R's own tensors) with shared
    gradients: optim.Adam against torch.optim.Adam(weight_decay=1e-4) over 3 steps."""
    from test_gpu_nyud2_model import inputs, loss_fn, make_model
    m = make_model(True)
    m.train()
    ps = list(m.parameters())
    assert len(ps) == 245 and sum(p.numel() for p in ps) == 67569473
    opt = optim().Adam(ps, 1e-4, weight_decay=1e-4)
    shadow = [p.detach().clone().requires_grad_(True) for p in ps]
    ref = torch.optim.Adam(shadow, 1e-4, weight_decay=1e-4)
    x, depth, weight = inputs(2, 228, 304, seed=11)
    for step in range(3):
        opt.zero_grad()
        out, _ = m(x, depth, 0)
        loss = loss_fn(out, depth, weight)
        loss.backward()
        for s, p in zip(shadow, ps):
            s.grad = p.grad.detach().clone()
        opt.step()
        ref.step()
        assert torch.isfinite(loss)
        for k, (s, p) in enumerate(zip(shadow, ps)):
            assert torch.allclose(s, p, rtol=RTOL, atol=ATOL), (step, k)


# ------------------------------------------------------------------------------------------ the driver
N_FDS, H, W = 4, 114, 152


@pytest.fixture(scope="module")
def run(tmp_path_factory):
    """One 3-epoch --fds --lds --reweight inverse run on a synthetic NYUD2 directory, with the FDS state before each
    collection pass and the collected (feature, depth) batches captured."""
    from fds_variants import FDSDepth
    import nyud2_train
    from test_gpu_nyud2_input_pipeline import write_dataset
    base = tmp_path_factory.mktemp("nyud2")
    data = str(base / "data")
    write_dataset(data, n_train=6, n_test=4)
    passes = []
    begin, acc = FDSDepth.begin_epoch_stats, FDSDepth.accumulate_map

    def spy_begin(self, labels):
        passes.append({'before': copy.deepcopy(self.state_dict()), 'feature': [], 'depth': []})
        return begin(self, labels)

    def spy_acc(self, features, labels):
        passes[-1]['feature'].append(features.float().clone())
        passes[-1]['depth'].append(labels.clone())
        return acc(self, features, labels)

    argv = ['--data_dir', data, '--store_root', str(base / "ckpt"), '--epochs', '3', '--fds', '--lds', '--reweight',
            'inverse', '--batch_size', '4', '--workers', '0']
    FDSDepth.begin_epoch_stats, FDSDepth.accumulate_map = spy_begin, spy_acc
    try:
        torch.manual_seed(0)
        nyud2_train.main(argv)
    finally:
        FDSDepth.begin_epoch_stats, FDSDepth.accumulate_map = begin, acc
    store = os.path.join(str(base / "ckpt"), nyud2_train.store_name(nyud2_train.build_parser().parse_args(argv)))
    return dict(data=data, base=base, argv=argv, store=store, passes=passes)


def load(path):
    return torch.load(path, map_location='cpu')


def test_driver_writes_the_reference_checkpoints(run):
    names = ['module.' + str(n) for n in golden("nyud2_model")["names"]]
    for f in ('checkpoint.pth.tar', 'checkpoint_best.pth.tar', 'checkpoint_final.pth.tar'):
        ck = load(os.path.join(run['store'], f))
        assert set(ck) == {'state_dict', 'epoch', 'error', 'metric'}, f
        assert list(ck['state_dict']) == names, f
        assert set(ck['metric']) == {'overall', 'many', 'medium', 'few'} and ck['error'] == ck['metric']['overall']['RMSE']
    final = load(os.path.join(run['store'], 'checkpoint_final.pth.tar'))
    assert final['epoch'] == 2
    sd = final['state_dict']
    assert sd['module.R.FDS.epoch'].item() == 2
    assert sd['module.R.FDS.num_samples_tracked'].double().sum().item() == 3 * N_FDS * H * W
    assert os.path.isfile(os.path.join(run['store'], 'training_log.log'))
    assert len(run['passes']) == 3 and all(sum(f.shape[0] for f in p['feature']) == N_FDS for p in run['passes'])


def test_fds_refresh_in_the_reference_order(run):
    """The last epoch's collected features replayed through a copy of the pre-pass FDSDepth in nyud2-dir/train.py's
    order -- update_last_epoch_stats(epoch), then one update_running_stats over all of them -- give the driver's 8
    buffers."""
    from fds_variants import FDSDepth
    p = run['passes'][2]
    ref = FDSDepth(feature_dim=128, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1, kernel='gaussian',
                   ks=5, sigma=2, momentum=0.9).to(DEV)
    ref.load_state_dict(p['before'])
    ref.update_last_epoch_stats(2)
    ref.update_running_stats(torch.cat(p['feature']), torch.cat(p['depth']), 2)
    got = load(os.path.join(run['store'], 'checkpoint_final.pth.tar'))['state_dict']
    want = ref.state_dict()
    assert len(want) == 8
    for k, v in want.items():
        g = got['module.R.FDS.' + k].to(DEV)
        assert torch.allclose(g, v, rtol=1e-5, atol=1e-5), (k, (g - v).abs().max().item())


def test_eval_entry_point_reproduces_the_stored_metrics(run):
    import depth_eval
    ckpt = os.path.join(run['store'], 'checkpoint.pth.tar')
    rmse, metric = depth_eval.main(['--eval_model', ckpt, '--data_dir', run['data']])
    stored = load(ckpt)['metric']
    assert set(metric) == set(stored)
    for shot in stored:
        for k, v in stored[shot].items():
            if k == 'NUM':
                assert metric[shot][k] == v, (shot, k)
            else:                                    # the fp64 accumulator is summed with atomics: order only
                assert metric[shot][k] == pytest.approx(v, rel=1e-12, abs=0, nan_ok=True), (shot, k)


def test_resume_continues_at_the_next_epoch(run):
    import nyud2_train
    nyud2_train.main(run['argv'][:run['argv'].index('--epochs')] + ['--epochs', '4', '--resume'] +
                     run['argv'][run['argv'].index('--epochs') + 2:])
    assert load(os.path.join(run['store'], 'checkpoint.pth.tar'))['epoch'] == 3
    with open(os.path.join(run['store'], 'training_log.log')) as f:
        log = f.read()
    assert 'Epoch: [3][0/2]' in log and log.count('Epoch: [0][0/2]') == 1


def test_retrain_fc_changes_only_R(run):
    import nyud2_train
    pre = os.path.join(run['store'], 'checkpoint_final.pth.tar')
    argv = ['--data_dir', run['data'], '--store_root', str(run['base'] / "rrt"), '--epochs', '1', '--batch_size', '4',
            '--workers', '0', '--retrain_fc', '--pretrained', pre]
    model = nyud2_train.main(argv)
    before = load(pre)['state_dict']
    changed = 0
    for name, p in model.named_parameters():
        b = before['module.' + name].to(DEV)
        if 'R' in name:
            changed += not torch.equal(p.detach(), b)
        else:
            assert torch.equal(p.detach(), b), name
    assert changed == len([n for n, _ in model.named_parameters() if 'R' in n])


def test_backbone_weights_load_E_exactly(tmp_path):
    import nyud2_train
    import resnet
    torch.manual_seed(5)
    src = resnet.E_resnet(resnet.resnet50()).state_dict()
    sd = {k: v.clone() for k, v in src.items()}
    sd['fc.weight'], sd['fc.bias'] = torch.randn(1000, 2048), torch.randn(1000)
    path = str(tmp_path / "resnet50.pth")
    torch.save(sd, path)
    args = nyud2_train.build_parser().parse_args(['--backbone_weights', path])
    torch.manual_seed(6)
    model = nyud2_train.define_model(args).cuda()
    got = model.E.state_dict()
    assert list(got) == list(src)
    for k, v in src.items():
        assert torch.equal(got[k].cpu(), v), k


# ------------------------------------------------------------------------------------------------- few SMs
@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_train_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process)."""
    if os.environ.get("DIRB200_TRAIN_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_TRAIN_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
