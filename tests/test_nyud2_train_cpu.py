"""CPU checks of the NYUD2-DIR training driver (nyud2_train.py, a mirror of nyud2-dir/train.py), depth_eval's test.py
table, and the host-side refusals of the multi-tensor Adam (dirb200_adam_step_multi, optim.Adam).  Every device pointer
below is a dummy that must never be dereferenced: a call that got past its checks would fault on a GPU machine and
fail without one."""
import ctypes

import numpy as np
import pytest
import torch

from util import golden

D = 16                                 # stands for a device buffer (16-byte aligned)

# nyud2-dir/train.py:18-56: flag -> default
REFERENCE_DEFAULTS = {
    'epochs': 10, 'start_epoch': 0, 'lr': 0.0001, 'weight_decay': 1e-4, 'batch_size': 32, 'store_root': 'checkpoint',
    'store_name': 'nyud2', 'data_dir': './data', 'resume': False,
    'lds': False, 'lds_kernel': 'gaussian', 'lds_ks': 5, 'lds_sigma': 2,
    'fds': False, 'fds_kernel': 'gaussian', 'fds_ks': 5, 'fds_sigma': 2, 'start_update': 0, 'start_smooth': 1,
    'bucket_num': 100, 'bucket_start': 7, 'fds_mmt': 0.9,
    'reweight': 'none', 'retrain_fc': False, 'pretrained': '',
}
EXTRA_DEFAULTS = {'workers': 8, 'print_freq': 1, 'gpu': 0, 'backbone_weights': ''}


def parse(*argv):
    import nyud2_train
    return nyud2_train.build_parser().parse_args(list(argv))


def test_parser_flags_and_defaults_are_the_reference():
    args = vars(parse())
    assert args == {**REFERENCE_DEFAULTS, **EXTRA_DEFAULTS}
    # the literal defaults keep their Python types (they decide the store name)
    assert type(args['lds_sigma']) is int and type(args['fds_sigma']) is int and type(args['fds_mmt']) is float
    assert parse('--learning-rate', '0.5').lr == 0.5 and parse('--wd', '0.5').weight_decay == 0.5
    for flag, bad in (('--lds_kernel', 'box'), ('--fds_kernel', 'box'), ('--reweight', 'sqrt')):
        with pytest.raises(SystemExit):
            parse(flag, bad)


@pytest.mark.parametrize("argv,want", [
    ((), 'nyud2_lr_0.0001_bs_32'),
    (('--reweight', 'inverse'), 'nyud2_inverse_lr_0.0001_bs_32'),
    (('--lds', '--reweight', 'inverse'), 'nyud2_lds_gau_5_2_lr_0.0001_bs_32'),
    (('--lds', '--reweight', 'inverse', '--lds_sigma', '2'), 'nyud2_lds_gau_5_2.0_lr_0.0001_bs_32'),
    (('--lds', '--lds_kernel', 'triang', '--reweight', 'sqrt_inv'), 'nyud2_lds_tri_5_lr_0.0001_bs_32'),
    (('--fds',), 'nyud2_fds_gau_5_2_0_1_0.9_lr_0.0001_bs_32'),
    (('--fds', '--fds_sigma', '2', '--fds_mmt', '0.9'), 'nyud2_fds_gau_5_2.0_0_1_0.9_lr_0.0001_bs_32'),
    (('--fds', '--fds_kernel', 'laplace', '--fds_ks', '7', '--start_update', '1', '--start_smooth', '2'),
     'nyud2_fds_lap_7_2_1_2_0.9_lr_0.0001_bs_32'),
    (('--lds', '--reweight', 'inverse', '--fds', '--batch_size', '8', '--lr', '1e-3'),
     'nyud2_lds_gau_5_2_fds_gau_5_2_0_1_0.9_lr_0.001_bs_8'),
    (('--retrain_fc', '--pretrained', 'x.pth.tar'), 'nyud2_retrain_fc_lr_0.0001_bs_32'),
    (('--store_name', 'run', '--reweight', 'sqrt_inv', '--retrain_fc'), 'run_sqrt_inv_retrain_fc_lr_0.0001_bs_32'),
])
def test_store_name(argv, want):
    import nyud2_train
    assert nyud2_train.store_name(parse(*argv)) == want


def test_lr_schedule():
    import nyud2_train
    args = parse('--lr', '0.01')
    got = [nyud2_train.lr_at(args, e) for e in range(12)]
    assert got == [0.01] * 5 + [0.01 * 0.1] * 5 + [0.01 * 0.1 ** 2] * 2


def test_shot_idx_is_the_reference_table():
    import depth_eval
    g = golden("depth_eval")
    for shot in ('many', 'medium', 'few'):
        assert depth_eval.SHOT_IDX[shot] == [int(b) for b in g["shot_" + shot]], shot
    assert sorted(sum(depth_eval.SHOT_IDX.values(), [])) == list(range(100))


def test_existing_store_dir_is_refused_without_a_terminal(tmp_path, monkeypatch):
    import io
    import nyud2_train
    argv = ['--store_root', str(tmp_path)]
    (tmp_path / nyud2_train.store_name(parse(*argv))).mkdir()
    monkeypatch.setattr('sys.stdin', io.StringIO('y\n'))
    with pytest.raises(RuntimeError, match='already exists'):
        nyud2_train.main(argv)


def test_strip_module():
    import depth_eval
    assert list(depth_eval.strip_module({'module.E.conv1.weight': 1, 'R.conv2.bias': 2})) == ['E.conv1.weight',
                                                                                            'R.conv2.bias']


# --------------------------------------------------------------------------------------- multi-tensor Adam refusals
def lib():
    import _lib
    import optim
    return _lib, optim


def table(n=3, edits=()):
    _, optim = lib()
    t = np.zeros(n, dtype=optim._SEGMENT)
    for k in ('param', 'grad', 'exp_avg', 'exp_avg_sq'):
        t[k] = D
    t['numel'], t['bc1'], t['bc2_sqrt'] = 4099, 0.1, 0.03
    for k, i, v in edits:
        t[k][i] = v
    return t


def refused_multi(t, nseg=None, msg="adam_step_multi"):
    L, _ = lib()
    ptr = None if t is None else t.ctypes.data_as(ctypes.c_void_p)
    rc = L.raw("dirb200_adam_step_multi")(ptr, len(t) if nseg is None else nseg, 1e-3, 0.9, 0.999, 1e-8, 1e-4, None)
    err = L.last_error()
    assert rc == -1 and msg in err, (rc, err)


def test_adam_multi_refuses_bad_arguments():
    _, optim = lib()
    assert optim._SEGMENT.itemsize == 48
    refused_multi(None, nseg=3, msg="bad arguments")
    for nseg in (0, -1):
        refused_multi(table(), nseg=nseg, msg="bad arguments")
    for k in ('param', 'grad', 'exp_avg', 'exp_avg_sq'):
        for i in (0, 2):                                      # the first and the last segment are both checked
            refused_multi(table(edits=[(k, i, 0)]), msg=f"segment {i} has a null pointer")
            refused_multi(table(edits=[(k, i, D + 2)]), msg=f"segment {i} is not 4-byte aligned")
    for v in (0, -1, 4096 * 2 ** 31 + 1):
        refused_multi(table(edits=[('numel', 1, v)]), msg="segment 1 has numel")
    for k in ('bc1', 'bc2_sqrt'):
        for v in (0.0, -0.5, np.inf, np.nan):
            refused_multi(table(edits=[(k, 2, v)]), msg="segment 2 has bias corrections")
    # a long table is checked in full before the first launch
    refused_multi(table(1500, [('numel', 1499, 0)]), msg="segment 1499 has numel")


def test_bias_corrections_in_double_from_fp32_betas():
    _, optim = lib()
    bc1, bc2s = optim._bias_corrections(0.9, 0.999, 3)
    b1, b2 = float(np.float32(0.9)), float(np.float32(0.999))
    assert bc1 == 1.0 - b1 ** 3 and bc2s == (1.0 - b2 ** 3) ** 0.5


def test_optim_adam_refuses_bad_options_and_cpu_tensors():
    L, optim = lib()
    p = torch.zeros(4, requires_grad=True)
    for kw in (dict(amsgrad=True), dict(maximize=True), dict(lr=-1.0), dict(eps=-1.0), dict(betas=(1.0, 0.999)),
               dict(betas=(0.9, -0.1)), dict(weight_decay=-1e-4)):
        with pytest.raises(ValueError):
            optim.Adam([p], **kw)
    p.grad = torch.ones(4)
    opt = optim.Adam([p], 1e-3)
    with pytest.raises(L.Dirb200Error, match="CUDA"):
        opt.step()
    assert len(opt.state) == 0                     # refused before any state was made
    opt.param_groups[0]['amsgrad'] = True          # e.g. loaded from a torch.optim.Adam(amsgrad=True) state_dict
    with pytest.raises(ValueError):
        opt.step()
    q = torch.zeros(4, requires_grad=True)         # no gradient: nothing to check, nothing stepped
    optim.Adam([q], 1e-3).step()
