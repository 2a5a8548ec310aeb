"""train.py (the reference-shaped driver) end to end on synthetic data: 3 tiny epochs with FDS + LDS, i.e. the
whole state machine -- epoch 0 collect, epoch 1 smooth with identity tables, epoch 2 live calibration -- plus
checkpoint writing and the validation pass; once with the datasets' float tensors and once with --device_transform (uint8
images, RandomCrop / flip / ToTensor / Normalize on the GPU per batch).

Then the driver against agedb-dir/train.py and imdb-wiki-dir/train.py: checkpoint files and keys, the lr schedule,
best_loss and the best checkpoint, the test pass with the best checkpoint and main's return, two identical runs giving
identical checkpoints, --resume (SGD, and Adam with FDS) equal to the uninterrupted run, --evaluate, --retrain_fc, each
--loss, and on-disk AgeDB / IMDB-WIKI sets with their scripts' LDS / FDS defaults."""
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("extra", [[], ["--device_transform"]], ids=["host_tensors", "device_transform"])
def test_train_script_runs_three_epochs(tmp_path, extra):
    import train
    argv = extra + ["--synthetic", "192", "--batch_size", "64", "--epoch", "3", "--fds", "--lds", "--reweight", "sqrt_inv",
            "--lds_ks", "5", "--lds_sigma", "2", "--fds_ks", "5", "--fds_sigma", "2", "--bucket_num", "101",
            "--bucket_start", "0", "--workers", "0", "--img_size", "64", "--print_freq", "1",
            "--store_root", str(tmp_path), "--lr", "1e-4"]
    train.main(argv)
    runs = os.listdir(tmp_path)
    assert len(runs) == 1
    ckpt = torch.load(os.path.join(tmp_path, runs[0], "ckpt.pth.tar"), map_location="cpu")
    assert ckpt["epoch"] == 3
    sd = ckpt["state_dict"]
    assert "module.FDS.smoothed_mean_last_epoch" in sd and "module.layer4.2.bn3.running_var" in sd
    assert int(sd["module.FDS.epoch"][0]) == 2                    # two update_last_epoch_stats transitions
    assert float(sd["module.FDS.num_samples_tracked"].sum()) == 3 * 192
    assert torch.isfinite(sd["module.conv1.weight"]).all()
    # the tables became non-trivial and smoothing changed them
    assert not torch.allclose(sd["module.FDS.smoothed_mean_last_epoch"], torch.zeros_like(sd["module.FDS.smoothed_mean_last_epoch"]))


# ------------------------------------------------------------------------------ the driver against the reference's
# Module-scoped runs of train.main on 192 synthetic samples (3 steps of 64 per epoch; val == test: 64 samples).  Every
# checkpoint the driver saves is kept (store/epoch<e>/ holds ckpt.pth.tar and ckpt.best.pth.tar as they were after
# epoch e), with what validate returned and the model's state at the test pass.
BASE = ["--synthetic", "192", "--img_size", "64", "--batch_size", "64", "--workers", "0"]
FDS_KEYS = ("epoch", "running_mean", "running_var", "running_mean_last_epoch", "running_var_last_epoch",
            "smoothed_mean_last_epoch", "smoothed_var_last_epoch", "num_samples_tracked")


def drive(argv, root, prepare=None):
    import shutil
    import train as T
    argv = list(argv) + ["--store_root", str(root)]
    store = os.path.join(str(root), T.store_name(T.build_parser().parse_known_args(argv)[0]))
    if prepare:
        prepare(store)
    rec = dict(store=store, val=[], test=[], train=[], epoch_host=[], saved=[])
    real_save, real_validate, real_train = T.save_checkpoint, T.validate, T.train

    def save(args, state, is_best, prefix=''):
        real_save(args, state, is_best, prefix)
        snap = os.path.join(store, f"epoch{state['epoch']}")
        os.makedirs(snap)
        for f in ("ckpt.pth.tar", "ckpt.best.pth.tar"):
            if os.path.exists(os.path.join(store, f)):
                shutil.copyfile(os.path.join(store, f), os.path.join(snap, f))
        rec["saved"].append((state["epoch"], is_best))

    def validate(loader, model, train_labels=None, prefix='Val'):
        out = real_validate(loader, model, train_labels=train_labels, prefix=prefix)
        if prefix == 'Test':
            rec["test_state"] = {k: v.detach().cpu().clone() for k, v in model.state_dict().items()}
        rec["val" if prefix == 'Val' else "test"].append(out)
        return out

    def train_epoch(loader, model, optimizer, epoch, args, stats_loader=None):
        fds = getattr(model.module, "FDS", None)
        rec["epoch_host"].append(None if fds is None else fds._epoch_host)
        rec["optimizer"], rec["model"] = optimizer, model
        out = real_train(loader, model, optimizer, epoch, args, stats_loader=stats_loader)
        rec["train"].append(out)
        return out

    with pytest.MonkeyPatch.context() as mp:
        mp.setattr(T, "save_checkpoint", save)
        mp.setattr(T, "validate", validate)
        mp.setattr(T, "train", train_epoch)
        torch.manual_seed(0)
        rec["ret"] = T.main(argv)
    return rec


def load(path):
    return torch.load(path, map_location="cpu")


def snap(rec, epoch, best=False):
    return os.path.join(rec["store"], f"epoch{epoch}", "ckpt.best.pth.tar" if best else "ckpt.pth.tar")


def resume_from(rec, epoch):
    """prepare(): the new store directory as rec's was after `epoch` (its ckpt.pth.tar and ckpt.best.pth.tar)."""
    import shutil

    def prepare(store):
        os.makedirs(store)
        for f in ("ckpt.pth.tar", "ckpt.best.pth.tar"):
            shutil.copyfile(os.path.join(rec["store"], f"epoch{epoch}", f), os.path.join(store, f))
    return prepare


def tensors_equal(a, b, what, skip=()):
    """Nested checkpoint pieces (dicts / lists of tensors and numbers) equal bit for bit, `skip` keys excepted."""
    if isinstance(a, dict):
        assert set(a) == set(b), what
        for k in a:
            if k not in skip:
                tensors_equal(a[k], b[k], f"{what}.{k}", skip)
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            tensors_equal(x, y, f"{what}[{i}]", skip)
    elif isinstance(a, torch.Tensor):
        assert a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b), what
    else:
        assert a == b, (what, a, b)


SGD_LDS = BASE + ["--optimizer", "sgd", "--lds", "--reweight", "sqrt_inv", "--epoch", "3", "--schedule", "1", "2"]
ADAM_FDS_LDS = BASE + ["--fds", "--lds", "--reweight", "sqrt_inv", "--epoch", "3"]


@pytest.fixture(scope="module")
def run_a(tmp_path_factory):
    return drive(SGD_LDS, tmp_path_factory.mktemp("a"))


def test_checkpoints_and_keys(run_a):
    import resnet
    names = ["module." + k for k in resnet.resnet50().state_dict()]
    assert sorted(os.listdir(run_a["store"])) == ["ckpt.best.pth.tar", "ckpt.pth.tar", "epoch1", "epoch2", "epoch3",
                                                  "training.log"]
    assert [e for e, _ in run_a["saved"]] == [1, 2, 3]
    for e in (1, 2, 3):
        ck = load(snap(run_a, e))
        assert set(ck) == {"epoch", "model", "best_loss", "state_dict", "optimizer"} and ck["epoch"] == e
        assert ck["model"] == "resnet50" and list(ck["state_dict"]) == names


def test_learning_rate_follows_the_schedule(run_a):
    """agedb-dir/utils.py:81-86 with --lr 1e-3 --schedule 1 2: each epoch's lr is the product of the drops."""
    for e in (1, 2, 3):
        lr = 1e-3
        for milestone in (1, 2):
            lr *= 0.1 if e - 1 >= milestone else 1.
        assert [g["lr"] for g in load(snap(run_a, e))["optimizer"]["param_groups"]] == [lr]


def test_best_loss_and_best_checkpoint(run_a):
    """best_loss is the running minimum of the validation L1 (--loss l1); ckpt.best.pth.tar is, byte for byte, the
    checkpoint of the epoch that reached it."""
    l1 = [v[1] for v in run_a["val"]]
    assert len(l1) == 3
    for e in (1, 2, 3):
        assert load(snap(run_a, e))["best_loss"] == min(l1[:e])
    assert [b for _, b in run_a["saved"]] == [l1[e] < min([1e5] + l1[:e]) for e in range(3)]
    best = int(np.argmin(l1)) + 1
    with open(os.path.join(run_a["store"], "ckpt.best.pth.tar"), "rb") as f, open(snap(run_a, best), "rb") as g:
        assert f.read() == g.read()


def test_test_pass_with_the_best_checkpoint(run_a):
    """After the epochs: the best checkpoint is loaded, tested, logged as the reference logs it, and returned."""
    best = load(os.path.join(run_a["store"], "ckpt.best.pth.tar"))
    tensors_equal({k: v for k, v in best["state_dict"].items()}, run_a["test_state"], "model at the test pass")
    assert len(run_a["test"]) == 1 and run_a["ret"] == run_a["test"][0]
    # the synthetic test split is the validation split: the test pass repeats the best epoch's validation bit for bit
    assert run_a["ret"] == run_a["val"][best["epoch"] - 1]
    log = open(os.path.join(run_a["store"], "training.log")).read()
    mse, l1, gm = run_a["ret"]
    assert f"Loaded best model, epoch {best['epoch']}, best val loss {best['best_loss']:.4f}" in log
    assert f"Test loss: MSE [{mse:.4f}], L1 [{l1:.4f}], G-Mean [{gm:.4f}]" in log


def test_identical_runs_write_identical_checkpoints(run_a, tmp_path):
    again = drive(SGD_LDS, tmp_path)
    for e in (1, 2, 3):
        a, b = load(snap(run_a, e)), load(snap(again, e))
        tensors_equal(a, b, f"epoch {e}")
    assert again["val"] == run_a["val"] and again["test"] == run_a["test"]


def test_resume_sgd_equals_the_uninterrupted_run(run_a, tmp_path):
    """--resume from the epoch-2 checkpoint, one more epoch: parameters, BN running statistics, the momentum buffer,
    best_loss and the test metrics are A's, bit for bit."""
    import train as T
    # the resume path is the copied epoch-2 checkpoint inside the new store directory (the usual layout)
    s = os.path.join(str(tmp_path), T.store_name(T.build_parser().parse_known_args(SGD_LDS)[0]))
    r = drive(SGD_LDS + ["--resume", os.path.join(s, "ckpt.pth.tar")], tmp_path, resume_from(run_a, 2))
    assert [e for e, _ in r["saved"]] == [3] and r["train"] and len(r["val"]) == 1
    tensors_equal(load(snap(run_a, 3)), load(snap(r, 3)), "epoch 3")
    assert r["val"][0] == run_a["val"][2] and r["ret"] == r["test"][0] == run_a["test"][0]


@pytest.fixture(scope="module")
def run_b(tmp_path_factory):
    return drive(ADAM_FDS_LDS, tmp_path_factory.mktemp("b"))


def test_resume_adam_fds_equals_the_uninterrupted_run(run_b, tmp_path):
    """--fds --lds with Adam: the same, except the eight FDS buffers, which agree to rtol 1e-6 only (the epoch-end
    statistics are summed with fp64 atomics, csrc/fds.cu).  FDS._epoch_host comes back from the checkpoint."""
    import train as T
    s = os.path.join(str(tmp_path), T.store_name(T.build_parser().parse_known_args(ADAM_FDS_LDS)[0]))
    r = drive(ADAM_FDS_LDS + ["--resume", os.path.join(s, "ckpt.pth.tar")], tmp_path, resume_from(run_b, 2))
    ck2 = load(snap(run_b, 2))
    assert r["epoch_host"] == [int(ck2["state_dict"]["module.FDS.epoch"][0])] == [run_b["epoch_host"][2]]
    a, b = load(snap(run_b, 3)), load(snap(r, 3))
    fds = {"module.FDS." + k for k in FDS_KEYS}
    assert fds <= set(a["state_dict"])
    tensors_equal(a, b, "epoch 3", skip=fds)
    for k in sorted(fds):
        assert torch.allclose(a["state_dict"][k], b["state_dict"][k], rtol=1e-6, atol=0.0), k
    assert r["val"][0] == run_b["val"][2] and r["ret"] == r["test"][0] == run_b["test"][0]


def test_evaluate_returns_the_test_metrics(run_a, tmp_path):
    """--evaluate --resume ckpt.best.pth.tar: every tensor of the checkpoint is in the model (the load is strict=False,
    as the reference's) and the test metrics are the training run's, bit for bit."""
    path = os.path.join(run_a["store"], "ckpt.best.pth.tar")
    r = drive(BASE + ["--evaluate", "--resume", path], tmp_path)
    assert r["saved"] == [] and r["val"] == [] and len(r["test"]) == 1
    tensors_equal(load(path)["state_dict"], r["test_state"], "model after the --evaluate load")
    assert r["ret"] == r["test"][0] == run_a["test"][0]


def test_retrain_fc_trains_only_the_regressor(run_a, tmp_path):
    """--retrain_fc --pretrained: the backbone parameters keep the pretrained bits, linear.* moves, the optimizer
    holds exactly those two tensors, and train-mode forwards move the BN running statistics."""
    path = os.path.join(run_a["store"], "ckpt.best.pth.tar")
    r = drive(BASE + ["--retrain_fc", "--pretrained", path, "--reweight", "sqrt_inv", "--epoch", "1"], tmp_path)
    pre, got = load(path)["state_dict"], load(snap(r, 1))["state_dict"]
    model = r["model"]
    params = {"module." + n for n, _ in model.module.named_parameters()}
    lin = {"module.linear.weight", "module.linear.bias"}
    for k in params - lin:
        assert torch.equal(pre[k], got[k]), k
    for k in lin:
        assert not torch.equal(pre[k], got[k]), k
    opt = [p for g in r["optimizer"].param_groups for p in g["params"]]
    assert len(opt) == 2 and opt[0] is model.module.linear.weight and opt[1] is model.module.linear.bias
    moved = [k for k in got if k.endswith("running_mean") or k.endswith("running_var")]
    assert moved and all(not torch.equal(pre[k], got[k]) for k in moved)


@pytest.mark.parametrize("loss", ["mse", "l1", "focal_l1", "focal_mse", "huber"])
def test_each_loss_trains_and_picks_its_metric(loss, tmp_path):
    """One epoch per --loss: a finite training loss; best_loss is the validation MSE for mse and the L1 for every
    other loss (agedb-dir/train.py:205)."""
    r = drive(BASE + ["--loss", loss, "--epoch", "1"], tmp_path)
    assert len(r["train"]) == 1 and np.isfinite(r["train"][0])
    mse, l1, _ = r["val"][0]
    assert mse != l1
    assert load(snap(r, 1))["best_loss"] == (mse if loss == "mse" else l1)


def write_ages(data, dataset, rng):
    """A small on-disk AgeDB / IMDB-WIKI set: Pillow-written JPEGs and <dataset>.csv with path, age, split.  Ages 0 to
    99 in training (0-2 included), the rest of the splits drawn from them."""
    from PIL import Image
    import pandas as pd
    os.makedirs(data)
    train_ages = np.concatenate([np.arange(100), rng.randint(0, 100, 200)])
    rows = []
    for split, ages in (("train", train_ages), ("val", rng.randint(0, 100, 40)), ("test", rng.randint(0, 100, 40))):
        for i, age in enumerate(ages):
            name = f"{split}_{i}.jpg"
            img = rng.randint(0, 256, size=(48 + i % 17, 40 + i % 23, 3)).astype(np.uint8)
            Image.fromarray(img).save(os.path.join(data, name), quality=90)
            rows.append((name, int(age), split))
    pd.DataFrame(rows, columns=["path", "age", "split"]).to_csv(os.path.join(data, f"{dataset}.csv"), index=False)
    return train_ages


@pytest.mark.parametrize("dataset,ks,bucket_start", [("agedb", 9, 3), ("imdb_wiki", 5, 0)])
def test_on_disk_sets_use_their_scripts_defaults(dataset, ks, bucket_start, tmp_path):
    """`--dataset <d> --fds --lds --reweight sqrt_inv` for 2 epochs with no LDS / FDS flags: the dataset's own FDS
    window (9 / 5 taps) and buckets (from age 3 / 0), and the reference's store name."""
    import json
    from util import GOLDEN
    flags = ["--dataset", dataset, "--fds", "--lds", "--reweight", "sqrt_inv"]
    case = next(c for c in json.load(open(os.path.join(GOLDEN, "train_flags.json")))["cases"] if c["argv"] == flags)
    ages = write_ages(str(tmp_path / "data"), dataset, np.random.RandomState(1))
    r = drive(flags + ["--data_dir", str(tmp_path / "data"), "--epoch", "2", "--img_size", "64", "--workers", "0"],
              tmp_path / "ckpt")
    assert os.path.basename(r["store"]) == case["store_name"]
    assert os.path.isfile(os.path.join(r["store"], "ckpt.best.pth.tar"))
    fds = r["model"].module.FDS
    assert fds.kernel_window.numel() == ks and fds.bucket_start == bucket_start
    sd = load(snap(r, 2))["state_dict"]
    assert sd["module.FDS.running_mean"].shape[0] == 100 - bucket_start
    # two refreshes (start_update 0) over every training sample, bucketed from bucket_start (lower ages fold into
    # the first bucket: age bucket_start is present)
    want = np.bincount(np.maximum(ages, bucket_start) - bucket_start, minlength=100 - bucket_start) * 2
    assert np.array_equal(sd["module.FDS.num_samples_tracked"].numpy(), want.astype(np.float32))
    assert all(np.isfinite(v) for v in r["ret"])
