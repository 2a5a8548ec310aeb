"""GPU checks of NYUD2-DIR's device input pipeline (loaddata.py, dirb200_depth_augment_batch) against the reference's
own transforms (nyud2-dir/nyu_transform.py, nyud2-dir/loaddata.py, loaded from oracle/_ref by oracle/nyu_transform_ref).

- Flip + rotate + crop: the uint8 crop (image and depth) byte for byte against RandomHorizontalFlip, RandomRotate and
  CenterCrop, at 0, +-1e-6, +-2.5, +-5, 4.999 degrees and random draws, flip on and off, on 240 x 320, 241 x 323 and
  portrait sources, random / near-constant / saturated images; the +-5 degree crops include the constant-fill band.
- Depth: the Pillow BICUBIC resize, ToTensor * 10 and _get_weights bit for bit, with LDS inverse / sqrt_inv tables and
  'none', over every uint8 depth value (so every bucket edge the 8-bit depth can reach).
- Training image: bit for bit against the reference's ops fed the device's Contrast mean; that mean within the bound
  of test_contrast_mean; the reference's seeded Compose within the per-element bound that mean difference allows.
- FDS and test chains bit for bit against the reference's Compose, image and depth.
- Determinism (bitwise repeats) and isolation (sample k alone gives the same bytes as in the batch).
- End to end on a synthetic on-disk set: the loaders' batches against the reference DataLoaders (keys, shapes, dtypes,
  and values where no random draw is involved), one net.model Adam step, depth_eval.test over the test loader.
Outputs are prefilled with NaN.  The file reruns itself with DIRB200_SMS=7."""
import os
import random
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from PIL import Image

pytestmark = pytest.mark.gpu
DEV = "cuda"
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
MEAN, STD = [0.485, 0.456, 0.406], [0.229, 0.224, 0.225]
PCA = {'eigval': torch.Tensor([0.2175, 0.0188, 0.0045]),
       'eigvec': torch.Tensor([[-0.5675, 0.7192, 0.4009], [-0.5808, -0.0045, -0.8140], [-0.5836, -0.6948, 0.4203]])}


def ref():
    from oracle import nyu_transform_ref
    if not nyu_transform_ref.available():
        pytest.fail("oracle/_ref has no copy of the reference's nyu_transform.py / loaddata.py: run __graft_entry__.build()")
    return nyu_transform_ref.load()


class Fixed:
    """Stands for nyu_transform's `random` module: hands out fixed draws."""

    def __init__(self, rnd=(), uni=()):
        self.rnd, self.uni = list(rnd), list(uni)

    def random(self):
        return self.rnd.pop(0)

    def uniform(self, a, b):
        return self.uni.pop(0)


def make_sources(n, h, w, kind, seed):
    r = np.random.RandomState(seed)
    if kind == "random":
        img = r.randint(0, 256, (n, h, w, 3))
        dep = r.randint(0, 256, (n, h, w))
    elif kind == "near_constant":                  # the spline overshoots around a few outliers in a flat field
        img = np.full((n, h, w, 3), 254) - (r.rand(n, h, w, 3) < 0.01) * 254
        dep = np.full((n, h, w), 1) + (r.rand(n, h, w) < 0.01) * 254
    else:                                          # saturated: 0 / 255 blocks, the overshoot hits both clips
        img = ((np.indices((h, w)).sum(0) // 3) % 2 * 255)[None, :, :, None].repeat(n, 0).repeat(3, 3)
        img[..., 1] = 255 - img[..., 1]
        dep = (r.rand(n, h, w) < 0.5) * 255
    return img.astype(np.uint8), dep.astype(np.uint8)


def device_batch(img, dep, split, params=None, table=None, debug=True):
    import loaddata
    out = loaddata.gpu_depth_transform_batch(torch.from_numpy(img).to(DEV), torch.from_numpy(dep).to(DEV), split,
                                             params=params, bucket_weights=table, debug=debug)
    torch.cuda.synchronize()
    return out


def params_for(n, angles, flips, seed=0):
    import loaddata
    p = loaddata.draw_nyud2_train_params(n, random.Random(seed), torch.Generator().manual_seed(seed))
    p["angle"] = torch.tensor(angles, dtype=torch.float64)
    p["flip"] = torch.tensor(flips, dtype=torch.uint8)
    return p


def ref_crop(nt, img, dep, angle, flip, size_depth=(304, 228)):
    """RandomHorizontalFlip -> RandomRotate -> CenterCrop of the reference on one sample -> (image u8, depth u8)."""
    s = {'image': Image.fromarray(img), 'depth': Image.fromarray(dep)}
    nt.random = Fixed(rnd=[0.0 if flip else 0.9], uni=[angle])
    try:
        s = nt.RandomHorizontalFlip()(s)
        s = nt.RandomRotate(5)(s)
    finally:
        nt.random = random
    s = nt.CenterCrop([304, 228], list(size_depth))(s)
    return np.asarray(s['image']), np.asarray(s['depth'])


# ------------------------------------------------------------------------------------------- rotate + crop, uint8
ANGLES = [0.0, 1e-6, -1e-6, 2.5, -2.5, 5.0, -5.0, 4.999]
GEOMS = [((240, 320), "random"), ((241, 323), "random"), ((400, 310), "random"), ((240, 320), "near_constant"),
         ((240, 320), "saturated"), ((229, 305), "random")]


@pytest.mark.parametrize("shape,kind", GEOMS, ids=[f"{s[0]}x{s[1]}-{k}" for s, k in GEOMS])
def test_rotate_crop_bit_exact(shape, kind):
    """Every byte of the flipped, rotated, cropped image and depth against the reference's own transforms."""
    nt, _ = ref()
    r = random.Random(shape[0] + shape[1])
    angles = ANGLES + [r.uniform(-5, 5) for _ in range(4)]
    n = len(angles)
    flips = [k % 2 for k in range(n)]
    img, dep = make_sources(n, *shape, kind, seed=shape[0])
    out = device_batch(img, dep, "train", params_for(n, angles, flips))
    crop = out["crop"].cpu().numpy()
    border = 0
    for k in range(n):
        ri, rd = ref_crop(nt, img[k], dep[k], angles[k], flips[k])
        assert np.array_equal(crop[k, ..., :3], ri), (k, angles[k], int((crop[k, ..., :3] != ri).sum()))
        assert np.array_equal(crop[k, ..., 3], rd), (k, angles[k], int((crop[k, ..., 3] != rd).sum()))
        if abs(angles[k]) >= 4.9 and shape == (240, 320):
            border += int((ri[:3, :3] == 0).all(-1).sum())
    if shape == (240, 320) and kind == "random":
        assert border > 0, "the +-5 degree crops should reach the constant-fill band"


# ------------------------------------------------------------------------------------------- depth and weights
def tables():
    import datasets
    import loaddata
    t = {"none": None}
    for rw, lds in (("inverse", True), ("sqrt_inv", True), ("inverse", False)):
        t[f"{rw}{'-lds' if lds else ''}"] = datasets.depth_bucket_weights(loaddata.TRAIN_BUCKET_NUM, rw, 100, 7, lds,
                                                                          'gaussian', 5, 2)
    return t


@pytest.mark.parametrize("table", ["none", "inverse-lds", "sqrt_inv-lds", "inverse"])
def test_depth_and_weight_bit_exact(table):
    """Depth resize byte for byte against Pillow's (the reference's CenterCrop), depth f32 against ToTensor * 10 and
    the weight against the reference's _get_weights, bit for bit.  The depth sources cover all 256 values."""
    nt, ld = ref()
    tab = tables()[table]
    n, h, w = 4, 240, 320
    img, dep = make_sources(n, h, w, "random", seed=3)
    dep[0] = (np.arange(h * w) % 256).reshape(h, w)                 # every value, hence every reachable bucket edge
    dep[1] = np.clip((np.indices((h, w))[1] // 8) * 7, 0, 255)      # smooth ramp: resize values between the inputs
    angles, flips = [0.0, 3.3, -4.2, 1.0], [0, 1, 0, 1]
    out = device_batch(img, dep, "train", params_for(n, angles, flips), table=tab)
    ds = ld.depthDataset.__new__(ld.depthDataset)
    ds.bucket_weights = None if tab is None else [np.float32(v) for v in tab]
    for k in range(n):
        _, rd = ref_crop(nt, img[k], dep[k], angles[k], flips[k], size_depth=(152, 114))
        s = nt.ToTensor()({'image': Image.fromarray(np.zeros((228, 304, 3), np.uint8)), 'depth': Image.fromarray(rd)})
        want_d = s['depth']
        want_w = ds._get_weights(want_d)
        got_d = out["depth"][k].cpu()
        assert got_d.shape == want_d.shape and torch.equal(got_d.view(torch.int32), want_d.view(torch.int32)), k
        assert torch.equal(out["weight"][k].cpu().view(torch.int32), want_w.view(torch.int32)), k


# ------------------------------------------------------------------------------------------- training image
def host_chain(crop_u8, rgb, order, alpha, mean):
    """The reference's own torch ops from ToTensor on (nyu_transform.py:151-347), with Contrast's mean given."""
    nt, _ = ref()
    img = torch.from_numpy(np.ascontiguousarray(crop_u8.transpose(2, 0, 1))).float().div(255)
    img = img.add(rgb.view(3, 1, 1).expand_as(img))
    for t, a in zip(order.tolist(), alpha.tolist()):
        if t == 0:
            img = img.lerp(img.new().resize_as_(img).zero_(), a)
        elif t == 1:
            gs = nt.Grayscale()(img)
            gs.fill_(mean)
            img = img.lerp(gs, a)
        else:
            img = img.lerp(nt.Grayscale()(img), a)
    for t, m, s in zip(img, MEAN, STD):
        t.sub_(m).div_(s)
    return img


def torch_mean_before_contrast(crop_u8, rgb, order, alpha):
    nt, _ = ref()
    img = torch.from_numpy(np.ascontiguousarray(crop_u8.transpose(2, 0, 1))).float().div(255)
    img = img.add(rgb.view(3, 1, 1).expand_as(img))
    for t, a in zip(order.tolist(), alpha.tolist()):
        if t == 1:
            gs = nt.Grayscale()(img)
            return gs.mean(), gs.abs().sum().item()
        img = img.lerp(img.new().resize_as_(img).zero_(), a) if t == 0 else img.lerp(nt.Grayscale()(img), a)


def mean_bound(abs_sum, count):
    """|device mean - torch mean|.  The device sums the fp32 grayscale values in fp64 (error below 2^-53 count sum|g|,
    negligible) and rounds the quotient to fp32 once: <= u |m|.  ATen reduces fp32 on the CPU in a cascade of
    ceil(log16 count) + 2 levels of at most 16 serial additions each (3 x 228 x 304 = 207 936 values: 7 levels), so
    its sum is within 16 (levels) u sum|g|, and its division adds u |m|.  Total <= (16 levels + 2) u sum|g| / count."""
    levels = int(np.ceil(np.log(count) / np.log(16))) + 2
    return (16 * levels + 2) * U * abs_sum / count


def test_contrast_mean_and_image_vs_host_restatement():
    """The device image equals the reference's ops fed the device's mean, bit for bit; the device mean is within
    mean_bound of torch's gs.mean() on the same image."""
    n, h, w = 6, 240, 320
    img, dep = make_sources(n, h, w, "random", seed=11)
    img[1] = 250                                                     # bright, near-constant: large mean
    p = params_for(n, [4.0, -2.0, 0.0, 5.0, -5.0, 1.5], [1, 0, 1, 0, 1, 0], seed=4)
    p["order"][:] = torch.tensor([[0, 1, 2], [1, 0, 2], [2, 1, 0], [0, 2, 1], [1, 2, 0], [2, 0, 1]], dtype=torch.int32)
    out = device_batch(img, dep, "train", p)
    crop = out["crop"].cpu().numpy()
    for k in range(n):
        m_dev = out["mean"][k].item()
        want = host_chain(crop[k, ..., :3], p["rgb"][k], p["order"][k], p["alpha"][k], m_dev)
        got = out["image"][k].cpu()
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (k, int((got != want).sum()))
        m_t, abs_sum = torch_mean_before_contrast(crop[k, ..., :3], p["rgb"][k], p["order"][k], p["alpha"][k])
        assert abs(m_dev - m_t.item()) <= mean_bound(abs_sum, 3 * 228 * 304), (k, m_dev, m_t.item())


def chain_bound(alpha, order, dm):
    """Per-element bound on |device - reference| when only Contrast's mean differs, by dm.  Contrast: |a| dm, plus a
    flipped rounding in its subtraction and its fma (2 x 2^-22 for values below 2).  Each later step multiplies the
    difference by at most (1 + |a|) (Brightness) or (1 + 2|a|) (Saturation: the grayscale is a convex combination of
    the channels) and adds 3 x 2^-22 of flipped roundings; Normalize divides by std and rounds twice more."""
    order, alpha = order.tolist(), alpha.tolist()
    k = order.index(1)
    e = abs(alpha[k]) * dm + 2 * 2.0 ** -22
    for t, a in zip(order[k + 1:], alpha[k + 1:]):
        e = e * ((1 + abs(a)) if t == 0 else (1 + 2 * abs(a))) + 3 * 2.0 ** -22
    return torch.tensor([(e + 2.0 ** -22) / s + 2.0 ** -21 for s in STD]).view(3, 1, 1)


def test_training_chain_vs_reference_compose():
    """The reference's seeded Compose (loaddata.py:110-125) against the device from the same seeds, every element
    within chain_bound of the mean difference mean_bound allows."""
    nt, _ = ref()
    import loaddata
    from torchvision import transforms
    n, h, w = 5, 240, 320
    img, dep = make_sources(n, h, w, "random", seed=21)
    chain = transforms.Compose([nt.RandomHorizontalFlip(), nt.RandomRotate(5), nt.CenterCrop([304, 228], [152, 114]),
                                nt.ToTensor(), nt.Lighting(0.1, PCA['eigval'], PCA['eigvec']),
                                nt.ColorJitter(0.4, 0.4, 0.4), nt.Normalize(MEAN, STD)])
    random.seed(5)
    torch.manual_seed(6)
    want = [chain({'image': Image.fromarray(img[k]), 'depth': Image.fromarray(dep[k])}) for k in range(n)]
    random.seed(5)
    torch.manual_seed(6)
    p = loaddata.draw_nyud2_train_params(n)
    out = device_batch(img, dep, "train", p)
    crop = out["crop"].cpu().numpy()
    for k in range(n):
        _, abs_sum = torch_mean_before_contrast(crop[k, ..., :3], p["rgb"][k], p["order"][k], p["alpha"][k])
        bound = chain_bound(p["alpha"][k], p["order"][k], mean_bound(abs_sum, 3 * 228 * 304))
        err = (out["image"][k].cpu().double() - want[k]['image'].double()).abs()
        assert bool((err <= bound).all()), (k, float((err - bound).max()))
        assert torch.equal(out["depth"][k].cpu(), want[k]['depth'])


# ------------------------------------------------------------------------------------------- FDS and test chains
@pytest.mark.parametrize("shape", [(240, 320), (241, 323)], ids=["240x320", "241x323"])
def test_fds_chain_bit_exact(shape):
    nt, _ = ref()
    from torchvision import transforms
    n = 3
    img, dep = make_sources(n, *shape, "random", seed=31)
    chain = transforms.Compose([nt.CenterCrop([304, 228], [152, 114]), nt.ToTensor(), nt.Normalize(MEAN, STD)])
    out = device_batch(img, dep, "fds")
    for k in range(n):
        want = chain({'image': Image.fromarray(img[k]), 'depth': Image.fromarray(dep[k])})
        assert torch.equal(out["image"][k].cpu().view(torch.int32), want['image'].view(torch.int32)), k
        assert torch.equal(out["depth"][k].cpu().view(torch.int32), want['depth'].view(torch.int32)), k
        assert bool((out["weight"][k] == 1).all())


def test_test_chain_bit_exact():
    nt, _ = ref()
    from torchvision import transforms
    n, h, w = 3, 240, 320
    img, _ = make_sources(n, h, w, "random", seed=41)
    dep = np.random.RandomState(42).randint(0, 12000, (n, h, w)).astype(np.uint16)
    dep[0, :2, :5] = [0, 1, 999, 1000, 32767]
    chain = transforms.Compose([nt.CenterCrop([304, 228], [304, 228]), nt.ToTensor(is_test=True),
                                nt.Normalize(MEAN, STD)])
    out = device_batch(img, dep.astype(np.int16), "test")
    for k in range(n):
        want = chain({'image': Image.fromarray(img[k]), 'depth': Image.fromarray(dep[k])})
        assert torch.equal(out["image"][k].cpu().view(torch.int32), want['image'].view(torch.int32)), k
        assert torch.equal(out["depth"][k].cpu().view(torch.int32), want['depth'].view(torch.int32)), k


# ------------------------------------------------------------------------------------------- determinism, isolation
def test_deterministic_and_batch_independent():
    import loaddata
    n, h, w = 8, 240, 320
    img, dep = make_sources(n, h, w, "random", seed=51)
    p = loaddata.draw_nyud2_train_params(n, random.Random(3), torch.Generator().manual_seed(3))
    tab = tables()["inverse-lds"]
    a = device_batch(img, dep, "train", p, tab)
    b = device_batch(img, dep, "train", p, tab)
    for key in ("image", "depth", "weight", "crop", "mean"):
        assert torch.equal(a[key], b[key]), key
        assert not a[key].float().isnan().any(), key
    k = 5
    one = device_batch(img[k:k + 1], dep[k:k + 1], "train", {q: v[k:k + 1] for q, v in p.items()}, tab)
    for key in ("image", "depth", "weight", "crop", "mean"):
        assert torch.equal(one[key][0], a[key][k]), key


def test_outputs_fully_written():
    """Outputs prefilled with NaN: every element of image, depth and weight is written by the kernels."""
    import _lib
    import ctypes
    import loaddata
    n, h, w = 3, 241, 323
    img, dep = make_sources(n, h, w, "random", seed=61)
    p = loaddata.draw_nyud2_train_params(n, random.Random(1), torch.Generator().manual_seed(1), (h, w))
    d = lambda t, dt: t.to(DEV, dt).contiguous()                      # noqa: E731
    imgs, deps = torch.from_numpy(img).to(DEV), torch.from_numpy(dep).to(DEV)
    out = [torch.full(s, float("nan"), device=DEV) for s in ((n, 3, 228, 304), (n, 1, 114, 152), (n, 1, 114, 152))]
    nb = _lib.raw("dirb200_depth_augment_workspace_bytes")(n, h, w, 228, 304)
    ws = torch.full((nb,), 255, dtype=torch.uint8, device=DEV)
    ms = (ctypes.c_float * 6)(*loaddata.MEAN_STD)
    tab = torch.tensor(tables()["inverse"], device=DEV)
    aff, flip, rgb, order, alpha = (d(p["affine"], torch.float64), d(p["flip"], torch.uint8), d(p["rgb"], torch.float32),
                                    d(p["order"], torch.int32), d(p["alpha"], torch.float32))
    _lib.call("dirb200_depth_augment_batch", _lib.ptr(imgs), _lib.ptr(deps), 0, n, h, w, 228, 304, 114, 152,
              _lib.ptr(flip), _lib.ptr(aff), _lib.ptr(rgb), _lib.ptr(order), _lib.ptr(alpha), ms, _lib.ptr(tab), 100,
              _lib.ptr(out[0]), _lib.ptr(out[1]), _lib.ptr(out[2]), None, None, _lib.ptr(ws), nb, _lib.stream_ptr())
    torch.cuda.synchronize()
    for t in out:
        assert not t.isnan().any()
    want = device_batch(img, dep, "train", p, tables()["inverse"])
    assert torch.equal(out[0], want["image"]) and torch.equal(out[1], want["depth"]) and torch.equal(out[2], want["weight"])


# ------------------------------------------------------------------------------------------- end to end
def write_dataset(root, n_train=6, n_test=4):
    r = np.random.RandomState(0)
    os.makedirs(os.path.join(root, "nyu2_train"))
    os.makedirs(os.path.join(root, "nyu2_test"))
    rows = {"nyu2_train.csv": [], "nyu2_test.csv": []}
    yy, xx = np.indices((480, 640))
    for k in range(n_train):
        im = (np.stack([xx * 255 // 639, yy * 255 // 479, (xx + yy) % 256], -1) + r.randint(0, 30, (480, 640, 3)))
        Image.fromarray(np.clip(im, 0, 255).astype(np.uint8)).save(os.path.join(root, "nyu2_train", f"{k}.jpg"))
        Image.fromarray(((xx // 3 + yy // 5 + 17 * k) % 256).astype(np.uint8)).save(
            os.path.join(root, "nyu2_train", f"{k}.png"))
        rows["nyu2_train.csv"].append(f"data/nyu2_train/{k}.jpg,data/nyu2_train/{k}.png")
    for k in range(n_test):
        Image.fromarray(r.randint(0, 256, (480, 640, 3)).astype(np.uint8)).save(os.path.join(root, "nyu2_test", f"{k}.jpg"))
        Image.fromarray((500 + xx * 13 + yy * 3 + k).astype(np.uint16)).save(os.path.join(root, "nyu2_test", f"{k}.png"))
        rows["nyu2_test.csv"].append(f"data/nyu2_test/{k}.jpg,data/nyu2_test/{k}.png")
    rows["nyu2_train_FDS_subset.csv"] = rows["nyu2_train.csv"][:4]
    for name, lines in rows.items():
        with open(os.path.join(root, name), "w") as f:
            f.write("\n".join(lines) + "\n")
    np.save(os.path.join(root, "test_balanced_mask.npy"), r.rand(n_test, 228, 304) < 0.7)


def test_loaders_end_to_end(tmp_path):
    _, ld = ref()
    import depth_eval
    import loaddata
    from test_gpu_nyud2_model import loss_fn, make_model
    root = str(tmp_path)
    write_dataset(root)
    args = SimpleNamespace(data_dir=root, reweight='inverse', lds=True, lds_kernel='gaussian', lds_ks=5, lds_sigma=2,
                           bucket_num=100, bucket_start=7)
    pairs = [(loaddata.getTrainingData(args, 2, num_workers=2), ld.getTrainingData(args, 2)),
             (loaddata.getTrainingFDSData(args, 2, num_workers=0), ld.getTrainingFDSData(args, 2)),
             (loaddata.getTestingData(args, 2), ld.getTestingData(args, 2))]
    batches = {}
    for (mine, theirs), split in zip(pairs, ("train", "fds", "test")):
        got, want = next(iter(mine)), next(iter(theirs))
        assert sorted(got) == sorted(want), (split, sorted(got), sorted(want))
        for k in want:
            assert got[k].shape == want[k].shape and got[k].dtype == want[k].dtype, (split, k)
            assert got[k].is_cuda, (split, k)
        if split != "train":                       # no random draws: the same values, bit for bit
            for k in want:
                assert torch.equal(got[k].cpu(), want[k]), (split, k)
        batches[split] = got
    # one net.model Adam step from a training batch
    m = make_model(True)
    m.train()
    opt = torch.optim.Adam(m.parameters(), 1e-4, weight_decay=1e-4)
    b = batches["train"]
    before = {n: p.detach().clone() for n, p in m.named_parameters()}
    opt.zero_grad()
    out, _ = m(b["image"], b["depth"], 1)
    loss = loss_fn(out, b["depth"], b["weight"])
    loss.backward()
    opt.step()
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    assert all(torch.isfinite(p).all() and not torch.equal(p.detach(), before[n]) for n, p in m.named_parameters())
    # depth_eval.test consumes the test loader
    shot_idx = dict(many=list(range(0, 30)), medium=list(range(30, 60)), few=list(range(60, 100)))
    rmse, metrics = depth_eval.test(loaddata.getTestingData(args, 2), m, shot_idx)
    assert np.isfinite(rmse) and 'overall' in metrics


# ------------------------------------------------------------------------------------------- few SMs
@pytest.mark.parametrize("env", [{"DIRB200_SMS": "7"}], ids=["sms7"])
def test_input_pipeline_file_with_few_sms(env):
    """This file once more with 7 SMs, in a subprocess (the switch is read once per process): the grid-stride loops
    run many times per thread."""
    if os.environ.get("DIRB200_INPUT_SUBRUN"):
        pytest.skip("already in a switched subprocess")
    e = dict(os.environ, DIRB200_INPUT_SUBRUN="1", **env)
    r = subprocess.run([sys.executable, "-m", "pytest", "-q", "-p", "no:cacheprovider", os.path.abspath(__file__),
                        "-k", "not with_few_sms"], env=e, cwd=ROOT, capture_output=True, text=True, timeout=1800)
    assert r.returncode == 0, f"{env}\n" + r.stdout[-5000:] + r.stderr[-2000:]
