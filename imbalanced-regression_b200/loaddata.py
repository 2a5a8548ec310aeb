"""NYUD2-DIR's data loaders (nyud2-dir/loaddata.py) with the per-sample transform chain on the device.

The reference decodes every sample and runs nyu_transform's chain one sample at a time on the CPU (flip, spline
rotation, crop, depth resize, Lighting, ColorJitter, Normalize), then maps a Python lambda over every depth pixel for
the loss weights (loaddata.py:58-67).  Here the host decodes and applies Scale(240) only, next to the decode; the rest
runs for the whole batch in dirb200_depth_augment_batch (csrc/depth_augment.cu) from the uint8 arrays.  The random
draws are made in the main process per batch, with the reference's own generators in its per-sample order, so a
seeded run does not depend on num_workers:

    python `random`:  flip (random() < 0.5), angle (uniform(-5, 5)), then the three jitter weights (uniform(-.4, .4))
    torch generator:  Lighting's three normal_(0, 0.1) draws, ColorJitter's randperm(3)

Everything but Contrast's grayscale mean is bit-identical to the reference for the same draws: rotate + crop and the
depth resize byte for byte, depth, weights, FDS and test images bit for bit.  The mean is reduced in fp64 on the device
in a fixed order where torch reduces in fp32; the training image differs from the reference's only through it.
"""
import csv
import ctypes
import os
import random

import numpy as np
import torch
from PIL import Image
from torch.utils.data import DataLoader, Dataset

import _lib
from datasets import depth_bucket_weights

# pixel counts per 0.1 m depth bucket of the training set (loaddata.py:11-19)
TRAIN_BUCKET_NUM = [0, 0, 0, 0, 0, 0, 0, 25848691, 24732940, 53324326, 69112955, 54455432, 95637682, 71403954,
                    117244217, 84813007, 126524456, 84486706, 133130272, 95464874, 146051415, 146133612, 96561379,
                    138366677, 89680276, 127689043, 81608990, 119121178, 74360607, 106839384, 97595765, 66718296,
                    90661239, 53103021, 83340912, 51365604, 71262770, 42243737, 65860580, 38415940, 53647559, 54038467,
                    28335524, 41485143, 32106001, 35936734, 23966211, 32018765, 19297203, 31503743, 21681574, 16363187,
                    25743420, 12769509, 17675327, 13147819, 15798560, 9547180, 14933200, 9663019, 12887283, 11803562,
                    7656609, 11515700, 7756306, 9046228, 5114894, 8653419, 6859433, 8001904, 6430700, 3305839, 6318461,
                    3486268, 5621065, 4030498, 3839488, 3220208, 4483027, 2555777, 4685983, 3145082, 2951048, 2762369,
                    2367581, 2546089, 2343867, 2481579, 1722140, 3018892, 2325197, 1952354, 2047038, 1858707, 2052729,
                    1348558, 2487278, 1314198, 3338550, 1132666]

PCA_EIGVAL = torch.Tensor([0.2175, 0.0188, 0.0045])
PCA_EIGVEC = torch.Tensor([[-0.5675, 0.7192, 0.4009],
                           [-0.5808, -0.0045, -0.8140],
                           [-0.5836, -0.6948, 0.4203]])
MEAN_STD = [0.485, 0.456, 0.406, 0.229, 0.224, 0.225]      # Normalize(mean, std) of all three chains
CROP = (228, 304)                                          # CenterCrop([304, 228], ...) as (h, w)
DEPTH_TRAIN = (114, 152)                                   # ... [152, 114]: the training / FDS depth size
SCALE = 240


def scale(img, size=SCALE, interpolation=Image.BILINEAR):
    """nyu_transform.Scale.changeScale: the smaller edge to `size` (image BILINEAR, depth NEAREST)."""
    w, h = img.size
    if (w <= h and w == size) or (h <= w and h == size):
        return img
    if w < h:
        return img.resize((size, int(size * h / w)), interpolation)
    return img.resize((int(size * w / h), size), interpolation)


class depthDataset(Dataset):
    """loaddata.py:21-93 up to Scale(240): the reference's CSV format (image path, depth path, the first path component
    stripped as :73-74 does) and its bucket weights; __getitem__ returns the decoded, scaled uint8 arrays
    {'image': [H, W, 3] u8, 'depth': [H, W] u8 (u16 for split='test'), 'idx'}.  The transform runs per batch on the
    device (gpu_depth_transform_batch)."""

    def __init__(self, data_dir, csv_file, mask_file=None, args=None, split='train'):
        assert split in ('train', 'fds', 'test')
        self.data_dir = data_dir
        self.split = split
        with open(csv_file, newline='') as f:
            self.frame = [row for row in csv.reader(f) if row]
        self.mask = torch.tensor(np.load(mask_file), dtype=torch.bool) if mask_file is not None else None
        self.bucket_weights = self._get_bucket_weights(args) if args is not None else None

    @staticmethod
    def _get_bucket_weights(args):
        if args.reweight == 'none':
            assert not args.lds, "Set reweight to 'sqrt_inv' or 'inverse' (default) when using LDS"
            return None
        return depth_bucket_weights(TRAIN_BUCKET_NUM, args.reweight, args.bucket_num, args.bucket_start, args.lds,
                                    args.lds_kernel, args.lds_ks, args.lds_sigma)

    def _path(self, name):
        return os.path.join(self.data_dir, '/'.join(name.split('/')[1:]))

    def __getitem__(self, idx):
        image = scale(Image.open(self._path(self.frame[idx][0])))
        depth = scale(Image.open(self._path(self.frame[idx][1])), interpolation=Image.NEAREST)
        image = np.asarray(image.convert('RGB') if image.mode != 'RGB' else image, dtype=np.uint8)
        depth = np.asarray(depth, dtype=np.uint16 if self.split == 'test' else np.uint8)
        return {'image': image, 'depth': depth, 'idx': idx}

    def __len__(self):
        return len(self.frame)


# ------------------------------------------------------------------------------------------------------- draws
def rotate_affine(angle, h, w):
    """The affine scipy.ndimage.rotate(a, angle, reshape=False) applies over an (h, w) plane, computed with rotate's
    own numpy expressions: float64 [6] = (m00, m01, m10, m11, offset0, offset1)."""
    from scipy import special
    c, s = special.cosdg(angle), special.sindg(angle)
    rot_matrix = np.array([[c, s], [-s, c]])
    in_plane_shape = np.asarray([h, w])
    out_center = rot_matrix @ ((in_plane_shape - 1) / 2)
    offset = (in_plane_shape - 1) / 2 - out_center
    return np.array([rot_matrix[0, 0], rot_matrix[0, 1], rot_matrix[1, 0], rot_matrix[1, 1], offset[0], offset[1]])


def lighting_offset(alpha, eigval=PCA_EIGVAL, eigvec=PCA_EIGVEC):
    """Lighting's per-channel offset (nyu_transform.py:228-232) from its three normal draws, with the same torch ops."""
    return eigvec.clone().mul(alpha.view(1, 3).expand(3, 3)).mul(eigval.view(1, 3).expand(3, 3)).sum(1).squeeze()


def draw_nyud2_train_params(n, rng=random, generator=None, shape=(SCALE, 320)):
    """The random draws of the training chain for n samples, consumed in exactly the reference's per-sample order:
    flip (rng.random()), angle (rng.uniform(-5, 5)), Lighting's 3 normals (torch), the jitter order (torch.randperm(3)),
    then one rng.uniform(-0.4, 0.4) per jitter transform in that order.  `generator`: the torch generator (None: the
    global one, as the reference).  Returns a dict of CPU tensors: flip u8 [n], angle f64 [n], affine f64 [n, 6] for
    a source of `shape` (h, w), rgb f32 [n, 3] (Lighting's offsets), order i32 [n, 3] (0 brightness, 1 contrast,
    2 saturation) and alpha f32 [n, 3] (the k-th applied transform's weight as torch's lerp uses it)."""
    flip = torch.zeros(n, dtype=torch.uint8)
    angle = torch.zeros(n, dtype=torch.float64)
    rgb = torch.zeros(n, 3, dtype=torch.float32)
    order = torch.zeros(n, 3, dtype=torch.int32)
    alpha = torch.zeros(n, 3, dtype=torch.float32)
    for k in range(n):
        flip[k] = 1 if rng.random() < 0.5 else 0                        # RandomHorizontalFlip
        angle[k] = rng.uniform(-5, 5)                                   # RandomRotate(5)
        a = torch.empty(3).normal_(0, 0.1, generator=generator)         # Lighting(0.1, ...)
        rgb[k] = lighting_offset(a)
        perm = torch.randperm(3, generator=generator)                   # ColorJitter: RandomOrder
        order[k] = perm.to(torch.int32)
        for j in range(3):
            alpha[k, j] = float(np.float32(rng.uniform(-0.4, 0.4)))
    affine = torch.from_numpy(np.stack([rotate_affine(float(a), *shape) for a in angle])) if n else \
        torch.zeros(0, 6, dtype=torch.float64)
    return {'flip': flip, 'angle': angle, 'affine': affine, 'rgb': rgb, 'order': order, 'alpha': alpha}


# ------------------------------------------------------------------------------------------------------- device
def gpu_depth_transform_batch(images_u8, depths, split='train', params=None, bucket_weights=None, rng=random,
                              generator=None, debug=False):
    """images_u8 u8 [N, H, W, 3], depths u8 [N, H, W] (u16 for split='test'), CUDA -> dict(image f32 [N, 3, 228, 304],
    depth f32 [N, 1, h, w], weight f32 [N, 1, h, w]) with (h, w) = (114, 152) for 'train' / 'fds' and (228, 304) for
    'test' (whose depths may be int16 or uint16: the kernel reads the bits as int16, as the reference's
    np.array(pic, np.int16) does).  split='train' draws the parameters (or takes `params` from draw_nyud2_train_params); bucket_weights: the
    100-entry table (None: ones).  debug=True adds 'crop' (u8 [N, 228, 304, 4]: R, G, B, depth after flip, rotation and
    crop) and, for 'train', 'mean' (f32 [N], Contrast's grayscale mean)."""
    assert split in ('train', 'fds', 'test')
    _lib.require_cuda(images_u8, depths)
    assert images_u8.dtype == torch.uint8 and images_u8.dim() == 4 and images_u8.shape[3] == 3
    n, h, w = images_u8.shape[:3]
    assert depths.shape == (n, h, w)
    dev = images_u8.device
    images_u8 = images_u8.contiguous()
    if split == 'test':
        assert depths.dtype in (torch.uint16, torch.int16), "the test chain takes 16-bit depths"
    else:
        assert depths.dtype == torch.uint8, "the training / FDS chains take 8-bit depths"
    depths = depths.contiguous()
    dh, dw = CROP if split == 'test' else DEPTH_TRAIN
    flip = affine = rgb = order = alpha = None
    if split == 'train':
        if params is None:
            params = draw_nyud2_train_params(n, rng, generator, (h, w))
        aff = torch.from_numpy(np.stack([rotate_affine(float(a), h, w) for a in params['angle']]))
        flip = params['flip'].to(device=dev, dtype=torch.uint8).contiguous()
        affine = aff.to(device=dev, dtype=torch.float64).contiguous()
        rgb = params['rgb'].to(device=dev, dtype=torch.float32).contiguous()
        order = params['order'].to(device=dev, dtype=torch.int32).contiguous()
        alpha = params['alpha'].to(device=dev, dtype=torch.float32).contiguous()
    table = None
    if bucket_weights is not None:
        table = torch.as_tensor(np.asarray(bucket_weights, dtype=np.float32), device=dev).contiguous()
    out = {'image': torch.empty(n, 3, *CROP, device=dev), 'depth': torch.empty(n, 1, dh, dw, device=dev),
           'weight': torch.empty(n, 1, dh, dw, device=dev)}
    crop = torch.empty(n, *CROP, 4, dtype=torch.uint8, device=dev) if debug else None
    mean = torch.empty(n, device=dev) if debug and split == 'train' else None
    nb = _lib.raw("dirb200_depth_augment_workspace_bytes")(n, h, w, *CROP)
    ws = torch.empty(nb, dtype=torch.uint8, device=dev)
    mean_std = (ctypes.c_float * 6)(*MEAN_STD)
    _lib.call("dirb200_depth_augment_batch", _lib.ptr(images_u8), _lib.ptr(depths), 1 if split == 'test' else 0, n, h,
              w, CROP[0], CROP[1], dh, dw, _lib.ptr(flip), _lib.ptr(affine), _lib.ptr(rgb), _lib.ptr(order),
              _lib.ptr(alpha), mean_std, _lib.ptr(table), 0 if table is None else table.numel(), _lib.ptr(out['image']),
              _lib.ptr(out['depth']), _lib.ptr(out['weight']), _lib.ptr(crop), _lib.ptr(mean), _lib.ptr(ws), nb,
              _lib.stream_ptr())
    if debug:
        out['crop'] = crop
        if mean is not None:
            out['mean'] = mean
    return out


# ------------------------------------------------------------------------------------------------------- loaders
def _collate(samples):
    return {'image': torch.from_numpy(np.stack([s['image'] for s in samples])),
            'depth': torch.from_numpy(np.stack([s['depth'].astype(np.int16) if s['depth'].dtype == np.uint16
                                                else s['depth'] for s in samples])),
            'idx': torch.tensor([s['idx'] for s in samples], dtype=torch.int64)}


class DeviceLoader:
    """Iterates a host DataLoader of decoded, scaled uint8 batches and transforms each batch on the device.  Yields the
    reference's batch dicts, already on the GPU: image f32 [B, 3, 228, 304], depth / weight f32 [B, 1, h, w], idx i64
    [B], and for the test set mask bool [B, 1, 228, 304]."""

    def __init__(self, dataset, batch_size, shuffle, num_workers, device=None, rng=random, generator=None):
        self.dataset = dataset
        self.loader = DataLoader(dataset, batch_size, shuffle=shuffle, num_workers=num_workers, collate_fn=_collate,
                                 pin_memory=torch.cuda.is_available())
        self.device = torch.device(device) if device is not None else torch.device('cuda')
        self.rng, self.generator = rng, generator

    def __len__(self):
        return len(self.loader)

    def __iter__(self):
        for b in self.loader:
            image = b['image'].to(self.device, non_blocking=True)
            depth = b['depth'].to(self.device, non_blocking=True)
            out = gpu_depth_transform_batch(image, depth, self.dataset.split, bucket_weights=self.dataset.bucket_weights,
                                            rng=self.rng, generator=self.generator)
            out['idx'] = b['idx'].to(self.device)
            if self.dataset.mask is not None:
                out['mask'] = self.dataset.mask[b['idx']].unsqueeze(1).to(self.device)
            yield out


def getTrainingData(args, batch_size=64, num_workers=8):
    """loaddata.py:96-130: nyu2_train.csv, the training chain with the bucket weights of `args`, shuffled."""
    ds = depthDataset(args.data_dir, os.path.join(args.data_dir, 'nyu2_train.csv'), args=args, split='train')
    return DeviceLoader(ds, batch_size, True, num_workers)


def getTrainingFDSData(args, batch_size=64, num_workers=8):
    """loaddata.py:132-148: nyu2_train_FDS_subset.csv, Scale -> CenterCrop with the depth resize -> ToTensor ->
    Normalize, weights all ones, in order."""
    ds = depthDataset(args.data_dir, os.path.join(args.data_dir, 'nyu2_train_FDS_subset.csv'), split='fds')
    return DeviceLoader(ds, batch_size, False, num_workers)


def getTestingData(args, batch_size=64, num_workers=0):
    """loaddata.py:151-170: nyu2_test.csv with test_balanced_mask.npy, the crop at full depth resolution, 16-bit depth
    / 1000, weights all ones, in order."""
    ds = depthDataset(args.data_dir, os.path.join(args.data_dir, 'nyu2_test.csv'),
                      mask_file=os.path.join(args.data_dir, 'test_balanced_mask.npy'), split='test')
    return DeviceLoader(ds, batch_size, False, num_workers)
