"""datasets.py -- mirror of agedb-dir/datasets.py / imdb-wiki-dir/datasets.py.

The hot-path piece is `_prepare_weights` (datasets.py:55-83): the label
histogram (int64, bit exact), the sqrt / clip re-weighting, the LDS
convolution and the per-sample weight gather run in libdirb200
(dirb200_lds_histogram / dirb200_lds_weights).  The image pipeline
(PIL decode, crop, flip, normalise; datasets.py:27-53) is out of scope of the
hot path (SURVEY.md §2a row 8) and kept as thin torchvision host code.
"""
import io
import logging
import os

import numpy as np
import torch
from torch.utils import data

import _lib
from utils import get_lds_kernel_window

print = logging.info


def lds_prepare_weights(labels, reweight, max_target=121, lds=False, lds_kernel='gaussian', lds_ks=5, lds_sigma=2,
                        device=None, return_hist=False, sharded=False):
    """GPU implementation of AgeDB._prepare_weights.  Returns a float32 CUDA
    tensor [N] (or None for reweight == 'none'); with return_hist also the
    int64 histogram.

    `labels` must be the WHOLE training label column (what the reference's dataset object holds) -- train.py builds
    the dataset over the whole split on every rank and shards by sampler.  `sharded=True` is for callers that hold
    only `rank::world` of the column: the int64 histogram and the sample count are then SUM-all-reduced over the
    default process group before the per-bin table and the len/sum(w) normaliser are formed, which gives every
    sample exactly the weight the unsharded call gives it (SURVEY.md section 8e(3))."""
    assert reweight in {'none', 'inverse', 'sqrt_inv'}
    assert reweight != 'none' if lds else True, \
        "Set reweight to 'sqrt_inv' (default) or 'inverse' when using LDS"
    if reweight == 'none' and not return_hist:       # the reference returns None before counting anything (datasets.py:59)
        return None
    device = device or torch.device('cuda')
    lab = torch.as_tensor(np.array(labels, dtype=np.float32)).reshape(-1).to(device).contiguous()
    n = lab.numel()
    hist = torch.zeros(max_target, dtype=torch.int64, device=device)
    st = _lib.stream_ptr()
    _lib.call("dirb200_lds_histogram", _lib.ptr(lab), n, max_target, _lib.ptr(hist), st)
    n_total = n
    if sharded:
        import torch.distributed as dist
        if dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1:
            cnt = torch.tensor([n], dtype=torch.int64, device=device)
            dist.all_reduce(hist, op=dist.ReduceOp.SUM)
            dist.all_reduce(cnt, op=dist.ReduceOp.SUM)
            n_total = int(cnt.item())
    if n == 0 or reweight == 'none':
        return (None, hist) if return_hist else None
    print(f"Using re-weighting: [{reweight.upper()}]")
    window, ks = None, 0
    if lds:
        window = np.ascontiguousarray(get_lds_kernel_window(lds_kernel, lds_ks, lds_sigma), dtype=np.float64)
        ks = len(window)
        print(f'Using LDS: [{lds_kernel.upper()}] ({lds_ks}/{lds_sigma})')
    scratch = torch.empty(2 * max_target + 2, dtype=torch.float64, device=device)
    weights = torch.empty(n, dtype=torch.float32, device=device)
    _lib.call("dirb200_lds_weights_sharded", _lib.ptr(lab), n, n_total, max_target, _lib.REWEIGHT[reweight],
              None if window is None else window.ctypes.data_as(_lib.P), ks, _lib.ptr(hist), _lib.ptr(scratch),
              _lib.ptr(weights), st)
    return (weights, hist) if return_hist else weights


class AgeDB(data.Dataset):
    label_column = 'age'

    def __init__(self, df, data_dir, img_size, split='train', reweight='none',
                 lds=False, lds_kernel='gaussian', lds_ks=5, lds_sigma=2, device_transform=False, device_decode=False):
        # device_transform (not in the reference): __getitem__ stops after the resize and returns the uint8 HWC image;
        # the rest of get_transform() runs on the GPU for the whole batch (gpu_transform_batch below).
        # device_decode (implies device_transform): __getitem__ returns a JPEG in the device decoder's supported set as
        # its bytes (EncodedJpeg); jpeg_collate + JpegBatch.cuda() decode and resize the batch on the GPU
        self.device_transform = device_transform or device_decode
        self.device_decode = device_decode
        self.df = df
        self.data_dir = data_dir
        self.img_size = img_size
        self.split = split
        w = self._prepare_weights(reweight=reweight, lds=lds, lds_kernel=lds_kernel, lds_ks=lds_ks,
                                  lds_sigma=lds_sigma)
        self.weights = None if w is None else w.cpu().numpy()

    def __len__(self):
        return len(self.df)

    def __getitem__(self, index):
        from PIL import Image
        index = index % len(self.df)
        row = self.df.iloc[index]
        path = os.path.join(self.data_dir, row['path'])
        img = None
        if self.device_decode:
            with open(path, 'rb') as f:
                raw = f.read()
            rc, desc, intervals = parse_jpeg(raw)
            if rc == 0:
                img = EncodedJpeg(raw, desc, intervals, self.img_size)
        if img is None:
            img = Image.open(path).convert('RGB')
            img = host_resize_u8(img, self.img_size) if self.device_transform else self.get_transform()(img)
        label = np.asarray([row[self.label_column]]).astype('float32')
        weight = np.asarray([self.weights[index]]).astype('float32') if self.weights is not None else \
            np.asarray([np.float32(1.)])
        return img, label, weight

    def get_transform(self):
        from torchvision import transforms
        norm = [transforms.ToTensor(), transforms.Normalize([.5, .5, .5], [.5, .5, .5])]
        size = (self.img_size, self.img_size)
        if self.split == 'train':
            return transforms.Compose([transforms.Resize(size), transforms.RandomCrop(self.img_size, padding=16),
                                       transforms.RandomHorizontalFlip()] + norm)
        return transforms.Compose([transforms.Resize(size)] + norm)

    def _prepare_weights(self, reweight, max_target=121, lds=False, lds_kernel='gaussian', lds_ks=5, lds_sigma=2):
        return lds_prepare_weights(self.df[self.label_column].values, reweight, max_target, lds, lds_kernel,
                                   lds_ks, lds_sigma)


class IMDBWIKI(AgeDB):
    pass


def host_resize_u8(img, size):
    """transforms.Resize((size, size)) of a PIL image as a uint8 HWC tensor: the device_transform sample."""
    from torchvision import transforms
    return torch.from_numpy(np.asarray(transforms.Resize((size, size))(img)).copy())


# ------------------------------------------------------------------ JPEG decode + resize on the device
# dirb200_jpeg_desc (include/dirb200.h), field for field
JPEG_DESC_DTYPE = np.dtype([(k, '<i4') for k in ('height', 'width', 'ncomp', 'hmax', 'vmax', 'mcus_x', 'mcus_y',
                                                 'restart_interval', 'n_intervals', 'scan_begin', 'scan_end')] +
                           [(k, '<i4', (3,)) for k in ('comp_h', 'comp_v', 'comp_tq', 'comp_td', 'comp_ta')] +
                           [('qt', '<u2', (4, 64)), ('huff_bits', 'u1', (2, 4, 16)), ('huff_vals', 'u1', (2, 4, 256))])
JPEG_DESC_BYTES = int(_lib.raw("dirb200_jpeg_desc_bytes")())
assert JPEG_DESC_DTYPE.itemsize == JPEG_DESC_BYTES, (JPEG_DESC_DTYPE.itemsize, JPEG_DESC_BYTES)


def parse_jpeg(raw):
    """dirb200_jpeg_parse on one file's bytes (host only, no CUDA call): (rc, desc uint8 [JPEG_DESC_BYTES],
    intervals int32 [n_intervals]).  rc 0: supported; > 0: not a supported JPEG; < 0: a malformed JPEG."""
    a = np.frombuffer(raw, dtype=np.uint8)
    desc = np.zeros(JPEG_DESC_BYTES, dtype=np.uint8)
    intervals = np.zeros((len(a) + 3) // 2, dtype=np.int32)
    rc = _lib.raw("dirb200_jpeg_parse")(a.ctypes.data_as(_lib.P) if len(a) else None, len(a),
                                        desc.ctypes.data_as(_lib.P), intervals.ctypes.data_as(_lib.P), len(intervals))
    if rc == _lib.DIRB200_ERR_ARG:
        raise _lib.Dirb200Error(f"dirb200_jpeg_parse: {_lib.last_error()}")
    n_iv = int(desc.view(JPEG_DESC_DTYPE)[0]['n_intervals']) if rc == 0 else 0
    return rc, desc, intervals[:n_iv].copy()


class EncodedJpeg:
    """One supported JPEG as AgeDB(device_decode=True) yields it: the file's bytes, its descriptor and restart-interval
    table, and the square size it is to be resized to."""
    __slots__ = ('raw', 'desc', 'intervals', 'size')

    def __init__(self, raw, desc, intervals, size):
        self.raw, self.desc, self.intervals, self.size = raw, desc, intervals, size

    @property
    def hw(self):
        d = self.desc.view(JPEG_DESC_DTYPE)[0]
        return int(d['height']), int(d['width'])


_DECODE_STATS = {'device': 0, 'flagged': 0, 'host': 0}


def take_device_decode_stats():
    """Images since the last call: decoded on the device, flagged by it (and decoded by Pillow after the batch's
    status read), and decoded by Pillow in the loader (outside the supported set)."""
    out = dict(_DECODE_STATS)
    for k in _DECODE_STATS:
        _DECODE_STATS[k] = 0
    return out


class JpegBatch:
    """A batch of AgeDB(device_decode=True) samples: the supported JPEGs packed for dirb200_jpeg_decode (bytes,
    offsets, descriptors, interval tables) and the images the loader already decoded and resized, with their batch
    positions.  .cuda() returns the uint8 [N, S, S, 3] tensor that stacking AgeDB(device_transform=True) items gives."""

    def __init__(self, items):
        self.n = len(items)
        self.jpeg_pos = [i for i, it in enumerate(items) if isinstance(it, EncodedJpeg)]
        self.host_pos = [i for i, it in enumerate(items) if not isinstance(it, EncodedJpeg)]
        jp = [items[i] for i in self.jpeg_pos]
        sizes = {it.size for it in jp} | {int(items[i].shape[0]) for i in self.host_pos}
        assert len(sizes) == 1, f"one image size per batch, got {sorted(sizes)}"
        self.size = sizes.pop()
        self.host = torch.stack([items[i] for i in self.host_pos]) if self.host_pos else None
        self.raw_lengths = [len(it.raw) for it in jp]
        lens = np.asarray(self.raw_lengths, dtype=np.int64)
        self.offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)]).astype(np.int64))
        self.data = torch.from_numpy(np.frombuffer(b''.join(it.raw for it in jp), dtype=np.uint8).copy())
        descs = np.stack([it.desc for it in jp]) if jp else np.zeros((0, JPEG_DESC_BYTES), np.uint8)
        self.descs = torch.from_numpy(descs)
        self.intervals = torch.from_numpy(np.concatenate([it.intervals for it in jp]) if jp else np.zeros(0, np.int32))
        hw = np.asarray([it.hw for it in jp], dtype=np.int32).reshape(-1, 2)
        self.hw = torch.from_numpy(hw)
        self.rgb_offsets = torch.from_numpy(np.concatenate([[0], np.cumsum(hw[:, 0].astype(np.int64) * hw[:, 1] * 3)])
                                            .astype(np.int64))
        m = len(jp)
        self.decode_ws = int(_lib.raw("dirb200_jpeg_decode_workspace_bytes")(descs.ctypes.data_as(_lib.P), m)) if m else 0
        self.resize_ws = int(_lib.raw("dirb200_resize_bilinear_workspace_bytes")(
            hw.ctypes.data_as(_lib.P), m, self.size, self.size)) if m else 0
        self.flagged = None

    def pin_memory(self):
        for k in ('data', 'offsets', 'descs', 'intervals', 'hw', 'rgb_offsets', 'host'):
            t = getattr(self, k)
            if t is not None and t.numel():
                setattr(self, k, t.pin_memory())
        return self

    def _host_decode(self, j):
        from PIL import Image
        lo = int(self.offsets[j])
        raw = self.data[lo:lo + self.raw_lengths[j]].numpy().tobytes()
        return host_resize_u8(Image.open(io.BytesIO(raw)).convert('RGB'), self.size)

    def cuda(self, device=None, non_blocking=False):
        dev = torch.device('cuda', torch.cuda.current_device()) if device is None else torch.device(device)
        S, m = self.size, len(self.jpeg_pos)
        out = torch.empty(self.n, S, S, 3, dtype=torch.uint8, device=dev)
        if self.host is not None:
            out[torch.tensor(self.host_pos, device=dev)] = self.host.to(dev, non_blocking=non_blocking)
        self.flagged = []
        if m:
            up = lambda t: t.to(dev, non_blocking=non_blocking)
            data, offsets, descs, intervals, hw, rgb_offsets = map(up, (self.data, self.offsets, self.descs,
                                                                       self.intervals, self.hw, self.rgb_offsets))
            rgb = torch.empty(int(self.rgb_offsets[-1]), dtype=torch.uint8, device=dev)
            status = torch.empty(m, dtype=torch.int32, device=dev)
            ws = torch.empty(self.decode_ws, dtype=torch.uint8, device=dev)
            st = _lib.stream_ptr()
            _lib.call("dirb200_jpeg_decode", _lib.ptr(data), _lib.ptr(offsets), _lib.ptr(descs), _lib.ptr(intervals), m,
                      _lib.ptr(rgb), _lib.ptr(rgb_offsets), _lib.ptr(status), _lib.ptr(ws), ws.numel(), st)
            dst = out if m == self.n else torch.empty(m, S, S, 3, dtype=torch.uint8, device=dev)
            rws = torch.empty(self.resize_ws, dtype=torch.uint8, device=dev)
            _lib.call("dirb200_resize_bilinear_u8", _lib.ptr(rgb), _lib.ptr(rgb_offsets), _lib.ptr(hw), m, S, S,
                      _lib.ptr(dst), _lib.ptr(rws), rws.numel(), st)
            if dst is not out:
                out[torch.tensor(self.jpeg_pos, device=dev)] = dst
            # the batch's one host sync: images the device flagged are decoded again by Pillow, so their pixels,
            # warnings and exceptions are Pillow's
            self.flagged = torch.nonzero(status.cpu()).flatten().tolist()
            for j in self.flagged:
                out[self.jpeg_pos[j]] = self._host_decode(j).to(dev)
        _DECODE_STATS['device'] += m - len(self.flagged)
        _DECODE_STATS['flagged'] += len(self.flagged)
        _DECODE_STATS['host'] += len(self.host_pos)
        return out


def jpeg_collate(batch):
    """collate_fn for AgeDB(device_decode=True): (JpegBatch, labels, weights), the labels and weights collated as the
    default collate does."""
    from torch.utils.data import default_collate
    labels, weights = default_collate([b[1:] for b in batch])
    return JpegBatch([b[0] for b in batch]), labels, weights


# ------------------------------------------------------------------ dense (NYUD2) LDS weights
def depth_bucket_weights(train_bucket_num, reweight, bucket_num=100, bucket_start=7, lds=False, lds_kernel='gaussian',
                         lds_ks=5, lds_sigma=2):
    """Per-bucket loss weights of nyud2-dir/loaddata.py:29-50 (host side, 100 numbers, once per run).
    `train_bucket_num`: pixel counts per 0.1 m depth bucket (the reference hard-codes its TRAIN_BUCKET_NUM)."""
    from scipy.ndimage import convolve1d
    assert reweight in {'none', 'inverse', 'sqrt_inv'}
    assert reweight != 'none' if lds else True, "Set reweight to 'sqrt_inv' or 'inverse' (default) when using LDS"
    if reweight == 'none':
        return None
    counts = list(train_bucket_num)
    if lds:
        values = counts[bucket_start:]
        if reweight == 'sqrt_inv':
            values = np.sqrt(values)
        window = get_lds_kernel_window(lds_kernel, lds_ks, lds_sigma)
        smoothed = convolve1d(np.asarray(values), weights=window, mode='reflect')
        per_bucket = [smoothed[0]] * bucket_start + list(smoothed)
    else:
        per_bucket = [counts[bucket_start]] * bucket_start + counts[bucket_start:]
        if reweight == 'sqrt_inv':
            per_bucket = np.sqrt(per_bucket)
    scaling = np.sum(counts) / np.sum(np.array(counts) / np.array(per_bucket))
    return np.asarray([np.float32(scaling / per_bucket[b]) for b in range(bucket_num)], dtype=np.float32)


def depth_pixel_weights(depth, bucket_weights):
    """weights[i] = bucket_weights[min(int(depth[i] * 10), 99)] for a whole depth map on the GPU (the reference maps a
    Python lambda over every pixel on the CPU, loaddata.py:52-64)."""
    _lib.require_cuda(depth)
    d = depth.detach().to(torch.float32).contiguous()
    table = torch.as_tensor(np.asarray(bucket_weights, dtype=np.float32), device=d.device)
    out = torch.empty_like(d)
    _lib.call("dirb200_lds_table_lookup", _lib.ptr(d), d.numel(), 10.0, table.numel() - 1, _lib.ptr(table),
              _lib.ptr(out), _lib.stream_ptr())
    return out


# ------------------------------------------------------------------ STS-B re-weighting / LDS
def stsb_weights_from_bins(bins, reweight, lds=False, lds_kernel='gaussian', lds_ks=5, lds_sigma=2, bucket_num=50):
    """Host part of sts-b-dir/tasks.py:44-73 (50 numbers + one gather over <= 6k sentence pairs, once per run): bin
    histogram, sqrt for 'sqrt_inv', LDS convolve (zero padded; scipy keeps an integer histogram integer, as the
    reference's call does), weight = float32(1 / value[bin]) rescaled to mean 1.  `bins`: int bucket index per sample.
    Returns (weights float32 [N], hist int64 [bucket_num])."""
    from scipy.ndimage import convolve1d
    assert reweight in {'inverse', 'sqrt_inv'}
    bins = np.asarray(bins, dtype=np.int64).reshape(-1)
    hist = np.bincount(bins, minlength=bucket_num).astype(np.int64)
    value_lst = np.sqrt(hist) if reweight == 'sqrt_inv' else hist
    print(f"Using re-weighting: [{reweight.upper()}]")
    if lds:
        window = get_lds_kernel_window(lds_kernel, lds_ks, lds_sigma)
        print(f'Using LDS: [{lds_kernel.upper()}] ({lds_ks}/{lds_sigma})')
        value_lst = convolve1d(value_lst, weights=window, mode='constant')
    with np.errstate(divide='ignore'):
        weights = (1.0 / np.asarray(value_lst)[bins]).astype(np.float32)
    scaling = np.float32(len(weights)) / np.sum(weights)
    return (np.float32(scaling) * weights).astype(np.float32), hist


def stsb_prepare_weights(scores, reweight, lds=False, lds_kernel='gaussian', lds_ks=5, lds_sigma=2, bucket_num=50,
                         device=None):
    """Loss weights of the STS-B loader (sts-b-dir/tasks.py:44-73).  The score -> bucket rule (np.histogram edges over
    [0, 5] in float32, 5.0 in the last bucket) is the same bit-exact kernel the STS-B FDS module bins with
    (dirb200_fds_bin_rows, DIRB200_BIN_EDGES5), so LDS and FDS can never disagree about a sample's bucket; the
    50-number table work stays on the host.  Returns a float32 CUDA tensor [N], or None for reweight == 'none'."""
    assert reweight in {'none', 'inverse', 'sqrt_inv'}
    assert reweight != 'none' if lds else True, "Set reweight to 'inverse' (default) or 'sqrt_inv' when using LDS"
    if reweight == 'none':
        return None
    device = device or torch.device('cuda')
    lab = torch.as_tensor(np.asarray(scores), dtype=torch.float32).reshape(-1).to(device).contiguous()
    _lib.require_cuda(lab)
    n = lab.numel()
    bins = torch.empty(n, dtype=torch.int32, device=device)
    flags = torch.zeros(2, dtype=torch.int32, device=device)
    _lib.call("dirb200_fds_bin_rows", _lib.ptr(lab), n, bucket_num, 0, _lib.BIN_EDGES5, _lib.ptr(flags), _lib.ptr(bins),
              _lib.stream_ptr())
    weights, _ = stsb_weights_from_bins(bins.cpu().numpy(), reweight, lds, lds_kernel, lds_ks, lds_sigma, bucket_num)
    return torch.from_numpy(weights).to(device)


# ---------------------------------------------------------------------------------------------------------------------
# Input pipeline on the device (SURVEY section 8f-4).  The reference transforms every sample on the host, one PIL image
# at a time (datasets.py:38-53).  Here everything after the resize -- RandomCrop(img_size, padding=16),
# RandomHorizontalFlip, ToTensor, Normalize -- runs as ONE kernel over the batch of uint8 images (a quarter of the bytes
# of the fp32 tensor cross PCIe).  With device_decode the JPEG decode and the resize run on the device too (JpegBatch
# above); images outside the decoder's supported set are decoded and resized on the host in the loader.
def draw_augment_params(n, size, pad=16, generator=None):
    """The random draws of RandomCrop(size, padding=pad) + RandomHorizontalFlip() for n samples, consumed from the torch
    generator in exactly the order the reference's per-sample Compose does (crop row, crop column, flip coin), so that
    a seeded run reproduces torchvision's choices: returns (crop_yx int32 [n, 2], flip uint8 [n])."""
    crop = torch.empty(n, 2, dtype=torch.int32)
    flip = torch.empty(n, dtype=torch.uint8)
    for k in range(n):
        # transforms.RandomCrop.get_params: the padded image is (size + 2 pad)^2, the crop size^2
        crop[k, 0] = int(torch.randint(0, 2 * pad + 1, size=(1,), generator=generator).item())
        crop[k, 1] = int(torch.randint(0, 2 * pad + 1, size=(1,), generator=generator).item())
        flip[k] = 1 if float(torch.rand(1, generator=generator)) < 0.5 else 0      # RandomHorizontalFlip(p=0.5)
    return crop, flip


def gpu_transform_batch(images_u8, train=True, pad=16, crop_yx=None, flip=None, generator=None, out=None):
    """images_u8: uint8 [N, S, S, 3] (RGB, HWC, already resized to img_size) on the GPU -> float32 [N, 3, S, S], the tensor
    the reference's train / val transform (datasets.py:38-53) produces, bit for bit for the same draws.
    train=True draws the crop origins / flips (or takes crop_yx / flip); train=False is the validation chain."""
    assert images_u8.is_cuda and images_u8.dtype == torch.uint8 and images_u8.dim() == 4 and images_u8.shape[3] == 3
    assert images_u8.shape[1] == images_u8.shape[2], "square images (Resize((img_size, img_size)))"
    images_u8 = images_u8.contiguous()
    n, size = images_u8.shape[0], images_u8.shape[1]
    dev = images_u8.device
    if train:
        if crop_yx is None or flip is None:
            crop_yx, flip = draw_augment_params(n, size, pad, generator)
        crop_yx = crop_yx.to(device=dev, dtype=torch.int32).contiguous()
        flip = flip.to(device=dev, dtype=torch.uint8).contiguous()
        assert crop_yx.shape == (n, 2) and flip.shape == (n,)
    else:
        crop_yx = flip = None
    if out is None:
        out = torch.empty(n, 3, size, size, dtype=torch.float32, device=dev)
    _lib.call("dirb200_augment_batch", _lib.ptr(images_u8), _lib.ptr(crop_yx) if crop_yx is not None else None,
              _lib.ptr(flip) if flip is not None else None, n, size, pad, 0.5, 0.5, _lib.ptr(out), _lib.stream_ptr())
    return out
