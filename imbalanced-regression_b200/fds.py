"""fds.FDS -- drop-in mirror of the reference module (agedb-dir/fds.py:14-144,
imdb-wiki-dir/fds.py) whose arithmetic runs in libdirb200's sm_90a kernels.

Same constructor, same eight registered buffers (identical state_dict keys and
shapes, fds.py:28-35), same methods and state machine -- including the
by-reference alias of `running_*_last_epoch` onto `running_*` (fds.py:55-56)
-- but:

  * `smooth` is ONE fused kernel (+ its backward) instead of ~93 masked
    gather/scatter rounds with host syncs per step;
  * `update_running_stats` is a counting sort of the rows by label bin plus ONE
    segmented fp64 (count, sum, sum^2) reduction that reads every feature once;
  * the epoch-end collection can be STREAMED batch by batch on the device
    (`begin_epoch_stats / accumulate_batch / finish_epoch_stats`), removing the
    GPU->CPU->GPU round trip of agedb-dir/train.py:276-279, and the
    accumulators all-reduce across ranks by plain addition.
"""
import logging

import numpy as np
import torch
import torch.nn as nn
from scipy.ndimage import gaussian_filter1d
from scipy.signal.windows import triang

import _lib
from utils import calibrate_mean_var  # noqa: F401  (re-exported like the reference does)

print = logging.info


class _CalibrateFn(torch.autograd.Function):
    """In-place FDS.smooth: y = x (untouched rows/channels) or
    (x - m1) * sqrt(clamp(v2 / v1)) + m2; backward scales the gradient."""

    @staticmethod
    def forward(ctx, x, labels, m1, v1, m2, v2, bucket_num, bucket_start, clip_min, clip_max, bin_rule=0):
        _lib.require_cuda(x, labels, m1, v1, m2, v2)
        assert x.dtype == torch.float32 and x.is_contiguous() and x.dim() == 2
        b, d = x.shape
        labels = labels.reshape(-1).to(torch.float32).contiguous()
        assert labels.numel() == b
        rowbin = torch.empty(b, dtype=torch.int32, device=x.device)
        scratch = torch.empty(2, dtype=torch.int32, device=x.device) if b > 2048 else None
        _lib.call("dirb200_fds_calibrate_fwd", _lib.ptr(x), _lib.ptr(labels), b, d, bucket_num, bucket_start,
                  bin_rule, _lib.ptr(m1), _lib.ptr(v1), _lib.ptr(m2), _lib.ptr(v2), clip_min, clip_max,
                  _lib.ptr(rowbin), _lib.ptr(scratch), _lib.stream_ptr())
        ctx.mark_dirty(x)
        ctx.save_for_backward(rowbin, v1, v2)
        ctx.clip = (clip_min, clip_max)
        ctx.bin_rule = bin_rule
        return x

    @staticmethod
    def backward(ctx, g):
        rowbin, v1, v2 = ctx.saved_tensors
        g = g.contiguous()
        out = torch.empty_like(g)
        b, d = g.shape
        _lib.call("dirb200_fds_calibrate_bwd", ctx.bin_rule, _lib.ptr(g), _lib.ptr(rowbin), b, d, _lib.ptr(v1),
                  _lib.ptr(v2), ctx.clip[0], ctx.clip[1], _lib.ptr(out), _lib.stream_ptr())
        return (out,) + (None,) * 10


class FDS(nn.Module):

    clip = (0.1, 10.0)      # calibrate_mean_var defaults, agedb-dir/utils.py:97
    bin_rule = _lib.BIN_AGE  # label -> bucket rule (see include/dirb200.h); variants in fds_variants.py
    fill_empty = False      # sts-b-dir/fds.py:112-125

    def __init__(self, feature_dim, bucket_num=100, bucket_start=3, start_update=0, start_smooth=1,
                 kernel='gaussian', ks=5, sigma=2, momentum=0.9):
        super(FDS, self).__init__()
        self.feature_dim = feature_dim
        self.bucket_num = bucket_num
        self.bucket_start = bucket_start
        self.kernel_window = self._get_kernel_window(kernel, ks, sigma)
        self.half_ks = (ks - 1) // 2
        self.momentum = momentum
        self.start_update = start_update
        self.start_smooth = start_smooth

        nb = bucket_num - bucket_start
        self.register_buffer('epoch', torch.zeros(1).fill_(start_update))
        for name, init in (('running_mean', 0.), ('running_var', 1.), ('running_mean_last_epoch', 0.),
                           ('running_var_last_epoch', 1.), ('smoothed_mean_last_epoch', 0.),
                           ('smoothed_var_last_epoch', 1.)):
            self.register_buffer(name, torch.full((nb, feature_dim), init))
        self.register_buffer('num_samples_tracked', torch.zeros(nb))
        # host copy of `epoch`: the reference's gates (`epoch == self.epoch + 1`,
        # `epoch < self.epoch`) would cost a device sync per call on a CUDA buffer
        self._epoch_host = int(start_update)
        self._acc = None

    # ------------------------------------------------------------------ windows
    @staticmethod
    def _get_kernel_window(kernel, ks, sigma):
        """float32, sum-normalised taps; same recipe as agedb-dir/fds.py:37-52."""
        assert kernel in ['gaussian', 'triang', 'laplace']
        half_ks = (ks - 1) // 2
        if kernel == 'gaussian':
            impulse = np.zeros(ks, dtype=np.float32)
            impulse[half_ks] = 1.
            resp = gaussian_filter1d(impulse, sigma=sigma)
            window = resp / sum(resp)
        elif kernel == 'triang':
            window = triang(ks) / sum(triang(ks))
        else:
            taps = [np.exp(-abs(x) / sigma) / (2. * sigma) for x in np.arange(-half_ks, half_ks + 1)]
            window = np.asarray(taps) / sum(taps)
        print(f'Using FDS: [{kernel.upper()}] ({ks}/{sigma})')
        w = torch.tensor(np.asarray(window), dtype=torch.float32)
        return w.cuda() if torch.cuda.is_available() else w

    def _window_host(self):
        return np.ascontiguousarray(self.kernel_window.detach().cpu().numpy(), dtype=np.float32)

    # ------------------------------------------------------------ state machine
    def _load_from_state_dict(self, state_dict, prefix, *args, **kwargs):
        super()._load_from_state_dict(state_dict, prefix, *args, **kwargs)
        if prefix + 'epoch' in state_dict:
            self._epoch_host = int(state_dict[prefix + 'epoch'].reshape(-1)[0].item())

    def _smooth_table(self, src):
        dst = torch.empty_like(src)
        w = self._window_host()
        nb, d = src.shape
        _lib.call("dirb200_fds_smooth_tables", _lib.ptr(src), nb, d, w.ctypes.data_as(_lib.P), len(w),
                  _lib.ptr(dst), _lib.stream_ptr())
        return dst

    def _update_last_epoch_stats(self):
        _lib.require_cuda(self.running_mean)
        # rebinding (not copying) on purpose: reference aliasing, fds.py:55-56
        self.running_mean_last_epoch = self.running_mean
        self.running_var_last_epoch = self.running_var
        self.smoothed_mean_last_epoch = self._smooth_table(self.running_mean_last_epoch)
        self.smoothed_var_last_epoch = self._smooth_table(self.running_var_last_epoch)

    def reset(self):
        self.running_mean.zero_()
        self.running_var.fill_(1)
        self.running_mean_last_epoch.zero_()
        self.running_var_last_epoch.fill_(1)
        self.smoothed_mean_last_epoch.zero_()
        self.smoothed_var_last_epoch.fill_(1)
        self.num_samples_tracked.zero_()

    def update_last_epoch_stats(self, epoch):
        if epoch == self._epoch_host + 1:
            self._epoch_host += 1
            self.epoch += 1
            self._update_last_epoch_stats()
            print(f"Updated smoothed statistics on Epoch [{epoch}]!")

    # --------------------------------------------------- streamed epoch statistics
    @staticmethod
    def _dist():
        import torch.distributed as dist
        return dist if (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1) else None

    def begin_epoch_stats(self, all_labels):
        """Start a streamed collection.  `all_labels`: every label this rank will
        feed (the edge-folding rule of fds.py:94-97 looks at the whole epoch's
        label set; flags are OR-reduced across ranks)."""
        dev = self.running_mean.device
        _lib.require_cuda(self.running_mean)
        nb, d = self.running_mean.shape
        lab = all_labels.reshape(-1).to(device=dev, dtype=torch.float32).contiguous()
        flags = torch.zeros(2, dtype=torch.int32, device=dev)
        _lib.call("dirb200_fds_label_flags", _lib.ptr(lab), lab.numel(), self.bucket_num, self.bucket_start,
                  self.bin_rule, _lib.ptr(flags), _lib.stream_ptr())
        dist = self._dist()
        if dist is not None:
            dist.all_reduce(flags, op=dist.ReduceOp.MAX)
        self._acc = dict(flags=flags, sums=torch.zeros(nb, d, dtype=torch.float64, device=dev),
                         sumsq=torch.zeros(nb, d, dtype=torch.float64, device=dev),
                         counts=torch.zeros(nb, dtype=torch.int64, device=dev), ws=None)

    def accumulate_batch(self, features, labels):
        acc = self._acc
        assert acc is not None, "call begin_epoch_stats first"
        _lib.require_cuda(features)
        assert self.feature_dim == features.size(1), "Input feature dimension is not aligned!"
        assert features.size(0) == labels.numel(), "Dimensions of features and labels are not aligned!"
        features = features.detach().to(torch.float32).contiguous()
        n, d = features.shape
        nb = self.bucket_num - self.bucket_start
        lab = labels.reshape(-1).to(device=features.device, dtype=torch.float32).contiguous()
        bins = torch.empty(n, dtype=torch.int32, device=features.device)
        st = _lib.stream_ptr()
        _lib.call("dirb200_fds_bin_rows", _lib.ptr(lab), n, self.bucket_num, self.bucket_start, self.bin_rule,
                  _lib.ptr(acc["flags"]), _lib.ptr(bins), st)
        need = _lib.raw("dirb200_fds_accumulate_workspace_bytes")(n, nb)
        if acc["ws"] is None or acc["ws"].numel() < need:
            acc["ws"] = torch.empty(need, dtype=torch.uint8, device=features.device)
        _lib.call("dirb200_fds_accumulate", _lib.ptr(features), _lib.ptr(bins), n, d, nb, _lib.ptr(acc["sums"]),
                  _lib.ptr(acc["sumsq"]), _lib.ptr(acc["counts"]), _lib.ptr(acc["ws"]), acc["ws"].numel(), st)

    def abort_epoch_stats(self):
        """Drop a streamed collection without touching the tables (update_running_stats' gate failed, fds.py:85)."""
        self._acc = None

    @classmethod
    def reduce_accumulators(cls, acc):
        """Merge the per-rank (count, sum x, sum x^2) accumulators: plain SUM all-reduces (the fp64 sums make
        the merge exact to rounding, independent of how rows were sharded)."""
        dist = cls._dist()
        if dist is not None:
            for k in ("sums", "sumsq", "counts"):
                dist.all_reduce(acc[k], op=dist.ReduceOp.SUM)
        return acc

    def finish_epoch_stats(self, epoch):
        acc, self._acc = self._acc, None
        assert acc is not None
        self.reduce_accumulators(acc)
        nb, d = self.running_mean.shape
        _lib.call("dirb200_fds_finalize", _lib.ptr(acc["sums"]), _lib.ptr(acc["sumsq"]), _lib.ptr(acc["counts"]),
                  nb, d, _lib.ptr(self.running_mean), _lib.ptr(self.running_var),
                  _lib.ptr(self.num_samples_tracked), -1.0 if self.momentum is None else float(self.momentum),
                  int(epoch == self.start_update), _lib.stream_ptr())
        if self.fill_empty:
            _lib.call("dirb200_fds_fill_empty", _lib.ptr(acc["counts"]), nb, d, _lib.ptr(self.running_mean),
                      _lib.ptr(self.running_var), _lib.stream_ptr())
        print(f"Updated running statistics with Epoch [{epoch}] features!")

    # ------------------------------------------------------------ reference API
    def update_running_stats(self, features, labels, epoch):
        if epoch < self._epoch_host:
            return
        assert self.feature_dim == features.size(1), "Input feature dimension is not aligned!"
        assert features.size(0) == labels.size(0), "Dimensions of features and labels are not aligned!"
        self.begin_epoch_stats(labels)
        self.accumulate_batch(features, labels)
        self.finish_epoch_stats(epoch)

    def smooth(self, features, labels, epoch):
        if epoch < self.start_smooth:
            return features
        return _CalibrateFn.apply(features, labels, self.running_mean_last_epoch, self.running_var_last_epoch,
                                  self.smoothed_mean_last_epoch, self.smoothed_var_last_epoch,
                                  self.bucket_num, self.bucket_start, self.clip[0], self.clip[1], self.bin_rule)
