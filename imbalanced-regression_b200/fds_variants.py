"""FDS variants of the other two sub-projects on the same kernels (SURVEY.md §8 rows f-2 / f-3):

* `FDSDepth`  -- nyud2-dir/models/fds.py: features are a dense map [B, C, H, W], labels a depth map
  [B, 1, H, W]; bucket = clamp(int(depth * 10), bucket_start, bucket_num - 1); calibration clip (0.2, 5)
  (nyud2-dir/util.py:151).  The reference bins pixel by pixel in a Python loop on the CPU
  (models/fds.py:110) -- here rows = pixels go through the same label-binning + segmented reduction kernels.
* `FDSSTSB`   -- sts-b-dir/fds.py: bucket from np.histogram edges over [0, 5] (50 buckets), empty buckets
  filled from their neighbours after every update, clip (0.5, 2) (sts-b-dir/util.py:63).
"""
import torch

import _lib
from fds import FDS


class FDSDepth(FDS):
    clip = (0.2, 5.0)
    bin_rule = _lib.BIN_DEPTH10

    def __init__(self, feature_dim, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1,
                 kernel='gaussian', ks=5, sigma=2, momentum=0.9):
        super().__init__(feature_dim, bucket_num, bucket_start, start_update, start_smooth, kernel, ks, sigma, momentum)

    def _update_last_epoch_stats(self):
        # the reference moves running_* to the CPU and back around every update (models/fds.py:88-96,105,126), which
        # on a GPU creates new tensors: running_*_last_epoch keeps the values it was bound to (no alias, unlike
        # the age / STS-B modules)
        super()._update_last_epoch_stats()
        self.running_mean_last_epoch = self.running_mean.clone()
        self.running_var_last_epoch = self.running_var.clone()

    @staticmethod
    def _rows(features, labels):
        b, c, h, w = features.shape
        return features.permute(0, 2, 3, 1).contiguous().view(-1, c), labels.reshape(-1)

    def accumulate_map(self, features, labels):
        """One batch of a streamed collection (begin_epoch_stats / finish_epoch_stats): features [N, C, h, w], labels
        the depth [N, 1, h, w], one row per pixel.  The depth rule ignores the edge flags, so begin_epoch_stats may be
        given no labels."""
        rows, lab = self._rows(features, labels)
        self.accumulate_batch(rows, lab)

    def update_running_stats(self, features, labels, epoch):
        if epoch < self._epoch_host:
            return
        assert self.feature_dim == features.size(1), "Input feature dimension is not aligned!"
        assert features.size(0) == labels.size(0), "Dimensions of features and labels are not aligned!"
        rows, lab = self._rows(features, labels)
        self.begin_epoch_stats(lab)
        self.accumulate_batch(rows, lab)
        self.finish_epoch_stats(epoch)

    def smooth(self, features, labels, epoch):
        if epoch < self.start_smooth:
            return features
        b, c, h, w = features.shape
        rows, lab = self._rows(features, labels)
        out = super().smooth(rows, lab, epoch)
        return out.view(b, h, w, c).permute(0, 3, 1, 2)


class FDSSTSB(FDS):
    clip = (0.5, 2.0)
    bin_rule = _lib.BIN_EDGES5
    fill_empty = True

    def __init__(self, feature_dim, bucket_num=50, bucket_start=0, start_update=0, start_smooth=1,
                 kernel='gaussian', ks=5, sigma=2, momentum=0.9):
        super().__init__(feature_dim, bucket_num, bucket_start, start_update, start_smooth, kernel, ks, sigma, momentum)
