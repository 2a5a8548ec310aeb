"""STS-B-DIR evaluation on the device: `STSShotAverage`, the scorer of sts-b-dir/util.py:101-172 that tasks.py:86 builds
with metric=['mse', 'l1', 'gmean', 'pearsonr', 'spearmanr'].

The interface is the reference's: `__call__(pred, label)` buffers one batch of host arrays (models.forward hands it the
batch's fp32 logits and labels), `get_metric(reset, type)` returns {'overall' | 'many' | 'medium' | 'few':
{metric: value, ..., 'num_samples': n}} (only the 'overall' dict when type == 'overall'), and `reset()` empties it.
The reference appends every value to Python lists and, per get_metric, bins each label with its own np.histogram
call and runs scipy on the host.  Here the batches go into one growing fp32 host array; get_metric copies it to the
device once and runs dirb200_stsb_shot_metrics, which computes every metric of every group in fp64
(include/dirb200.h).  The values are fp32 as the model produces them; other dtypes are converted to fp32.  The
kernel ranks by an O(N^2) pair count and takes up to 2^22 values per call (the reference's default validation
interval gathers 400 x 128 = 51 200).

Differences from the reference: a label above 5 goes to the last bin (the reference raises IndexError); NaN labels
count as few.  Otherwise the definitions are the reference's: x = 5 pred in fp64, the np.histogram bins over [0, 5],
the many / medium / few table, 1e-10 for an exact zero difference in the G-mean, scipy's Pearson and Spearman (NaN
for a constant group), 0 for an empty group and 0 correlations for a group of one.
"""
import numpy as np
import torch

import _lib

SHOTS = ('overall', 'many', 'medium', 'few')          # the rows of dirb200_stsb_shot_metrics's output
METRICS = ('num_samples', 'mse', 'l1', 'gmean', 'pearsonr', 'spearmanr')   # its columns


def shot_metrics(preds, labels):
    """dirb200_stsb_shot_metrics over CUDA fp32 vectors: a float64 [4, 6] CPU array, rows SHOTS, columns METRICS."""
    _lib.require_cuda(preds, labels)
    if preds.dtype is not torch.float32 or labels.dtype is not torch.float32 or not preds.is_contiguous() \
            or not labels.is_contiguous() or preds.numel() != labels.numel() or preds.device != labels.device:
        raise _lib.Dirb200Error("stsb shot metrics: preds and labels must be contiguous fp32 CUDA tensors of one size "
                                "on one device")
    n = preds.numel()
    out = torch.empty(len(SHOTS) * len(METRICS), dtype=torch.float64, device=preds.device)
    ws = torch.empty(max(1, _lib.raw("dirb200_stsb_shot_metrics_workspace_bytes")(n)), dtype=torch.uint8,
                     device=preds.device)
    with torch.cuda.device(preds.device):
        _lib.call("dirb200_stsb_shot_metrics", _lib.ptr(preds), _lib.ptr(labels), n, _lib.ptr(ws), ws.numel(),
                  _lib.ptr(out), _lib.stream_ptr())
    return out.view(len(SHOTS), len(METRICS)).cpu().numpy()


class STSShotAverage:
    def __init__(self, metric):
        self._metric = metric
        self._buf = np.empty((2, 1024), dtype=np.float32)       # [pred; label], grown by doubling
        self._count = 0

    def __call__(self, pred, label):
        pred = np.asarray(pred, dtype=np.float32).reshape(-1)
        label = np.asarray(label, dtype=np.float32).reshape(-1)
        if pred.size != label.size:
            raise ValueError(f"STSShotAverage: {pred.size} predictions for {label.size} labels")
        end = self._count + pred.size
        if end > self._buf.shape[1]:
            grown = np.empty((2, max(end, 2 * self._buf.shape[1])), dtype=np.float32)
            grown[:, :self._count] = self._buf[:, :self._count]
            self._buf = grown
        self._buf[0, self._count:end] = pred
        self._buf[1, self._count:end] = label
        self._count = end

    def get_metric(self, reset=False, type=None):
        dev = torch.device("cuda", torch.cuda.current_device())
        both = torch.from_numpy(np.ascontiguousarray(self._buf[:, :self._count])).to(dev)
        table = shot_metrics(both[0], both[1])
        metric = {}
        for row, shot in zip(table, SHOTS):
            metric[shot] = {k: float(v) for k, v in zip(METRICS[1:], row[1:]) if k in self._metric}
            metric[shot]['num_samples'] = int(row[0])
        if reset:
            self.reset()
        return metric['overall'] if type == 'overall' else metric

    def reset(self):
        self._count = 0
