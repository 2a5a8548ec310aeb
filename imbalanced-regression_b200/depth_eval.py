"""NYUD2-DIR test-time evaluation on the device (nyud2-dir/test.py:39-60, nyud2-dir/util.py:35-133).

The reference up-samples each test prediction with F.interpolate(align_corners=True), selects the balanced test
mask, copies the selected pixels to the host (one sync per image), bins every pixel with a Python map and computes
RMSE / ABS_REL / LG10 / MAE / delta1-3 on CPU tensors, overall and per many / medium / few-shot group.  Here one
kernel (dirb200_depth_metrics_accumulate) does the up-sampling, the mask, the binning and the error sums per batch
and adds them into a [4][10] fp64 device accumulator; evaluate_shot() copies that accumulator to the host once.
"""
import logging

import numpy as np
import torch

import _lib

SHOTS = ('overall', 'many', 'medium', 'few')
METRICS = ('MSE', 'RMSE', 'ABS_REL', 'LG10', 'MAE', 'DELTA1', 'DELTA2', 'DELTA3', 'NUM')
NBINS = 100                         # Evaluator.get_bin_idx clamps to 99
_INT_MAX = 2 ** 31 - 1


def group_table(shot_idx):
    """u8[100]: the shot group (1 many, 2 medium, 3 few, 0 none) of each depth bin of `shot_idx`."""
    table = np.zeros(NBINS, dtype=np.uint8)
    for g, shot in enumerate(SHOTS[1:], start=1):
        for b in shot_idx.get(shot, ()):
            b = int(b)
            if not 0 <= b < NBINS:
                raise ValueError(f"shot_idx['{shot}'] holds bin {b}, outside [0, {NBINS})")
            if table[b]:
                raise ValueError(f"bin {b} is in two shot groups")
            table[b] = g
    return table


def metrics_from_acc(acc):
    """The reference's metric_dict (util.py:89-133 per row) from a host [4][10] accumulator."""
    acc = np.asarray(acc, dtype=np.float64).reshape(4, 10)
    out = {}
    for row, shot in enumerate(SHOTS):
        errors = {'MSE': 0, 'RMSE': 0, 'ABS_REL': 0, 'LG10': 0, 'MAE': 0, 'DELTA1': 0, 'DELTA2': 0, 'DELTA3': 0,
                  'NUM': 0}
        n = acc[row, 0]
        if n > 0:
            with np.errstate(divide='ignore', invalid='ignore'):
                errors['MSE'] = float(acc[row, 1] / n)
                errors['MAE'] = float(acc[row, 2] / n)
                errors['ABS_REL'] = float(acc[row, 3] / n)
                errors['LG10'] = float(acc[row, 4] / n)
            # the reference divides fp32 sums of 0/1 by the fp32 count
            for k, name in enumerate(('DELTA1', 'DELTA2', 'DELTA3')):
                errors[name] = float(np.float32(acc[row, 5 + k]) / np.float32(n))
            errors['NUM'] = int(n)
        with np.errstate(invalid='ignore'):
            errors['RMSE'] = np.sqrt(errors['MSE'])
        out[shot] = errors
    return out


class Evaluator:
    """util.py:35-133 with the pixels accumulated on the device.  `shot_idx` maps 'many' / 'medium' / 'few' to the
    depth bins (0.1 m buckets, 0..99) of each group, as the reference's Evaluator hard-codes them."""

    def __init__(self, shot_idx):
        self.shot_idx = {k: [int(b) for b in v] for k, v in shot_idx.items()}
        self._table_host = group_table(self.shot_idx)
        self._table = None
        self._acc = None
        self._ws = None

    def _state(self, device):
        if self._acc is None or self._acc.device != device:
            self._acc = torch.zeros(4, 10, dtype=torch.float64, device=device)
            self._table = torch.from_numpy(self._table_host).to(device)
            self._ws = None
        return self._acc

    def _launch(self, pred, ph, pw, target, mask, n, h, w, table, nbins, acc):
        need = _lib.raw("dirb200_depth_metrics_workspace_bytes")(n, h, w)
        ws = self._ws
        if ws is None or ws.numel() < need or ws.device != target.device:
            ws = self._ws = torch.empty(max(need, 1), dtype=torch.uint8, device=target.device)
        _lib.call("dirb200_depth_metrics_accumulate", _lib.ptr(pred), ph, pw, _lib.ptr(target), _lib.ptr(mask), n, h,
                  w, _lib.ptr(table), nbins, _lib.ptr(acc), _lib.ptr(ws), ws.numel(), _lib.stream_ptr())

    def _flat(self, output, depth, table, nbins, acc):
        o = output.detach().reshape(-1).to(torch.float32).contiguous()
        t = depth.detach().reshape(-1).to(torch.float32).contiguous()
        if o.numel() != t.numel():
            raise ValueError(f"output has {o.numel()} values, depth {t.numel()}")
        for lo in range(0, t.numel(), _INT_MAX):
            k = min(_INT_MAX, t.numel() - lo)
            self._launch(o[lo:lo + k], 1, k, t[lo:lo + k], None, 1, 1, k, table, nbins, acc)

    def __call__(self, output, depth):
        """util.py:47-51: add the (already masked) predictions and targets to the running sums, on the device."""
        _lib.require_cuda(output, depth)
        acc = self._state(depth.device)
        self._flat(output, depth, self._table, NBINS, acc)

    def add(self, output, depth, mask):
        """The fused form of test.py:52-54: equivalent to
        self(F.interpolate(output, size=(H, W), mode='bilinear', align_corners=True)[mask], depth[mask]) for
        output [B,1,ph,pw], depth [B,1,H,W] and a bool mask [B,1,H,W] (None: every pixel), in one kernel launch."""
        _lib.require_cuda(output, depth, mask)
        if output.dim() != 4 or depth.dim() != 4 or output.shape[1] != 1 or depth.shape[1] != 1 \
                or output.shape[0] != depth.shape[0]:
            raise ValueError(f"add expects output [B,1,ph,pw] and depth [B,1,H,W], got {tuple(output.shape)} and "
                             f"{tuple(depth.shape)}")
        if mask is not None and (mask.dtype != torch.bool or tuple(mask.shape) != tuple(depth.shape)):
            raise ValueError(f"mask must be a bool tensor shaped like depth {tuple(depth.shape)}")
        b, _, ph, pw = output.shape
        _, _, h, w = depth.shape
        acc = self._state(depth.device)
        o = output.detach().to(torch.float32).contiguous()
        t = depth.detach().to(torch.float32).contiguous()
        m = None if mask is None else mask.contiguous()
        self._launch(o, ph, pw, t, m, b, h, w, self._table, NBINS, acc)

    def counts_and_sums(self):
        """The raw [4][10] accumulator (device tensor): rows overall / many / medium / few; columns NUM, sum d^2,
        sum d, sum d/t, sum lg10 error, delta1-3 counts, NaN targets, inf targets."""
        if self._acc is None:
            return torch.zeros(4, 10, dtype=torch.float64)
        return self._acc

    def evaluate_shot(self):
        """util.py:53-78: the metric dict of every group from one device-to-host copy, logged as the reference does.
        The reference's get_bin_idx calls int() on every target; like it, this raises ValueError when a NaN target
        was seen and OverflowError for an infinite one (the NaN check comes first when both occur)."""
        acc = self.counts_and_sums().cpu().numpy()
        if acc[0, 8] > 0:
            raise ValueError(f"cannot convert float NaN to integer ({int(acc[0, 8])} NaN depth values)")
        if acc[0, 9] > 0:
            raise OverflowError(f"cannot convert float infinity to integer ({int(acc[0, 9])} infinite depth values)")
        metric_dict = metrics_from_acc(acc)
        logging.info('\n***** TEST RESULTS *****')
        for shot in ['Overall', 'Many', 'Medium', 'Few']:
            logging.info(f" * {shot}: RMSE {metric_dict[shot.lower()]['RMSE']:.3f}\t"
                         f"ABS_REL {metric_dict[shot.lower()]['ABS_REL']:.3f}\t"
                         f"LG10 {metric_dict[shot.lower()]['LG10']:.3f}\t"
                         f"MAE {metric_dict[shot.lower()]['MAE']:.3f}\t"
                         f"DELTA1 {metric_dict[shot.lower()]['DELTA1']:.3f}\t"
                         f"DELTA2 {metric_dict[shot.lower()]['DELTA2']:.3f}\t"
                         f"DELTA3 {metric_dict[shot.lower()]['DELTA3']:.3f}\t"
                         f"NUM {metric_dict[shot.lower()]['NUM']}")
        return metric_dict

    def reset(self):
        if self._acc is not None:
            self._acc.zero_()

    @staticmethod
    def get_bin_idx(x):
        return min(int(x * np.float32(10)), 99)

    @staticmethod
    def evaluate(output, target):
        """util.py:88-133: the overall metrics of two flat tensors; NaN targets are left out as setNanToZero does."""
        _lib.require_cuda(output, target)
        acc = torch.zeros(4, 10, dtype=torch.float64, device=target.device)
        Evaluator({})._flat(output, target, None, 0, acc)
        return metrics_from_acc(acc.cpu().numpy())['overall']


def test(test_loader, model, shot_idx):
    """test.py:39-60: eval-mode forward over the loader ({'image', 'depth', 'mask'} batches), fused up-sampling +
    mask + metrics per batch on the device, one host copy at the end.  Returns (overall RMSE, metric_dict)."""
    model.eval()
    logging.info('Starting testing...')
    evaluator = Evaluator(shot_idx)
    with torch.no_grad():
        for sample_batched in test_loader:
            image, depth, mask = sample_batched['image'], sample_batched['depth'], sample_batched['mask']
            depth = depth.cuda(non_blocking=True)
            mask = mask.cuda(non_blocking=True)
            image = image.cuda()
            output = model(image)
            evaluator.add(output, depth, mask)
    logging.info('Finished testing. Start printing statistics below...')
    metric_dict = evaluator.evaluate_shot()
    return metric_dict['overall']['RMSE'], metric_dict
