"""train.py -- host driver mirroring agedb-dir/train.py / imdb-wiki-dir/train.py
(same flags, same store-name rule, same train / validate / checkpoint flow)
on top of the H100-native modules of this directory.

Differences that matter:
  * one process per GPU (`torchrun --nproc-per-node N train.py ...`): the
    gradient all-reduce goes over NCCL (parallel.DataParallel), the optimizer
    is the fused flat-buffer Adam / SGD (optim.py);
  * the epoch-end FDS refresh (train.py:269-281 of the reference) streams each
    batch's features into the on-device per-bin accumulators -- no
    GPU->CPU->GPU round trip of the feature matrix, statistics all-reduced
    across ranks -- in the reference's order: collection pass with the old
    tables, then update_last_epoch_stats, then the running-statistics update;
  * LDS weights always come from the WHOLE training label column (every rank
    computes the same table); shards are equal-length index slices;
  * arguments are parsed inside main() (importing this file has no side
    effects) and `--synthetic N` trains on N synthetic samples (no dataset /
    network needed);
  * tensorboard_logger is optional.
"""
import argparse
import logging
import os
import time
from collections import defaultdict

import numpy as np
import torch
from torch.utils.data import DataLoader, Dataset

from resnet import resnet50
from loss import *  # noqa: F401,F403  (looked up by name, as the reference does at train.py:255)
from datasets import AgeDB, IMDBWIKI, gpu_transform_batch, jpeg_collate, lds_prepare_weights, take_device_decode_stats
from utils import AverageMeter, ProgressMeter, adjust_learning_rate, nvtx_range, prepare_folders, save_checkpoint
from optim import FusedAdam, FusedSGD
from parallel import DataParallel, ShardSampler, is_distributed

print = logging.info


# The defaults that agedb-dir/train.py and imdb-wiki-dir/train.py do not share (lines 29, 35 and 40 of each): the
# parser takes them from the script of the --dataset given, so `--dataset imdb_wiki` trains with IMDB-WIKI-DIR's LDS /
# FDS windows and FDS buckets from age 0.  Flags given explicitly still win.
DATASET_DEFAULTS = {'agedb': dict(lds_ks=9, fds_ks=9, bucket_start=3),
                    'imdb_wiki': dict(lds_ks=5, fds_ks=5, bucket_start=0)}


class _Parser(argparse.ArgumentParser):
    def parse_known_args(self, args=None, namespace=None):
        pre = argparse.ArgumentParser(add_help=False, allow_abbrev=False)
        pre.add_argument('--dataset', type=str, default='agedb')
        dataset = pre.parse_known_args(args)[0].dataset
        self.set_defaults(**DATASET_DEFAULTS.get(dataset, DATASET_DEFAULTS['agedb']))
        return super().parse_known_args(args, namespace)


def build_parser():
    p = _Parser(formatter_class=argparse.ArgumentDefaultsHelpFormatter)
    p.add_argument('--lds', action='store_true', default=False, help='whether to enable LDS')
    p.add_argument('--lds_kernel', type=str, default='gaussian', choices=['gaussian', 'triang', 'laplace'])
    p.add_argument('--lds_ks', type=int, default=9, help='LDS kernel size: should be odd number')
    p.add_argument('--lds_sigma', type=float, default=1, help='LDS gaussian/laplace kernel sigma')
    p.add_argument('--fds', action='store_true', default=False, help='whether to enable FDS')
    p.add_argument('--fds_kernel', type=str, default='gaussian', choices=['gaussian', 'triang', 'laplace'])
    p.add_argument('--fds_ks', type=int, default=9, help='FDS kernel size: should be odd number')
    p.add_argument('--fds_sigma', type=float, default=1, help='FDS gaussian/laplace kernel sigma')
    p.add_argument('--start_update', type=int, default=0, help='which epoch to start FDS updating')
    p.add_argument('--start_smooth', type=int, default=1, help='which epoch to start using FDS to smooth features')
    p.add_argument('--bucket_num', type=int, default=100, help='maximum bucket considered for FDS')
    p.add_argument('--bucket_start', type=int, default=3, choices=[0, 3], help='0 for IMDBWIKI, 3 for AgeDB')
    p.add_argument('--fds_mmt', type=float, default=0.9, help='FDS momentum')
    p.add_argument('--reweight', type=str, default='none', choices=['none', 'sqrt_inv', 'inverse'])
    p.add_argument('--retrain_fc', action='store_true', default=False, help='retrain last regression layer only')
    p.add_argument('--dataset', type=str, default='agedb', choices=['imdb_wiki', 'agedb'])
    p.add_argument('--data_dir', type=str, default='./data')
    p.add_argument('--model', type=str, default='resnet50')
    p.add_argument('--store_root', type=str, default='checkpoint')
    p.add_argument('--store_name', type=str, default='')
    p.add_argument('--gpu', type=int, default=None)
    p.add_argument('--optimizer', type=str, default='adam', choices=['adam', 'sgd'])
    p.add_argument('--loss', type=str, default='l1', choices=['mse', 'l1', 'focal_l1', 'focal_mse', 'huber'])
    p.add_argument('--lr', type=float, default=1e-3)
    p.add_argument('--epoch', type=int, default=90)
    p.add_argument('--momentum', type=float, default=0.9)
    p.add_argument('--weight_decay', type=float, default=1e-4)
    p.add_argument('--schedule', type=int, nargs='*', default=[60, 80])
    p.add_argument('--batch_size', type=int, default=256, help='batch size PER GPU (one process per GPU)')
    p.add_argument('--print_freq', type=int, default=10)
    p.add_argument('--img_size', type=int, default=224)
    p.add_argument('--workers', type=int, default=32)
    p.add_argument('--resume', type=str, default='')
    p.add_argument('--pretrained', type=str, default='')
    p.add_argument('--evaluate', action='store_true')
    p.add_argument('--synthetic', type=int, default=0, help='train on this many synthetic samples (no dataset needed)')
    p.add_argument('--device_transform', action='store_true', default=False,
                   help='(not a reference flag) the dataset yields the resized uint8 image; crop / flip / ToTensor / '
                        'Normalize (datasets.py:38-53) run on the GPU for the whole batch (datasets.gpu_transform_batch)')
    p.add_argument('--device_decode', action='store_true', default=False,
                   help='(not a reference flag; implies --device_transform) the JPEG decode and Resize((img_size, '
                        'img_size)) run on the GPU per batch too (datasets.JpegBatch); files outside the device '
                        "decoder's supported set are decoded by Pillow in the loader")
    return p


def store_name(args):
    """Experiment directory name, same rule as the reference (train.py:78-93)."""
    name = f'_{args.store_name}' if len(args.store_name) else ''
    if not args.lds and args.reweight != 'none':
        name += f'_{args.reweight}'
    if args.lds:
        name += f'_lds_{args.lds_kernel[:3]}_{args.lds_ks}'
        if args.lds_kernel in ['gaussian', 'laplace']:
            name += f'_{args.lds_sigma}'
    if args.fds:
        name += f'_fds_{args.fds_kernel[:3]}_{args.fds_ks}'
        if args.fds_kernel in ['gaussian', 'laplace']:
            name += f'_{args.fds_sigma}'
        name += f'_{args.start_update}_{args.start_smooth}_{args.fds_mmt}'
    if args.retrain_fc:
        name += '_retrain_fc'
    return f"{args.dataset}_{args.model}{name}_{args.optimizer}_{args.loss}_{args.lr}_{args.batch_size}"


class SyntheticAges(Dataset):
    """N(0,1) images with an age-like skewed label column; weights from the GPU LDS path."""

    def __init__(self, n, img_size, args, seed=0, train=True):
        self.device_transform = bool(getattr(args, 'device_transform', False))
        rng = np.random.RandomState(seed)
        self.labels = np.clip(np.round(rng.gamma(6.0, 6.5, size=n)), 0, 100).astype(np.float32)
        self.img_size, self.seed = img_size, seed
        w = lds_prepare_weights(self.labels, args.reweight, lds=args.lds, lds_kernel=args.lds_kernel,
                                lds_ks=args.lds_ks, lds_sigma=args.lds_sigma) if train else None
        self.weights = None if w is None else w.cpu().numpy()

    def __len__(self):
        return len(self.labels)

    def __getitem__(self, i):
        g = torch.Generator().manual_seed(self.seed * 1000003 + i)
        w = np.float32(1.) if self.weights is None else self.weights[i]
        if self.device_transform:            # a "resized RGB image": uint8 HWC, transformed on the GPU per batch
            img = torch.randint(0, 256, (self.img_size, self.img_size, 3), generator=g, dtype=torch.uint8)
        else:
            img = torch.randn(3, self.img_size, self.img_size, generator=g)
        return img, np.asarray([self.labels[i]], np.float32), np.asarray([w], np.float32)


def _label_column(loader):
    """Every label the loader will yield this epoch (its sampler's indices of the dataset's label column)."""
    ds = loader.dataset
    col = np.asarray(ds.labels if hasattr(ds, 'labels') else ds.df[ds.label_column].values, dtype=np.float32)
    sampler = getattr(loader, 'sampler', None)
    if isinstance(sampler, ShardSampler):
        return col[sampler.indices()]
    return col


def train(train_loader, model, optimizer, epoch, args, stats_loader=None):
    """One epoch (agedb-dir/train.py:234-283).  `stats_loader`: loader of the epoch-end FDS collection pass when it
    differs from `train_loader` (N > 1: the training sampler pads the shards to equal length so that every rank runs
    the same number of all-reduces; the collection pass must see every sample exactly once, so it uses the exact
    shards)."""
    if isinstance(getattr(train_loader, 'sampler', None), ShardSampler):
        train_loader.sampler.set_epoch(epoch)
    batch_time, data_time = AverageMeter('Time', ':6.2f'), AverageMeter('Data', ':6.4f')
    losses = AverageMeter(f'Loss ({args.loss.upper()})', ':.3f')
    progress = ProgressMeter(len(train_loader), [batch_time, data_time, losses], prefix="Epoch: [{}]".format(epoch))
    loss_fn = globals()[f"weighted_{args.loss}_loss"]
    model.train()
    end = time.time()
    for idx, (inputs, targets, weights) in enumerate(train_loader):
        data_time.update(time.time() - end)
        inputs, targets, weights = (t.cuda(non_blocking=True) for t in (inputs, targets, weights))
        if inputs.dtype == torch.uint8:           # --device_transform: RandomCrop(padding=16) / flip / ToTensor / Normalize
            inputs = gpu_transform_batch(inputs, train=True)
        with nvtx_range("dirb200/forward"):
            outputs = model(inputs, targets, epoch)
            if args.fds:
                outputs, _ = outputs
            loss = loss_fn(outputs, targets, weights)
        optimizer.zero_grad()
        with nvtx_range("dirb200/backward"):
            loss.backward()
        with nvtx_range("dirb200/grad_allreduce"):
            model.reduce_gradients()
        with nvtx_range("dirb200/optimizer"):
            optimizer.step()
        if idx % args.print_freq == 0:            # the only host sync of the loop (reference: every step)
            value = loss.item()
            assert not (np.isnan(value) or value > 1e6), f"Loss explosion: {value}"
            losses.update(value, inputs.size(0))
            batch_time.update(time.time() - end)
            progress.display(idx)
        end = time.time()

    if args.fds and epoch >= args.start_update:
        print(f"Create Epoch [{epoch}] features of all training data...")
        # Reference order (agedb-dir/train.py:269-281): FIRST the collection pass -- train-mode forward under no_grad,
        # so FDS.smooth still calibrates with the tables of the PREVIOUS refresh and the collected features are the
        # smoothed ones -- THEN update_last_epoch_stats (rebinding + stencil), THEN update_running_stats.  The
        # per-bin sums are streamed into device accumulators batch by batch (no GPU->CPU->GPU round trip) and only
        # finalised after the last-epoch tables have moved, exactly where the reference calls update_running_stats.
        fds = model.module.FDS
        loader = stats_loader if stats_loader is not None else train_loader
        fds.begin_epoch_stats(torch.as_tensor(_label_column(loader), dtype=torch.float32).cuda())
        with torch.no_grad(), nvtx_range("dirb200/fds_collection_pass"):
            for (inputs, targets, _) in loader:
                targets = targets.cuda(non_blocking=True)
                inputs = inputs.cuda(non_blocking=True)
                if inputs.dtype == torch.uint8:   # the collection pass iterates the TRAIN loader: its transform
                    inputs = gpu_transform_batch(inputs, train=True)
                _, feature = model(inputs, targets, epoch)
                fds.accumulate_batch(feature, targets)
        fds.update_last_epoch_stats(epoch)
        if epoch >= fds._epoch_host:            # gate of update_running_stats (fds.py:85), evaluated after the update
            fds.finish_epoch_stats(epoch)
        else:
            fds.abort_epoch_stats()
    return losses.avg


def shot_metrics(preds, labels, train_labels, many_shot_thr=100, low_shot_thr=20):
    """Many / median / low-shot MSE, L1 and G-Mean (agedb-dir/train.py:338-391), reduced on the GPU in one pass:
    an exact int64 histogram of int(train_label) + dirb200_shot_metrics over the predictions.  `preds` / `labels`
    may be torch tensors (any device) or numpy arrays; returns the reference's nested dict (+ 'overall')."""
    import _lib
    dev = torch.device('cuda', torch.cuda.current_device())
    as_dev = lambda a: torch.as_tensor(np.asarray(a) if not isinstance(a, torch.Tensor) else a,
                                       dtype=torch.float32).reshape(-1).to(dev).contiguous()
    if not isinstance(preds, (torch.Tensor, np.ndarray)):
        raise TypeError(f'Type ({type(preds)}) of predictions not supported')
    p, l, t = as_dev(preds), as_dev(labels), as_dev(train_labels)
    assert p.numel() == l.numel()
    # NaN training labels are skipped by the histogram (a NaN max would not convert to a bin count)
    top = lambda x: float(torch.nan_to_num(x, nan=0.0).max()) if x.numel() else 0.0
    nbins = int(max(top(t), top(l), 0.0)) + 2
    hist = torch.zeros(nbins, dtype=torch.int64, device=dev)
    _lib.call("dirb200_int_label_histogram", _lib.ptr(t), t.numel(), nbins, _lib.ptr(hist), _lib.stream_ptr())
    out = torch.empty(4, 4, dtype=torch.float64, device=dev)
    _lib.call("dirb200_shot_metrics", _lib.ptr(p), _lib.ptr(l), p.numel(), _lib.ptr(hist), nbins, int(many_shot_thr),
              int(low_shot_thr), _lib.ptr(out), _lib.stream_ptr())
    o = out.cpu().numpy()
    shot_dict = defaultdict(dict)
    with np.errstate(divide='ignore', invalid='ignore'):
        for row, name in enumerate(('overall', 'many', 'median', 'low')):
            cnt = o[row, 0]
            shot_dict[name]['mse'] = float(o[row, 1] / cnt)          # plain floats: they end up in checkpoints
            shot_dict[name]['l1'] = float(o[row, 2] / cnt)
            shot_dict[name]['gmean'] = float(np.exp(o[row, 3] / cnt))
    return shot_dict


def validate(val_loader, model, train_labels=None, prefix='Val'):
    """agedb-dir/train.py:286-335: eval-mode forward over the loader; predictions stay on the device and the
    overall + shot metrics come from ONE reduction kernel at the end (the reference copies every batch to the host
    and loops over np.unique(labels) there)."""
    model.eval()
    preds, labels = [], []
    with torch.no_grad():
        for (inputs, targets, _) in val_loader:
            inputs, targets = inputs.cuda(non_blocking=True), targets.cuda(non_blocking=True)
            if inputs.dtype == torch.uint8:       # --device_transform: the val / test chain (ToTensor + Normalize)
                inputs = gpu_transform_batch(inputs, train=False)
            preds.append(model(inputs).reshape(-1).float())
            labels.append(targets.reshape(-1).float())
    if not preds:
        return float('nan'), float('nan'), float('nan')
    preds, labels = torch.cat(preds), torch.cat(labels)
    shot = shot_metrics(preds, labels, train_labels if train_labels is not None else labels.new_zeros(0))
    ov = shot['overall']
    print(f" * Overall: MSE {ov['mse']:.3f}\tL1 {ov['l1']:.3f}\tG-Mean {ov['gmean']:.3f}")
    if train_labels is not None:
        for name in ('many', 'median', 'low'):
            d = shot[name]
            print(f" * {name.capitalize()}: MSE {d['mse']:.3f}\tL1 {d['l1']:.3f}\tG-Mean {d['gmean']:.3f}")
    return ov['mse'], ov['l1'], ov['gmean']


def main(argv=None):
    """Trains, then tests the best checkpoint; returns the test split's (MSE, L1, G-Mean).  With --evaluate: only
    the test pass of the --resume checkpoint, same return."""
    args, _ = build_parser().parse_known_args(argv)
    args.device_transform = args.device_transform or args.device_decode
    args.start_epoch, args.best_loss = 0, 1e5
    args.store_name = store_name(args)
    rank = int(os.environ.get("RANK", "0"))
    world = int(os.environ.get("WORLD_SIZE", "1"))
    torch.cuda.set_device(int(os.environ.get("LOCAL_RANK", args.gpu or 0)))
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.distributed.init_process_group("nccl")
    prepare_folders(args)
    handlers = [logging.StreamHandler()] if rank else \
        [logging.FileHandler(os.path.join(args.store_root, args.store_name, 'training.log')), logging.StreamHandler()]
    logging.root.handlers = []
    logging.basicConfig(level=logging.INFO if rank == 0 else logging.WARNING, format="%(asctime)s | %(message)s",
                        handlers=handlers)
    print(f"Args: {args}")
    print(f"Store name: {args.store_name}")

    print('=====> Preparing data...')
    # Every rank builds the dataset over the WHOLE training split, so the LDS histogram, clip, smoothing and the
    # len/sum(w) normaliser see the same label column the reference sees (datasets.py:55-83); the mini-batches are
    # sharded by the sampler (rank::world of one global permutation per epoch).
    if args.synthetic:
        train_dataset = SyntheticAges(args.synthetic, args.img_size, args, seed=0)
        val_dataset = SyntheticAges(max(args.synthetic // 8, args.batch_size), args.img_size, args, seed=999, train=False)
        test_dataset = val_dataset
    else:
        import pandas as pd
        df = pd.read_csv(os.path.join(args.data_dir, f"{args.dataset}.csv"))
        cls = AgeDB if args.dataset == 'agedb' else IMDBWIKI
        parts = {s: df[df['split'] == s] for s in ('train', 'val', 'test')}
        dt = dict(device_transform=args.device_transform, device_decode=args.device_decode)
        train_dataset = cls(data_dir=args.data_dir, df=parts['train'], img_size=args.img_size, split='train',
                            reweight=args.reweight, lds=args.lds, lds_kernel=args.lds_kernel, lds_ks=args.lds_ks,
                            lds_sigma=args.lds_sigma, **dt)
        val_dataset = cls(data_dir=args.data_dir, df=parts['val'], img_size=args.img_size, split='val', **dt)
        test_dataset = cls(data_dir=args.data_dir, df=parts['test'], img_size=args.img_size, split='test', **dt)
    mk = lambda ds, sampler: DataLoader(ds, batch_size=args.batch_size, sampler=sampler, shuffle=False,
                                        num_workers=args.workers, pin_memory=True, drop_last=False,
                                        collate_fn=jpeg_collate if args.device_decode else None)
    n_train = len(train_dataset)
    train_loader = mk(train_dataset, ShardSampler(n_train, rank, world, shuffle=True, pad=True))
    stats_loader = train_loader if world == 1 else mk(train_dataset, ShardSampler(n_train, rank, world, shuffle=False,
                                                                                  pad=False))
    val_loader, test_loader = mk(val_dataset, None), mk(test_dataset, None)
    print(f"Training data size: {len(train_dataset)}")
    # shot metrics compare against the WHOLE training label column (reference: df_train['age'], train.py:121)
    train_labels = np.asarray(train_dataset.labels if args.synthetic else parts['train']['age'].values)

    print('=====> Building model...')
    model = resnet50(fds=args.fds, bucket_num=args.bucket_num, bucket_start=args.bucket_start,
                     start_update=args.start_update, start_smooth=args.start_smooth,
                     kernel=args.fds_kernel, ks=args.fds_ks, sigma=args.fds_sigma, momentum=args.fds_mmt)
    model = DataParallel(model.cuda())
    model.broadcast_parameters()

    if args.evaluate:
        assert args.resume, 'Specify a trained model using [args.resume]'
        checkpoint = torch.load(args.resume)
        model.load_state_dict(checkpoint['state_dict'], strict=False)
        print(f"===> Checkpoint '{args.resume}' loaded (epoch [{checkpoint['epoch']}]), testing...")
        return validate(test_loader, model, train_labels=train_labels, prefix='Test')

    if args.retrain_fc:
        assert args.reweight != 'none' and args.pretrained
        for name, param in model.named_parameters():
            if 'fc' not in name and 'linear' not in name:
                param.requires_grad = False

    params = [p for p in model.parameters() if p.requires_grad]
    gs = 1.0 / world
    optimizer = FusedAdam(params, lr=args.lr, grad_scale=gs) if args.optimizer == 'adam' else \
        FusedSGD(params, lr=args.lr, momentum=args.momentum, weight_decay=args.weight_decay, grad_scale=gs)

    if args.pretrained:
        checkpoint = torch.load(args.pretrained, map_location="cpu")
        state = {k: v for k, v in checkpoint['state_dict'].items() if 'linear' not in k and 'fc' not in k}
        model.load_state_dict(state, strict=False)
        print(f'===> Pre-trained model loaded: {args.pretrained} ({len(state)} tensors)')
    if args.resume and os.path.isfile(args.resume):
        checkpoint = torch.load(args.resume, map_location='cuda')
        args.start_epoch, args.best_loss = checkpoint['epoch'], checkpoint['best_loss']
        model.load_state_dict(checkpoint['state_dict'])
        optimizer.load_state_dict(checkpoint['optimizer'])
        print(f"===> Loaded checkpoint '{args.resume}' (Epoch [{checkpoint['epoch']}])")

    for epoch in range(args.start_epoch, args.epoch):
        adjust_learning_rate(optimizer, epoch, args)
        train_loss = train(train_loader, model, optimizer, epoch, args, stats_loader=stats_loader)
        val_mse, val_l1, val_gmean = validate(val_loader, model, train_labels=train_labels)
        metric = val_mse if args.loss == 'mse' else val_l1
        is_best = metric < args.best_loss
        args.best_loss = min(metric, args.best_loss)
        print(f"Best {'L1' if 'l1' in args.loss else 'MSE'} Loss: {args.best_loss:.3f}")
        if rank == 0:
            save_checkpoint(args, {'epoch': epoch + 1, 'model': args.model, 'best_loss': args.best_loss,
                                   'state_dict': model.state_dict(), 'optimizer': optimizer.state_dict()}, is_best)
        print(f"Epoch #{epoch}: Train loss [{train_loss:.4f}]; Val loss: MSE [{val_mse:.4f}], L1 [{val_l1:.4f}], "
              f"G-Mean [{val_gmean:.4f}]")
        if args.device_decode:
            st = take_device_decode_stats()
            print(f"Epoch #{epoch}: images decoded on the device {st['device']}, flagged by it and decoded by Pillow "
                  f"{st['flagged']}, outside its supported set (decoded by Pillow in the loader) {st['host']}")

    # test with the best checkpoint (agedb-dir/train.py:224-231); only rank 0 writes it
    print("=" * 120)
    print("Test best model on testset...")
    if is_distributed():
        torch.distributed.barrier()
    checkpoint = torch.load(os.path.join(args.store_root, args.store_name, 'ckpt.best.pth.tar'), map_location='cuda')
    model.load_state_dict(checkpoint['state_dict'])
    print(f"Loaded best model, epoch {checkpoint['epoch']}, best val loss {checkpoint['best_loss']:.4f}")
    test_mse, test_l1, test_gmean = validate(test_loader, model, train_labels=train_labels, prefix='Test')
    print(f"Test loss: MSE [{test_mse:.4f}], L1 [{test_l1:.4f}], G-Mean [{test_gmean:.4f}]\nDone")
    if is_distributed():
        torch.distributed.destroy_process_group()
    return test_mse, test_l1, test_gmean


if __name__ == '__main__':
    main()
