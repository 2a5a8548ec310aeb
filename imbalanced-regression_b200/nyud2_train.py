"""nyud2_train.py -- NYUD2-DIR's training driver (nyud2-dir/train.py) on the native path: the same flags and defaults,
the same store-name rule, the same epoch loop, log lines and checkpoints, on net.model, loaddata's device loaders,
loss.weighted_mse_loss, optim.Adam and depth_eval.

    python nyud2_train.py --data_dir DATA [--fds] [--lds --reweight inverse] ...

Differences from the reference:
  * one process on one GPU (--gpu).  The default batch of 32 is one BatchNorm batch of 32, where the reference's
    4-GPU DataParallel normalises over 8 samples per replica;
  * the optimizer is optim.Adam, one multi-tensor launch per step over net.model's 245 parameters;
  * the epoch-end FDS refresh streams each batch's unsmoothed R features and depths into R.FDS's device accumulators
    instead of concatenating them on the host (train.py:216-228), in the reference's order: the collection pass in train
    mode with the old tables, update_last_epoch_stats(epoch), then the running-statistics update gated on the epoch
    counter after that update;
  * `resnet50(pretrained=True)` downloads ImageNet weights; here --backbone_weights PATH loads a torchvision-layout
    ResNet-50 state_dict into E (fc.* dropped), and without it E starts from a random initialisation;
  * tensorboardX is optional; checkpoint metrics are stored as plain Python numbers.
Checkpoints keep DataParallel's `module.` prefix, so the reference's test.py loads them.
"""
import argparse
import logging
import os
import shutil
import sys
import time

import torch

import depth_eval
import loaddata
import net
from loss import weighted_mse_loss
from optim import Adam
from resnet import E_resnet, resnet50
from utils import AverageMeter


def build_parser():
    parser = argparse.ArgumentParser(description='')
    # training/optimization related
    parser.add_argument('--epochs', default=10, type=int, help='number of total epochs to run')
    parser.add_argument('--start_epoch', default=0, type=int, help='manual epoch number (useful on restarts)')
    parser.add_argument('--lr', '--learning-rate', default=0.0001, type=float, help='initial learning rate')
    parser.add_argument('--weight_decay', '--wd', default=1e-4, type=float, help='weight decay (default: 1e-4)')
    parser.add_argument('--batch_size', default=32, type=int, help='batch size number')
    parser.add_argument('--store_root', type=str, default='checkpoint')
    parser.add_argument('--store_name', type=str, default='nyud2')
    parser.add_argument('--data_dir', type=str, default='./data', help='data directory')
    parser.add_argument('--resume', action='store_true', default=False, help='whether to resume training')
    # LDS
    parser.add_argument('--lds', action='store_true', default=False, help='whether to enable LDS')
    parser.add_argument('--lds_kernel', type=str, default='gaussian', choices=['gaussian', 'triang', 'laplace'],
                        help='LDS kernel type')
    parser.add_argument('--lds_ks', type=int, default=5, help='LDS kernel size: should be odd number')
    parser.add_argument('--lds_sigma', type=float, default=2, help='LDS gaussian/laplace kernel sigma')
    # FDS
    parser.add_argument('--fds', action='store_true', default=False, help='whether to enable FDS')
    parser.add_argument('--fds_kernel', type=str, default='gaussian', choices=['gaussian', 'triang', 'laplace'],
                        help='FDS kernel type')
    parser.add_argument('--fds_ks', type=int, default=5, help='FDS kernel size: should be odd number')
    parser.add_argument('--fds_sigma', type=float, default=2, help='FDS gaussian/laplace kernel sigma')
    parser.add_argument('--start_update', type=int, default=0, help='which epoch to start FDS updating')
    parser.add_argument('--start_smooth', type=int, default=1, help='which epoch to start using FDS to smooth features')
    parser.add_argument('--bucket_num', type=int, default=100, help='maximum bucket considered for FDS')
    parser.add_argument('--bucket_start', type=int, default=7, help='minimum(starting) bucket for FDS, 7 for NYUDv2')
    parser.add_argument('--fds_mmt', type=float, default=0.9, help='FDS momentum')
    # re-weighting: SQRT_INV / INV
    parser.add_argument('--reweight', type=str, default='none', choices=['none', 'inverse', 'sqrt_inv'],
                        help='cost-sensitive reweighting scheme')
    # two-stage training: RRT
    parser.add_argument('--retrain_fc', action='store_true', default=False,
                        help='whether to retrain last regression layer (regressor)')
    parser.add_argument('--pretrained', type=str, default='',
                        help='pretrained checkpoint file path to load backbone weights for RRT')
    # not in the reference
    parser.add_argument('--workers', type=int, default=8,
                        help='[not in the reference] host decode workers of the training and FDS loaders')
    parser.add_argument('--print_freq', type=int, default=1,
                        help='[not in the reference] log every N-th training batch (1: every batch, as the reference)')
    parser.add_argument('--gpu', type=int, default=0, help='[not in the reference] the CUDA device to train on')
    parser.add_argument('--backbone_weights', type=str, default='',
                        help='[not in the reference] torchvision-layout ResNet-50 state_dict loaded into E (fc.* '
                             'dropped), in place of resnet50(pretrained=True)\'s download; without it E starts random')
    return parser


def store_name(args):
    """train.py:74-87.  The defaults of --lds_sigma / --fds_sigma / --fds_mmt are the literals 2, 2 and 0.9, so the
    defaults give `_2` where a typed `--lds_sigma 2` gives `_2.0`."""
    name = args.store_name
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
    name += f'_lr_{args.lr}_bs_{args.batch_size}'
    return name


def lr_at(args, epoch):
    """train.py:230-234"""
    return args.lr * (0.1 ** (epoch // 5))


def query_yes_no(question):
    """util.py:136-149: ask on stdin, empty answer is yes."""
    valid = {"yes": True, "y": True, "ye": True, "no": False, "n": False}
    while True:
        print(question + " [Y/n] ", end=':')
        choice = input().lower()
        if choice == '':
            return True
        if choice in valid:
            return valid[choice]
        print("Please respond with 'yes' or 'no' (or 'y' or 'n').\n")


def load_backbone(model, path):
    """A torchvision-layout ResNet-50 state_dict (optionally under 'state_dict') into E, fc.* dropped, strictly."""
    sd = torch.load(path, map_location='cpu')
    if 'state_dict' in sd:
        sd = sd['state_dict']
    model.E.load_state_dict({k: v for k, v in sd.items() if not k.startswith('fc.')})


def define_model(args):
    """train.py:59-64 on the native modules; E from --backbone_weights, or random with a warning."""
    model = net.model(args, E_resnet(resnet50()), num_features=2048, block_channel=[256, 512, 1024, 2048])
    if args.backbone_weights:
        load_backbone(model, args.backbone_weights)
        logging.info(f'===> Backbone weights loaded: {args.backbone_weights}')
    else:
        logging.warning('No --backbone_weights: the encoder starts from a random initialisation (the reference starts '
                        'from ImageNet weights)')
    return model


def with_module(state_dict):
    """state_dict keys as DataParallel writes them."""
    return {'module.' + k: v for k, v in state_dict.items()}


def plain(metric_dict):
    """The metric dict with plain Python numbers (a checkpoint that torch.load reads with weights_only=True)."""
    return {shot: {k: (int(v) if k == 'NUM' else float(v)) for k, v in m.items()} for shot, m in metric_dict.items()}


def save_checkpoint(args, state_dict, epoch, error, metric_dict, filename='checkpoint.pth.tar'):
    """train.py:256-263"""
    path = os.path.join(args.store_dir, filename)
    logging.info(f'Saving checkpoint to {path}...')
    torch.save({'state_dict': with_module(state_dict), 'epoch': epoch, 'error': float(error),
                'metric': plain(metric_dict)}, path)


def train(train_loader, train_fds_loader, model, optimizer, epoch, args, writer=None):
    """train.py:180-228: one epoch, then (with --fds, from --start_update on) the FDS collection pass."""
    batch_time = AverageMeter('Time')
    losses = AverageMeter('Loss')
    model.train()
    end = time.time()
    for i, sample_batched in enumerate(train_loader):
        image, depth, weight = sample_batched['image'], sample_batched['depth'], sample_batched['weight']
        optimizer.zero_grad()
        if args.fds:
            output, feature = model(image, depth, epoch)
        else:
            output = model(image, depth, epoch)
        loss = weighted_mse_loss(output, depth, weight)          # torch.mean(((output - depth) ** 2) * weight)
        losses.update(loss.item(), image.size(0))
        loss.backward()
        optimizer.step()
        batch_time.update(time.time() - end)
        end = time.time()
        if writer is not None:
            writer.add_scalar('data/loss', loss.item(), i + epoch * len(train_loader))
        if i % args.print_freq == 0:
            logging.info('Epoch: [{0}][{1}/{2}]\t'
                         'Time {batch_time.val:.3f} ({batch_time.sum:.3f})\t'
                         'Loss {loss.val:.4f} ({loss.avg:.4f})\t'
                         .format(epoch, i, len(train_loader), batch_time=batch_time, loss=losses))

    if args.fds and epoch >= args.start_update:
        fds = model.R.FDS
        logging.info(f"Starting Creating Epoch [{epoch}] features of subsampled training data...")
        fds.begin_epoch_stats(torch.empty(0, device=fds.running_mean.device))
        n = 0
        with torch.no_grad():
            for sample_batched in train_fds_loader:
                image, depth = sample_batched['image'], sample_batched['depth']
                _, feature = model(image, depth, epoch)
                fds.accumulate_map(feature, depth)
                n += image.size(0)
        logging.info(f"Created Epoch [{epoch}] features of subsampled training data (size: {n})!")
        fds.update_last_epoch_stats(epoch)
        if epoch < int(fds.epoch.item()):                     # update_running_stats' gate (models/fds.py:99)
            fds.abort_epoch_stats()
        else:
            fds.finish_epoch_stats(epoch)


def main(argv=None):
    """train.py:66-178.  Returns the trained model."""
    args = build_parser().parse_args(argv)
    args.store_name = store_name(args)
    args.store_dir = os.path.join(args.store_root, args.store_name)

    if not args.resume:
        if os.path.exists(args.store_dir):
            if sys.stdin is not None and sys.stdin.isatty() and \
                    query_yes_no('overwrite previous folder: {} ?'.format(args.store_dir)):
                shutil.rmtree(args.store_dir)
                print(args.store_dir + ' removed.')
            else:
                raise RuntimeError('Output folder {} already exists'.format(args.store_dir))
        print(f"===> Creating folder: {args.store_dir}")
        os.makedirs(args.store_dir)

    logging.root.handlers = []
    logging.basicConfig(level=logging.INFO, format="%(asctime)s | %(message)s",
                        handlers=[logging.FileHandler(os.path.join(args.store_dir, 'training_log.log')),
                                  logging.StreamHandler()])
    logging.info(args)

    try:
        from tensorboardX import SummaryWriter
        writer = SummaryWriter(args.store_dir)
    except ImportError:
        writer = None

    torch.cuda.set_device(args.gpu)
    model = define_model(args).cuda()

    error_best, metric_dict_best, epoch_best = 1e5, {}, -1
    if args.resume:
        path = os.path.join(args.store_dir, 'checkpoint.pth.tar')
        model_state = torch.load(path, map_location='cpu')
        logging.info(f"Loading checkpoint from {path} (Epoch [{model_state['epoch']}], RMSE: {model_state['error']:.3f})")
        model.load_state_dict(depth_eval.strip_module(model_state['state_dict']))
        args.start_epoch = model_state['epoch'] + 1
        epoch_best = model_state['epoch']
        error_best = model_state['error']
        metric_dict_best = model_state['metric']

    if args.retrain_fc:
        assert os.path.isfile(args.pretrained), f"No checkpoint found at '{args.pretrained}'"
        model_state = torch.load(args.pretrained, map_location='cpu')
        new_state_dict = {k: v for k, v in model_state['state_dict'].items() if 'R' not in k}
        model.load_state_dict(depth_eval.strip_module(new_state_dict), strict=False)
        logging.info(f'===> Pretrained weights found in total: [{len(new_state_dict)}]')
        logging.info(f'===> Pre-trained model loaded: {args.pretrained}')
        for name, param in model.named_parameters():
            if 'R' not in name:
                param.requires_grad = False
        logging.info(f'Only optimize parameters: {[n for n, p in model.named_parameters() if p.requires_grad]}')

    params = [p for p in model.parameters() if p.requires_grad] if args.retrain_fc else model.parameters()
    optimizer = Adam(params, args.lr, weight_decay=args.weight_decay)

    train_loader = loaddata.getTrainingData(args, args.batch_size, num_workers=args.workers)
    train_fds_loader = loaddata.getTrainingFDSData(args, args.batch_size, num_workers=args.workers)
    test_loader = loaddata.getTestingData(args, 1)

    if args.start_epoch >= args.epochs:
        logging.info(f'Nothing to train: start epoch {args.start_epoch}, {args.epochs} epochs')
        return model
    for epoch in range(args.start_epoch, args.epochs):
        for group in optimizer.param_groups:
            group['lr'] = lr_at(args, epoch)
        train(train_loader, train_fds_loader, model, optimizer, epoch, args, writer)
        error, metric_dict = depth_eval.test(test_loader, model, depth_eval.SHOT_IDX)
        if error < error_best:
            error_best, metric_dict_best, epoch_best = error, metric_dict, epoch
            save_checkpoint(args, model.state_dict(), epoch, error, metric_dict, 'checkpoint_best.pth.tar')
        save_checkpoint(args, model.state_dict(), epoch, error, metric_dict, 'checkpoint.pth.tar')

    save_checkpoint(args, model.state_dict(), epoch, error, metric_dict, 'checkpoint_final.pth.tar')
    logging.info(f'Best epoch: {epoch_best}; RMSE: {error_best:.3f}')
    logging.info('***** TEST RESULTS *****')
    for shot in ['Overall', 'Many', 'Medium', 'Few']:
        m = metric_dict_best[shot.lower()]
        logging.info(f" * {shot}: RMSE {m['RMSE']:.3f}\t"
                     f"ABS_REL {m['ABS_REL']:.3f}\t"
                     f"LG10 {m['LG10']:.3f}\t"
                     f"MAE {m['MAE']:.3f}\t"
                     f"DELTA1 {m['DELTA1']:.3f}\t"
                     f"DELTA2 {m['DELTA2']:.3f}\t"
                     f"DELTA3 {m['DELTA3']:.3f}\t"
                     f"NUM {m['NUM']}")
    if writer is not None:
        writer.close()
    return model


if __name__ == '__main__':
    main()
