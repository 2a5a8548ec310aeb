"""net.model -- NYUD2-DIR's depth network (nyud2-dir/models/net.py:5-22) on the native path: the multi-scale encoder E
(resnet.E_resnet), the decoder D and multi-scale fusion MFF (dense_ops.D / MFF) and the refinement module R
(dense_ops.RefinementR, with R's FDS as fds_variants.FDSDepth).  state_dict keys and shapes are the reference's, so its
checkpoints load (after stripping DataParallel's `module.` prefix):

    model = net.model(args, resnet.E_resnet(resnet.resnet50()), num_features=2048, block_channel=[256, 512, 1024, 2048])

(nyud2-dir/train.py:59-64).  forward(x, depth, epoch): x fp32 NCHW [N, 3, H, W] (H, W multiples of 4) -> the depth
prediction fp32 [N, 1, H/2, W/2]; in training with FDS also the unsmoothed 128-channel feature map of R, the input of
R.FDS.update_running_stats (nyud2-dir/train.py:216-228)."""
import torch.nn as nn

import dense_ops
from fds_variants import FDSDepth
from resnet import E_resnet


class model(nn.Module):
    def __init__(self, args, Encoder, num_features, block_channel):
        super(model, self).__init__()
        if not isinstance(Encoder, E_resnet):
            raise TypeError(f"net.model needs a resnet.E_resnet encoder, got {type(Encoder).__name__}")
        self.E = Encoder
        self.D = dense_ops.D(num_features)
        self.MFF = dense_ops.MFF(block_channel)
        num_r = 64 + block_channel[3] // 32                 # modules.py:134
        fds = None
        if args is not None and args.fds:                    # modules.py:149-152
            fds = FDSDepth(feature_dim=num_r, bucket_num=args.bucket_num, bucket_start=args.bucket_start,
                           start_update=args.start_update, start_smooth=args.start_smooth, kernel=args.fds_kernel,
                           ks=args.fds_ks, sigma=args.fds_sigma, momentum=args.fds_mmt)
        self.R = dense_ops.RefinementR(num_r, fds=fds)

    def forward(self, x, depth=None, epoch=None):
        x_block1, x_block2, x_block3, x_block4 = self.E(x)
        x_decoder = self.D(x_block1, x_block2, x_block3, x_block4)
        x_mff = self.MFF(x_block1, x_block2, x_block3, x_block4, [x_decoder.size(1), x_decoder.size(2)])
        out = self.R(dense_ops.cat_channels([x_decoder, x_mff]), depth, epoch)
        if isinstance(out, tuple):
            # NHWC [N, h, w, 1] and NCHW [N, 1, h, w] are the same bytes; the feature is a view of the NHWC bf16 map
            pred, feature = out
            return pred.view(pred.shape[0], 1, pred.shape[1], pred.shape[2]), feature.permute(0, 3, 1, 2)
        return out.view(out.shape[0], 1, out.shape[1], out.shape[2])
