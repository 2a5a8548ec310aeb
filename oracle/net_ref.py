"""NYUD2-DIR's assembled depth network net.model (nyud2-dir/models/net.py:5-22) as a pure function over a parameter dict
-- TEST INFRASTRUCTURE ONLY (see oracle/dir_oracle.py for the rules).

forward(p, x, depth, epoch, fds) = R(cat(D(E(x)), MFF(E(x))), depth, epoch) in training mode (batch statistics), built
from encoder_ref.forward_blocks (E), the decoder_d / mff restatement of tests/test_nyud2_decoder_cpu.py (D, MFF) and
refinement() below (R, modules.py:128-174, with R.FDS.smooth of nyud2-dir/models/fds.py:129-149 and
calibrate_mean_var of nyud2-dir/util.py:151-162).  Pinned against the reference's own net.model by
tests/test_nyud2_model_cpu.py (fixture tests/golden/nyud2_model.npz, made by tests/golden/make_golden_nyud2_model.py).
Any float dtype; the GPU tests run refinement() in float64 on the native bf16 storage points (`force`).

install() copies the reference's nyud2-dir/models/net.py next to the modules oracle/encoder_ref.install() copies into
the git-ignored oracle/_ref/nyud2-dir/models/, for the reference arm of tools/nyud2_model_bench.py.
"""
import os

import torch
import torch.nn.functional as F

from oracle import encoder_ref

NET_PY = os.path.join(encoder_ref.REF_DIR, "models", "net.py")


def available():
    return encoder_ref.available() and os.path.exists(NET_PY)


def install(reference_root="/root/reference"):
    """Copy nyud2-dir/models/net.py into oracle/_ref (called by __graft_entry__.build() after encoder_ref.install())."""
    import shutil
    src = os.path.join(reference_root, "nyud2-dir", "models", "net.py")
    if not os.path.isfile(src) or not os.path.isdir(os.path.dirname(NET_PY)):
        return False
    shutil.copyfile(src, NET_PY)
    return True


def bn_train(x, w, b, eps=1e-5):
    mean = x.mean((0, 2, 3), keepdim=True)
    var = ((x - mean) ** 2).mean((0, 2, 3), keepdim=True)
    return (x - mean) / torch.sqrt(var + eps) * w.view(1, -1, 1, 1).to(x.dtype) + b.view(1, -1, 1, 1).to(x.dtype)


def fds_smooth(feature, depth, tables, bucket_num=100, bucket_start=7, clip=(0.2, 5.0)):
    """FDS.smooth on an NCHW feature map: every pixel's channels re-coloured with its depth bucket's statistics
    (bucket = clamp(floor(10 depth), bucket_start, bucket_num - 1)); tables: the four *_last_epoch [nb, C] tables."""
    n, c, h, w = feature.shape
    rows = feature.permute(0, 2, 3, 1).reshape(-1, c)
    lab = depth.reshape(-1).to(torch.float32)
    bucket = torch.clamp(torch.floor(lab * 10).long(), bucket_start, bucket_num - 1) - bucket_start
    m1, v1 = tables["running_mean_last_epoch"][bucket], tables["running_var_last_epoch"][bucket]
    m2, v2 = tables["smoothed_mean_last_epoch"][bucket], tables["smoothed_var_last_epoch"][bucket]
    factor = torch.clamp(v2 / v1, clip[0], clip[1]).to(rows.dtype)
    out = (rows - m1.to(rows.dtype)) * torch.sqrt(factor) + m2.to(rows.dtype)
    return out.view(n, h, w, c).permute(0, 3, 1, 2)


def refinement(p, x, depth=None, epoch=None, fds=None, force=None, taps=None):
    """R (modules.py:128-174) in training mode: returns (x2, x1).  fds: None, or dict(tables=..., start_smooth=...);
    force: {"x0", "x1", "x1_s"} -> values that replace those activations in the forward (teacher forcing, gradients
    pass straight through); taps receives them."""
    def tap(name, t):
        if force is not None and name in force:
            t = t + (force[name] - t).detach()
        if taps is not None:
            taps[name] = t
        return t
    x0 = tap("x0", torch.relu(bn_train(F.conv2d(x, p["conv0.weight"], padding=2), p["bn0.weight"], p["bn0.bias"])))
    x1 = tap("x1", torch.relu(bn_train(F.conv2d(x0, p["conv1.weight"], padding=2), p["bn1.weight"], p["bn1.bias"])))
    x1_s = x1
    if fds is not None and epoch >= fds["start_smooth"]:
        x1_s = tap("x1_s", fds_smooth(x1, depth, fds["tables"]))
    x2 = F.conv2d(x1_s, p["conv2.weight"], p["conv2.bias"], padding=2)
    return x2, x1


def forward(p, x, depth=None, epoch=None, fds=None):
    """p: parameters by net.model name ("E.conv1.weight", "D.up1.conv1.weight", "R.conv2.bias", ...); x NCHW
    [N, 3, H, W] -> (out [N, 1, H/2, W/2], feature [N, 128, H/2, W/2] = R's unsmoothed x1)."""
    from test_nyud2_decoder_cpu import decoder_d, mff
    sub = lambda pre: {k[len(pre):]: v for k, v in p.items() if k.startswith(pre)}
    blocks = encoder_ref.forward_blocks(sub("E."), x)
    x_decoder = decoder_d(sub("D."), blocks)
    x_mff = mff(sub("MFF."), blocks, x_decoder.shape[2:])
    return refinement(sub("R."), torch.cat((x_decoder, x_mff), 1), depth, epoch, fds)
