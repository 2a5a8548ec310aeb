"""Golden fixture for NYUD2-DIR's decoder D and multi-scale fusion MFF, produced by running the REFERENCE's own modules.

Run in the build container only (needs the reference tree, read-only):

    python tests/golden/make_golden_nyud2_decoder.py

nyud2-dir/models/modules.py (D, modules.py:61-94; MFF, modules.py:96-128) is imported unmodified and run on the CPU in
fp32, in training mode (batch statistics).  Parameters are filled as make_golden_nyud2_encoder.fill_params does; the
inputs are block maps of the 36 x 44 encoder geometry (batch 2):
  x_block{s} = relu(det_param("x_nyud2_decoder_{s}", (2, C_s, H_s, W_s), 1)),  C = 256, 512, 1024, 2048,
  (H, W) = 9x11, 5x6, 3x3, 2x2
(non-negative like E_resnet's outputs).  D returns 64 channels at 18 x 22 (twice block1); MFF runs at that size.  The
loss is <D(x), gD> + <MFF(x, (18, 22)), gM> with gD, gM = det_param("g_nyud2_decoder_D" / "_MFF", output shape, 1).

Stored (kept small: inputs and output gradients are regenerated from det_param by the test):
  d_names / d_shapes, m_names / m_shapes   state_dict keys and shapes of D(2048) and MFF([256, 512, 1024, 2048])
  d_out, m_out                             the outputs (NCHW, float16)
  dx{s} (s = 1..4)                         d loss / d x_block{s}: norm and the values at SAMPLE flat indices
  grad sample / norm per parameter         "{d|m}g:{name}" = values at the parameter's sample indices, "{d|m}n:{name}" =
                                           the full gradient's L2 norm
Sample indices of a tensor with `numel` elements: numpy.linspace(0, numel - 1, min(numel, SAMPLE)).astype(int64).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_nyud2_encoder import det_param, fill_params  # noqa: E402

REF = "/root/reference/nyud2-dir"
CHANNELS = (256, 512, 1024, 2048)
SIZES = ((9, 11), (5, 6), (3, 3), (2, 2))
BATCH = 2
SAMPLE = 512


def sample_idx(numel):
    return np.linspace(0, numel - 1, min(numel, SAMPLE)).astype(np.int64)


def inputs():
    return [torch.relu(det_param(f"x_nyud2_decoder_{s + 1}", (BATCH, c, h, w), 1.0))
            for s, (c, (h, w)) in enumerate(zip(CHANNELS, SIZES))]


def main():
    sys.path.insert(0, REF)                 # `from models import ...`; models/fds.py imports the top-level util.py
    from models import modules
    torch.manual_seed(0)
    Dm, Mm = modules.D(2048), modules.MFF(list(CHANNELS))
    fill_params([("D." + n, p) for n, p in Dm.named_parameters()])
    fill_params([("MFF." + n, p) for n, p in Mm.named_parameters()])
    Dm.train()
    Mm.train()
    xs = [x.clone().requires_grad_(True) for x in inputs()]
    d = Dm(*xs)
    size = (d.shape[2], d.shape[3])
    m = Mm(*xs, size)
    gD = det_param("g_nyud2_decoder_D", tuple(d.shape), 1.0)
    gM = det_param("g_nyud2_decoder_MFF", tuple(m.shape), 1.0)
    ((d * gD).sum() + (m * gM).sum()).backward()
    out = dict(d_out=d.detach().numpy().astype(np.float16), m_out=m.detach().numpy().astype(np.float16))
    for tag, mod in (("d", Dm), ("m", Mm)):
        sd = mod.state_dict()
        names = list(sd.keys())
        shapes = np.full((len(names), 4), -1, dtype=np.int64)
        for i, k in enumerate(names):
            shapes[i, :sd[k].dim()] = sd[k].shape
        out[f"{tag}_names"] = np.array(names)
        out[f"{tag}_shapes"] = shapes
        for n, p in mod.named_parameters():
            g = p.grad.detach().reshape(-1)
            out[f"{tag}g:{n}"] = g.numpy()[sample_idx(g.numel())].astype(np.float32)
            out[f"{tag}n:{n}"] = np.float64(g.double().norm())
    for s, x in enumerate(xs):
        g = x.grad.detach().reshape(-1)
        out[f"dx{s + 1}"] = g.numpy()[sample_idx(g.numel())].astype(np.float32)
        out[f"dxn{s + 1}"] = np.float64(g.double().norm())
    path = os.path.join(HERE, "nyud2_decoder.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", tuple(d.shape), tuple(m.shape))


if __name__ == "__main__":
    main()
