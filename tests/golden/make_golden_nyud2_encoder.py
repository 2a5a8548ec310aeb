"""Golden fixture for the NYUD2-DIR multi-scale encoder, produced by running the REFERENCE's own modules.

Run in the build container only (needs /root/reference, read-only):

    python tests/golden/make_golden_nyud2_encoder.py

nyud2-dir/models/resnet.py (resnet50) and nyud2-dir/models/modules.py (E_resnet, modules.py:33-58) are imported
unmodified and run on the CPU in fp32.  Every parameter is overwritten with tests/util.det_param values (so that a test
regenerates them without the reference):
  conv weights  det_param(name, shape, sqrt(2 / (k * k * cout)))   (the scale of resnet.py's initialisation)
  BN weights    1 + 0.1 * det_param(name, shape, 1)
  BN biases     0.1 * det_param(name, shape, 1)
and E is run in training mode (batch statistics) on x = det_param("x_nyud2_encoder", (2, 3, 36, 44), 1): H and W are
multiples of 4 but not of 32, so every stage map (18x22, 9x11, 5x6, 3x3, 2x2) has an odd side.

Stored: E.state_dict() key names and shapes, x, and the four block outputs (NCHW fp32).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/nyud2-dir"
X_SHAPE = (2, 3, 36, 44)


def det_param(name, shape, scale):
    """tests/util.det_param (the reference's nyud2-dir/util.py takes the module name `util` here)."""
    seed = sum((i + 1) * ord(c) for i, c in enumerate(name)) % (2 ** 31)
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def fill_params(named):
    """(name, tensor) pairs in named_parameters() order -> the fixture's deterministic values (in place)."""
    with torch.no_grad():
        for name, p in named:
            if p.dim() == 4:
                cout, _, k, _ = p.shape
                p.copy_(det_param(name, p.shape, (2.0 / (k * k * cout)) ** 0.5))
            elif name.endswith("weight"):
                p.copy_(1.0 + 0.1 * det_param(name, p.shape, 1.0))
            else:
                p.copy_(0.1 * det_param(name, p.shape, 1.0))


def main():
    sys.path.insert(0, REF)                 # `from models import ...`; models/fds.py imports the top-level util.py
    from models import modules, resnet
    torch.manual_seed(0)
    E = modules.E_resnet(resnet.resnet50())
    fill_params(list(E.named_parameters()))
    E.train()
    x = det_param("x_nyud2_encoder", X_SHAPE, 1.0)
    with torch.no_grad():
        blocks = E(x)
    sd = E.state_dict()
    names = list(sd.keys())
    shapes = np.full((len(names), 4), -1, dtype=np.int64)
    for i, k in enumerate(names):
        shapes[i, :sd[k].dim()] = sd[k].shape
    out = dict(names=np.array(names), shapes=shapes, x=x.numpy())
    for s, b in enumerate(blocks):
        out[f"block{s + 1}"] = b.numpy().astype(np.float32)
    path = os.path.join(HERE, "nyud2_encoder.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes;", [tuple(b.shape) for b in blocks])


if __name__ == "__main__":
    main()
