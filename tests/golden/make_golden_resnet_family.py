"""Generate tests/golden/resnet_family.npz by running the REFERENCE's own agedb-dir/resnet.py.

Run in the build container only (needs /root/reference, read-only):

    python tests/golden/make_golden_resnet_family.py

Stores
  * one fp32 CPU training-mode forward + backward of ResNet(BasicBlock, [2, 2, 2, 2]) (ResNet-18 with the 1-output
    regressor, FDS idle) on a seeded 4 x 3 x 224 x 224 batch (the reference's AvgPool2d(7) needs the 7 x 7 map of a
    224^2 input): the encoding, the prediction, the loss, bn1's running statistics and, for every parameter, its
    gradient's sum, absolute sum and 64 elements at fixed positions (the whole gradient of every parameter with at most
    4096 elements);
  * the state_dict keys and shapes of ResNet-18 / 34 / 101 / 152 (layer lists of nyud2-dir/models/resnet.py:153-205)
    with and without FDS.
The same shim as make_golden.py: fds.FDS calls .cuda() unconditionally (fds.py:52), so torch.Tensor.cuda is the
identity here.  Nothing is copied from the reference; only its outputs on seeded inputs are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
REF = "/root/reference/agedb-dir"
torch.Tensor.cuda = lambda self, *a, **k: self
sys.path.insert(0, REF)
import resnet as ref_resnet      # noqa: E402
import loss as ref_loss          # noqa: E402

FDS_ARGS = dict(bucket_num=100, bucket_start=3, start_update=0, start_smooth=1, kernel="gaussian", ks=5, sigma=2,
                momentum=0.9)
DEPTHS = {18: ("BasicBlock", [2, 2, 2, 2]), 34: ("BasicBlock", [3, 4, 6, 3]), 101: ("Bottleneck", [3, 4, 23, 3]),
          152: ("Bottleneck", [3, 8, 36, 3])}
SAMPLES = 64


def det_param(name: str, shape, scale: float) -> torch.Tensor:
    """Deterministic parameter generator shared with tests (see tests/util.py)."""
    seed = sum((i + 1) * ord(c) for i, c in enumerate(name)) % (2 ** 31)
    g = torch.Generator().manual_seed(seed)
    return torch.randn(*shape, generator=g) * scale


def sample_index(numel):
    """The gradient positions stored per parameter: all of a small one, else SAMPLES spread over the tensor."""
    if numel <= 4096:
        return np.arange(numel)
    return np.unique(np.linspace(0, numel - 1, SAMPLES).round().astype(np.int64))


def make(depth, fds):
    block, layers = DEPTHS[depth]
    return ref_resnet.ResNet(getattr(ref_resnet, block), layers, fds=fds, **FDS_ARGS)


def basic_case(out):
    torch.manual_seed(0)
    torch.set_num_threads(8)
    m = make(18, False)
    with torch.no_grad():
        for n, p in m.named_parameters():
            if p.dim() == 4:
                fan = p.shape[0] * p.shape[2] * p.shape[3]
                p.copy_(det_param(n, p.shape, (2.0 / fan) ** 0.5))
            elif n == "linear.weight":
                p.copy_(det_param(n, p.shape, 0.05))
            elif n == "linear.bias":
                p.fill_(0.1)
            elif n.endswith("weight"):        # BN gamma
                p.copy_(1.0 + 0.1 * det_param(n, p.shape, 1.0))
            else:                             # BN beta
                p.copy_(0.1 * det_param(n, p.shape, 1.0))
    m.train()
    x = det_param("input18", (4, 3, 224, 224), 1.0)
    t = torch.tensor([[31.0], [44.0], [5.0], [70.0]])
    w = torch.tensor([[0.5], [1.5], [1.0], [2.0]])
    enc = {}

    def keep(mod, inp, o):                   # returns None: the forward's own output is kept
        enc["enc"] = o.reshape(o.shape[0], -1).detach().clone()
    m.avgpool.register_forward_hook(keep)
    pred = m(x, t, 0)
    loss = ref_loss.weighted_l1_loss(pred, t, w)
    loss.backward()
    out["basic/pred"] = pred.detach().numpy()
    out["basic/enc"] = enc["enc"].numpy()
    out["basic/loss"] = loss.detach().numpy()
    out["basic/bn1_running_mean"] = m.bn1.running_mean.numpy().copy()
    out["basic/bn1_running_var"] = m.bn1.running_var.numpy().copy()
    for n, p in m.named_parameters():
        g = p.grad.reshape(-1)
        out[f"grad_sum/{n}"] = g.double().sum().numpy()
        out[f"grad_abs/{n}"] = g.double().abs().sum().numpy()
        out[f"grad_at/{n}"] = g[torch.from_numpy(sample_index(g.numel()))].numpy().copy()


def layouts(out):
    for depth in DEPTHS:
        for fds in (False, True):
            m = make(depth, fds)
            sd = m.state_dict()
            tag = f"resnet{depth}" + ("_fds" if fds else "")
            out[f"keys/{tag}"] = np.array(list(sd.keys()))
            shapes = np.full((len(sd), 4), -1, np.int64)
            for i, v in enumerate(sd.values()):
                shapes[i, :v.dim()] = v.shape
            out[f"shapes/{tag}"] = shapes
            out[f"n_params/{tag}"] = np.array(sum(p.numel() for p in m.parameters()))


if __name__ == "__main__":
    import logging
    logging.disable(logging.CRITICAL)
    out = {}
    basic_case(out)
    layouts(out)
    np.savez_compressed(os.path.join(HERE, "resnet_family.npz"), **out)
    print("resnet_family.npz", os.path.getsize(os.path.join(HERE, "resnet_family.npz")), "bytes")
