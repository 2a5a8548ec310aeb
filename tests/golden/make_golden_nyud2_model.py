"""Golden fixture for NYUD2-DIR's assembled depth network net.model (nyud2-dir/models/net.py:5-22), produced by running
the REFERENCE's own modules.

Run in the build container only (needs the reference tree, read-only):

    python tests/golden/make_golden_nyud2_model.py

nyud2-dir/models/{net,modules,resnet,fds}.py are imported unmodified and run on the CPU in fp32 (one shim:
Tensor.cuda -> identity, because fds.py calls .cuda() unconditionally).  The model is
net.model(args, E_resnet(resnet50()), 2048, [256, 512, 1024, 2048]) with args.fds on (FDS defaults of
nyud2-dir/train.py: 100 buckets from 7, gaussian window ks 5 / sigma 2, momentum 0.9, start_update 0, start_smooth 1).
  parameters      make_golden_nyud2_encoder.fill_params over named_parameters() ("E.conv1.weight", ...)
  FDS tables      running_mean_last_epoch = 0.3 det_param("fds.rm"), running_var_last_epoch = 0.5 + |det_param("fds.rv")|,
                  smoothed_mean_last_epoch = 0.3 det_param("fds.sm"), smoothed_var_last_epoch = 0.5 + |det_param("fds.sv")|
                  (each [93, 128]); the rest as constructed
  input           x = det_param("x_nyud2_model", (2, 3, 36, 44), 1)
  depth, weight   0.5 + 9.5 u_d and 0.5 + u_w, u = torch.rand from torch.Generator().manual_seed(11) ([2, 1, 18, 22] each,
                  depth first)
  epoch           1 (= start_smooth: R's features are smoothed)
The train-mode forward returns (out, feature); loss = torch.mean(((out - depth) ** 2) * weight) (train.py:200) is
back-propagated; then eval() and one forward on the same x (running statistics updated once by the training forward).

Stored:
  names / shapes, names_nofds / shapes_nofds   state_dict keys and shapes with and without args.fds
  out, eval_out                                the train-mode and the eval-mode output [2, 1, 18, 22], fp32
  feature, feature_norm                        feature [2, 128, 18, 22] at sample_idx(numel, 8192), and its L2 norm
  loss                                         the loss
  g:{name}, n:{name}                           every parameter gradient at sample_idx(numel, 128), and its L2 norm
Sample indices: numpy.linspace(0, numel - 1, min(numel, k)).astype(int64).
"""
import os
import sys
from types import SimpleNamespace

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from make_golden_nyud2_encoder import det_param, fill_params  # noqa: E402

REF = "/root/reference/nyud2-dir"
X_SHAPE = (2, 3, 36, 44)
OUT_SHAPE = (2, 1, 18, 22)
FEATURE_SAMPLE = 8192
GRAD_SAMPLE = 128


def sample_idx(numel, k):
    return np.linspace(0, numel - 1, min(numel, k)).astype(np.int64)


def make_args(fds=True):
    return SimpleNamespace(fds=fds, bucket_num=100, bucket_start=7, start_update=0, start_smooth=1,
                           fds_kernel="gaussian", fds_ks=5, fds_sigma=2.0, fds_mmt=0.9)


def fds_tables(nb=93, c=128):
    return {"running_mean_last_epoch": 0.3 * det_param("fds.rm", (nb, c), 1.0),
            "running_var_last_epoch": 0.5 + det_param("fds.rv", (nb, c), 1.0).abs(),
            "smoothed_mean_last_epoch": 0.3 * det_param("fds.sm", (nb, c), 1.0),
            "smoothed_var_last_epoch": 0.5 + det_param("fds.sv", (nb, c), 1.0).abs()}


def depth_and_weight():
    g = torch.Generator().manual_seed(11)
    depth = 0.5 + 9.5 * torch.rand(OUT_SHAPE, generator=g)
    weight = 0.5 + torch.rand(OUT_SHAPE, generator=g)
    return depth, weight


def layout(sd):
    names = list(sd.keys())
    shapes = np.full((len(names), 4), -1, dtype=np.int64)
    for i, k in enumerate(names):
        shapes[i, :sd[k].dim()] = sd[k].shape
    return np.array(names), shapes


def main():
    torch.Tensor.cuda = lambda self, *a, **k: self
    sys.path.insert(0, REF)                 # `from models import ...`; models/fds.py imports the top-level util.py
    from models import modules, net, resnet
    torch.manual_seed(0)
    m = net.model(make_args(True), modules.E_resnet(resnet.resnet50()), 2048, [256, 512, 1024, 2048])
    fill_params(list(m.named_parameters()))
    for k, v in fds_tables().items():
        setattr(m.R.FDS, k, v.clone())
    out = {}
    out["names"], out["shapes"] = layout(m.state_dict())
    m_nofds = net.model(make_args(False), modules.E_resnet(resnet.resnet50()), 2048, [256, 512, 1024, 2048])
    out["names_nofds"], out["shapes_nofds"] = layout(m_nofds.state_dict())
    x = det_param("x_nyud2_model", X_SHAPE, 1.0)
    depth, weight = depth_and_weight()
    m.train()
    pred, feature = m(x, depth, 1)
    loss = torch.mean(((pred - depth) ** 2) * weight)
    loss.backward()
    out["out"] = pred.detach().numpy().astype(np.float32)
    f = feature.detach().reshape(-1)
    out["feature"] = f.numpy()[sample_idx(f.numel(), FEATURE_SAMPLE)].astype(np.float32)
    out["feature_norm"] = np.float64(f.double().norm())
    out["loss"] = np.float64(loss.item())
    for n, p in m.named_parameters():
        g = p.grad.detach().reshape(-1)
        out[f"g:{n}"] = g.numpy()[sample_idx(g.numel(), GRAD_SAMPLE)].astype(np.float32)
        out[f"n:{n}"] = np.float64(g.double().norm())
    m.eval()
    with torch.no_grad():
        out["eval_out"] = m(x).numpy().astype(np.float32)
    path = os.path.join(HERE, "nyud2_model.npz")
    np.savez_compressed(path, **out)
    print(path, os.path.getsize(path), "bytes; loss", loss.item(), tuple(pred.shape), tuple(feature.shape))


if __name__ == "__main__":
    main()
