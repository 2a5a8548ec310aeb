"""CPU restatement of one reference training step (agedb-dir/train.py:246-262:
forward through ResNet-50 with FDS.smooth, weighted L1, backward, Adam) in
plain PyTorch fp32 -- TEST INFRASTRUCTURE / CPU BASELINE ONLY (bench.py's
`cpu_baseline` and `--impl reference` legs; see oracle/dir_oracle.py's header).
It is the "port" kind of baseline: where no copy of the reference's own
modules is installed (oracle/_ref), the timed CPU arm is this restatement, which uses the same
torch CPU kernels (MKL-DNN convolutions, ATen BN/ReLU, autograd, torch.optim.Adam)
the reference's own modules would dispatch to.
"""
import torch

from oracle import resnet_ref as R


def init_params(seed=0, layers=R.LAYERS):
    """He-normal convs / BN (1, 0) / Linear default, as agedb-dir/resnet.py:103-109."""
    g = torch.Generator().manual_seed(seed)
    p = {}
    for name, shape in R.param_shapes(layers):
        if len(shape) == 4:
            n = shape[2] * shape[3] * shape[0]
            v = torch.randn(*shape, generator=g) * (2.0 / n) ** 0.5
        elif name.startswith("linear"):
            bound = 1 / 2048 ** 0.5
            v = (torch.rand(*shape, generator=g) * 2 - 1) * bound
        elif name.endswith("weight"):
            v = torch.ones(*shape)
        else:
            v = torch.zeros(*shape)
        p[name] = v.requires_grad_(True)
    return p


def fds_smooth_torch(enc, labels, bucket_num, bucket_start, m1, v1, m2, v2, clip=(0.1, 10.0)):
    """Differentiable FDS.smooth (agedb-dir/fds.py:115-144 + utils.py:97-107), vectorised over rows."""
    lab = labels.reshape(-1)
    lo, hi = float(bucket_start), float(bucket_num - 1)
    has_lo, has_hi = bool((lab == lo).any()), bool((lab == hi).any())
    bins = (lab - lo).long().clamp(0, bucket_num - bucket_start - 1)
    active = (lab >= lo) & (lab <= hi)
    if has_lo:
        active = active | (lab < lo)
    if has_hi:
        active = active | (lab > hi)
    rv1, rv2, rm1, rm2 = v1[bins], v2[bins], m1[bins], m2[bins]
    row_ok = active & ~(v1.sum(1)[bins] < 1e-10)
    ok = row_ok[:, None] & (rv1 != 0)
    fac = torch.clamp(rv2 / torch.where(rv1 != 0, rv1, torch.ones_like(rv1)), clip[0], clip[1])
    return torch.where(ok, (enc - rm1) * torch.sqrt(fac) + rm2, enc)


class RefTrainer:
    def __init__(self, bucket_num=101, bucket_start=0, lr=1e-3, seed=0, fds_tables=None):
        self.p = init_params(seed)
        self.opt = torch.optim.Adam(list(self.p.values()), lr=lr)
        self.bucket_num, self.bucket_start = bucket_num, bucket_start
        self.tables = fds_tables          # (m1, v1, m2, v2) or None

    def step(self, x, targets, weights):
        pred_in = R.forward_encoding(self.p, x)
        if self.tables is not None:
            pred_in = fds_smooth_torch(pred_in, targets, self.bucket_num, self.bucket_start, *self.tables)
        pred = pred_in @ self.p["linear.weight"].t() + self.p["linear.bias"]
        loss = ((pred - targets).abs() * weights).mean()
        self.opt.zero_grad()
        loss.backward()
        self.opt.step()
        return float(loss.detach())
