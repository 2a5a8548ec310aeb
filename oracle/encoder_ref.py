"""NYUD2-DIR's multi-scale encoder (nyud2-dir/models/modules.py:33-58, E_resnet.forward) as a pure function over a
state_dict -- TEST INFRASTRUCTURE ONLY (see oracle/dir_oracle.py for the rules).

oracle/resnet_ref.forward_encoding computes the same network but hands its block outputs out only as detached taps.
forward_blocks runs the identical computation (resnet_ref's own helpers, tap names and teacher forcing) and returns the
four layer-group outputs with their autograd history, so that a loss sum_s <x_block_s, d_s> can be back-propagated.
Both are pinned against the reference's own E_resnet by tests/test_nyud2_encoder_cpu.py (fixture
tests/golden/nyud2_encoder.npz, made by tests/golden/make_golden_nyud2_encoder.py).

install() copies the reference's nyud2-dir/models/ into the git-ignored oracle/_ref/nyud2-dir/models/ (next to the
util.py oracle/ref_nyud2.install() copies) for the reference arm of tools/nyud2_encoder_bench.py.
"""
import os

import torch.nn.functional as F

from oracle import resnet_ref as R

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_DIR = os.path.join(ROOT, "oracle", "_ref", "nyud2-dir")
MODELS = ("__init__.py", "resnet.py", "modules.py", "fds.py")


def last_blocks(layers=R.LAYERS):
    """Block index (forward_encoding's tap numbering) of the last block of every layer group."""
    out, bi = [], 0
    for nblocks in layers:
        bi += nblocks
        out.append(bi - 1)
    return out


def forward_blocks(p, x, layers=R.LAYERS, stats=None, quant=False, taps=None, force=None):
    """x [B,3,H,W] -> (x_block1, ..., x_block4) NCHW, train-mode BN; arguments as resnet_ref.forward_encoding."""
    def tap(name, t):
        if force is not None and name in force:
            t = t + (force[name] - t).detach()
        if taps is not None:
            taps[name] = t.detach()
        return t
    x = R._q(x, quant)
    x = tap("stem.y", R._conv(x, p["conv1.weight"], 2, 3, quant))
    x = tap("stem.a", R._q(F.relu(R._bn(x, p, "bn1.", stats, quant)), quant))
    x = tap("stem.pool", F.max_pool2d(R._rb(x, quant), 3, 2, 1))
    outs, bi = [], 0
    for li, nblocks in enumerate(layers):
        for b in range(nblocks):
            stride = 2 if (b == 0 and li > 0) else 1
            pre = f"layer{li + 1}.{b}."
            idn = R._rb(x, quant)
            o = tap(f"{bi}.0", R._conv(x, p[pre + "conv1.weight"], 1, 0, quant))
            o = tap(f"{bi}.1", R._q(F.relu(R._bn(o, p, pre + "bn1.", stats, quant)), quant))
            o = tap(f"{bi}.2", R._conv(o, p[pre + "conv2.weight"], stride, 1, quant))
            o = tap(f"{bi}.3", R._q(F.relu(R._bn(o, p, pre + "bn2.", stats, quant)), quant))
            o = tap(f"{bi}.4", R._conv(o, p[pre + "conv3.weight"], 1, 0, quant))
            o = R._bn(o, p, pre + "bn3.", stats, quant)
            if pre + "downsample.0.weight" in p:
                idn = tap(f"{bi}.5", R._conv(x, p[pre + "downsample.0.weight"], stride, 0, quant))
                idn = R._bn(idn, p, pre + "downsample.1.", stats, quant)
            x = tap(f"{bi}.6", R._q(F.relu(o + idn), quant))
            bi += 1
        outs.append(x)
    return tuple(outs)


def available():
    return all(os.path.exists(os.path.join(REF_DIR, "models", f)) for f in MODELS) and \
        os.path.exists(os.path.join(REF_DIR, "util.py"))


def install(reference_root="/root/reference"):
    """Copy nyud2-dir/models/{__init__,resnet,modules,fds}.py into oracle/_ref (called by __graft_entry__.build())."""
    import shutil
    src = os.path.join(reference_root, "nyud2-dir", "models")
    if not all(os.path.isfile(os.path.join(src, f)) for f in MODELS):
        return False
    os.makedirs(os.path.join(REF_DIR, "models"), exist_ok=True)
    for f in MODELS:
        shutil.copyfile(os.path.join(src, f), os.path.join(REF_DIR, "models", f))
    return True
