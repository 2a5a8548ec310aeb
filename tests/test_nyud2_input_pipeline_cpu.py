"""CPU-only companions of tests/test_gpu_nyud2_input_pipeline.py (the NYUD2-DIR input pipeline, loaddata.py).

1. draw_nyud2_train_params consumes Python `random` and the torch generator exactly as the reference's per-sample
   training chain does: the draws recorded from the reference's own transforms (tests/golden/nyud2_transform.npz, made
   by tests/golden/make_golden_nyud2_transform.py) come back bit for bit from the same seeds.
2. The affine the host hands the kernel is rotate's: scipy's affine_transform with it equals scipy's rotate bit for bit
   (float64 and uint8), at the angles and source shapes the GPU tests use.
3. dirb200_depth_augment_batch refuses bad arguments on the host, with a message, before any CUDA call.  Every device
   pointer below is a dummy that must never be dereferenced."""
import ctypes
import os
import random

import numpy as np
import pytest
import scipy.ndimage as nd
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
D = ctypes.c_void_p(16)               # stands for a device buffer
MEAN_STD = (ctypes.c_float * 6)(0.485, 0.456, 0.406, 0.229, 0.224, 0.225)


def test_draws_reproduce_the_reference_chain():
    import loaddata
    g = np.load(os.path.join(HERE, "golden", "nyud2_transform.npz"))
    n = len(g["angle"])
    random.seed(int(g["py_seed"]))
    torch.manual_seed(int(g["torch_seed"]))
    p = loaddata.draw_nyud2_train_params(n)
    assert p["flip"].tolist() == [1 if u < 0.5 else 0 for u in g["flip_u"]]
    assert p["angle"].numpy().tobytes() == g["angle"].tobytes()
    assert p["order"].tolist() == g["perm"].tolist()
    assert p["alpha"].numpy().tobytes() == g["jitter"].astype(np.float32).tobytes()
    want_rgb = torch.stack([loaddata.lighting_offset(torch.from_numpy(a)) for a in g["normal"]])
    assert torch.equal(p["rgb"], want_rgb)
    # and the same stream with an explicit generator / Random instance
    rng, gen = random.Random(int(g["py_seed"])), torch.Generator().manual_seed(int(g["torch_seed"]))
    q = loaddata.draw_nyud2_train_params(n, rng, gen)
    assert all(torch.equal(p[k], q[k]) for k in p)


SHAPES = [(240, 320), (241, 323), (320, 240), (13, 17)]
ANGLES = [0.0, 1e-6, -1e-6, 2.5, -2.5, 5.0, -5.0, 4.999, 3.7318]


@pytest.mark.parametrize("shape", SHAPES, ids=["x".join(map(str, s)) for s in SHAPES])
def test_affine_is_rotates(shape):
    import loaddata
    a = np.random.RandomState(shape[0]).randint(0, 256, shape).astype(np.uint8)
    for ang in ANGLES:
        m = loaddata.rotate_affine(ang, *shape)
        for src in (a, a.astype(np.float64)):
            want = nd.rotate(src, ang, reshape=False, order=2)
            got = nd.affine_transform(src, m[:4].reshape(2, 2), m[4:], order=2, mode="constant")
            assert got.dtype == want.dtype and got.tobytes() == want.tobytes(), (shape, ang)


def _args(**kw):
    a = dict(images=D, depths=D, depth_u16=0, n=2, h=240, w=320, crop_h=228, crop_w=304, depth_h=114, depth_w=152,
             flip=D, affine=D, rgb=D, order=D, alpha=D, mean_std=MEAN_STD, table=D, nb=100, image_out=D, depth_out=D,
             weight_out=D, debug_crop=None, debug_mean=None, ws=D, ws_bytes=1 << 40, stream=None)
    a.update(kw)
    return list(a.values())


BAD = [dict(images=None), dict(depths=None), dict(image_out=None), dict(depth_out=None), dict(ws=None),
       dict(mean_std=None), dict(n=0), dict(n=-1), dict(h=0), dict(w=-3), dict(crop_h=0), dict(depth_w=0),
       dict(h=227), dict(w=303), dict(depth_h=229), dict(depth_w=305), dict(n=8000, h=400, w=400),
       dict(depth_u16=2), dict(depth_u16=1), dict(depth_u16=1, affine=None, flip=None),
       dict(order=None), dict(alpha=None), dict(nb=99), dict(nb=0), dict(weight_out=None), dict(ws_bytes=1000),
       dict(mean_std=(ctypes.c_float * 6)(0.485, 0.456, 0.406, 0.229, 0.0, 0.225))]


@pytest.mark.parametrize("kw", BAD, ids=[",".join(f"{k}={v if not hasattr(v, '_type_') else 'p'}" for k, v in b.items())
                                         for b in BAD])
def test_depth_augment_refuses_bad_arguments(kw):
    import _lib
    got = _lib.raw("dirb200_depth_augment_batch")(*_args(**kw))
    assert got == -1 and "depth_augment_batch" in _lib.last_error(), (kw, got, _lib.last_error())


def test_workspace_bytes():
    import _lib
    f = _lib.raw("dirb200_depth_augment_workspace_bytes")
    assert f(8, 240, 320, 228, 304) == 8 * 4 * 240 * 320 * 8 + 8 * 228 * 304 * 4 + 8 * 16 * 8
    assert f(0, 240, 320, 228, 304) == 0 and f(8, 240, 320, 0, 304) == 0
