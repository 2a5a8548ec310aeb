"""CPU-only companions of tests/test_gpu_dense_and_step_kernels.py.

1. Its float64 up-sampling reference builds the interpolation weights from a restatement of the align_corners=False
   index rule (src_index).  Here that restatement is pinned to the rule F.interpolate applies in float64: the weight
   matrix read off F.interpolate of an identity agrees with it entry by entry to a few fp32 ulps of the source position
   (the restatement forms the position in fp32, as the kernel does), so both pick the same source rows and the same
   lambda wherever the choice matters.
2. The up-sampling, channel-copy, pooling, regressor and optimizer entry points refuse bad arguments on the host, with a
   message, before any CUDA call.  Every pointer below is a dummy that must never be dereferenced, so a call that got past
   its checks would fault on a GPU machine and fail without one.

Found by these tests: dirb200_copy_channels accepted negative channel offsets (src_off + c <= src_stride holds for
src_off = -8), and dirb200_linear1_fwd / _bwd narrowed a row count above 2^31 - 1 to the launch's 32-bit grid size or
loop bound, computing a different, smaller problem without an error."""
import ctypes

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_dense_and_step_kernels import interp_matrix, src_index

D = ctypes.c_void_p(16)               # stands for a device buffer (16-byte aligned)
D8 = ctypes.c_void_p(24)              # 8-byte aligned only
BAD_C = (0, -8, 12)


def lib():
    import _lib
    import resnet  # noqa: F401  (registers the linear1 / optimizer entry points)
    return _lib


def refused(name, *args, msg, rc=-1):
    L = lib()
    got = L.raw(name)(*args)
    err = L.last_error()
    assert got == rc and msg in err, (name, args, got, err)


# ------------------------------------------------------------------------------------------- the index rule, pinned
# every (in, out) of the GPU file's up-sampling shapes, per axis, and a few ratios near integers
AXES = sorted({(8, 15), (10, 19), (15, 29), (19, 38), (29, 57), (38, 76), (57, 114), (76, 152), (29, 114), (38, 152),
               (15, 114), (19, 152), (8, 114), (10, 152), (15, 15), (19, 19), (37, 7), (41, 5), (12, 5), (9, 4),
               (1, 13), (1, 17), (13, 1), (17, 1), (1, 5), (20, 33), (7, 14), (1, 1), (5, 11), (7, 9),
               (3, 7), (7, 3), (100, 301), (301, 100), (64, 63), (63, 64)})


def aten_matrix(in_size, out_size):
    """float64 [out, in] weights of F.interpolate(mode='bilinear', align_corners=False) along one axis (the other
    axis has size 1 -> 1, weight 1)"""
    eye = torch.eye(in_size, dtype=torch.float64).view(1, in_size, in_size, 1)
    return F.interpolate(eye, size=(out_size, 1), mode="bilinear", align_corners=False)[0, :, :, 0].t().numpy()


@pytest.mark.parametrize("in_size,out_size", AXES, ids=[f"{a}-to-{b}" for a, b in AXES])
def test_index_rule_restatement_matches_interpolate(in_size, out_size):
    i0, i1, lam = src_index(in_size, out_size)
    assert (i0 >= 0).all() and (i1 <= in_size - 1).all() and ((i1 == i0) | (i1 == i0 + 1)).all()
    assert ((lam >= 0) & (lam < 1)).all()
    W, ref = interp_matrix(in_size, out_size), aten_matrix(in_size, out_size)
    assert np.allclose(W.sum(1), 1.0, rtol=0, atol=1e-12)
    # the source position s is formed in fp32 (scale = fp32(in / out) and the fma): up to a few ulps of s from
    # float64's; lambda (and 1 - lambda) move by that much
    s = i0 + lam.astype(np.float64)
    tol = 4 * np.spacing(np.maximum(s, 1.0).astype(np.float32)).astype(np.float64)
    err = np.abs(W - ref).max(1)
    assert (err <= tol).all(), (np.argmax(err - tol), err.max(), tol.max())
    # the same source rows wherever lambda is not within tol of 0 or 1 (where the row choice carries no weight)
    nz, nz_ref = W > tol[:, None], ref > tol[:, None]
    assert (nz == nz_ref).all()


def test_index_rule_needs_the_clamp_at_zero():
    """The first output positions of an up-sampling map to s < 0 before the clamp: without it, lambda would be
    negative and the weights would not form a convex combination (the kernel's upsample_src_index clamps too)."""
    scale = np.float32(8) / np.float32(15)
    assert np.float32(0.5 * float(scale) - 0.5) < 0
    i0, i1, lam = src_index(8, 15)
    assert i0[0] == 0 and lam[0] == 0


# ---------------------------------------------------------------------------------------------- host-side refusals
def up_calls(n, h, w, c, ho, wo, x=D, out=D):
    return [(name, (x, n, h, w, c, ho, wo, out, None))
            for name in ("dirb200_upsample_bilinear_fwd", "dirb200_upsample_bilinear_bwd")]


def test_upsample_refuses_bad_arguments():
    cases = [up_calls(2, 8, 10, c, 15, 19) for c in BAD_C]
    for k in range(6):                                        # n, h, w, (c), ho, wo each 0 and -1
        if k == 3:
            continue
        for v in (0, -1):
            a = [2, 8, 10, 64, 15, 19]
            a[k] = v
            cases.append(up_calls(*a))
    cases += [up_calls(2, 8, 10, 64, 15, 19, x=None), up_calls(2, 8, 10, 64, 15, 19, out=None)]
    for calls in cases:
        for name, args in calls:
            refused(name, *args, msg=name[len("dirb200_"):])


def copy_args(src_stride=64, src_off=16, dst_stride=128, dst_off=32, c=16, pixels=100, src=D, dst=D):
    return (src, src_stride, src_off, dst, dst_stride, dst_off, c, pixels, None)


@pytest.mark.parametrize("kw", [
    dict(c=0), dict(c=-8), dict(c=12),
    dict(src_stride=60), dict(dst_stride=100),                # strides not multiples of 8
    dict(src_off=4), dict(dst_off=12),                        # offsets not multiples of 8
    dict(src_off=56), dict(dst_off=120),                      # range past the row
    dict(src_stride=8, src_off=0),                            # row narrower than the copy
    dict(src_off=-8), dict(dst_off=-16),                      # negative offsets (were accepted)
    dict(src_off=-64, src_stride=0, c=64),
    dict(pixels=-1),
    dict(src=None), dict(dst=None),
], ids=lambda kw: "-".join(f"{k}={v}" for k, v in kw.items()))
def test_copy_channels_refuses_bad_arguments(kw):
    refused("dirb200_copy_channels", *copy_args(**kw), msg="copy_channels")


def test_avgpool_refuses_bad_arguments():
    for name, p0 in (("dirb200_avgpool_fwd", D), ("dirb200_avgpool_bwd", D)):
        for c in BAD_C:
            refused(name, p0, 4, 49, c, D, None, msg="avgpool")
        for n, hw in ((0, 49), (-1, 49), (4, 0), (4, -1)):
            refused(name, p0, n, hw, 64, D, None, msg="avgpool")
        refused(name, None, 4, 49, 64, D, None, msg="avgpool")
        refused(name, p0, 4, 49, 64, None, None, msg="avgpool")


BIG_ROWS = (2 ** 31, 2 ** 32 + 1)        # rows past a 32-bit grid size / loop bound (were narrowed silently)


def test_linear1_refuses_bad_arguments():
    for n, d in ((0, 2048), (-1, 2048), (4, 0), (4, -1)) + tuple((n, 1) for n in BIG_ROWS):
        refused("dirb200_linear1_fwd", D, D, D, n, d, D, None, msg="linear1_fwd")
        refused("dirb200_linear1_bwd", D, D, D, n, d, D, D, D, None, msg="linear1_bwd")
        refused("dirb200_linear1_bwd", D, D, D, n, d, None, D, D, None, msg="linear1_bwd")
    for k in range(4):                                         # x, w, bias, pred
        a = [D, D, D, 4, 2048, D, None]
        a[(0, 1, 2, 5)[k]] = None
        refused("dirb200_linear1_fwd", *a, msg="linear1_fwd")
    for k in (0, 1, 2, 6, 7):                                  # grad_pred, x, w, dw, dbias (dx may be NULL)
        a = [D, D, D, 4, 2048, D, D, D, None]
        a[k] = None
        refused("dirb200_linear1_bwd", *a, msg="linear1_bwd")


def adam_args(p=D, g=D, m=D, v=D, n=4099, step=1):
    return (p, g, m, v, n, 1e-3, 0.9, 0.999, 1e-8, 0.0, step, 1.0, None, None)


def test_adam_refuses_bad_arguments():
    for kw in (dict(p=None), dict(g=None), dict(m=None), dict(v=None), dict(n=0), dict(n=-1), dict(step=0),
               dict(step=-1)):
        refused("dirb200_adam_step", *adam_args(**kw), msg="bad arguments")
    for k in ("p", "g", "m", "v"):                             # float4 accesses: 16-byte aligned buffers
        refused("dirb200_adam_step", *adam_args(**{k: D8}), msg="16-byte aligned")


def test_sgd_refuses_bad_arguments():
    base = [D, D, D, 4099, 0.05, 0.9, 1e-4, 1, 1.0, None, None]
    for k, v in ((0, None), (1, None), (3, 0), (3, -1), (2, None)):     # ... and momentum != 0 without a buffer
        a = list(base)
        a[k] = v
        refused("dirb200_sgd_step", *a, msg="sgd_step")


def test_grad_clip_refuses_bad_arguments():
    L = lib()
    need = L.raw("dirb200_grad_clip_workspace_bytes")()
    assert need >= 8 * 1024 + 16
    base = [D, 4099, 1.0, 1.0, D, need, D, None]
    for k, v in ((0, None), (4, None), (6, None), (1, 0), (1, -1), (3, 0.0), (3, -1.0)):
        a = list(base)
        a[k] = v
        refused("dirb200_grad_clip_coef", *a, msg="bad arguments")
    a = list(base)
    a[0] = D8
    refused("dirb200_grad_clip_coef", *a, msg="16-byte aligned")
    a = list(base)
    a[5] = need - 1
    refused("dirb200_grad_clip_coef", *a, msg="workspace too small", rc=-3)
