"""CPU-only: the BatchNorm entry points and the layer-kernel test aids (include/dirb200.h, "Test aids: BatchNorm /
pooling layer kernels") refuse unsupported arguments on the host, with rc -1 and a message, before any CUDA call.  Every
pointer below is a dummy that must never be dereferenced, so a call that got past its checks would fault on a GPU
machine and fail without one.

c = 0 used to divide by c / 8 = 0 in the channel check (SIGFPE), c = -8 passed that check, and c = 24 (three channel
groups, which do not divide the 256 threads of a CTA) is refused by the kernels' dispatch."""
import ctypes

import pytest

D = ctypes.c_void_p(16)               # stands for a device buffer
BAD_C = (0, -8, 24)


def lib():
    import _lib
    return _lib


def refused(name, *args, msg):
    L = lib()
    rc = L.raw(name)(*args)
    err = L.last_error()
    assert rc == -1 and msg in err, (name, args, rc, err)


def nblk():
    return ctypes.byref(ctypes.c_int(-1))


# one call per entry point with (rows, c) substituted; every other argument is valid for rows = 64, c = 64
def bn_calls(rows, c):
    return [
        ("dirb200_bn_train_fwd", (D, rows, c, D, D, 1e-5, 0.1, D, D, 1, D, D, D, D, D, None)),
        ("dirb200_bn_train_fwd", (D, rows, c, D, D, 1e-5, 0.1, None, None, 0, D, D, D, D, D, None)),
        ("dirb200_bn_train_bwd", (D, D, rows, c, D, D, D, D, 1, D, D, D, D, None)),
        ("dirb200_bn_train_bwd", (D, D, rows, c, D, D, D, None, 0, D, D, D, D, None)),
        ("dirb200_layer_bn_stats", (D, rows, c, D, nblk(), None)),
        ("dirb200_layer_bn_apply", (D, D, D, None, None, None, None, 1, rows, c, D, None, None)),
        ("dirb200_layer_bn_apply", (D, D, D, D, None, None, None, 1, rows, c, D, D, None)),
        ("dirb200_layer_bn_bwd_reduce", (D, None, None, D, None, D, D, None, rows, c, 0, 0, None, D, nblk(), None)),
        ("dirb200_layer_bn_bwd_reduce", (D, D, D, D, None, None, None, D, rows, c, 0, 0, D, D, nblk(), None)),
        ("dirb200_layer_bn_bwd_coeffs", (D, 4, 2, 1, rows, c, D, D, D, D, D, D, None)),
        ("dirb200_layer_bn_bwd_apply", (D, None, D, D, None, None, D, D, None, rows, c, 0, 0, D, None, None, None)),
        ("dirb200_layer_bn_bwd_apply", (D, D, D, D, D, D, None, None, D, rows, c, 0, 0, D, D, None, None)),
    ]


@pytest.mark.parametrize("c", BAD_C)
def test_bn_entry_points_refuse_unsupported_channel_counts(c):
    for name, args in bn_calls(64, c):
        refused(name, *args, msg="channel count")


@pytest.mark.parametrize("rows", (0, -1))
def test_bn_entry_points_refuse_empty_row_counts(rows):
    for name, args in bn_calls(rows, 64):
        refused(name, *args, msg="rows")


def test_pool_aids_refuse_bad_channel_counts_and_sizes():
    """The pool kernels take any positive multiple of 8 channels (one thread per pixel block and channel group)."""
    for c in (0, -8, 12):
        refused("dirb200_layer_bn_relu_maxpool_fwd", D, D, D, 2, 8, 8, c, D, D, None, msg="channel count")
        refused("dirb200_layer_maxpool_bwd", D, None, D, 2, 8, 8, c, D, None, msg="channel count")
    refused("dirb200_layer_bn_relu_maxpool_fwd", D, D, D, 0, 8, 8, 64, D, D, None, msg="map size")
    refused("dirb200_layer_bn_relu_maxpool_fwd", D, D, D, 2, 8, -2, 64, D, D, None, msg="map size")
    refused("dirb200_layer_maxpool_bwd", D, D, D, 2, 0, 8, 64, D, None, msg="map size")
    # the backward needs an even map (a thread owns a 2x2 input block)
    refused("dirb200_layer_maxpool_bwd", D, D, D, 2, 9, 8, 64, D, None, msg="even")
    refused("dirb200_layer_maxpool_bwd", D, None, D, 2, 8, 7, 64, D, None, msg="even")
    refused("dirb200_layer_bn_relu_maxpool_fwd", D, None, D, 2, 8, 8, 64, D, D, None, msg="null")
    refused("dirb200_layer_maxpool_bwd", D, D, None, 2, 8, 8, 64, D, None, msg="null")


def test_layer_aids_refuse_invalid_operand_combinations():
    rows, c = 2 * 8 * 8, 64
    # a third gradient only in the two-gradient identity forms (with g2 and dz_out)
    refused("dirb200_layer_bn_bwd_reduce", D, None, D, D, None, None, None, D, rows, c, 0, 0, D, D, nblk(), None,
            msg="third gradient")
    refused("dirb200_layer_bn_bwd_reduce", D, D, D, D, None, None, None, D, rows, c, 0, 0, None, D, nblk(), None,
            msg="third gradient")
    # compact second gradient: odd map sides, one side only, maps that do not tile the rows, together with y2
    for h2, w2, r in ((9, 8, 2 * 9 * 8), (8, 9, 2 * 8 * 9), (8, 0, rows), (0, 8, rows), (-8, 8, rows), (8, 8, rows + 32)):
        refused("dirb200_layer_bn_bwd_reduce", D, D, None, D, None, None, None, D, r, c, h2, w2, D, D, nblk(), None,
                msg="compact")
        refused("dirb200_layer_bn_bwd_apply", D, D, D, D, None, None, None, None, D, r, c, h2, w2, D, None, D, None,
                msg="compact")
    refused("dirb200_layer_bn_bwd_reduce", D, D, None, D, D, None, None, D, rows, c, 8, 8, None, D, nblk(), None,
            msg="compact")
    refused("dirb200_layer_bn_bwd_apply", D, D, D, D, D, D, None, None, D, rows, c, 8, 8, D, D, None, None,
            msg="compact")
    # the compact form of the apply pass also stores dz
    refused("dirb200_layer_bn_bwd_apply", D, D, D, D, None, None, None, None, D, rows, c, 8, 8, D, None, None, None,
            msg="compact")
    # mask-from-y / no-ReLU forms take one gradient and one BN; dz_out is stored in mask forms only, never with y2
    refused("dirb200_layer_bn_bwd_reduce", D, D, None, D, None, D, D, None, rows, c, 0, 0, None, D, nblk(), None,
            msg="one gradient")
    refused("dirb200_layer_bn_bwd_reduce", D, None, None, D, None, D, None, None, rows, c, 0, 0, None, D, nblk(), None,
            msg="one gradient")
    refused("dirb200_layer_bn_bwd_reduce", D, None, None, D, D, None, None, D, rows, c, 0, 0, D, D, nblk(), None,
            msg="identity blocks")
    refused("dirb200_layer_bn_bwd_apply", D, None, D, D, None, None, D, D, None, rows, c, 0, 0, D, None, D, None,
            msg="one gradient")
    refused("dirb200_layer_bn_bwd_apply", D, None, D, D, D, D, None, None, D, rows, c, 0, 0, D, D, D, None,
            msg="either a downsample branch")
    refused("dirb200_layer_bn_bwd_apply", D, None, D, D, D, None, None, None, D, rows, c, 0, 0, D, D, None, None,
            msg="coef2")
    # bn_apply: one shortcut operand; the downsample branch needs its coefficients
    refused("dirb200_layer_bn_apply", D, D, D, D, D, D, D, 1, rows, c, D, D, None, msg="one shortcut operand")
    refused("dirb200_layer_bn_apply", D, D, D, None, D, None, D, 1, rows, c, D, D, None, msg="res_scale")
    # the mask bits mean "> 0" only behind the ReLU
    refused("dirb200_layer_bn_apply", D, D, D, D, None, None, None, 0, rows, c, D, D, None, msg="needs relu")
    refused("dirb200_layer_bn_apply", D, D, D, None, None, None, None, 0, rows, c, D, D, None, msg="needs relu")
    # coefficients: K = 2 or 3, dgamma from slot 1 .. K-1, at least one partial row
    for nb, k, gslot in ((4, 4, 1), (4, 1, 1), (4, 2, 0), (4, 2, 2), (4, 3, 3), (0, 2, 1)):
        refused("dirb200_layer_bn_bwd_coeffs", D, nb, k, gslot, rows, c, D, D, D, D, D, D, None, msg="layer_bn_bwd_coeffs")
    # null pointers
    refused("dirb200_layer_bn_stats", None, rows, c, D, nblk(), None, msg="null")
    refused("dirb200_layer_bn_stats", D, rows, c, D, None, None, msg="null")
    refused("dirb200_layer_bn_apply", D, None, D, None, None, None, None, 1, rows, c, D, None, None, msg="null")
    refused("dirb200_layer_bn_bwd_reduce", D, None, None, D, None, D, D, None, rows, c, 0, 0, None, None, nblk(), None,
            msg="null")
    refused("dirb200_layer_bn_bwd_coeffs", D, 4, 2, 1, rows, c, D, D, D, None, D, D, None, msg="null")
    refused("dirb200_layer_bn_bwd_apply", D, None, D, None, None, None, D, D, None, rows, c, 0, 0, D, None, None, None,
            msg="null")
