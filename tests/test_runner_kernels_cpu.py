"""CPU-only: the test aids of the ResNet runner's batched kernels (include/dirb200.h, "Test aids: the runner's batched
kernels") and dirb200_resnet_peek_conv refuse bad arguments on the host, with rc -1 and a message, before any CUDA
call.  Every pointer below is a dummy that must never be dereferenced, so a call that got past its checks would fault
on a GPU machine and fail without one."""
import ctypes

import pytest

D = ctypes.c_void_p(16)               # stands for a device buffer
DF = ctypes.cast(D, ctypes.POINTER(ctypes.c_float))
NULLF = ctypes.POINTER(ctypes.c_float)()


class PrepJob(ctypes.Structure):
    _fields_ = [("w_off", ctypes.c_int64), ("cout", ctypes.c_int), ("cin", ctypes.c_int), ("kh", ctypes.c_int),
                ("kw", ctypes.c_int), ("stem", ctypes.c_int), ("w_fprop", ctypes.c_void_p), ("w_dgrad", ctypes.c_void_p)]


class ReduceJob(ctypes.Structure):
    _fields_ = [("partial", ctypes.c_void_p), ("w_off", ctypes.c_int64), ("splits", ctypes.c_int), ("cout", ctypes.c_int),
                ("cin", ctypes.c_int), ("kh", ctypes.c_int), ("kw", ctypes.c_int), ("stem", ctypes.c_int)]


class BnJob(ctypes.Structure):
    _fields_ = [("c", ctypes.c_int), ("gamma_off", ctypes.c_int64), ("beta_off", ctypes.c_int64),
                ("rm_off", ctypes.c_int64), ("rv_off", ctypes.c_int64), ("scale", ctypes.c_void_p),
                ("shift", ctypes.c_void_p)]


class ConvPeek(ctypes.Structure):
    _fields_ = [("w_fprop", ctypes.c_void_p), ("w_dgrad", ctypes.c_void_p), ("partial", ctypes.c_void_p),
                ("scale", ctypes.c_void_p), ("shift", ctypes.c_void_p), ("w_off", ctypes.c_int64)] + \
               [(k, ctypes.c_int) for k in ("cout", "cin", "kh", "kw", "stride", "pad", "stem", "splits")]


def lib():
    import _lib
    return _lib


def refused(name, *args, msg):
    L = lib()
    rc = L.raw(name)(*args)
    err = L.last_error()
    assert rc == -1 and msg in err, (name, args, rc, err)


def arr(cls, *jobs):
    return (cls * len(jobs))(*jobs)


GOOD_PREP = dict(w_off=0, cout=64, cin=64, kh=3, kw=3, stem=0, w_fprop=16, w_dgrad=16)
GOOD_REDUCE = dict(partial=16, w_off=0, splits=3, cout=64, cin=64, kh=3, kw=3, stem=0)
GOOD_BN = dict(c=64, gamma_off=0, beta_off=64, rm_off=0, rv_off=64, scale=16, shift=16)


def prep(**kw):
    return PrepJob(**{**GOOD_PREP, **kw})


def red(**kw):
    return ReduceJob(**{**GOOD_REDUCE, **kw})


def bn(**kw):
    return BnJob(**{**GOOD_BN, **kw})


def test_job_layouts_match_the_header():
    """The ctypes mirrors used here and in the GPU tests have the C structs' sizes (natural alignment, LP64)."""
    assert ctypes.sizeof(PrepJob) == 48
    assert ctypes.sizeof(ReduceJob) == 40
    assert ctypes.sizeof(BnJob) == 56
    assert ctypes.sizeof(ConvPeek) == 80


# (field overrides, message) refused by both conv-job aids
BAD_SHAPES = [
    (dict(cout=0), "non-positive"), (dict(cin=-64), "non-positive"), (dict(kh=0), "non-positive"),
    (dict(kw=-1), "non-positive"),
    (dict(stem=1, cin=3, kh=7, kw=5), "3x7x7"), (dict(stem=1, cin=4, kh=7, kw=7), "3x7x7"),
    (dict(stem=1, cin=3, kh=3, kw=3), "3x7x7"),
    (dict(cout=1 << 16, cin=1 << 15, kh=1, kw=1), "2^31"),                # exactly 2^31 weights
    (dict(cout=65536, cin=4096, kh=3, kw=3), "2^31"),
    (dict(cout=1 << 23, cin=3, kh=7, kw=7, stem=1), "2^31"),              # the stem's 256-wide operand overflows
    (dict(w_off=-1), "negative w_off"),
]


@pytest.mark.parametrize("bad,msg", BAD_SHAPES, ids=[f"{i}" for i in range(len(BAD_SHAPES))])
def test_conv_job_aids_refuse_bad_jobs(bad, msg):
    # the bad job is the second of three: every job is checked before the first CUDA call
    stem_ok = dict(w_dgrad=None) if bad.get("stem") else {}
    refused("dirb200_prep_weights_all", DF, arr(PrepJob, prep(), prep(**bad, **stem_ok), prep()), 3, None, msg=msg)
    refused("dirb200_wgrad_reduce_all", arr(ReduceJob, red(), red(**bad), red()), 3, DF, None, msg=msg)


def test_conv_job_aids_accept_the_largest_filter_below_2_31():
    """2^31 - 1 weights is within FastDiv's range: the shape check passes, so a null pointer in a LATER job is what is
    refused (no CUDA call is reached)."""
    big = dict(cout=(1 << 31) - 1, cin=1, kh=1, kw=1)
    refused("dirb200_prep_weights_all", DF, arr(PrepJob, prep(**big), prep(w_fprop=None)), 2, None, msg="null w_fprop")
    refused("dirb200_wgrad_reduce_all", arr(ReduceJob, red(**big), red(partial=None)), 2, DF, None, msg="null partial")


def test_prep_weights_all_refuses_bad_arguments():
    jobs = arr(PrepJob, prep())
    refused("dirb200_prep_weights_all", NULLF, jobs, 1, None, msg="null")
    refused("dirb200_prep_weights_all", DF, None, 1, None, msg="null")
    refused("dirb200_prep_weights_all", DF, arr(PrepJob, prep(), prep(w_fprop=None)), 2, None, msg="null w_fprop")
    for n in (0, -1, 65536):
        refused("dirb200_prep_weights_all", DF, jobs, n, None, msg="njobs")
    # the stem has no dgrad operand
    refused("dirb200_prep_weights_all", DF, arr(PrepJob, prep(stem=1, cin=3, kh=7, kw=7)), 1, None, msg="w_dgrad")


def test_wgrad_reduce_all_refuses_bad_arguments():
    jobs = arr(ReduceJob, red())
    refused("dirb200_wgrad_reduce_all", None, 1, DF, None, msg="null")
    refused("dirb200_wgrad_reduce_all", jobs, 1, NULLF, None, msg="null")
    refused("dirb200_wgrad_reduce_all", arr(ReduceJob, red(), red(partial=None)), 2, DF, None, msg="null partial")
    for n in (0, -3, 65536):
        refused("dirb200_wgrad_reduce_all", jobs, n, DF, None, msg="njobs")
    for s in (0, -1):
        refused("dirb200_wgrad_reduce_all", arr(ReduceJob, red(), red(splits=s)), 2, DF, None, msg="splits")
        refused("dirb200_wgrad_reduce_all", arr(ReduceJob, red(stem=1, cin=3, kh=7, kw=7, splits=s)), 1, DF, None,
                msg="splits")


def test_bn_eval_coeffs_all_refuses_bad_arguments():
    jobs = arr(BnJob, bn())
    f = "dirb200_bn_eval_coeffs_all"
    refused(f, None, 1, DF, DF, 1e-5, None, msg="null")
    refused(f, jobs, 1, NULLF, DF, 1e-5, None, msg="null")
    refused(f, jobs, 1, DF, NULLF, 1e-5, None, msg="null")
    refused(f, arr(BnJob, bn(), bn(scale=None)), 2, DF, DF, 1e-5, None, msg="null scale")
    refused(f, arr(BnJob, bn(), bn(shift=None)), 2, DF, DF, 1e-5, None, msg="null scale")
    for n in (0, -1, 65536):
        refused(f, jobs, n, DF, DF, 1e-5, None, msg="njobs")
    for c in (0, -64):
        refused(f, arr(BnJob, bn(), bn(c=c)), 2, DF, DF, 1e-5, None, msg="channel count")
    for k in ("gamma_off", "beta_off", "rm_off", "rv_off"):
        refused(f, arr(BnJob, bn(**{k: -1})), 1, DF, DF, 1e-5, None, msg="negative offset")


def test_peek_conv_refuses_a_null_net_or_output():
    import resnet  # noqa: F401  (registers the runner bindings)
    out = ConvPeek()
    for block, conv in ((-1, 0), (0, 0), (0, 3)):
        refused("dirb200_resnet_peek_conv", None, block, conv, ctypes.byref(out), msg="null")
    refused("dirb200_resnet_peek_conv", D, 0, 0, None, msg="null")


def test_peek_bn_stats_refuses_a_null_net_or_output():
    import resnet  # noqa: F401  (registers the runner bindings)
    p = ctypes.c_void_p()
    for block, conv in ((-1, 0), (0, 0), (0, 3)):
        refused("dirb200_resnet_peek_bn_stats", None, block, conv, ctypes.byref(p), ctypes.byref(p), msg="null")
        refused("dirb200_resnet_peek_bn_stats", D, block, conv, None, ctypes.byref(p), msg="null")
        refused("dirb200_resnet_peek_bn_stats", D, block, conv, ctypes.byref(p), None, msg="null")


def test_peek_refuses_bad_selectors_before_reading_the_net():
    """dirb200_resnet_peek checks its selector before it reads the net (the null net here would otherwise be
    refused as a null pointer): 0 .. 7 for a block, 0, 1, 6 and 7 for the stem."""
    import resnet  # noqa: F401  (registers the runner bindings)
    ptr, rows, ch = ctypes.c_void_p(), ctypes.c_int64(), ctypes.c_int()
    out = (ctypes.byref(ptr), ctypes.byref(rows), ctypes.byref(ch))
    for block, which in ((0, 8), (0, -1), (-1, 8), (3, 100), (-1, -2)):
        refused("dirb200_resnet_peek", None, block, which, *out, msg=f"bad selector {which}")
    for which in (2, 3, 4, 5):
        refused("dirb200_resnet_peek", None, -1, which, *out, msg="for the stem")
    for block, which in ((-1, 0), (-1, 7), (0, 6), (0, 7)):
        refused("dirb200_resnet_peek", None, block, which, *out, msg="null")
        refused("dirb200_resnet_peek", D, block, which, None, ctypes.byref(rows), ctypes.byref(ch), msg="null")
