"""ctypes signatures of the convolution-stack entry points (include/dirb200.h)."""
from ctypes import c_float, c_int, c_int64, c_size_t, c_void_p

import _lib

P = c_void_p
_I9 = [c_int] * 9

_lib.register({
    "dirb200_conv_prep_weights": (c_int, [P, c_int, c_int, c_int, c_int, c_int, P, P, P]),
    "dirb200_input_to_s2d": (c_int, [P, c_int, c_int, c_int, P, P]),
    "dirb200_conv_fprop": (c_int, [P, P, P] + _I9 + [c_int, P]),
    "dirb200_conv_dgrad": (c_int, [P, P, P] + _I9 + [P]),
    "dirb200_conv_wgrad_workspace_bytes": (c_size_t, _I9 + [c_int]),
    "dirb200_conv_wgrad": (c_int, [P, P, P, P, c_size_t] + _I9 + [c_int, c_int, P]),
    "dirb200_conv_plan": (c_int, _I9 + [c_int, c_int, P]),
    "dirb200_bn_eval_coeffs": (c_int, [c_int, P, P, c_float, P, P, P, P, P]),
    # test aids: the fused BatchNorm epilogues and their consumers
    "dirb200_conv_fprop_bn_stats": (c_int, [P, P, P] + _I9 + [c_int, P, P, P]),
    "dirb200_conv_fprop_affine": (c_int, [P, P, P] + _I9 + [P, P, P, c_int, P]),
    "dirb200_conv_dgrad_bn_moments": (c_int, [P, P, P] + _I9 + [P, P, P, P, P, P]),
    "dirb200_bn_finalize_layout": (c_int, [P, P, c_int64, c_int, P, P, c_float, c_float, P, P, P, P, P, P, P]),
    "dirb200_bn_bwd_coeffs_layout": (c_int, [P, P, c_int64, c_int, P, P, P, P, P, P, P]),
})
