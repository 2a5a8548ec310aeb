"""ctypes binding of libdirb200.so (the C ABI declared in include/dirb200.h).

Product-path plumbing: loads the in-tree shared library and fails loudly when
it is missing or when a call reports an error -- there is no CPU / eager
fallback anywhere in this package.
"""
import ctypes
import os
from ctypes import c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libdirb200.so")

BIN_AGE, BIN_DEPTH10, BIN_EDGES5 = 0, 1, 2
LOSS_KINDS = {"mse": 0, "l1": 1, "focal_mse": 2, "focal_l1": 3, "huber": 4}
ACTIVATE = {"sigmoid": 0, "tanh": 1}
REWEIGHT = {"sqrt_inv": 1, "inverse": 2}
DIRB200_ERR_ARG = -1


class Dirb200Error(RuntimeError):
    pass


def _load():
    if not os.path.exists(LIB_PATH):
        raise Dirb200Error(
            f"{LIB_PATH} not found: build it with `make -C {os.path.join(_HERE, 'csrc')}` "
            "(or __graft_entry__.build()); there is no fallback path")
    return ctypes.CDLL(LIB_PATH)


_lib = _load()
P = c_void_p

_SIGS = {
    "dirb200_last_error": (c_char_p, []),
    "dirb200_version": (c_int, []),
    "dirb200_launch_count": (c_int64, []),
    "dirb200_fds_label_flags": (c_int, [P, c_int64, c_int, c_int, c_int, P, P]),
    "dirb200_fds_bin_rows": (c_int, [P, c_int64, c_int, c_int, c_int, P, P, P]),
    "dirb200_fds_accumulate_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "dirb200_fds_accumulate": (c_int, [P, P, c_int64, c_int, c_int, P, P, P, P, c_size_t, P]),
    "dirb200_fds_set_profiling": (c_int, [c_int]),
    "dirb200_fds_last_accumulate_kernel_ms": (c_int, [P]),
    "dirb200_fds_finalize": (c_int, [P, P, P, c_int, c_int, P, P, P, c_double, c_int, P]),
    "dirb200_fds_smooth_tables": (c_int, [P, c_int, c_int, P, c_int, P, P]),
    "dirb200_fds_calibrate_fwd": (c_int, [P, P, c_int64, c_int, c_int, c_int, c_int, P, P, P, P,
                                          c_float, c_float, P, P, P]),
    "dirb200_fds_calibrate_bwd": (c_int, [c_int, P, P, c_int64, c_int, P, P, c_float, c_float, P, P]),
    "dirb200_fds_fill_empty": (c_int, [P, c_int, c_int, P, P, P]),
    "dirb200_loss_workspace_bytes": (c_size_t, [c_int64]),
    "dirb200_loss_fwd_bwd": (c_int, [c_int, P, P, P, c_int64, c_float, c_float, c_int, c_float, P, P, P,
                                     c_size_t, P]),
    "dirb200_lds_histogram": (c_int, [P, c_int64, c_int, P, P]),
    "dirb200_lds_table_lookup": (c_int, [P, c_int64, c_float, c_int, P, P, P]),
    "dirb200_lds_weights": (c_int, [P, c_int64, c_int, c_int, P, c_int, P, P, P, P]),
    "dirb200_lds_weights_sharded": (c_int, [P, c_int64, c_int64, c_int, c_int, P, c_int, P, P, P, P]),
    "dirb200_int_label_histogram": (c_int, [P, c_int64, c_int, P, P]),
    "dirb200_shot_metrics": (c_int, [P, P, c_int64, P, c_int, c_int, c_int, P, P]),
    "dirb200_stsb_shot_metrics_workspace_bytes": (c_size_t, [c_int64]),
    "dirb200_stsb_shot_metrics": (c_int, [P, P, c_int64, P, c_size_t, P, P]),
    "dirb200_depth_metrics_workspace_bytes": (c_size_t, [c_int64, c_int, c_int]),
    "dirb200_depth_metrics_accumulate": (c_int, [P, c_int, c_int, P, P, c_int64, c_int, c_int, P, c_int, P, P,
                                                 c_size_t, P]),
    "dirb200_bn_workspace_bytes": (c_size_t, [c_int]),
    "dirb200_bn_train_fwd": (c_int, [P, c_int64, c_int, P, P, c_float, c_float, P, P, c_int, P, P, P, P, P, P]),
    "dirb200_bn_train_bwd": (c_int, [P, P, c_int64, c_int, P, P, P, P, c_int, P, P, P, P, P]),
    "dirb200_maxpool3x3s2_fwd": (c_int, [P, c_int, c_int, c_int, c_int, P, P, P]),
    "dirb200_maxpool3x3s2_bwd": (c_int, [P, P, c_int, c_int, c_int, c_int, P, P]),
    "dirb200_avgpool_fwd": (c_int, [P, c_int, c_int, c_int, P, P]),
    "dirb200_avgpool_bwd": (c_int, [P, c_int, c_int, c_int, P, P]),
    # test aids: the BatchNorm / pooling layer kernels one launch at a time
    "dirb200_layer_bn_stats": (c_int, [P, c_int64, c_int, P, P, P]),
    "dirb200_layer_bn_apply": (c_int, [P, P, P, P, P, P, P, c_int, c_int64, c_int, P, P, P]),
    "dirb200_layer_bn_bwd_reduce": (c_int, [P, P, P, P, P, P, P, P, c_int64, c_int, c_int, c_int, P, P, P, P]),
    "dirb200_layer_bn_bwd_coeffs": (c_int, [P, c_int, c_int, c_int, c_int64, c_int, P, P, P, P, P, P, P]),
    "dirb200_layer_bn_bwd_apply": (c_int, [P, P, P, P, P, P, P, P, P, c_int64, c_int, c_int, c_int, P, P, P, P]),
    "dirb200_layer_bn_relu_maxpool_fwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P, P, P]),
    "dirb200_layer_maxpool_bwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P, P]),
    # test aids: the runner's batched weight re-layout, split-K reduction and eval-BatchNorm kernels
    "dirb200_prep_weights_all": (c_int, [P, P, c_int, P]),
    "dirb200_wgrad_reduce_all": (c_int, [P, c_int, P, P]),
    "dirb200_bn_eval_coeffs_all": (c_int, [P, c_int, P, P, c_float, P]),
    "dirb200_upsample_bilinear_fwd": (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_int, P, P]),
    "dirb200_upsample_bilinear_bwd": (c_int, [P, c_int, c_int, c_int, c_int, c_int, c_int, P, P]),
    "dirb200_copy_channels": (c_int, [P, c_int, c_int, P, c_int, c_int, c_int, c_int64, P]),
    "dirb200_depth_head_fwd": (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, P]),
    "dirb200_depth_head_dgrad": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    "dirb200_depth_head_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "dirb200_depth_head_wgrad": (c_int, [P, P, P, P, P, c_size_t, c_int, c_int, c_int, c_int, P]),
    "dirb200_augment_batch": (c_int, [P, P, P, c_int, c_int, c_int, c_float, c_float, P, P]),
    "dirb200_depth_augment_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "dirb200_depth_augment_batch": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P, P, P, P,
                                            P, P, P, c_int, P, P, P, P, P, P, c_size_t, P]),
    # STS-B-DIR sentence-pair encoder (csrc/lstm.cu, csrc/pair_encoder.cu)
    "dirb200_lstm_prep_weights": (c_int, [P] * 8 + [c_int] * 5 + [P] * 6),
    "dirb200_lstm_scatter_grads": (c_int, [P] * 3 + [c_int] * 5 + [P] * 9),
    "dirb200_lstm_fwd_step": (c_int, [P, P, P, P] + [c_int] * 5 + [P] * 5),
    "dirb200_lstm_layer_fwd": (c_int, [P, P, P, P] + [c_int] * 4 + [P] * 5),
    "dirb200_lstm_bwd_step": (c_int, [P] * 5 + [c_int] * 4 + [P] * 4),
    "dirb200_lstm_layer_bwd": (c_int, [P] * 5 + [c_int] * 3 + [P] * 4),
    "dirb200_col_sum_bf16": (c_int, [P, c_int64, c_int, P, P]),
    "dirb200_embed_gather": (c_int, [P, P, P, P, c_int64, c_int, c_int, c_int, c_int, P, P]),
    "dirb200_embed_grad": (c_int, [P, P, P, P, c_int64, c_int, c_int, c_int, c_int, c_int64, P, P]),
    "dirb200_pair_maxpool_fwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P, P, P]),
    "dirb200_pair_maxpool_bwd": (c_int, [P, P, P, P, c_int, c_int, c_int, c_int, P, P]),
    "dirb200_stsb_gather_batch": (c_int, [P, P, P, P, c_int64, c_int, P, c_int64, c_int, c_int, P, P, P, P, P]),
    # JPEG decode + Pillow bilinear resize (csrc/jpeg.cu); the parse and the two size queries are host-only
    "dirb200_jpeg_desc_bytes": (c_size_t, []),
    "dirb200_jpeg_parse": (c_int, [P, c_int64, P, P, c_int64]),
    "dirb200_jpeg_decode_workspace_bytes": (c_size_t, [P, c_int]),
    "dirb200_jpeg_decode": (c_int, [P, P, P, P, c_int, P, P, P, P, c_size_t, P]),
    "dirb200_resize_bilinear_workspace_bytes": (c_size_t, [P, c_int, c_int, c_int]),
    "dirb200_resize_bilinear_u8": (c_int, [P, P, P, c_int, c_int, c_int, P, P, c_size_t, P]),
}


def _bind(sigs):
    for name, (res, args) in sigs.items():
        fn = getattr(_lib, name)     # AttributeError here == header/library mismatch: fail loudly
        fn.restype = res
        fn.argtypes = args


_bind(_SIGS)


def exported_symbols():
    return sorted(_SIGS)


def register(sigs):
    """Used by sibling modules (conv stack) to bind further entry points."""
    _SIGS.update(sigs)
    _bind(sigs)


def last_error() -> str:
    return (_lib.dirb200_last_error() or b"").decode()


def call(name, *args):
    rc = getattr(_lib, name)(*args)
    if rc != 0:
        raise Dirb200Error(f"{name} failed (rc={rc}): {last_error()}")


def raw(name):
    return getattr(_lib, name)


def launch_count() -> int:
    return int(_lib.dirb200_launch_count())


def ptr(t):
    """Device pointer of a torch tensor (None -> NULL)."""
    return None if t is None else c_void_p(t.data_ptr())


def stream_ptr():
    import torch
    return c_void_p(torch.cuda.current_stream().cuda_stream)


def require_cuda(*tensors):
    for t in tensors:
        if t is not None and not t.is_cuda:
            raise Dirb200Error("dirb200 kernels need CUDA tensors; there is no CPU path")
