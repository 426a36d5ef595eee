"""ctypes binding of libfpd_b200.so (the C ABI declared in include/fpd_b200.h).

There is deliberately no fallback: if the shared library is missing or a call fails, this raises.
"""
import ctypes
import os
from ctypes import c_char_p, c_float, c_int, c_int64, c_size_t, c_void_p, POINTER

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfpd_b200.so")


class NativeLibraryMissing(RuntimeError):
    pass


_lib = None

P = c_void_p  # every device / host pointer travels as void*

_SIGNATURES = {
    "fpd_last_error": (c_char_p, []),
    "fpd_version": (c_int, []),
    "fpd_sm_count": (c_int, []),
    "fpd_launch_count": (ctypes.c_longlong, []),
    "fpd_conv2d_tc_ts_supported": (c_int, [c_int, c_int, c_int]),
    "fpd_conv2d_tc_ts": (c_int, [P, P, P, P, c_int, P, P, P, P, P, P, c_float, c_int, c_int, c_int, c_int, c_int,
                                 c_int, P]),
    "fpd_conv2d_tc_h_supported": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "fpd_conv2d_tc_h": (c_int, [P, P, P, P, c_int, P, P, c_int, P, P, P, P, c_float, P, c_int, c_int, c_int, c_int, c_int,
                                c_int, P]),
    "fpd_conv2d_tc_f16x1_kernel": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "fpd_conv2d_tc_f16x1": (c_int, [P, P, P, P, c_int, P, P, P, P, P, c_float, c_int, c_int, c_int, c_int, c_int, c_int,
                                    P]),
    "fpd_conv2d_tc_f16x1_train_plan": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, POINTER(c_int)]),
    "fpd_conv2d_tc_f16x1_train": (c_int, [P, P, P, P, c_int, P, P, P, P, P, c_float, P, c_int, c_int, c_int, c_int, c_int,
                                          c_int, P, P, P]),
    "fpd_conv2d_tc_f16x1_io": (c_int, [P, c_int, P, P, P, c_int, P, P, P, P, c_int, c_float, c_int, c_int, c_int, c_int,
                                       c_int, c_int, P]),
    "fpd_set_conv1x1": (c_int, [c_int]),
    "fpd_set_conv_halo": (c_int, [c_int]),
    "fpd_set_wgrad_halo": (c_int, [c_int]),
    "fpd_conv2d_tc_h_stats_blocks": (c_int, [c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "fpd_conv2d_tc_h_stats": (c_int, [P, P, P, P, c_int, P, P, c_int, P, P, P, c_float, c_int, c_int, c_int, c_int, c_int,
                                      c_int, P, P, P]),
    "fpd_bn_finalize_sums": (c_int, [P, c_int, P, c_int64, c_int, P, P, c_float, c_float, P, P, P, P, P, P, P, P]),
    "fpd_channel_sum_fused": (c_int, [P, c_int64, c_int, c_float, P, P, P, c_size_t, P, P]),
    "fpd_bn_bwd_reduce_fused": (c_int, [P, P, P, P, P, P, c_int, c_int64, c_int, P, P, c_size_t, P, P]),
    "fpd_bn_stats_fused": (c_int, [P, c_int64, c_int, P, P, c_float, c_float, P, P, P, P, P, P, P, P, c_size_t, P, P]),
    "fpd_weight_prep_f16_both": (c_int, [P, P, P, P, P, c_int, c_int, c_int, P]),
    "fpd_weight_prep_f16": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_conv2d_wgrad_tc3_supported": (c_int, [c_int, c_int, c_int, c_int, c_int]),
    "fpd_conv2d_wgrad_tc_supported": (c_int, [c_int, c_int, c_int]),
    "fpd_conv2d_wgrad_tc_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int]),
    "fpd_conv2d_wgrad_tc_fused": (c_int, [P, P, P, P, c_int, P, c_int, P, c_float, c_int, c_int, c_int, c_int, c_int,
                                          c_int, P, c_size_t, P]),
    "fpd_conv2d_simt_fwd": (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_conv2d_simt_dgrad": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_conv2d_simt_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int]),
    "fpd_conv2d_simt_wgrad": (c_int, [P, P, P, c_float, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P,
                                      c_size_t, P]),
    "fpd_weight_prep": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_bn_stats_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "fpd_bn_stats": (c_int, [P, c_int64, c_int, P, P, P, c_size_t, P]),
    "fpd_bn_finalize": (c_int, [P, P, P, P, c_float, c_int64, P, P, P, P, P, c_float, c_int, P]),
    "fpd_affine_act_split": (c_int, [P, P, P, P, c_int, P, P, c_int64, c_int, P]),
    "fpd_affine_act": (c_int, [P, P, P, P, c_int, P, c_int64, c_int, P]),
    "fpd_affine_add_act": (c_int, [P, P, P, P, P, c_int, P, c_int64, c_int, P]),
    "fpd_fuse_sum": (c_int, [POINTER(c_void_p), POINTER(c_int), c_int, c_int, P, c_int, c_int, c_int, c_int, P]),
    "fpd_upsample_bwd": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_im2col": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_channel_reduce_workspace_bytes": (c_size_t, [c_int64, c_int]),
    "fpd_channel_sum": (c_int, [P, c_int64, c_int, c_float, P, P, c_size_t, P]),
    "fpd_bn_bwd_reduce": (c_int, [P, P, P, P, P, P, c_int, c_int64, c_int, P, P, c_size_t, P]),
    "fpd_bn_bwd_apply_sum": (c_int, [P, P, P, P, P, P, P, c_int, P, P, P, P, c_int64, c_int, P, c_size_t, P]),
    "fpd_bn_bwd_apply": (c_int, [P, P, P, P, P, P, P, c_int, P, c_int, P, c_int64, c_int, P]),
    "fpd_affine_act_bwd": (c_int, [P, P, P, P, P, c_int, c_int, P, c_int64, c_int, P]),
    "fpd_maxpool2x2_fwd": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_maxpool2x2_bwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_upsample2x_add": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_upsample2x_bwd": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_maxpool3x3s2_fwd": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_maxpool3x3s2_bwd": (c_int, [P, P, P, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_depth_space2": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_deconv_weight_map": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_subsample2": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_upsample_zero2": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_affine_act_f16": (c_int, [P, P, P, P, c_int, P, c_int64, c_int, P]),
    "fpd_affine_add_act_f16": (c_int, [P, P, P, P, P, c_int, P, c_int64, c_int, P]),
    "fpd_fuse_sum_f16": (c_int, [POINTER(c_void_p), POINTER(c_int), c_int, c_int, P, c_int, c_int, c_int, c_int, P]),
    "fpd_maxpool2x2_fwd_f16": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_upsample2x_add_f16": (c_int, [P, P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_subsample2_f16": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_half_to_float": (c_int, [P, P, c_int64, P]),
    "fpd_nchw_to_nhwc": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_nchw_to_nhwc_flipw": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_nhwc_to_nchw": (c_int, [P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_add": (c_int, [P, P, P, c_int64, P]),
    "fpd_loss_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int]),
    "fpd_loss_fused": (c_int, [POINTER(c_void_p), c_int, P, P, P, c_float, POINTER(c_void_p), c_float, P, c_int, c_int,
                               c_int, c_int, P, c_size_t, P]),
    "fpd_joints_mse": (c_int, [P, P, P, P, P, c_int, c_int, c_int, P, c_size_t, P]),
    "fpd_loss_ohkm_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "fpd_loss_ohkm_fused": (c_int, [POINTER(c_void_p), c_int, P, P, P, c_float, POINTER(c_void_p), c_float, P, c_int,
                                    c_int, c_int, c_int, c_int, c_int, P, c_size_t, P]),
    "fpd_joints_ohkm_workspace_bytes": (c_size_t, [c_int, c_int]),
    "fpd_joints_ohkm": (c_int, [P, P, P, c_int, P, P, c_int, c_int, c_int, P, c_size_t, P]),
    "fpd_loss_kl_workspace_bytes": (c_size_t, [c_int, c_int, c_int, c_int, c_int]),
    "fpd_loss_kl_fused": (c_int, [POINTER(c_void_p), c_int, P, P, P, c_float, POINTER(c_void_p), c_float, P, c_int,
                                  c_int, c_int, c_int, c_int, c_int, c_float, c_float, P, c_size_t, P]),
    "fpd_joints_kld_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "fpd_joints_kld": (c_int, [P, P, P, c_float, P, P, c_int, c_int, c_int, P, c_size_t, P]),
    "fpd_kd_weights": (c_int, [P, P, c_float, P, c_int, c_int, c_int, c_int, P]),
    "fpd_loss_kdw_fused": (c_int, [POINTER(c_void_p), c_int, P, P, P, P, c_float, POINTER(c_void_p), c_float, P, c_int,
                                   c_int, c_int, c_int, c_int, c_int, c_float, c_float, P, c_size_t, P]),
    "fpd_feature_mse_workspace_bytes": (c_size_t, [c_int64]),
    "fpd_feature_mse": (c_int, [P, P, c_int, c_float, P, P, P, c_int64, P, c_size_t, P]),
    "fpd_flip_merge_argmax": (c_int, [P, P, P, c_int, P, P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_argmax_nchw": (c_int, [P, P, P, c_int, c_int, P]),
    "fpd_final_preds": (c_int, [P, P, P, P, c_int, P, c_int, c_int, c_int, c_int, P]),
    "fpd_final_preds_dark": (c_int, [P, P, P, P, c_int, P, c_int, c_int, c_int, c_int, P]),
    "fpd_pck_counts": (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, P]),
    "fpd_heatmap_resample": (c_int, [P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_nms_workspace_bytes": (c_size_t, [c_int]),
    "fpd_nms_device": (c_int, [P, c_int, c_int, c_float, P, P, P, c_size_t, P]),
    "fpd_nms_host": (c_int, [P, P, P, c_int, c_int, c_float, c_int]),
    "fpd_oks_nms_device": (c_int, [P, c_int, P, P, c_int, c_int, ctypes.c_double, c_int, ctypes.c_double, P, P, P, c_size_t,
                                   P]),
    "fpd_oks_rescore": (c_int, [P, c_int, P, c_int, c_int, ctypes.c_double, P, P]),
    "fpd_gaussian_targets": (c_int, [P, P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_gaussian_targets_unbiased": (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_gaussian_targets_udp": (c_int, [P, P, P, P, P, c_int, c_int, c_int, c_int, c_int, c_int, c_int, P]),
    "fpd_crop_affine_normalize": (c_int, [P, c_size_t, P, P, P, P, P, P, c_int, c_int, c_int, P]),
    "fpd_adam_flat": (c_int, [P, P, P, P, c_int64, c_float, c_float, c_float, c_float, c_float, c_int, c_float, P]),
}

EXPORTED_SYMBOLS = tuple(_SIGNATURES)


def lib():
    """Load (once) and return the ctypes handle. Raises NativeLibraryMissing if the .so is not built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise NativeLibraryMissing(
                "libfpd_b200.so not found at %s -- run `python -c 'import __graft_entry__ as g; g.build()'` "
                "(there is no CPU / PyTorch fallback for the H100 kernels)" % LIB_PATH)
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in _SIGNATURES.items():
            fn = getattr(h, name)  # AttributeError here = header/library mismatch: fail loudly
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def last_error():
    return lib().fpd_last_error().decode("utf-8", "replace")


def check(rc, what=""):
    if rc != 0:
        raise RuntimeError("libfpd_b200 %s failed (rc=%d): %s" % (what, rc, last_error()))
