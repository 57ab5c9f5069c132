"""ctypes binding of libfsb200.so (C ABI in include/fsb200.h).

The product path has NO fallback: if the shared library is missing or a call fails, an exception is
raised (never a silent PyTorch/CPU substitute)."""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfsb200.so")

FSB_CONV_RELU = 1
FSB_CONV_AFFINE = 2
FSB_CONV_FORCE_DIRECT = 4
FSB_CONV_STATS = 8
FSB_CONV_OUT_F32 = 16
FSB_ACT_IN_F32 = 32
FSB_CONV_X_DOWN2 = 64
FSB_CONV_Y_UP2 = 128
ABI_VERSION = 2
FSB_ERR_UNSUPPORTED = -3


class FsbError(RuntimeError):
    pass


class ConvDesc(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("N", "H", "W", "Cin", "Cout", "ksize", "stride", "pad", "dil", "off_h", "off_w",
                                         "Ho", "Wo", "x_cstride", "y_cstride")] + [("flags", C.c_uint32), ("stats_C", C.c_int32),
                                                                                    ("stats_off", C.c_int32)]


class BnSel(C.Structure):
    """fsb_bn_sel: one BatchNorm parameter set of a slimmable unit, selected on the device by a width index"""
    _fields_ = [("gamma", C.c_void_p), ("beta", C.c_void_p), ("running_mean", C.c_void_p), ("running_var", C.c_void_p),
                ("num_batches_tracked", C.c_void_p), ("dgamma", C.c_void_p), ("dbeta", C.c_void_p), ("C", C.c_int32),
                ("reserved", C.c_int32)]


class TrainPreDesc(C.Structure):
    """fsb_train_pre_desc: batch geometry of the training augmentation"""
    _fields_ = [(n, C.c_int32) for n in ("n", "crop_h", "crop_w", "label_h", "label_w")]


_P = C.c_void_p
_SIGS = {
    "fsb_abi_version": (C.c_int, []),
    "fsb_last_error_string": (C.c_char_p, []),
    "fsb_device_info": (C.c_int, [C.POINTER(C.c_int)] * 3),
    "fsb_set_pdl": (C.c_int, [C.c_int]),
    "fsb_set_option": (C.c_int, [C.c_char_p, C.c_int]),
    "fsb_get_option": (C.c_int, [C.c_char_p]),
    "fsb_conv_kernel_id": (C.c_int, [C.POINTER(ConvDesc), _P, C.c_int]),
    "fsb_conv_stats_rows": (C.c_int, [C.POINTER(ConvDesc)]),
    "fsb_conv_residency": (C.c_int, [C.POINTER(ConvDesc)]),
    "fsb_stat_rows": (C.c_int, [C.c_int64]),
    "fsb_wsum_rows": (C.c_int, [C.c_int64, C.c_int]),
    "fsb_rowsum": (C.c_int, [C.c_int, _P, C.c_int, C.c_int, _P, _P]),
    "fsb_debug_set_buffer": (C.c_int, [_P]),
    "fsb_conv_packed_bytes": (C.c_size_t, [C.POINTER(ConvDesc)]),
    "fsb_pack_conv_weight": (C.c_int, [C.POINTER(ConvDesc), _P, C.c_int64, C.c_int64, _P, _P]),
    "fsb_bn_fold": (C.c_int, [C.c_int, _P, _P, _P, _P, C.c_float, _P, _P, _P, _P]),
    "fsb_conv_fwd": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, _P]),
    "fsb_conv_fwd_half": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P, _P, _P, _P, C.c_int, _P]),
    "fsb_stem_conv_nchw": (C.c_int, [C.c_int] * 4 + [_P, C.c_int, _P, _P, _P, _P, C.c_int, C.c_uint32, _P]),
    "fsb_stem_conv_u8hwc": (C.c_int, [C.c_int] * 4 + [_P, _P, _P, _P, _P, _P, C.c_int, C.c_uint32, _P]),
    "fsb_stem_fused": (C.c_int, [C.c_int] * 4 + [_P, _P, C.c_int, _P, _P, _P, C.c_int, _P, _P, _P, _P, C.c_int, _P]),
    "fsb_confusion_matrix": (C.c_int, [C.c_int64, _P, _P, C.c_int, C.c_int, _P, _P]),
    "fsb_bilinear_fwd": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, C.c_uint32, _P]),
    "fsb_bilinear_fwd_half": (C.c_int, [C.c_int] * 4 + [_P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_uint32, _P]),
    "fsb_upsample_logits_nchw": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P]),
    "fsb_upsample_argmax": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, _P]),
    "fsb_upsample_argmax_confusion": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P, _P]),
    "fsb_upsample_argmax_map": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, _P, _P, _P, _P, _P]),
    "fsb_nearest_fwd": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P]),
    "fsb_upsample_logits_nearest_nchw": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P]),
    "fsb_upsample_argmax_nearest": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, _P]),
    "fsb_nchw_to_nhwc_f16": (C.c_int, [C.c_int] * 4 + [_P, C.c_int, _P, C.c_int, _P]),
    "fsb_nhwc_f16_to_nchw": (C.c_int, [C.c_int] * 4 + [_P, C.c_int, _P, C.c_int, _P]),
    "fsb_copy_channels": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "fsb_bn_stats": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, _P]),
    "fsb_bn_finalize": (C.c_int, [C.c_int, _P, C.c_int, C.c_int, C.c_double, _P, _P, C.c_float, C.c_float, _P, _P, _P, _P, _P, _P, _P]),
    "fsb_affine_act": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, _P, _P, C.c_int, C.c_uint32, _P]),
    "fsb_bn_bwd_reduce": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_int, _P, _P]),
    "fsb_bn_bwd_apply": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_double,
                                   C.c_int, _P, C.c_int, _P, _P, C.c_float, C.c_int, _P]),
    "fsb_bn_finalize_sel": (C.c_int, [C.c_int, _P, C.c_int, C.c_int, C.c_double, C.c_float, C.c_float, _P, _P, _P, _P, _P, _P, C.c_int, _P]),
    "fsb_affine_act_sel": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, _P, _P, C.c_int, C.c_uint32, _P, _P, C.c_int, _P]),
    "fsb_bn_bwd_reduce_sel": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, C.c_int, _P,
                                        _P, _P, C.c_int, _P]),
    "fsb_bn_bwd_apply_sel": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, C.c_int, _P, _P, _P, _P, C.c_double,
                                       C.c_int, _P, C.c_int, C.c_float, _P, _P, C.c_int, _P]),
    "fsb_relu_bwd": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "fsb_conv_packed_dgrad_bytes": (C.c_size_t, [C.POINTER(ConvDesc)]),
    "fsb_pack_conv_weight_dgrad": (C.c_int, [C.POINTER(ConvDesc), _P, C.c_int64, C.c_int64, _P, _P]),
    "fsb_conv_dgrad": (C.c_int, [C.POINTER(ConvDesc), _P, C.c_int, _P, _P, C.c_int64, C.c_int64, _P, C.c_int, _P]),
    "fsb_conv_wgrad": (C.c_int, [C.POINTER(ConvDesc), _P, _P, C.c_int, _P, C.c_int64, C.c_int64, C.c_int, C.c_float, _P]),
    "fsb_bilinear_bwd": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "fsb_upsample_logits_bwd": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, C.c_float, _P]),
    "fsb_nchw_grad_to_nhwc": (C.c_int, [C.c_int] * 4 + [_P, C.c_int, _P, C.c_int, C.c_float, _P]),
    "fsb_wsum_fwd": (C.c_int, [C.c_int, C.c_int64, C.c_int, _P, _P, _P, _P, C.c_int, _P]),
    "fsb_wsum_bwd": (C.c_int, [C.c_int, C.c_int64, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, _P, C.c_float, _P]),
    "fsb_add_inplace": (C.c_int, [C.c_int64, C.c_int, _P, C.c_int, _P, C.c_int, _P]),
    "fsb_conv_bn_act_train_fwd": (C.c_int, [C.POINTER(ConvDesc), _P, _P, _P, _P, C.c_float, C.c_float, _P, _P, _P, _P, C.c_int, _P,
                                            C.c_int, _P, C.c_int, _P, _P, _P]),
    "fsb_conv_bn_act_train_bwd": (C.c_int, [C.POINTER(ConvDesc), _P, _P, C.c_int, _P, C.c_int, _P, C.c_int, _P, _P, C.c_int, _P, _P,
                                            C.c_int64, C.c_int64, _P, C.c_int, _P, _P, C.c_int, _P, C.c_float, _P, _P, _P]),
    "fsb_loss_logp_fwd": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P, _P, _P]),
    "fsb_kth_workspace_bytes": (C.c_size_t, []),
    "fsb_kth_smallest_f32": (C.c_int, [_P, C.c_int64, C.c_int64, _P, _P, _P]),
    "fsb_loss_rows": (C.c_int, []),
    "fsb_ohem_reduce": (C.c_int, [_P, _P, C.c_int64, C.c_int, C.c_int, _P, _P, _P, _P]),
    "fsb_loss_ce_bwd": (C.c_int, [C.c_int] * 6 + [_P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P, C.c_int, C.c_float, C.c_int, _P]),
    "fsb_loss_kl_fwd": (C.c_int, [C.c_int] * 8 + [_P, C.c_int, _P, C.c_int, _P, _P, _P, _P, _P]),
    "fsb_loss_kl_bwd": (C.c_int, [C.c_int] * 8 + [_P, C.c_int, _P, C.c_int, _P, _P, _P, _P, C.c_int, C.c_float, C.c_int, _P]),
    "fsb_flat_chunk": (C.c_int, []),
    "fsb_flat_grad_norm": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P, C.c_float, _P, _P]),
    "fsb_flat_scale": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, _P]),
    "fsb_flat_sgd": (C.c_int, [_P, C.c_int, _P, _P, _P, _P, C.c_float, C.c_float, C.c_float, _P]),
    "fsb_dp_unique_id": (C.c_int, [_P]),
    "fsb_dp_init": (C.c_int, [_P, C.c_int, C.c_int]),
    "fsb_dp_world": (C.c_int, []),
    "fsb_dp_enable": (C.c_int, [C.c_int]),
    "fsb_dp_allreduce_f32": (C.c_int, [_P, C.c_int64, _P]),
    "fsb_dp_shutdown": (C.c_int, []),
    "fsb_peer_alloc": (C.c_int, [_P]),
    "fsb_peer_open": (C.c_int, [_P, C.c_int, C.c_int]),
    "fsb_peer_world": (C.c_int, []),
    "fsb_peer_enable": (C.c_int, [C.c_int]),
    "fsb_peer_begin": (C.c_int, [C.c_int, _P]),
    "fsb_peer_allreduce_f32": (C.c_int, [_P, C.c_int64, _P]),
    "fsb_peer_shutdown": (C.c_int, []),
    "fsb_supernet_latency_workspace_bytes": (C.c_size_t, [_P]),
    "fsb_supernet_latency_fwd": (C.c_int, [_P] * 13 + [_P]),
    "fsb_supernet_latency_bwd": (C.c_int, [_P] * 12 + [_P]),
    "fsb_train_pre": (C.c_int, [C.POINTER(TrainPreDesc)] + [_P] * 7),
}
EXPORTED_SYMBOLS = tuple(_SIGS)

_lib = None


def lib():
    """Load libfsb200.so (once).  Raises FsbError loudly if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise FsbError("libfsb200.so not found at %s -- run `python -m fasterseg_b200.build` (needs nvcc); "
                           "there is no CPU/PyTorch fallback" % LIB_PATH)
        l = C.CDLL(LIB_PATH)
        for name, (res, args) in _SIGS.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        if l.fsb_abi_version() != ABI_VERSION:
            raise FsbError("libfsb200.so ABI version mismatch")
        _lib = l
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().fsb_last_error_string()
        raise FsbError("%s failed (%d): %s" % (what or "fsb call", rc, msg.decode() if msg else "?"))


def set_option(name: str, value: int):
    """tuning / validation switch of the library (named like its environment variable, e.g. "FSB_CONV_TC2")"""
    check(lib().fsb_set_option(name.encode(), int(value)), "fsb_set_option(%s)" % name)


def get_option(name: str) -> int:
    return lib().fsb_get_option(name.encode())
