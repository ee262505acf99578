"""ctypes binding of libbdbnn_b200.so (the C ABI in include/bdbnn.h).

There is NO CPU fallback and no PyTorch-eager fallback: if the shared library is missing or a call
fails, a RuntimeError is raised."""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libbdbnn_b200.so")

_lock = threading.Lock()
_lib = None

c_void_p, c_int, c_int64, c_size_t = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_size_t


class ConvShape(ctypes.Structure):
    """Mirror of `bdbnn_conv_shape` (include/bdbnn.h)."""
    _fields_ = [(n, ctypes.c_int32) for n in
                ("N", "H", "W", "Cin", "Cout", "kh", "kw", "stride", "pad", "Ho", "Wo")]


_P = c_void_p
_SH = ctypes.POINTER(ConvShape)
# name -> (restype, argtypes); MUST list every symbol include/bdbnn.h declares (tests check this).
SIGNATURES = {
    "bdbnn_version": (c_int, []),
    "bdbnn_last_error_string": (ctypes.c_char_p, []),
    "bdbnn_tc_supported": (c_int, [_SH]),
    "bdbnn_debug_trace": (c_int, [_P]),
    "bdbnn_act_pack": (c_int, [_P, c_int64, c_int, _P, _P, _P, c_int, _P]),
    "bdbnn_weight_pack": (c_int, [_P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P, _P, c_int, _P]),
    "bdbnn_weight_pack_multi": (c_int, [c_int] + [_P] * 12 + [c_int, _P]),
    "bdbnn_weight_unpack_multi": (c_int, [c_int] + [_P] * 6 + [c_int, _P]),
    "bdbnn_bits_to_fp8": (c_int, [_P, c_int64, c_int, _P, _P]),
    "bdbnn_ede_scale": (c_int, [_P, _P, _P, _P, c_int64, _P]),
    "bdbnn_ce_topk_fwd_bwd": (c_int, [_P, _P, c_int, c_int, c_int, c_int, _P, _P, _P, _P, _P, _P, _P]),
    "bdbnn_optim_adam_multi": (c_int, [_P, _P, _P, _P, _P, _P, _P, c_int, ctypes.c_float, ctypes.c_float,
                                       ctypes.c_float, c_int64, ctypes.c_float, _P]),
    "bdbnn_optim_sgd_multi": (c_int, [_P, _P, _P, _P, _P, _P, c_int, ctypes.c_float, c_int, ctypes.c_float, _P]),
    "bdbnn_optim_step_inc": (c_int, [_P, _P]),
    "bdbnn_optim_adam_multi_graph": (c_int, [_P, _P, _P, _P, _P, _P, c_int, ctypes.c_float, ctypes.c_float,
                                             ctypes.c_float, _P, _P, ctypes.c_float, _P]),
    "bdbnn_optim_sgd_multi_graph": (c_int, [_P, _P, _P, _P, _P, c_int, ctypes.c_float, _P, ctypes.c_float, _P]),
    "bdbnn_real_conv_pack": (c_int, [_P, c_int, c_int, c_int, c_int, c_int, _P, c_int] + [_P] * 8),
    "bdbnn_stem_supported": (c_int, [c_int, c_int, c_int]),
    "bdbnn_stem_xw_bytes": (c_size_t, [c_int, c_int, c_int]),
    "bdbnn_stem_wgrad_workspace_bytes": (c_size_t, [c_int, c_int, c_int]),
    "bdbnn_stem_pack": (c_int, [_P, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, _P, _P, _P, _P, _P, _P]),
    "bdbnn_stem_conv_fwd": (c_int, [_P, _P, _P, _P, c_int, c_int, c_int, _P, _P, _P]),
    "bdbnn_stem_conv_wgrad": (c_int, [_P, _P, _P, _P, _P, c_int, c_int, c_int, _P, c_size_t, _P]),
    "bdbnn_binconv_fwd_tc8": (c_int, [_P, _P, _P, _P, _SH, _P, _P, _P]),
    "bdbnn_binconv_fwd_xnor": (c_int, [_P, _P, _P, _P, _SH, _P]),
    "bdbnn_binconv_fwd_tc": (c_int, [_P, _P, c_int, _P, _P, _SH, _P, _P, _P]),
    "bdbnn_binconv_dgrad": (c_int, [_P, _P, _P, _P, _P, _SH, _P]),
    "bdbnn_binconv_wgrad": (c_int, [_P, _P, _P, _P, _SH, _P]),
    "bdbnn_grad_pack": (c_int, [_P, _P, c_int64, c_int, c_int, _P, _P, _P]),
    "bdbnn_binconv_dgrad_tc": (c_int, [_P, c_int, _P, _P, _P, _P, _P, _SH, _P]),
    "bdbnn_wgrad_tc_workspace_bytes": (c_size_t, [_SH]),
    "bdbnn_debug_wgrad_plan": (c_int, [_SH, c_int, _P, c_int]),
    "bdbnn_debug_conv_plan": (c_int, [_SH, c_int, c_int, _P, c_int]),
    "bdbnn_debug_tc_conv_ctas_per_sm": (c_int, [c_int, c_int, c_int, c_int, _P]),
    "bdbnn_binconv_wgrad_tc": (c_int, [_P, c_int, _P, _P, _P, _P, _P, _SH, _P, c_size_t, _P]),
    "bdbnn_kurtosis_multi_fwd": (c_int, [_P, _P, _P, c_int, _P, _P, _P, _P]),
    "bdbnn_kurtosis_multi_bwd": (c_int, [_P, _P, _P, c_int, _P, _P, _P, c_int, _P]),
    "bdbnn_sign_flips_multi": (c_int, [_P, _P, _P, c_int, _P, _P, c_int, _P]),
    "bdbnn_weight_stats_multi": (c_int, [_P, _P, _P, c_int, _P, _P, _P, _P, _P]),
    "bdbnn_binconv_fwd_b1_eval": (c_int, [_P] * 8 + [_SH, _P]),
    "bdbnn_binconv_fwd_b1_i16": (c_int, [_P] * 4 + [_SH, _P]),
    "bdbnn_b1_popc_table": (c_int, [_P, c_int, c_int, c_int, _P, _P]),
    "bdbnn_debug_b1_mma": (c_int, [_P] * 4),
    "bdbnn_kd_logits_fwd_bwd": (c_int, [_P, _P, c_int, c_int, _P, _P, _P, _P]),
    "bdbnn_kd_layer_multi_fwd": (c_int, [_P, _P, _P, c_int, _P, _P, _P]),
    "bdbnn_kd_layer_multi_bwd": (c_int, [_P, _P, c_int, _P, _P, c_int, _P]),
    "bdbnn_bn_fwd": (c_int, [_P, _P, _P, _P, c_int64, c_int, ctypes.c_float, ctypes.c_float] + [_P] * 12 + [c_int, c_int, _P]),
    "bdbnn_bn_bwd_pack": (c_int, [_P] * 7 + [c_int64, c_int, c_int] + [_P] * 8),
    "bdbnn_bn_fwd_i16": (c_int, [_P] * 5 + [c_int64, c_int, ctypes.c_float, ctypes.c_float] + [_P] * 12 + [c_int, _P]),
    "bdbnn_bn_bwd_pack_i16": (c_int, [_P] * 8 + [c_int64, c_int, c_int] + [_P] * 7 + [c_int, _P]),
    "bdbnn_binconv_dgrad_tc_stats": (c_int, [_P, c_int, _P, _P, _P, _P, _P, _SH] + [_P] * 7),
    "bdbnn_binconv_fwd_tc_i16": (c_int, [_P, _P, c_int, _P, _P, _SH, _P, _P, _P]),
    "bdbnn_bn_pool_fwd": (c_int, [_P, _P, _P] + [c_int] * 9 + [ctypes.c_float, ctypes.c_float] + [_P] * 14 + [c_int, c_int, _P]),
    "bdbnn_bn_pool_bwd": (c_int, [_P] * 9 + [c_int] * 9 + [_P] * 9),
    "bdbnn_maxpool_fwd": (c_int, [_P, _P, _P] + [c_int] * 9 + [_P]),
    "bdbnn_maxpool_bwd": (c_int, [_P, _P, _P] + [c_int] * 9 + [_P]),
    "bdbnn_bn_eval_fold": (c_int, [_P] * 5 + [c_int, ctypes.c_float, _P, _P, _P]),
    "bdbnn_binconv_fwd_tc_eval": (c_int, [_P, _P, c_int] + [_P] * 6 + [_SH, _P]),
    "bdbnn_stem_conv_fwd_eval": (c_int, [_P] * 5 + [c_int] * 3 + [_P]),
    "bdbnn_stem_conv_fwd_eval_relu": (c_int, [_P] * 6 + [c_int] * 3 + [_P]),
    "bdbnn_real_act_pack": (c_int, [_P, c_int64, c_int, _P, c_int, _P, _P]),
    "bdbnn_real_weight_pack_multi": (c_int, [c_int] + [_P] * 8 + [_P]),
    "bdbnn_real_weight_pack_multi_grad": (c_int, [c_int] + [_P] * 11 + [_P]),
    "bdbnn_real_conv_fwd_eval": (c_int, [_P] * 6 + [c_int, _P, _P, _SH, _P]),
    "bdbnn_real_gconv_supported": (c_int, [_SH, c_int]),
    "bdbnn_real_gconv_fwd": (c_int, [_P, _P, _P, _P, _SH, c_int, _P, _P, _P]),
    "bdbnn_real_gconv_fwd_eval": (c_int, [_P] * 6 + [c_int, _P, _P, _SH, c_int, _P]),
    "bdbnn_real_gconv_dgrad": (c_int, [_P] * 6 + [_SH, c_int, _P]),
    "bdbnn_real_gconv_wgrad_workspace_bytes": (c_size_t, [_SH, c_int]),
    "bdbnn_real_gconv_wgrad": (c_int, [_P] * 6 + [_SH, c_int, _P, c_size_t, _P]),
    "bdbnn_real_weight_pack_multi_grouped": (c_int, [c_int] + [_P] * 12 + [_P]),
    "bdbnn_bn_fwd_pad_shortcut": (c_int, [_P, _P] + [c_int] * 5 + [_P, _P, c_int, ctypes.c_float, ctypes.c_float] +
                                  [_P] * 12 + [c_int, c_int, _P]),
    "bdbnn_bn_fwd_i16_pad_shortcut": (c_int, [_P, _P, _P] + [c_int] * 5 + [_P, _P, c_int, ctypes.c_float,
                                                                          ctypes.c_float] + [_P] * 12 + [c_int, _P]),
    "bdbnn_pad_shortcut_bwd": (c_int, [_P, _P] + [c_int] * 6 + [_P]),
    "bdbnn_cifar_stem_fwd": (c_int, [_P, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, _P, c_int, _P, _P, _P,
                                     _P]),
    "bdbnn_cifar_stem_fwd_eval": (c_int, [_P, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, _P, c_int] +
                                  [_P] * 5),
    "bdbnn_binconv_fwd_tc_eval_pad_shortcut": (c_int, [_P, _P, c_int, _P, _P, _P] + [c_int] * 4 + [_P, _P, _P, _SH,
                                                                                                 _P]),
    "bdbnn_real_conv_fwd_eval_pad_shortcut": (c_int, [_P] * 6 + [c_int] * 5 + [_P, _P, _SH, _P]),
    "bdbnn_cifar_stem_fwd_eval_hardtanh": (c_int, [_P, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, _P,
                                                   c_int] + [_P] * 5),
    "bdbnn_cifar_stem_wgrad_workspace_bytes": (c_size_t, [c_int] * 4),
    "bdbnn_cifar_stem_wgrad": (c_int, [_P, c_int, c_int, c_int, c_int64, c_int64, c_int64, c_int64, _P, _P, c_int, _P,
                                       _P, c_size_t, _P]),
    "bdbnn_bn_fwd_hardtanh": (c_int, [_P] * 4 + [c_int64, c_int, ctypes.c_float, ctypes.c_float] + [_P] * 12 +
                              [c_int, c_int, _P]),
    "bdbnn_bn_bwd_pack_hardtanh": (c_int, [_P] * 9 + [c_int64, c_int, c_int] + [_P] * 8),
    "bdbnn_bn_fwd_relu": (c_int, [_P] * 4 + [c_int64, c_int, ctypes.c_float, ctypes.c_float] + [_P] * 10 + [c_int, _P]),
    "bdbnn_bn_bwd_pack_relu": (c_int, [_P] * 8 + [c_int64, c_int, c_int] + [_P] * 9),
    "bdbnn_bn_pool_fwd_relu": (c_int, [_P, _P, _P] + [c_int] * 9 + [ctypes.c_float, ctypes.c_float] + [_P] * 12 +
                               [c_int, _P]),
    "bdbnn_bn_pool_bwd_relu": (c_int, [_P] * 10 + [c_int] * 9 + [_P] * 9),
    "bdbnn_real_scale_fold": (c_int, [_P, _P, _P, c_int, _P, _P, _P]),
    "bdbnn_pool2_i16": (c_int, [_P, _P] + [c_int] * 4 + [_P] * 5),
    "bdbnn_pool2_bn_bwd_pack": (c_int, [_P] * 10 + [c_int] * 5 + [_P] * 8),
    "bdbnn_pool2_bn_eval_hardtanh": (c_int, [_P] * 3 + [c_int] * 4 + [_P] * 3 + [c_int, _P]),
    "bdbnn_real_pool2_bn_eval_hardtanh": (c_int, [_P] * 3 + [c_int] * 4 + [_P] * 3),
    "bdbnn_real_bn_fwd_hardtanh": (c_int, [_P] * 3 + [c_int64, c_int, ctypes.c_float, ctypes.c_float] + [_P] * 9 +
                                   [c_int, _P]),
    "bdbnn_real_pool2": (c_int, [_P] + [c_int] * 4 + [_P] * 5),
    "bdbnn_real_pool2_bn_bwd_pack": (c_int, [_P] * 9 + [c_int] * 4 + [_P] * 8),
    "bdbnn_cifar_batch": (c_int, [_P, _P, c_int64, ctypes.c_uint64, ctypes.c_uint32, c_int64, c_int, c_int, _P, _P, _P,
                                  c_int64, c_int64, c_int64, c_int64, _P, _P]),
    "bdbnn_imagenet_batch": (c_int, [_P, _P, c_int, _P, _P, _P, c_int64, c_int64, c_int64, c_int64, _P, _P]),
    "bdbnn_jpeg_parse": (c_int, [ctypes.c_char_p, c_int64, _P, _P, c_int64, _P, c_int]),
    "bdbnn_jpeg_subseq_bits": (c_int, []),
    "bdbnn_debug_jpeg_subseq_bits": (c_int, [c_int]),
    "bdbnn_jpeg_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "bdbnn_jpeg_check_batch": (c_int, [_P, c_int, _P, c_int, c_int64, c_int64, c_size_t]),
    "bdbnn_jpeg_decode_batch": (c_int, [_P, _P, c_int, _P, _P, c_int, _P, _P, c_int64, _P, c_size_t, _P, c_int64, _P,
                                        _P, _P, _P]),
    "bdbnn_jpeg_index_scratch_bytes": (c_size_t, [c_int64]),
    "bdbnn_debug_jpeg_index_entry": (c_int, [c_int, c_int, c_int, c_int, c_int, _P, _P]),
    "bdbnn_jpeg_index_file": (c_int, [ctypes.c_char_p, c_int64, c_int, _P, c_size_t, _P, c_int64, _P, _P]),
    "bdbnn_jpeg_decode_batch_indexed": (c_int, [_P, _P, c_int, _P, _P, c_int, _P, _P, c_int64, _P, _P, c_int64, _P,
                                                c_size_t, _P, c_int64, _P, _P, _P, _P]),
    "bdbnn_jpeg_decode_batch_files": (c_int, [_P, _P, c_int64, _P, _P, _P, _P, c_int, _P, _P, c_int, _P, c_int64, _P,
                                              _P, c_int64, _P, c_size_t, _P, c_int64, _P, _P, _P]),
}


def lib():
    """Load (once) and return the ctypes handle. Raises RuntimeError if the library is absent."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"bdbnn_b200: {LIB_PATH} not found. Build it with `python -m bdbnn_b200.build` "
                "(nvcc, sm_90a). There is no CPU / eager fallback.")
        h = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(h, name)
            fn.restype = res
            fn.argtypes = args
        _lib = h
    return _lib


def check(rc, what):
    if rc != 0:
        msg = lib().bdbnn_last_error_string().decode("utf-8", "replace")
        raise RuntimeError(f"bdbnn_b200: {what} failed with code {rc}: {msg}")


def launch_count():
    """Number of kernels this process launched through the C ABI (bench.py reports it)."""
    return _launches[0]


_launches = [0]


def count(n=1):
    _launches[0] += n
