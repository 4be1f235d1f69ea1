"""ctypes binding of libian_b200.so (C-ABI: include/ian_b200.h).  No CPU fallback: if the library is
missing or no sm_90 (H100) GPU is present, construction fails loudly."""
from __future__ import annotations

import ctypes as C
import os

HERE = os.path.dirname(os.path.abspath(__file__))
# IAN_B200_LIB: another in-tree BUILD of the same sources/ABI (to compare two builds in one process run); the
# default is the library build.py produces.  It is never a different implementation: there is no fallback.
LIB_PATH = os.environ.get("IAN_B200_LIB") or os.path.join(HERE, "libian_b200.so")

IAN_OK = 0
IAN_PATH_TC, IAN_PATH_SIMT = 0, 1
IAN_MODEL_SIMPLE, IAN_MODEL_FULL, IAN_MODEL_V1 = 0, 1, 2

_F = C.POINTER(C.c_float)
_I = C.POINTER(C.c_int32)
_H = C.c_void_p

# every symbol include/ian_b200.h declares: name -> (restype, argtypes)
SIGNATURES = {
    "ian_create": (C.c_int, [C.c_int, C.c_int, C.POINTER(_H)]),
    "ian_set_param": (C.c_int, [_H, C.c_char_p, _F, C.POINTER(C.c_int64), C.c_int]),
    "ian_model_param_count": (C.c_int, [C.c_int]),
    "ian_model_param_spec": (C.c_int, [C.c_int, C.c_int, C.POINTER(C.c_char_p), C.POINTER(C.c_int64), C.POINTER(C.c_int)]),
    "ian_set_made_ordering": (C.c_int, [_H, _I, C.c_int]),
    "ian_made_mask": (C.c_int, [_I, C.c_int, C.c_int, C.c_void_p]),
    "ian_debug_made_weights": (C.c_int, [_H, _F]),
    "ian_finalize": (C.c_int, [_H]),
    "ian_destroy": (C.c_int, [_H]),
    "ian_last_error": (C.c_char_p, [_H]),
    "ian_get_zdim": (C.c_int, [_H]),
    "ian_set_path": (C.c_int, [_H, C.c_int]),
    "ian_set_precision": (C.c_int, [_H, C.c_int]),
    "ian_launch_count": (C.c_int64, [_H]),
    "ian_encode_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_encode_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_decode_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_decode_host": (C.c_int, [_H, _F, C.c_int, _F]),
    "ian_reconstruct_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_reconstruct_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_reconstruct_submit": (C.c_int, [_H, _F, C.c_int, _F, _F, C.POINTER(C.c_int)]),
    "ian_reconstruct_wait": (C.c_int, [_H, C.c_int]),
    "ian_host_alloc": (C.c_int, [_H, C.c_size_t, C.POINTER(C.c_void_p)]),
    "ian_host_free": (C.c_int, [_H, C.c_void_p]),
    "ian_gather_create": (C.c_int, [_H, C.c_int, C.c_int, C.c_int, C.c_void_p]),
    "ian_gather_connect": (C.c_int, [_H, C.c_void_p]),
    "ian_reconstruct_gather_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.POINTER(C.c_void_p), C.c_void_p]),
    "ian_reconstruct_gather_async_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_gather_wait_dev": (C.c_int, [_H, C.POINTER(C.c_void_p), C.c_void_p]),
    "ian_encode_pre_host": (C.c_int, [_H, _F, C.c_int, _F]),
    "ian_flow_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_encode_pre_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_flow_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_flow_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_flow_vjp_host": (C.c_int, [_H, _F, _F, C.c_int, _F]),
    "ian_flow_jvp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_flow_jvp_host": (C.c_int, [_H, _F, _F, C.c_int, _F, _F]),
    "ian_encode_pre_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_encode_pre_vjp_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_encode_pre_jvp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_encode_pre_jvp_host": (C.c_int, [_H, _F, _F, C.c_int, _F, _F]),
    "ian_grad_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_grad_host": (C.c_int, [_H, _F, _I, _F, C.c_int, C.c_int, _F]),
    "ian_decode_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_decode_vjp_host": (C.c_int, [_H, _F, _F, C.c_int, _F]),
    "ian_decode_jvp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_decode_jvp_host": (C.c_int, [_H, _F, _F, C.c_int, _F, _F]),
    "ian_encode_jvp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_encode_jvp_host": (C.c_int, [_H, _F, _F, C.c_int, _F, _F, _F]),
    "ian_decode_gauss_newton_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p,
                                              C.c_void_p]),
    "ian_decode_gauss_newton_host": (C.c_int, [_H, _F, _F, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double),
                                               C.POINTER(C.c_double)]),
    "ian_fit_latent_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p]),
    "ian_fit_latent_host": (C.c_int, [_H, _F, C.c_int, _F, C.c_int, _F]),
    "ian_map_gauss_newton_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p,
                                           C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_map_gauss_newton_host": (C.c_int, [_H, _F, _F, _F, C.c_double, C.c_int, C.POINTER(C.c_double),
                                            C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "ian_fit_latent_map_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_void_p, C.c_int,
                                         C.c_void_p, C.c_void_p]),
    "ian_fit_latent_map_host": (C.c_int, [_H, _F, _F, C.c_double, C.c_int, _F, _F, C.c_int, _F]),
    "ian_robust_gauss_newton_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_int]
                                    + [C.c_void_p] * 5),
    "ian_robust_gauss_newton_host": (C.c_int, [_H, _F, _F, _F, C.c_double, C.c_int, C.POINTER(C.c_double), C.c_int]
                                     + [C.POINTER(C.c_double)] * 4),
    "ian_fit_latent_robust_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_double, C.c_int, C.c_void_p, C.c_int, C.c_void_p,
                                            C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_fit_latent_robust_host": (C.c_int, [_H, _F, _F, C.c_double, C.c_int, C.POINTER(C.c_double), C.c_int, _F, _F, C.c_int,
                                             _F, C.POINTER(C.c_double), _F]),
    "ian_introspect_dev": (C.c_int, [_H, C.c_void_p, C.c_int] + [C.c_void_p] * 5),
    "ian_introspect_host": (C.c_int, [_H, _F, C.c_int, _F, _F, _F, _F]),
    "ian_introspect_jvp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int] + [C.c_void_p] * 9),
    "ian_introspect_jvp_host": (C.c_int, [_H, _F, _F, C.c_int] + [_F] * 8),
    "ian_introspect_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_int] + [C.c_void_p] * 6),
    "ian_introspect_vjp_host": (C.c_int, [_H, _F, C.c_int] + [_F] * 5),
    "ian_feature_gauss_newton_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_double, C.c_double, C.c_void_p,
                                               C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_feature_gauss_newton_host": (C.c_int, [_H, _F, _F, C.c_int, C.c_double, C.c_double, C.POINTER(C.c_double),
                                                C.POINTER(C.c_double), C.POINTER(C.c_double)]),
    "ian_fit_latent_features_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_int, C.c_double, C.c_double,
                                              C.c_void_p, C.c_void_p]),
    "ian_fit_latent_features_host": (C.c_int, [_H, _F, C.c_int, _F, C.c_int, C.c_double, C.c_double, _F]),
    "ian_set_discriminator_param": (C.c_int, [_H, C.c_char_p, _F, C.POINTER(C.c_int64), C.c_int]),
    "ian_discriminate_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_discriminate_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_discriminate_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_discriminate_vjp_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_discriminate_train_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_discriminate_train_host": (C.c_int, [_H, _F, C.c_int, _F, _F, _F]),
    "ian_discriminate_train_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_discriminate_train_vjp_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_param_vjp_supported": (C.c_int, [C.c_int, C.c_int]),
    "ian_decode_param_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_decode_param_vjp_host": (C.c_int, [_H, _F, _F, C.c_int, _F, C.c_void_p]),
    "ian_decode_train_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_decode_train_host": (C.c_int, [_H, _F, C.c_int, _F, _F]),
    "ian_decode_train_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_decode_train_vjp_host": (C.c_int, [_H, _F, _F, C.c_int, _F, C.c_void_p]),
    "ian_update_param_host": (C.c_int, [_H, C.c_char_p, _F, C.POINTER(C.c_int64), C.c_int]),
    "ian_encode_vjp_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_encode_vjp_host": (C.c_int, [_H, _F, C.c_int, _F, _F, _F]),
    "ian_edit_loop_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_float,
                                    C.c_void_p]),
    "ian_edit_loop_host": (C.c_int, [_H, _F, _I, _F, C.c_int, C.c_int, C.c_int, C.c_float]),
    "ian_paint_stroke_host": (C.c_int, [_H, _F, _I, _F, C.c_float, C.c_void_p, _F, C.c_void_p, C.c_void_p]),
    "ian_bn_batch_stats_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_bn_train_normalize_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_double,
                                             C.c_void_p, C.c_void_p, C.c_float, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p,
                                             C.c_void_p]),
    "ian_minibatch_discrim_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int, C.c_int,
                                            C.c_void_p, C.c_void_p]),
    "ian_bn_backward_sums_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                           C.c_double, C.c_float, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_bn_backward_dx_dev": (C.c_int, [_H, C.c_void_p, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_double, C.c_void_p, C.c_void_p, C.c_void_p, C.c_float, C.c_void_p, C.c_void_p]),
    "ian_minibatch_discrim_bwd_dev": (C.c_int, [_H, C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_int,
                                                C.c_int, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]),
    "ian_set_layer_timing": (C.c_int, [_H, C.c_int]),
    "ian_layer_time_ms": (C.c_double, [_H, C.c_char_p, C.c_int]),
}

_lib = None


def load():
    """dlopen the in-tree library and type every entry point."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError(
            "libian_b200.so is not built (%s). Run `python neural-photo-editor_b200/build.py`; "
            "there is no CPU or PyTorch fallback for the IAN hot path." % LIB_PATH)
    lib = C.CDLL(LIB_PATH)
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)          # AttributeError if the .so lacks a declared symbol
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


class IanError(RuntimeError):
    pass


def check(lib, handle, rc):
    if rc != IAN_OK:
        msg = lib.ian_last_error(handle)
        raise IanError("libian_b200 error %d: %s" % (rc, msg.decode() if msg else "?"))
