"""ctypes binding of libcgvc.so (the C ABI declared in include/cgvc.h).

There is deliberately no fallback: if the shared library is missing or fails to load, importing the
package's compute classes raises.  PyTorch is used by callers for device storage only.
"""
from __future__ import annotations

import ctypes as C
import os

from . import build as _build

_LIB = None

ARENA_PARAM, ARENA_GRAD, ARENA_ADAM_M, ARENA_ADAM_V, ARENA_WORK = range(5)
PREC_FP32_SIMT, PREC_BF16X3, PREC_BF16, PREC_F16F8 = 0, 1, 2, 3
PRECISIONS = {"fp32": PREC_FP32_SIMT, "fp32_simt": PREC_FP32_SIMT, "bf16x3": PREC_BF16X3, "bf16": PREC_BF16, "f16f8": PREC_F16F8}
ERR_ARG = -1
ERR_UNBOUND = -3
ERR_DIRECTION = -4
ERR_UNSUPPORTED = -5

LOSS_NAMES = ("cycle_loss", "identity_loss", "generator_loss_A2B", "generator_loss_B2A", "generator_loss",
              "discriminator_loss_A", "discriminator_loss_B", "discriminator_loss")


class Config(C.Structure):
    _fields_ = [("num_features", C.c_int), ("max_batch", C.c_int), ("max_frames", C.c_int),
                ("precision", C.c_int), ("device", C.c_int), ("train", C.c_int)]


LOSS_SCALE_MODES = {"static": 0, "monitor": 1, "dynamic": 2}


class LossScaleInfo(C.Structure):
    """cgvc_loss_scale_info of include/cgvc.h"""
    _fields_ = [("scale", C.c_float), ("good_steps", C.c_int), ("skipped", C.c_longlong), ("last_skipped", C.c_int),
                ("nonfinite", C.c_uint), ("sat_grad", C.c_ulonglong), ("sat_act", C.c_ulonglong)]


class LossScaleNetInfo(C.Structure):
    """cgvc_loss_scale_net_info of include/cgvc.h: index 0 the generators, 1 the discriminators"""
    _fields_ = [("scale", C.c_float), ("good_steps", C.c_int), ("sat_grad", C.c_ulonglong), ("ufl_grad", C.c_ulonglong),
                ("groups", C.c_ulonglong)]


class WeightLayerInfo(C.Structure):
    """cgvc_weight_layer_info of include/cgvc.h"""
    _fields_ = [(n, C.c_int) for n in ("n_layers", "kh", "kw", "cin", "cout", "gated", "shuffle", "fold")] + \
               [(n, C.c_longlong) for n in ("ka", "kg", "ba", "bg")] + \
               [(n, C.c_int) for n in ("nt_n", "cin_k", "cin_n", "nt_k", "cin_q", "nt_q", "q_ok")]


class CgvcError(RuntimeError):
    def __init__(self, code, msg):
        super().__init__("libcgvc error %d: %s" % (code, msg))
        self.code = code


def _declare(lib):
    vp, ci, cf, sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
    P = C.POINTER
    sig = {
        "cgvc_abi_version": (ci, []),
        "cgvc_create": (ci, [P(Config), P(vp)]),
        "cgvc_destroy": (ci, [vp]),
        "cgvc_last_error": (C.c_char_p, [vp]),
        "cgvc_arena_bytes": (ci, [vp, ci, P(sz)]),
        "cgvc_bind_arena": (ci, [vp, ci, vp, sz]),
        "cgvc_param_count": (ci, [vp, P(ci), P(sz)]),
        "cgvc_param_info": (ci, [vp, ci, P(C.c_char_p), P(sz), P(ci), P(ci * 4)]),
        "cgvc_params_updated": (ci, [vp, vp]),
        "cgvc_set_adam_step": (ci, [vp, C.c_longlong]),
        "cgvc_get_adam_step": (ci, [vp, P(C.c_longlong)]),
        "cgvc_loss_scale_state": (ci, [vp, vp, vp]),
        "cgvc_set_loss_scale_state": (ci, [vp, cf, ci, C.c_longlong, vp]),
        "cgvc_loss_scale_net_state": (ci, [vp, vp, vp]),
        "cgvc_set_loss_scale_net_state": (ci, [vp, ci, cf, ci, vp]),
        "cgvc_set_plane_counters": (ci, [vp, vp]),
        "cgvc_train_step": (ci, [vp, vp, vp, ci, ci, cf, cf, cf, cf, vp, vp, vp, vp]),
        "cgvc_compute_gradients": (ci, [vp, vp, vp, ci, ci, cf, cf, vp, vp, vp, vp]),
        "cgvc_adam_step": (ci, [vp, cf, cf, cf, vp]),
        "cgvc_apply_gradients": (ci, [vp, cf, cf, vp]),
        "cgvc_generator_forward": (ci, [vp, ci, vp, vp, ci, ci, vp]),
        "cgvc_generator_forward_packed": (ci, [vp, ci, vp, vp, P(C.c_longlong), ci, vp]),
        "cgvc_discriminator_forward_packed": (ci, [vp, ci, vp, vp, P(C.c_longlong), ci, vp]),
        "cgvc_discriminator_forward": (ci, [vp, ci, vp, vp, ci, ci, vp]),
        "cgvc_debug_activation": (ci, [vp, C.c_char_p, vp, sz, P(sz), vp]),
        "cgvc_weight_planes": (ci, [vp, ci, P(WeightLayerInfo), C.c_char_p, vp, sz, P(sz), vp]),
        "cgvc_comm_unique_id": (ci, [vp, vp]),
        "cgvc_comm_init": (ci, [vp, vp, ci, ci]),
        "cgvc_comm_destroy": (ci, [vp]),
        "cgvc_allreduce_grads": (ci, [vp, vp]),
        "cgvc_sample_plan": (ci, [vp, vp, ci, vp, ci, C.c_ulonglong, C.c_longlong, ci, vp, vp, vp]),
        "cgvc_gather_minibatch": (ci, [vp, vp, vp, vp, vp, vp, ci, ci, ci, ci, vp, vp, vp]),
        "cgvc_kernel_launches": (ci, [P(C.c_ulonglong)]),
        "cgvc_set_option": (ci, [vp, C.c_char_p, ci]),
        "cgvc_profile_enable": (ci, [ci]),
        "cgvc_profile_collect": (ci, [P(C.c_double), P(C.c_double), P(C.c_longlong)]),
        "cgvc_profile_launches": (ci, [P(C.c_double), P(C.c_double), P(C.c_longlong), ci, P(ci)]),
        "cgvc_conv_forward": (ci, [vp, ci, vp, vp, vp, vp] + [ci] * 9 + [vp]),
        "cgvc_conv_backward": (ci, [vp, ci, vp, vp, vp, vp, vp, vp] + [ci] * 9 + [vp]),
        "cgvc_in_glu_forward": (ci, [vp] * 8 + [ci] * 4 + [vp]),
        "cgvc_in_glu_backward": (ci, [vp] * 13 + [ci] * 4 + [vp]),
        "cgvc_split_planes": (ci, [vp, ci, vp, C.c_longlong, ci, vp, vp, vp, vp]),
        "cgvc_im2col_planes": (ci, [vp, ci, vp, C.c_longlong, ci, ci, ci, ci, vp, vp, vp, vp]),
        "cgvc_in_glu_forward_planes": (ci, [vp] * 8 + [ci] * 6 + [vp] * 5),
        "cgvc_in_glu_backward_planes": (ci, [vp] * 13 + [ci] * 6 + [vp] * 4),
        "cgvc_in_glu_forward_packed": (ci, [vp] * 8 + [ci] * 5 + [vp] * 2 + [ci] * 3 + [vp] * 4),
        "cgvc_in_glu_backward_bias": (ci, [vp] * 15 + [ci] * 6 + [vp] * 4),
        "cgvc_conv_in_forward": (ci, [vp, ci] + [vp] * 15 + [ci] * 8 + [P(ci), vp]),
        "cgvc_conv_in_backward": (ci, [vp, ci] + [vp] * 16 + [ci] * 8 + [P(ci), vp]),
        "cgvc_glu_forward_planes": (ci, [vp] * 3 + [ci] * 4 + [vp] * 4),
        "cgvc_glu_backward_planes": (ci, [vp] * 6 + [ci] * 4 + [vp] * 4),
        "cgvc_disc_input_forward": (ci, [vp, ci] + [vp] * 10 + [ci] * 9 + [P(ci), vp]),
        "cgvc_disc_input_backward": (ci, [vp] * 11 + [ci] * 9 + [P(ci), vp]),
        "cgvc_head_forward": (ci, [vp, vp, C.c_longlong, vp, vp, vp, vp]),
        "cgvc_head_loss_backward": (ci, [vp, vp, vp, C.c_longlong, vp, cf, cf] + [vp] * 6),
        "cgvc_head_backward": (ci, [vp, vp, vp, C.c_longlong] + [vp] * 7),
        "cgvc_l1_loss_grad": (ci, [vp, vp, vp, C.c_longlong] + [vp] * 4 + [ci, vp]),
        "cgvc_edge_h1_forward": (ci, [vp, ci, vp, ci, ci] + [vp] * 6),
        "cgvc_edge_o1_forward": (ci, [vp, ci, vp, ci, ci] + [vp] * 4),
        "cgvc_edge_o1_backward": (ci, [vp, ci, vp, vp, ci, ci] + [vp] * 4),
        "cgvc_edge_h1_backward": (ci, [vp, ci, vp, vp, vp, ci, ci] + [vp] * 4),
        "cgvc_tape_bytes": (ci, [vp, ci, ci, ci, P(sz)]),
        "cgvc_generator_forward_tape": (ci, [vp, ci, vp, vp, ci, ci, vp, sz, vp]),
        "cgvc_generator_forward_packed_tape": (ci, [vp, ci, vp, vp, P(C.c_longlong), ci, vp, sz, vp]),
        "cgvc_discriminator_forward_packed_tape": (ci, [vp, ci, vp, vp, P(C.c_longlong), ci, vp, sz, vp]),
        "cgvc_discriminator_forward_tape": (ci, [vp, ci, vp, vp, ci, ci, vp, sz, vp]),
        "cgvc_generator_backward_tape": (ci, [vp, vp, vp, vp, vp]),
        "cgvc_discriminator_backward_tape": (ci, [vp, vp, vp, vp, vp]),
    }
    for name, (res, args) in sig.items():
        fn = getattr(lib, name)          # AttributeError here = the library does not export a declared symbol
        fn.restype = res
        fn.argtypes = args
    return sig


EXPORTED_SYMBOLS = None


def lib_path():
    return _build.LIB


def load(build_if_missing=True):
    """Load libcgvc.so, building it in-tree with nvcc first if it is missing or stale."""
    global _LIB, EXPORTED_SYMBOLS
    if _LIB is not None:
        return _LIB
    path = _build.LIB
    if build_if_missing and _build.is_stale():
        _build.build()
    if not os.path.exists(path):
        raise RuntimeError("libcgvc.so not found at %s (run __graft_entry__.build()); there is no CPU fallback" % path)
    lib = C.CDLL(path, mode=C.RTLD_GLOBAL)
    EXPORTED_SYMBOLS = sorted(_declare(lib).keys())
    if lib.cgvc_abi_version() != 1:
        raise RuntimeError("libcgvc.so ABI version mismatch")
    _LIB = lib
    return lib


def check(handle, code):
    if code != 0:
        msg = _LIB.cgvc_last_error(handle)
        raise CgvcError(code, msg.decode() if msg else "?")
