"""ctypes binding of libfcsa_b200.so - the declarations of include/fcsa_b200.h, nothing more.

This plays the role of the reference's pybind11 module import
(flash_cosine_sim_attention.py:15-23).  There the import failure was swallowed with a printed
hint and the package then broke later; here a missing or unloadable library raises
immediately and there is no other code path (no CPU fallback).
"""
import ctypes
import os
from ctypes import POINTER, Structure, byref, c_char_p, c_float, c_int32, c_int64, c_size_t, c_void_p

FCSA_F16 = 0
FCSA_BF16 = 1

FCSA_OK = 0
FCSA_ERR_INVALID = 1
FCSA_ERR_UNSUPPORTED = 2
FCSA_ERR_CUDA = 3
FCSA_ERR_WORKSPACE = 4

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libfcsa_b200.so")

# every symbol include/fcsa_b200.h declares (tests check the library exports exactly these)
EXPORTED_SYMBOLS = (
    "fcsa_version",
    "fcsa_last_error",
    "fcsa_debug",
    "fcsa_forward",
    "fcsa_backward_workspace_bytes",
    "fcsa_backward_zeroed_bytes",
    "fcsa_zeroed_init",
    "fcsa_backward",
    "fcsa_l2norm_forward",
    "fcsa_l2norm_backward",
    "fcsa_set_kernel_events",
    "fcsa_forward_fused",
    "fcsa_backward_fused",
    "fcsa_forward_bias",
    "fcsa_backward_bias",
    "fcsa_f32_cast",
    "fcsa_f32_cast_backward",
    "fcsa_decode_workspace_bytes",
    "fcsa_decode",
    "fcsa_decode_varlen_workspace_bytes",
    "fcsa_decode_varlen",
    "fcsa_decode_rolling_workspace_bytes",
    "fcsa_decode_rolling",
    "fcsa_forward_fused_varlen",
    "fcsa_backward_fused_varlen_workspace_bytes",
    "fcsa_backward_fused_varlen_zeroed_bytes",
    "fcsa_backward_fused_varlen",
    "fcsa_backward_fused_deterministic_workspace_bytes",
    "fcsa_backward_fused_deterministic",
    "fcsa_backward_fused_deterministic_varlen_workspace_bytes",
    "fcsa_backward_fused_deterministic_varlen",
)


class FcsaTensor(Structure):
    _fields_ = [("ptr", c_void_p), ("sb", c_int64), ("sh", c_int64), ("sn", c_int64)]


class FcsaProblem(Structure):
    _fields_ = [
        ("dtype", c_int32),
        ("batch", c_int32),
        ("heads", c_int32),
        ("kv_heads", c_int32),
        ("seq_q", c_int32),
        ("seq_k", c_int32),
        ("head_dim", c_int32),
        ("causal", c_int32),
        ("scale", c_float),
        ("shift", c_float),
        ("key_mask", c_void_p),
        ("key_mask_stride", c_int64),
        ("out_f32", c_int32),
        ("window", c_int32),
    ]


class FcsaL2Norm(Structure):
    _fields_ = [("groups", c_int32), ("q_hat", FcsaTensor), ("k_hat", FcsaTensor), ("q_rnorm", c_void_p),
                ("k_rnorm", c_void_p)]


class FcsaBias(Structure):
    _fields_ = [("ptr", c_void_p), ("sb", c_int64), ("sh", c_int64), ("sn", c_int64), ("amax", c_void_p)]


class FcsaVarlen(Structure):
    _fields_ = [("cu_seqlens_q", c_void_p), ("cu_seqlens_k", c_void_p), ("total_q", c_int32), ("total_k", c_int32)]


class FcsaError(RuntimeError):
    def __init__(self, code, message):
        super().__init__(f"libfcsa_b200 error {code}: {message}")
        self.code = code


_lib = None


def load():
    """Load (once) and return the ctypes handle.  Raises if the library is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise ImportError(
            f"{LIB_PATH} is missing: build it with `python -m flash_cosine_sim_attention_b200.build` "
            "(needs nvcc; sm_90a only).  There is no CPU fallback."
        )
    lib = ctypes.CDLL(LIB_PATH)
    PT = POINTER(FcsaTensor)
    PP = POINTER(FcsaProblem)
    lib.fcsa_version.restype = c_int32
    lib.fcsa_version.argtypes = []
    lib.fcsa_last_error.restype = c_char_p
    lib.fcsa_last_error.argtypes = []
    lib.fcsa_debug.restype = c_int64
    lib.fcsa_debug.argtypes = []
    lib.fcsa_forward.restype = c_int32
    lib.fcsa_forward.argtypes = [PP, PT, PT, PT, PT, c_void_p, c_void_p]
    lib.fcsa_backward_workspace_bytes.restype = c_size_t
    lib.fcsa_backward_workspace_bytes.argtypes = [PP]
    lib.fcsa_backward.restype = c_int32
    lib.fcsa_backward_zeroed_bytes.restype = c_size_t
    lib.fcsa_backward_zeroed_bytes.argtypes = [PP]
    lib.fcsa_zeroed_init.restype = c_int32
    lib.fcsa_zeroed_init.argtypes = [c_void_p, c_size_t, c_void_p]
    lib.fcsa_backward.argtypes = [PP, PT, PT, PT, PT, PT, c_void_p, PT, PT, PT, c_void_p, c_size_t, c_void_p, c_size_t,
                                  c_void_p]
    lib.fcsa_l2norm_forward.restype = c_int32
    lib.fcsa_l2norm_forward.argtypes = [c_int32] * 6 + [PT, PT, c_void_p, c_void_p]
    lib.fcsa_l2norm_backward.restype = c_int32
    lib.fcsa_l2norm_backward.argtypes = [c_int32] * 6 + [PT, PT, c_void_p, PT, c_void_p]
    PN = POINTER(FcsaL2Norm)
    lib.fcsa_forward_fused.restype = c_int32
    lib.fcsa_forward_fused.argtypes = [PP, PT, PT, PT, PN, PT, c_void_p, c_void_p]
    lib.fcsa_backward_fused.restype = c_int32
    lib.fcsa_backward_fused.argtypes = [PP, PN, PT, PT, PT, c_void_p, PT, PT, PT, c_void_p, c_size_t, c_void_p, c_size_t,
                                        c_void_p]
    PB = POINTER(FcsaBias)
    lib.fcsa_forward_bias.restype = c_int32
    lib.fcsa_forward_bias.argtypes = [PP, PT, PT, PT, PB, PT, c_void_p, c_void_p]
    lib.fcsa_backward_bias.restype = c_int32
    lib.fcsa_backward_bias.argtypes = [PP, PT, PT, PT, PT, PT, c_void_p, PB, c_void_p, c_int64, c_int64,
                                       PT, PT, PT, c_void_p, c_size_t, c_void_p, c_size_t, c_void_p]
    lib.fcsa_f32_cast.restype = c_int32
    lib.fcsa_f32_cast.argtypes = [c_int32] * 6 + [PT, PT, c_void_p, c_void_p, c_int32, c_void_p]
    lib.fcsa_f32_cast_backward.restype = c_int32
    lib.fcsa_f32_cast_backward.argtypes = [c_int32] * 6 + [PT, PT, c_void_p, PT, c_void_p, c_int32, c_void_p]
    lib.fcsa_decode_workspace_bytes.restype = c_size_t
    lib.fcsa_decode_workspace_bytes.argtypes = [PP, c_int32]
    lib.fcsa_decode.restype = c_int32
    lib.fcsa_decode.argtypes = [PP, PT, PT, PT, c_void_p, PT, PT, c_int32, c_int32, PT, c_void_p, c_size_t, c_void_p]
    lib.fcsa_decode_varlen_workspace_bytes.restype = c_size_t
    lib.fcsa_decode_varlen_workspace_bytes.argtypes = [PP, c_int32]
    lib.fcsa_decode_varlen.restype = c_int32
    lib.fcsa_decode_varlen.argtypes = [PP, c_void_p, c_int32, PT, PT, PT, c_void_p, PT, PT, c_int32, PT, c_void_p,
                                       c_size_t, c_void_p]
    lib.fcsa_decode_rolling_workspace_bytes.restype = c_size_t
    lib.fcsa_decode_rolling_workspace_bytes.argtypes = [PP, c_void_p, c_int32]
    lib.fcsa_decode_rolling.restype = c_int32
    lib.fcsa_decode_rolling.argtypes = [PP, c_void_p, c_int32, PT, PT, PT, c_void_p, PT, PT, c_int32, PT, c_void_p,
                                        c_size_t, c_void_p]
    PV = POINTER(FcsaVarlen)
    lib.fcsa_forward_fused_varlen.restype = c_int32
    lib.fcsa_forward_fused_varlen.argtypes = [PP, PV, PT, PT, PT, PN, PT, c_void_p, c_void_p]
    lib.fcsa_backward_fused_varlen_workspace_bytes.restype = c_size_t
    lib.fcsa_backward_fused_varlen_workspace_bytes.argtypes = [PP, PV]
    lib.fcsa_backward_fused_varlen_zeroed_bytes.restype = c_size_t
    lib.fcsa_backward_fused_varlen_zeroed_bytes.argtypes = [PP, PV]
    lib.fcsa_backward_fused_varlen.restype = c_int32
    lib.fcsa_backward_fused_varlen.argtypes = [PP, PV, PN, PT, PT, PT, c_void_p, PT, PT, PT, c_void_p, c_size_t,
                                               c_void_p, c_size_t, c_void_p]
    lib.fcsa_backward_fused_deterministic_workspace_bytes.restype = c_size_t
    lib.fcsa_backward_fused_deterministic_workspace_bytes.argtypes = [PP]
    lib.fcsa_backward_fused_deterministic.restype = c_int32
    lib.fcsa_backward_fused_deterministic.argtypes = [PP, PN, PT, PT, PT, c_void_p, PT, PT, PT, c_void_p, c_size_t,
                                                      c_void_p]
    lib.fcsa_backward_fused_deterministic_varlen_workspace_bytes.restype = c_size_t
    lib.fcsa_backward_fused_deterministic_varlen_workspace_bytes.argtypes = [PP, PV]
    lib.fcsa_backward_fused_deterministic_varlen.restype = c_int32
    lib.fcsa_backward_fused_deterministic_varlen.argtypes = [PP, PV, PN, PT, PT, PT, c_void_p, PT, PT, PT, c_void_p,
                                                             c_size_t, c_void_p]
    lib.fcsa_set_kernel_events.restype = c_int32
    lib.fcsa_set_kernel_events.argtypes = [c_int32, c_void_p, c_void_p]
    _lib = lib
    return lib


def check(code):
    if code != FCSA_OK:
        msg = load().fcsa_last_error()
        raise FcsaError(code, msg.decode() if msg else "")


def ref(x):
    return byref(x)
