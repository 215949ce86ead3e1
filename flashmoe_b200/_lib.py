"""ctypes binding of the C-ABI in include/flashmoe_b200.h (the only way Python reaches the CUDA code).

There is NO CPU or eager fallback: if the native library is missing or fails to load, every entry point raises.
"""
from __future__ import annotations

import ctypes
from pathlib import Path
from typing import Optional

from . import config as _config

LIB_PATH = Path(__file__).resolve().parent / "libflashmoe_b200.so"
FM_MAX_WORLD = 16
FM_IPC_HANDLE_BYTES = 64
FM_HOST_SLOTS = 3

# enum fm_buffer
BUF_TOPK_IDX, BUF_TOPK_W, BUF_MCW, BUF_SLOT, BUF_COUNTS, BUF_RECV_X, BUF_HIDDEN, BUF_RET_Y, BUF_GATE_OUT, BUF_RECV_CNT, BUF_TRACE, BUF_AUX_LOSS = range(12)
BUF_SHARED_Y = 12
BUF_SHARED_HIDDEN = 13

# every symbol include/flashmoe_b200.h declares (tests check the library exports all of them)
EXPORTED_SYMBOLS = (
    "fm_compiled_config", "fm_create", "fm_destroy", "fm_get_dims", "fm_num_local_experts", "fm_symm_size",
    "fm_symm_local_ptr", "fm_symm_export", "fm_symm_attach_ipc", "fm_symm_attach_ptrs", "fm_symm_use_external",
    "fm_moe_forward", "fm_moe_forward_tokens", "fm_moe_forward_tokens_dev", "fm_moe_forward_routed", "fm_moe_forward_gated", "fm_shared_reserve", "fm_moe_forward_shared", "fm_last_launch", "fm_output_buffer", "fm_moe_forward_host", "fm_host_submit", "fm_host_wait", "fm_check", "fm_set_timeout_ms", "fm_set_trace", "fm_set_weight_on_input", "fm_launch_count",
    "fm_buffer_bytes",
    "fm_read_buffer", "fm_last_error", "fm_version",
)


class FmConfig(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in _config.ALL_KEYS]

    @classmethod
    def from_config(cls, cfg: _config.MoEConfig) -> "FmConfig":
        return cls(**cfg.raw())

    def to_config(self) -> _config.MoEConfig:
        return _config.MoEConfig(**{k: int(getattr(self, k)) for k in _config.ALL_KEYS})


class FmDims(ctypes.Structure):
    _fields_ = [(k, ctypes.c_int32) for k in (
        "S", "H", "E", "P", "PX", "element_size", "k", "EC", "pEC", "TCM", "world", "rank", "num_local_experts",
        "num_sms", "smem_bytes", "grid")]


class FmRouter(ctypes.Structure):
    """fm_router_t: the router rule of fm_moe_forward_gated (flashmoe_b200.router.RouterSpec builds one)."""
    _fields_ = [("scoring", ctypes.c_int32), ("n_group", ctypes.c_int32), ("topk_group", ctypes.c_int32),
                ("group_top", ctypes.c_int32), ("renormalize", ctypes.c_int32), ("scale", ctypes.c_float)]


class FmSharedExpert(ctypes.Structure):
    """fm_shared_expert_t: the shared expert of fm_moe_forward_shared (device pointers and its intermediate size Ps)."""
    _fields_ = [("w", ctypes.c_void_p), ("bias_up", ctypes.c_void_p), ("bias_down", ctypes.c_void_p),
                ("inter", ctypes.c_int32)]


_lib: Optional[ctypes.CDLL] = None


def load() -> ctypes.CDLL:
    """Load libflashmoe_b200.so; raises RuntimeError (never falls back) when it is missing."""
    global _lib
    if _lib is not None:
        return _lib
    if not LIB_PATH.exists():
        raise RuntimeError(
            f"native library {LIB_PATH} not found: build it with `python -m flashmoe_b200._build` "
            "(there is no CPU fallback for the MoE forward path)")
    L = ctypes.CDLL(str(LIB_PATH))
    vp, cvp = ctypes.c_void_p, ctypes.c_void_p
    L.fm_last_error.restype = ctypes.c_char_p
    L.fm_version.restype = ctypes.c_char_p
    L.fm_compiled_config.argtypes = [ctypes.POINTER(FmConfig)]
    L.fm_create.argtypes = [ctypes.POINTER(FmConfig), ctypes.c_int, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp)]
    L.fm_destroy.argtypes = [vp]
    L.fm_get_dims.argtypes = [vp, ctypes.POINTER(FmDims)]
    L.fm_num_local_experts.argtypes = [vp]
    L.fm_symm_size.argtypes = [vp, ctypes.POINTER(ctypes.c_size_t)]
    L.fm_symm_local_ptr.argtypes = [vp, ctypes.POINTER(vp)]
    L.fm_symm_export.argtypes = [vp, vp]
    L.fm_symm_attach_ipc.argtypes = [vp, cvp]
    L.fm_symm_attach_ptrs.argtypes = [vp, ctypes.POINTER(vp)]
    L.fm_symm_use_external.argtypes = [vp, vp, ctypes.c_size_t]
    L.fm_moe_forward.argtypes = [vp, cvp, cvp, cvp, cvp, cvp, vp, vp]
    L.fm_moe_forward_tokens.argtypes = [vp, cvp, ctypes.c_int, cvp, cvp, cvp, cvp, vp, vp]
    L.fm_moe_forward_tokens_dev.argtypes = [vp, cvp, cvp, cvp, cvp, cvp, cvp, vp, vp]
    L.fm_moe_forward_routed.argtypes = [vp, cvp, ctypes.c_int, cvp, cvp, cvp, cvp, cvp, cvp, vp, vp]
    L.fm_moe_forward_gated.argtypes = [vp, cvp, ctypes.c_int, cvp, cvp, ctypes.POINTER(FmRouter), cvp, cvp, cvp, cvp,
                                       vp, vp]
    L.fm_shared_reserve.argtypes = [vp, ctypes.c_int32]
    L.fm_moe_forward_shared.argtypes = [vp, cvp, ctypes.c_int, cvp, cvp, ctypes.POINTER(FmRouter), cvp, cvp, cvp, cvp,
                                        cvp, cvp, ctypes.POINTER(FmSharedExpert), vp, vp]
    L.fm_last_launch.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_int32)]
    L.fm_moe_forward_host.argtypes = [vp, cvp, cvp, cvp, cvp, cvp, vp, vp]
    L.fm_output_buffer.argtypes = [vp, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_size_t)]
    L.fm_host_submit.argtypes = [vp, cvp, cvp, cvp, cvp, cvp, vp, vp, ctypes.POINTER(ctypes.c_uint64)]
    L.fm_host_wait.argtypes = [vp, ctypes.c_uint64]
    L.fm_check.argtypes = [vp]
    L.fm_set_timeout_ms.argtypes = [vp, ctypes.c_uint32]
    L.fm_set_trace.argtypes = [vp, ctypes.c_int]
    L.fm_set_weight_on_input.argtypes = [vp, ctypes.c_int]
    L.fm_launch_count.argtypes = [vp]
    L.fm_launch_count.restype = ctypes.c_uint64
    L.fm_buffer_bytes.argtypes = [vp, ctypes.c_int, ctypes.POINTER(ctypes.c_size_t)]
    L.fm_read_buffer.argtypes = [vp, ctypes.c_int, vp, ctypes.c_size_t]
    for name in EXPORTED_SYMBOLS:
        fn = getattr(L, name)
        if fn.restype is ctypes.c_int or name not in ("fm_last_error", "fm_version", "fm_launch_count"):
            fn.restype = ctypes.c_int
    _lib = L
    return L


class FlashMoEError(RuntimeError):
    """A C-ABI call returned a negative status; the message is fm_last_error()."""

    def __init__(self, code: int, message: str):
        super().__init__(f"[flashmoe_b200 {code}] {message}")
        self.code = code


def check(rc: int) -> int:
    if rc < 0:
        raise FlashMoEError(rc, load().fm_last_error().decode(errors="replace"))
    return rc


def compiled_config() -> _config.MoEConfig:
    c = FmConfig()
    check(load().fm_compiled_config(ctypes.byref(c)))
    return c.to_config()
