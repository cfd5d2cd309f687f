"""ctypes binding of libptk.so (the C-ABI declared in include/ptk.h).

There is exactly one way to compute in this package: through these entry points.  If the shared library is missing
or no H100 is present, every compute call raises — there is no CPU or PyTorch fallback anywhere in the product path.
"""

from __future__ import annotations

import ctypes
import os
import threading
from ctypes import POINTER, byref, c_char_p, c_double, c_float, c_int, c_int64, c_size_t, c_uint, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libptk.so")


class PtkError(RuntimeError):
    """An error reported by libptk (status != 0)."""


# dtype codes of include/ptk.h
DTYPE_CODE = {
    "bool": 0, "int8": 1, "int16": 2, "int32": 3, "int64": 4,
    "uint8": 5, "uint16": 6, "uint32": 7, "uint64": 8,
    "float16": 9, "float32": 10, "float64": 11,
}

_i64p = POINTER(c_int64)

# name -> (restype, argtypes); every symbol include/ptk.h declares must be listed here (tests check both ways).
SIGNATURES = {
    "ptk_version": (c_int, []),
    "ptk_last_error": (c_char_p, []),
    "ptk_init": (c_int, [c_int]),
    "ptk_sm_count": (c_int, []),
    "ptk_device": (c_int, []),
    "ptk_sync_stream": (c_int, [c_void_p]),
    "ptk_memcpy_h2d_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptk_memcpy_d2h_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptk_memcpy_d2d_async": (c_int, [c_void_p, c_void_p, c_size_t, c_void_p]),
    "ptk_memset_async": (c_int, [c_void_p, c_int, c_size_t, c_void_p]),
    "ptk_host_alloc_pinned": (c_int, [POINTER(c_void_p), c_size_t]),
    "ptk_host_free_pinned": (c_int, [c_void_p]),
    "ptk_jit_compile": (c_int, [c_char_p, POINTER(c_char_p), c_int, POINTER(c_void_p), POINTER(c_size_t),
                                POINTER(c_void_p)]),
    "ptk_free": (None, [c_void_p]),
    "ptk_module_load": (c_int, [c_void_p, c_size_t, POINTER(c_void_p)]),
    "ptk_module_unload": (c_int, [c_void_p]),
    "ptk_module_get_function": (c_int, [c_void_p, c_char_p, POINTER(c_void_p)]),
    "ptk_func_set_max_dynamic_smem": (c_int, [c_void_p, c_int]),
    "ptk_func_max_active_blocks": (c_int, [c_void_p, c_int, c_int, POINTER(c_int)]),
    "ptk_launch": (c_int, [c_void_p, c_uint, c_uint, c_uint, c_uint, c_uint, c_uint, c_uint, c_void_p,
                           POINTER(c_void_p), c_int, c_int]),
    "ptk_graph_begin_capture": (c_int, [c_void_p]),
    "ptk_graph_end_capture": (c_int, [c_void_p, POINTER(c_void_p)]),
    "ptk_graph_launch": (c_int, [c_void_p, c_void_p]),
    "ptk_graph_destroy": (c_int, [c_void_p]),
    "ptk_event_create": (c_int, [POINTER(c_void_p)]),
    "ptk_event_record": (c_int, [c_void_p, c_void_p]),
    "ptk_event_elapsed_ms": (c_int, [c_void_p, c_void_p, POINTER(c_float)]),
    "ptk_event_destroy": (c_int, [c_void_p]),
    "ptk_stream_wait_event": (c_int, [c_void_p, c_void_p]),
    "ptk_copy_strided": (c_int, [c_void_p, _i64p, c_void_p, _i64p, _i64p, c_int, c_int, c_void_p]),
    "ptk_inc_strided": (c_int, [c_void_p, _i64p, c_void_p, _i64p, _i64p, c_int, c_int, c_int, c_void_p]),
    "ptk_take": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_void_p,
                         c_void_p]),
    "ptk_put": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_void_p,
                        c_void_p]),
    "ptk_put_rows_workspace_bytes": (c_size_t, [c_int64, c_int64]),
    "ptk_put_rows": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_void_p, c_size_t, c_void_p,
                             c_void_p]),
    "ptk_linearize_index": (c_int, [c_int, POINTER(c_void_p), _i64p, c_int64, c_void_p, c_void_p, c_void_p]),
    "ptk_nonzero_workspace_bytes": (c_size_t, [c_int64]),
    "ptk_nonzero_count": (c_int, [c_void_p, c_int64, c_void_p, c_size_t, c_void_p]),
    "ptk_nonzero_fill": (c_int, [c_void_p, c_int64, c_void_p, c_void_p, c_void_p]),
    "ptk_random_fill": (c_int, [c_int, c_int, c_void_p, c_int64, ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_int64, c_void_p,
                                c_int64, c_void_p, c_int64, c_void_p]),
    "ptk_random_count": (c_int, [c_int, c_int, c_void_p, c_int64, ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_int64,
                                 c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_void_p]),
    "ptk_random_rows": (c_int, [c_int, c_int, c_void_p, c_int64, c_int64, ctypes.c_uint64, ctypes.c_uint64, c_void_p, c_int64,
                                c_void_p, c_int64, c_void_p, c_void_p]),
    "ptk_arange": (c_int, [c_int, c_void_p, c_int64, c_double, c_double, c_int64, c_int64, c_void_p]),
    "ptk_argmax": (c_int, [c_int, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "ptk_cumop": (c_int, [c_int, c_int, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_void_p]),
    "ptk_gemm_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64, c_int]),
    "ptk_gemm": (c_int, [c_int, c_int64, c_int64, c_int64, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int64,
                         c_int64, c_double, c_void_p, c_int64, c_int64, c_int, c_void_p, c_size_t, c_void_p]),
    "ptk_gemm_bias_act": (c_int, [c_int, c_int64, c_int64, c_int64, c_void_p, c_int64, c_int64, c_void_p, c_int64,
                                  c_int64, c_void_p, c_int, c_void_p, c_int64, c_int64, c_int, c_void_p, c_size_t,
                                  c_void_p]),
    "ptk_gemm_tc_ex": (c_int, [c_int64, c_int64, c_int64, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_void_p,
                               c_int64, c_int64, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int, c_void_p, c_int64,
                               c_void_p, c_size_t, c_void_p]),
    "ptk_gemm_split_workspace_bytes": (c_size_t, [c_int64, c_int64, c_int64]),
    "ptk_gemm_tc_split": (c_int, [c_int64, c_int64, c_int64, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64,
                                  c_double, c_void_p, c_int64, c_int64, c_void_p, c_int, c_int, c_void_p, c_size_t, c_void_p]),
    "ptk_stage_bytes": (c_size_t, [c_int64, c_int64, c_int]),
    "ptk_stage_operand": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_void_p, c_int64, c_int64,
                                  c_void_p]),
    "ptk_gemm_tc_staged": (c_int, [c_int64, c_int64, c_int64, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_int64,
                                   c_int, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int, c_void_p, c_int64, c_int64,
                                   c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "ptk_gemm_exact_main_default": (c_int, []),
    "ptk_gemm_lead_bits": (c_int, [c_int64]),
    "ptk_mlp_chain": (c_int, [c_void_p, c_int64, c_void_p, c_int64, c_int64, c_int, POINTER(c_void_p), POINTER(c_void_p),
                              POINTER(c_int), POINTER(c_int), POINTER(c_int), c_void_p]),
    "ptk_gemv": (c_int, [c_int, c_int64, c_int64, c_double, c_void_p, c_int64, c_int64, c_void_p, c_int64, c_double,
                         c_void_p, c_int64, c_void_p]),
    "ptk_ger": (c_int, [c_int, c_int64, c_int64, c_double, c_void_p, c_int64, c_void_p, c_int64, c_void_p, c_int64,
                        c_int64, c_void_p]),
    "ptk_allreduce_oneshot_buffer_bytes": (c_size_t, [c_int, c_int64, c_int]),
    "ptk_allreduce_oneshot": (c_int, [c_int, c_void_p, c_void_p, c_int64, POINTER(ctypes.c_uint64), c_int, c_int, c_int64,
                                      c_void_p, c_void_p]),
    "ptk_potrf": (c_int, [c_int, c_void_p, c_int64, c_int64, c_int, c_void_p]),
    "ptk_trsm": (c_int, [c_int, c_void_p, c_void_p, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_void_p]),
    "ptk_potrs": (c_int, [c_int, c_void_p, c_void_p, c_int64, c_int64, c_int, c_int, _i64p, _i64p, c_void_p]),
}

_lock = threading.Lock()
_lib = None
_inited_device = None

# Trace-only mode (build-time): no device, no arithmetic, no results.  Buffers are torch "meta" tensors and every
# C-ABI call is skipped; the only effect of running a function is that the kernels it WOULD launch get generated and
# compiled by NVRTC into the on-disk cubin cache.  Used by __graft_entry__.build() (CPU-only box) and by the CPU test
# suite to exercise the launch logic.  It is not an execution path: outputs are meaningless zeros.
TRACE_ONLY = os.environ.get("PTK_TRACE_ONLY") == "1"


class _TraceLib:
    def __getattr__(self, name):
        if name == "ptk_sm_count":
            return lambda: 132  # H100 SXM
        if name == "ptk_put_rows_workspace_bytes":
            return lambda n_dst, n_idx: 4 * (n_dst + 1 + n_idx) + 64
        if name == "ptk_stage_bytes":
            return lambda r, c, p: (r if p <= 1 else 3 * ((r + 255) // 256 * 256)) * ((c + 7) // 8 * 8) * 2 + 512 + 4 * r
        if name == "ptk_gemm_exact_main_default":
            return lambda: 1
        if name == "ptk_gemm_lead_bits":
            return lambda K: 7
        if name == "ptk_nonzero_workspace_bytes":
            return lambda n: 8 * ((n + 4095) // 4096 + 1)
        if name == "ptk_last_error":
            return lambda: b""
        return lambda *a, **k: 0


def set_trace_only(flag: bool) -> None:
    global TRACE_ONLY
    TRACE_ONLY = bool(flag)


def load_library() -> ctypes.CDLL:
    """dlopen libptk.so and attach prototypes.  Does not touch the GPU (safe on a CPU-only box)."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise PtkError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(make -C pytensor_b200/csrc). The CUDA backend has no fallback path."
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError here = header/library drift; tests pin this
            fn.restype = res
            fn.argtypes = args
        _lib = lib
    return _lib


def last_error() -> str:
    msg = load_library().ptk_last_error()
    return msg.decode("utf-8", "replace") if msg else ""


def check(status: int, what: str = "") -> None:
    if status != 0:
        raise PtkError(f"{what + ': ' if what else ''}{last_error()} (status {status})")


def init(device: int | None = None) -> ctypes.CDLL:
    """Load the library and bind it to `device` (default: torch's current CUDA device). Raises without a GPU."""
    global _inited_device
    lib = load_library()
    if device is None:
        device = int(os.environ.get("LOCAL_RANK", "0")) if _inited_device is None else _inited_device
    if _inited_device == device:
        return lib
    check(lib.ptk_init(int(device)), "ptk_init")
    _inited_device = device
    return lib


def lib() -> ctypes.CDLL:
    """The initialised library (initialises on first use)."""
    if TRACE_ONLY:
        return _TraceLib()
    if _inited_device is None:
        return init()
    return _lib


def sm_count() -> int:
    return int(lib().ptk_sm_count())


__all__ = [
    "PtkError", "DTYPE_CODE", "SIGNATURES", "LIB_PATH", "load_library", "init", "lib", "check", "last_error",
    "sm_count", "byref", "c_void_p", "c_int", "c_int64", "c_double", "c_float", "c_size_t",
]
