"""Device-buffer plumbing.  torch.cuda tensors are used ONLY as containers (allocation through torch's caching
allocator, shape/stride/dtype bookkeeping, views) — never for arithmetic: every byte that moves or changes on the
device does so in a libptk kernel or a cudaMemcpy issued through the C-ABI.
"""

from __future__ import annotations

import ctypes

import numpy as np
import torch

from . import lib as _lib

NP_TO_TORCH = {
    "bool": torch.bool, "int8": torch.int8, "int16": torch.int16, "int32": torch.int32, "int64": torch.int64,
    "uint8": torch.uint8, "uint16": torch.uint16, "uint32": torch.uint32, "uint64": torch.uint64,
    "float16": torch.float16, "float32": torch.float32, "float64": torch.float64,
}
TORCH_TO_NP = {v: k for k, v in NP_TO_TORCH.items()}


def require_cuda() -> None:
    if _lib.TRACE_ONLY:
        return
    if not torch.cuda.is_available():
        raise _lib.PtkError("the CUDA backend needs an H100 (torch.cuda.is_available() is False); there is no CPU fallback")


_device = None


def device() -> torch.device:
    global _device
    if _lib.TRACE_ONLY:
        return torch.device("meta")
    if _device is None:
        require_cuda()
        _lib.init(torch.cuda.current_device())
        _device = torch.device("cuda", torch.cuda.current_device())
        # The backend runs on its own (capturable) stream, which it also makes torch's current stream so that the
        # caching allocator, the caller's torch ops and our kernels are all ordered on one stream. The legacy default
        # stream cannot be captured into a CUDA graph.
        global _vm_stream
        _vm_stream = torch.cuda.Stream(device=_device)
        torch.cuda.set_stream(_vm_stream)
    return _device


_vm_stream = None


def vm_stream():
    device()
    return _vm_stream


def stream_ptr() -> int:
    if _lib.TRACE_ONLY:
        return 0
    return torch.cuda.current_stream().cuda_stream


def is_dev(x) -> bool:
    return isinstance(x, torch.Tensor)


def np_dtype_name(x) -> str:
    if isinstance(x, torch.Tensor):
        return TORCH_TO_NP[x.dtype]
    return np.asarray(x).dtype.name


class GraphUnsupported(RuntimeError):
    """Raised when something that cannot be part of a CUDA graph (a device->host read, a blocking copy) is attempted
    while the VM is capturing; the VM then abandons the capture and runs the call eagerly."""


class Arena:
    """Bump allocator over one device buffer: gives the captured CUDA graph stable addresses (no allocator calls while
    capturing, same pointers on every replay)."""

    ALIGN = 256

    def __init__(self, nbytes: int):
        self.buf = torch.empty((max(int(nbytes), 1),), dtype=torch.uint8, device=device())
        self.off = 0

    def alloc(self, shape, tdtype):
        n = 1
        for s in shape:
            n *= int(s)
        nbytes = n * torch.empty((), dtype=tdtype, device="meta").element_size()
        start = self.off
        self.off = (start + nbytes + self.ALIGN - 1) // self.ALIGN * self.ALIGN
        if self.off > self.buf.numel():
            raise GraphUnsupported("arena exhausted (allocation pattern changed between the measuring run and capture)")
        if nbytes == 0:
            return torch.empty(tuple(shape), dtype=tdtype, device=self.buf.device)
        return self.buf[start:start + nbytes].view(tdtype).view(tuple(shape))


class _AllocState:
    arena = None        # Arena while capturing
    measuring = False   # count bytes of every allocation (the eager run that precedes a capture)
    measured = 0
    capturing = False


alloc_state = _AllocState()


def empty_t(shape, tdtype) -> torch.Tensor:
    """The single device-allocation point of the backend."""
    shape = tuple(int(s) for s in shape)
    st = alloc_state
    if st.arena is not None:
        return st.arena.alloc(shape, tdtype)
    if st.measuring:
        n = 1
        for s in shape:
            n *= s
        nbytes = n * torch.empty((), dtype=tdtype, device="meta").element_size()
        st.measured += (nbytes + Arena.ALIGN - 1) // Arena.ALIGN * Arena.ALIGN + Arena.ALIGN
    return torch.empty(shape, dtype=tdtype, device=device())


def empty(shape, dtype: str) -> torch.Tensor:
    return empty_t(shape, NP_TO_TORCH[dtype])


def empty_like_layout(shape, dtype: str, order) -> torch.Tensor:
    """Dense buffer whose dims are laid out in `order` (a permutation, slowest first); C order = range(ndim)."""
    shape = tuple(int(s) for s in shape)
    if order is None or tuple(order) == tuple(range(len(shape))):
        return empty(shape, dtype)
    perm_shape = [shape[i] for i in order]
    base = empty(perm_shape, dtype)
    inv = [0] * len(order)
    for pos, dim in enumerate(order):
        inv[dim] = pos
    return base.permute(inv)


def ptr(t: torch.Tensor) -> int:
    return t.data_ptr()


def i64_array(values):
    n = max(1, len(values))
    arr = (ctypes.c_int64 * n)(*[int(v) for v in values])
    return arr


def copy_strided(dst: torch.Tensor, src: torch.Tensor) -> None:
    """dst[...] = src[...] (same shape; src may carry 0 strides for broadcast) with the libptk copy kernel."""
    assert dst.dtype == src.dtype and tuple(dst.shape) == tuple(src.shape), (dst.shape, src.shape)
    if dst.numel() == 0:
        return
    L = _lib.lib()
    nd = dst.dim()
    _lib.check(
        L.ptk_copy_strided(ptr(dst), i64_array(dst.stride()), ptr(src), i64_array(src.stride()),
                           i64_array(dst.shape), nd, dst.element_size(), stream_ptr()),
        "ptk_copy_strided",
    )


def contiguous(t: torch.Tensor) -> torch.Tensor:
    """C-contiguous version of `t` (itself when already contiguous); the copy runs in the libptk copy kernel."""
    if t.is_contiguous():
        return t
    out = empty_t(t.shape, t.dtype)
    copy_strided(out, t)
    return out


def clone(t: torch.Tensor) -> torch.Tensor:
    out = empty_t(t.shape, t.dtype)
    copy_strided(out, t)
    return out


def to_device(arr) -> torch.Tensor:
    """Host -> device copy (cudaMemcpyAsync on the current stream; pinned sources stay asynchronous)."""
    if isinstance(arr, torch.Tensor):
        if arr.is_cuda or arr.is_meta:
            return arr
        arr = arr.numpy()
    a = np.asarray(arr)
    if not a.flags.c_contiguous:
        a = np.ascontiguousarray(a)
    out = empty(a.shape, a.dtype.name)
    if a.size and alloc_state.capturing:
        # a host value that is a function of the call signature only (shape integers, constants): upload it NOW on a
        # side stream into its arena slot so that the captured graph finds it there on every replay
        side = _side_stream()
        _lib.check(_lib.lib().ptk_memcpy_h2d_async(ptr(out), a.ctypes.data, a.nbytes, side.cuda_stream), "h2d")
        _lib.check(_lib.lib().ptk_sync_stream(side.cuda_stream), "sync")
        return out
    if a.size:
        _lib.check(_lib.lib().ptk_memcpy_h2d_async(ptr(out), a.ctypes.data, a.nbytes, stream_ptr()), "h2d")
        # The source may be pageable and freed/mutated by the caller right after we return: make the copy complete.
        # (cudaMemcpyAsync from pageable memory has already staged it; for pinned memory we must wait.)
        _lib.check(_lib.lib().ptk_sync_stream(stream_ptr()), "sync")
    return out


_side = None


def _side_stream():
    global _side
    if _side is None:
        _side = torch.cuda.Stream()
    return _side


def to_device_async(arr: np.ndarray, out: torch.Tensor | None = None) -> torch.Tensor:
    """H2D without the trailing synchronise: the caller guarantees `arr` outlives the copy (e.g. pinned staging)."""
    a = np.asarray(arr)
    if not a.flags.c_contiguous:
        a = np.ascontiguousarray(a)
    if out is None:
        out = empty(a.shape, a.dtype.name)
    if a.size:
        _lib.check(_lib.lib().ptk_memcpy_h2d_async(ptr(out), a.ctypes.data, a.nbytes, stream_ptr()), "h2d")
    return out


class _PinnedPool:
    """Page-locked host blocks for function outputs.  A block is handed out inside a NumPy array and returns to the
    pool when that array (and every view of it) has been garbage collected, so each call still yields a fresh object
    (the `no_recycling` contract, pytensor/link/vm.py:860-885) without paying page faults + a pageable D2H per call."""

    MIN_BYTES = 1 << 20

    def __init__(self):
        self.free = {}
        self.total = 0

    def take(self, nbytes):
        cap = 1 << max(20, (int(nbytes) - 1).bit_length())
        lst = self.free.get(cap)
        if lst:
            return lst.pop(), cap
        p = ctypes.c_void_p()
        _lib.check(_lib.lib().ptk_host_alloc_pinned(ctypes.byref(p), cap), "ptk_host_alloc_pinned")
        self.total += cap
        return p.value, cap

    def give(self, ptr, cap):
        self.free.setdefault(cap, []).append(ptr)


_pinned_pool = _PinnedPool()
PINNED_POOL_LIMIT = 8 << 30


def pinned_empty(shape, dtype) -> np.ndarray:
    import weakref

    dt = np.dtype(dtype)
    n = 1
    for s in shape:
        n *= int(s)
    nbytes = n * dt.itemsize
    ptr_, cap = _pinned_pool.take(nbytes)
    buf = (ctypes.c_char * nbytes).from_address(ptr_)
    weakref.finalize(buf, _pinned_pool.give, ptr_, cap)
    return np.frombuffer(buf, dtype=dt).reshape(tuple(int(s) for s in shape))


def host_empty(shape, dtype, always_pinned: bool = False) -> np.ndarray:
    """Host array for a function output: page-locked (pooled) when large enough to matter, else plain NumPy.
    `always_pinned`: also pin small arrays — a device->host copy into pageable memory blocks the calling thread until the
    copy has run, which would stall a software pipeline that wants to keep enqueueing work."""
    dt = np.dtype(dtype)
    nbytes = dt.itemsize
    for s in shape:
        nbytes *= int(s)
    if ((nbytes >= _PinnedPool.MIN_BYTES or (always_pinned and nbytes > 0)) and _pinned_pool.total < PINNED_POOL_LIMIT
            and not _lib.TRACE_ONLY):
        return pinned_empty(tuple(shape), dt)
    return np.empty(tuple(int(s) for s in shape), dtype=dt)


def to_host(t, sync: bool = True) -> np.ndarray:
    """Device -> host copy into a fresh numpy array (C order)."""
    if not isinstance(t, torch.Tensor):
        return np.asarray(t)
    if t.is_meta:
        return np.zeros(tuple(t.shape), dtype=TORCH_TO_NP[t.dtype])
    if alloc_state.capturing:
        raise GraphUnsupported("device->host read inside a graph capture")
    src = contiguous(t)
    out = host_empty(tuple(src.shape), TORCH_TO_NP[src.dtype])
    if out.size:
        _lib.check(_lib.lib().ptk_memcpy_d2h_async(out.ctypes.data, ptr(src), out.nbytes, stream_ptr()), "d2h")
    if sync:
        _lib.check(_lib.lib().ptk_sync_stream(stream_ptr()), "sync")
    return out


def synchronize() -> None:
    _lib.check(_lib.lib().ptk_sync_stream(stream_ptr()), "sync")


def bump_version(t) -> None:
    """Tell torch (and the VM's staged-operand cache, which keys on `Tensor._version`) that `t` was written through a raw
    pointer (a libptk kernel or memcpy)."""
    if isinstance(t, torch.Tensor) and not t.is_meta:
        try:
            torch.autograd.graph.increment_version(t)
        except Exception:  # noqa: BLE001  (inference tensors)
            pass


class unmanaged:
    """Context: allocations inside live outside any capture arena / measuring pass (persistent buffers)."""

    def __enter__(self):
        st = alloc_state
        self._saved = (st.arena, st.measuring)
        st.arena, st.measuring = None, False
        return self

    def __exit__(self, *a):
        alloc_state.arena, alloc_state.measuring = self._saved
