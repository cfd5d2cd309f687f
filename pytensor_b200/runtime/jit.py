"""NVRTC-backed kernel cache.

The reference compiles one C++ module per Apply node with g++ and caches it on disk keyed by op/type signature
(pytensor/link/c/cmodule.py:612 ModuleCache, :1181-1260 module_from_key).  The H100 analogue: one sm_90a cubin per
generated kernel source, cached in memory per process and on disk keyed by the SHA-256 of (architecture, source,
options).  Two disk caches: the in-tree `_kcache/` that `__graft_entry__.build()` fills (read-only afterwards, so that a
run from a read-only tree still starts with cache hits) and a per-user directory under the system temporary directory
(PTK_KCACHE overrides it) that receives everything compiled at run time.  A cached cubin is trusted by its file name, so
the shared-temp default is used only when it is a real directory owned by this user and closed to everyone else (it is
created with mode 0700); otherwise kernels compiled at run time are cached in memory only.
"""

from __future__ import annotations

import ctypes
import hashlib
import os
import stat
import tempfile
import threading

from . import lib as _lib

ARCH = "sm_90a"  # the architecture ptk_jit_compile targets (csrc/ptk_runtime.cu)
BUILD_CACHE_DIR = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "_kcache")
DEFAULT_CACHE_DIR = os.path.join(tempfile.gettempdir(), f"ptk_kcache_{os.getuid()}")
CACHE_DIR = os.environ.get("PTK_KCACHE") or DEFAULT_CACHE_DIR

_lock = threading.Lock()
_cubins: dict[str, bytes] = {}
_modules: dict[str, int] = {}
_functions: dict[tuple[str, str], int] = {}
stats = {"compiled": 0, "disk_hits": 0, "mem_hits": 0, "launches": 0}


def _key(src: str, opts: tuple[str, ...]) -> str:
    h = hashlib.sha256()
    h.update(("ptk-jit-v2\0" + ARCH + "\0" + "\0".join(opts) + "\0").encode())
    h.update(src.encode())
    return h.hexdigest()[:32]


def _usable_cache_dir() -> str | None:
    """CACHE_DIR, created (mode 0700) if missing; None when it is the shared-temp default but not a directory that only
    this user can write (someone else could have planted cubins there)."""
    d = CACHE_DIR
    try:
        os.makedirs(d, mode=0o700, exist_ok=True)
        st = os.lstat(d)
    except OSError:
        return None
    if d == DEFAULT_CACHE_DIR and (not stat.S_ISDIR(st.st_mode) or st.st_uid != os.getuid() or st.st_mode & 0o077):
        return None
    return d


def compile_cubin(src: str, opts: tuple[str, ...] = ()) -> tuple[str, bytes]:
    """Source -> (key, cubin bytes). Needs no GPU (NVRTC cross-compiles), so it also runs in the CPU-only build check."""
    key = _key(src, opts)
    with _lock:
        if key in _cubins:
            stats["mem_hits"] += 1
            return key, _cubins[key]
    cache_dir = _usable_cache_dir()
    candidates = [os.path.join(BUILD_CACHE_DIR, key + ".cubin")]
    if cache_dir is not None:
        candidates.insert(0, os.path.join(cache_dir, key + ".cubin"))
    for p in dict.fromkeys(candidates):
        if os.path.exists(p):
            with open(p, "rb") as f:
                data = f.read()
            with _lock:
                _cubins[key] = data
                stats["disk_hits"] += 1
            return key, data
    L = _lib.load_library()
    cubin = ctypes.c_void_p()
    size = ctypes.c_size_t()
    log = ctypes.c_void_p()
    c_opts = (ctypes.c_char_p * max(1, len(opts)))(*[o.encode() for o in opts])
    st = L.ptk_jit_compile(src.encode(), c_opts, len(opts), ctypes.byref(cubin), ctypes.byref(size), ctypes.byref(log))
    log_txt = ""
    if log.value:
        log_txt = ctypes.string_at(log.value).decode("utf-8", "replace")
        L.ptk_free(log)
    if st != 0:
        numbered = "\n".join(f"{i + 1:4d}: {line}" for i, line in enumerate(src.split("\n")))
        raise _lib.PtkError(f"NVRTC failed: {_lib.last_error()}\n{log_txt}\n--- source ---\n{numbered}")
    data = ctypes.string_at(cubin.value, size.value)
    L.ptk_free(cubin)
    if cache_dir is not None:
        try:
            path = os.path.join(cache_dir, key + ".cubin")
            tmp = path + f".tmp{os.getpid()}"
            with open(tmp, "wb") as f:
                f.write(data)
            os.replace(tmp, path)
            with open(os.path.join(cache_dir, key + ".cu"), "w") as f:
                f.write(src)
        except OSError:
            pass
    with _lock:
        _cubins[key] = data
        stats["compiled"] += 1
    return key, data


def get_function(src: str, name: str, opts: tuple[str, ...] = ()) -> int:
    """Source + kernel name -> CUfunction handle (loads the module on the current device on first use)."""
    key, data = compile_cubin(src, opts)
    fkey = (key, name)
    f = _functions.get(fkey)
    if f is not None:
        return f
    L = _lib.lib()
    with _lock:
        mod = _modules.get(key)
        if mod is None:
            m = ctypes.c_void_p()
            buf = ctypes.create_string_buffer(data, len(data))
            _lib.check(L.ptk_module_load(buf, len(data), ctypes.byref(m)), "ptk_module_load")
            mod = m.value
            _modules[key] = mod
        fn = ctypes.c_void_p()
        _lib.check(L.ptk_module_get_function(mod, name.encode(), ctypes.byref(fn)), f"get_function({name})")
        _functions[fkey] = fn.value
    return fn.value


def get_function_gen(gen, prefix: str, opts: tuple[str, ...] = ()):
    """`gen(kernel_name) -> source`.  The kernel is named after the hash of its own source so that the same generated
    kernel has the same name (and disk-cache key) in every process — cubins built by `build()` are hits on the GPU box.
    Returns (function handle, kernel name)."""
    placeholder = "PTKKERNELNAMEPLACEHOLDER"
    src = gen(placeholder)
    name = f"{prefix}_{hashlib.sha256(src.encode()).hexdigest()[:16]}"
    src = src.replace(placeholder, name)
    if _lib.TRACE_ONLY:
        compile_cubin(src, opts)
        return 0, name
    return get_function(src, name, opts), name


def precompile_gen(gen, prefix: str, opts: tuple[str, ...] = ()) -> str:
    """CPU-side half of get_function_gen (NVRTC only, no device): used by build() to warm the disk cache."""
    placeholder = "PTKKERNELNAMEPLACEHOLDER"
    src = gen(placeholder)
    name = f"{prefix}_{hashlib.sha256(src.encode()).hexdigest()[:16]}"
    compile_cubin(src.replace(placeholder, name), opts)
    return name


class KernelArgs:
    """Packs kernel parameters for ptk_launch: keeps the ctypes scalars alive and exposes the void*[] array."""

    __slots__ = ("_vals", "array")

    def __init__(self, vals):
        self._vals = vals
        n = len(vals)
        self.array = (ctypes.c_void_p * n)(*[ctypes.cast(ctypes.pointer(v), ctypes.c_void_p) for v in vals])


def launch(func: int, grid, block, args: KernelArgs, smem: int = 0, stream: int = 0, cooperative: bool = False,
           cluster: int = 1) -> None:
    gx, gy, gz = (tuple(grid) + (1, 1))[:3]
    bx, by, bz = (tuple(block) + (1, 1))[:3]
    stats["launches"] += 1
    if _lib.TRACE_ONLY:
        return
    _lib.check(
        _lib.lib().ptk_launch(func, gx, gy, gz, bx, by, bz, smem, stream, args.array, 1 if cooperative else 0, cluster),
        "ptk_launch",
    )
