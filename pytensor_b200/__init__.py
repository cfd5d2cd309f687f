"""pytensor_b200 — an H100-native (sm_90a) graph-execution backend for PyTensor.

    import pytensor_b200            # registers mode="CUDA" / "CUDA_BF16" with the host PyTensor
    f = pytensor.function([x], y, mode="CUDA")

Layout: `csrc/` hand-written CUDA + the C-ABI (libptk.so), `runtime/` ctypes + NVRTC cache + device buffers,
`codegen/` scalar-graph -> CUDA source, `vm/` executable nodes + VM (pytensor-free), `link/cuda/` the Linker plugin.
"""

__version__ = "0.1.0"


def register():
    from pytensor_b200._host import ensure_pytensor

    ensure_pytensor()
    from pytensor_b200.link import cuda

    cuda.register()
    return cuda


def shared(value, **kwargs):
    """Device-resident `pytensor.shared` (see pytensor_b200/sharedvar.py)."""
    from pytensor_b200.sharedvar import shared as _shared

    return _shared(value, **kwargs)


try:  # registration is best-effort at import: the runtime/vm layers work without the host framework
    register()
except ImportError:  # pragma: no cover - host not present
    pass
