"""Values held in the CUDA VM's storage cells.

A `Val` is what a storage cell (`storage_map[var][0]`, pytensor/link/utils.py:40-141) holds under the CUDALinker:
a device buffer (torch.cuda tensor used as a container), a host array, or both views of the same data.  Host copies
exist only for (a) function inputs as the caller handed them over, (b) constants, (c) integer shape plumbing
(`Shape_i`, `MakeVector`, slice bounds, `n_steps`) that sizes allocations and launches and therefore has to be known
on the host.  Floating-point tensor math never happens on the host.
"""

from __future__ import annotations

import numpy as np
import torch

from ..runtime import device as dev


class Val:
    __slots__ = ("h", "d", "aux", "key", "fresh")

    def __init__(self, h=None, d=None, aux=None, key=None, fresh=False):
        self.h = h
        self.d = d
        # optional companion of `d`: the same matrix staged as the A operand of the next tensor-core product
        # (a nodes_blas.Staged written by the epilogue of the product that computed `d`), or None
        self.aux = aux
        # identity of the CONTENT when the VM knows it cannot have changed since it last saw this key (a graph constant;
        # a caller-owned device tensor that is the same object at the same torch version as in the previous calls):
        # lets a tensor-core GEMM reuse the staged copy of a weight matrix instead of re-staging it (nodes_blas.py)
        self.key = key
        # `h` was filled for this call alone (the chunked host pipeline's page-locked results): handed out without a copy
        self.fresh = fresh

    # ---- metadata without forcing a transfer ----
    @property
    def shape(self):
        return tuple(self.d.shape) if self.d is not None else tuple(np.shape(self.h))

    @property
    def ndim(self):
        return self.d.dim() if self.d is not None else np.ndim(self.h)

    @property
    def dtype(self) -> str:
        return dev.TORCH_TO_NP[self.d.dtype] if self.d is not None else np.asarray(self.h).dtype.name

    @property
    def size(self) -> int:
        n = 1
        for s in self.shape:
            n *= int(s)
        return n

    def on_host(self) -> bool:
        return self.h is not None

    def on_dev(self) -> bool:
        return self.d is not None

    # ---- materialisation (cached) ----
    def dev(self) -> torch.Tensor:
        if self.d is None:
            self.d = dev.to_device(np.asarray(self.h))
        return self.d

    def host(self) -> np.ndarray:
        if self.h is None:
            self.h = dev.to_host(self.d)
        return self.h

    def item(self):
        return self.host().item() if isinstance(self.host(), np.ndarray) else self.host()

    def __repr__(self):
        where = ("H" if self.h is not None else "") + ("D" if self.d is not None else "")
        return f"Val<{where} {self.dtype}{list(self.shape)}>"


def wrap(x) -> Val:
    """Anything the caller put in an input cell -> Val (no copy, no transfer)."""
    if isinstance(x, Val):
        return x
    if isinstance(x, torch.Tensor):
        if x.is_cuda or x.is_meta:
            return Val(d=x)
        return Val(h=x.numpy())
    if isinstance(x, np.random.Generator):
        return Val(h=x)   # RNG state stays a host object (vm/nodes_random.py)
    return Val(h=np.asarray(x))
