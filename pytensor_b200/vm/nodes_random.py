"""RandomVariable on the device (reference: pytensor/tensor/random/op.py:49; perform :457-468 = `rng_fn(rng, *params, size)`
on a host numpy Generator, returning (the advanced generator, the draws)).

The generator stays a HOST object: each call takes 128 bits from it (which advances it exactly as a draw would, so the
`updates={rng: next_rng}` contract and copy-vs-inplace semantics are the reference's), and those bits key a counter-based
Philox stream on the device (csrc/ptk_random.cu).  Shapes, dtypes and parameter broadcasting follow the reference; the
VALUES are a different (equally distributed) stream — parity is distributional, see tests/test_gpu_random.py.
A graph with RandomVariable nodes is never captured into a CUDA graph (the key changes on every call)."""

from __future__ import annotations

import copy

import numpy as np

from ..runtime import device as dev
from ..runtime import lib as _lib
from .nodes_basic import _broadcast_view, _err_flag
from .nodes_elemwise import Node
from .values import Val

# reference op name -> (ptk_random_fill code, number of distribution parameters it takes)
DIST = {"uniform": (0, 2), "normal": (1, 2), "halfnormal": (2, 2), "lognormal": (3, 2), "exponential": (4, 1), "laplace": (5, 2),
        "logistic": (6, 2), "gumbel": (7, 2), "cauchy": (8, 2), "bernoulli": (9, 1), "gamma": (10, 2), "beta": (11, 2),
        "integers": (12, 2), "weibull": (13, 1), "pareto": (14, 2), "halfcauchy": (15, 2), "invgamma": (16, 2),
        "studentt": (17, 3), "t": (17, 3)}


def _generator(v: Val):
    g = v.h
    if isinstance(g, np.ndarray):
        g = g.item()
    if not isinstance(g, np.random.Generator):
        raise TypeError(f"RandomVariable: expected a numpy Generator, got {type(g).__name__}")
    return g


# discrete counts through ptk_random_count: reference op name -> (ptk_random_count code, number of parameters)
COUNT = {"poisson": (0, 1), "binomial": (1, 2), "negative_binomial": (2, 2), "geometric": (3, 1), "beta_binomial": (4, 3)}
# row samplers through ptk_random_rows: reference op name -> (ptk_random_rows kind, number of parameters)
ROWS = {"categorical": (0, 1), "multinomial": (1, 2), "dirichlet": (2, 1)}
# samplers whose number of trials NumPy casts to int64 with the "safe" rule (multinomial: only in its unbatched call)
INT_N = ("binomial",)

_PARAM_ERROR = ("{}: a parameter is outside the distribution's domain (or an integer n exceeds 2**53, which the float64 "
                "parameter path cannot carry exactly)")


def _draw_key(vals, inplace):
    """(generator to return, key, seed): 128 bits from the host Generator, which advances as a draw would."""
    gen = _generator(vals[0])
    if not inplace:
        gen = copy.deepcopy(gen)
    key, seed = (int(w) for w in gen.bit_generator.random_raw(2))   # advances the generator: the next call differs
    return gen, key, seed


def _check_int_n(name, t):
    if dev.TORCH_TO_NP[t.dtype].startswith("float"):
        raise TypeError(f"{name}: cannot cast n of dtype {dev.TORCH_TO_NP[t.dtype]} to int64 according to the rule 'safe'")


def _f64(t):
    if dev.TORCH_TO_NP[t.dtype] != "float64":
        from .nodes_cast import cast_to

        t = cast_to(t, "float64")
    return t


def _rows_f64(t, batch, k, keep):
    """float64 parameter rows of length k (k None: one value per row) over the batch shape: (pointer, row stride), the
    stride 0 when one row serves the whole batch."""
    t = _f64(t)
    keep.append(t)
    width = 1 if k is None else k
    if t.numel() == width and t.is_contiguous():
        return dev.ptr(t), 0
    tb = _broadcast_view(t, tuple(batch) + (() if k is None else (k,)))
    tb = tb if tb.is_contiguous() else dev.contiguous(tb)
    keep.append(tb)
    return dev.ptr(tb), width


def _check_broadcast_to(shape, target, what):
    if tuple(np.broadcast_shapes(tuple(shape), tuple(target))) != tuple(target):
        raise ValueError(f"{what}: cannot broadcast a parameter of shape {tuple(shape)} to {tuple(target)}")


class RandomVariableNode(Node):
    def __init__(self, dist_name, dtype, inplace, size_is_none, name="RandomVariable"):
        self.count = dist_name in COUNT   # discrete counts: ptk_random_count with an error word
        self.code, self.n_params = COUNT[dist_name] if self.count else DIST[dist_name]
        self.dist_name, self.dtype, self.inplace, self.size_is_none, self.name = dist_name, dtype, inplace, size_is_none, name

    def run(self, vals):
        if dev.alloc_state.capturing:
            raise dev.GraphUnsupported("random draws are keyed per call")
        gen, key, seed = _draw_key(vals, self.inplace)
        params = vals[2:2 + self.n_params]
        if self.dist_name in INT_N:
            _check_int_n(self.name, params[0].dev())
        pshapes = [tuple(p.shape) for p in params]
        if self.size_is_none:
            shape = tuple(np.broadcast_shapes(*pshapes)) if pshapes else ()
        else:
            shape = tuple(int(s) for s in np.asarray(vals[1].host()).reshape(-1))
            if pshapes:
                np.broadcast_shapes(shape, *pshapes)   # raises like numpy when the parameters do not fit `size`
        n = int(np.prod(shape, dtype=np.int64)) if shape else 1
        out = dev.empty(shape, self.dtype)
        ptrs, strides, keep = [], [], []
        for p in params:
            t = p.dev()
            if dev.TORCH_TO_NP[t.dtype] != "float64":
                from .nodes_cast import cast_to

                t = cast_to(t, "float64")
            if t.numel() == 1:
                ptrs.append(dev.ptr(t))
                strides.append(0)
            else:
                tb = _broadcast_view(t, shape)
                tb = tb if tb.is_contiguous() else dev.contiguous(tb)
                ptrs.append(dev.ptr(tb))
                strides.append(1)
                keep.append(tb)
            keep.append(t)
        while len(ptrs) < 3:
            ptrs.append(None)
            strides.append(0)
        if n and self.count:
            _lib.check(_lib.lib().ptk_random_count(self.code, _lib.DTYPE_CODE[self.dtype], dev.ptr(out), n, key, seed, ptrs[0],
                                                   strides[0], ptrs[1], strides[1], ptrs[2], strides[2],
                                                   _err_flag(_PARAM_ERROR.format(self.name), ValueError), dev.stream_ptr()),
                       "ptk_random_count")
        elif n:
            _lib.check(_lib.lib().ptk_random_fill(self.code, _lib.DTYPE_CODE[self.dtype], dev.ptr(out), n, key, seed, ptrs[0],
                                                  strides[0], ptrs[1], strides[1], ptrs[2], strides[2], dev.stream_ptr()),
                       "ptk_random_fill")
        return [Val(h=gen), Val(d=out)]


class RandomRowsNode(Node):
    """categorical `(p)->()`, multinomial `(),(p)->(p)` and dirichlet `(a)->(a)`: a batch row is k contiguous float64
    parameters (reference rng_fn: pytensor/tensor/random/basic.py, DirichletRV / MultinomialRV / CategoricalRV).  The batch
    shape follows each rng_fn; the draws come from ptk_random_rows."""

    def __init__(self, dist_name, dtype, inplace, size_is_none, name="RandomVariable"):
        self.kind, self.n_params = ROWS[dist_name]
        self.dist_name, self.dtype, self.inplace, self.size_is_none, self.name = dist_name, dtype, inplace, size_is_none, name

    def run(self, vals):
        if dev.alloc_state.capturing:
            raise dev.GraphUnsupported("random draws are keyed per call")
        gen, key, seed = _draw_key(vals, self.inplace)
        params = [v.dev() for v in vals[2:2 + self.n_params]]
        size = None if self.size_is_none else tuple(int(s) for s in np.asarray(vals[1].host()).reshape(-1))
        p = params[-1]
        if p.dim() < 1:
            raise ValueError(f"{self.name}: the probabilities / concentrations need at least one dimension")
        k = int(p.shape[-1])
        pbatch = tuple(p.shape[:-1])
        nv = None
        if self.dist_name == "categorical":
            if size is None:
                batch = pbatch
            else:   # basic.py CategoricalRV.rng_fn: `size` must not broadcast against p's batch shape
                if len(size) < len(pbatch) or any(s == 1 and q != 1 for s, q in zip(reversed(size), reversed(pbatch))):
                    raise ValueError("`size` is incompatible with the shape of `p`")
                batch = tuple(np.broadcast_shapes(size, pbatch))
            out_shape = batch
        elif self.dist_name == "multinomial":
            nv = params[0]
            if size is None and nv.dim() == 0 and p.dim() == 1:
                _check_int_n(self.name, nv)   # NumPy's unbatched call casts n "safe"ly; batched rows truncate a float n
            if size is None:
                batch = tuple(np.broadcast_shapes(tuple(nv.shape), pbatch))
            else:
                batch = size
                _check_broadcast_to(nv.shape, batch, self.name)
                _check_broadcast_to(p.shape, batch + (k,), self.name)
            out_shape = batch + (k,)
        else:
            batch = pbatch if size is None else size
            _check_broadcast_to(p.shape, batch + (k,), self.name)
            out_shape = batch + (k,)
        rows = int(np.prod(batch, dtype=np.int64)) if batch else 1
        out = dev.empty(out_shape, self.dtype)
        if rows and (k or self.dist_name == "categorical"):
            keep = []
            pp, ps = _rows_f64(p, batch, k, keep)
            np_, ns = _rows_f64(nv, batch, None, keep) if nv is not None else (None, 0)
            err = _err_flag(_PARAM_ERROR.format(self.name), ValueError)
            _lib.check(_lib.lib().ptk_random_rows(self.kind, _lib.DTYPE_CODE[self.dtype], dev.ptr(out), rows, k, key, seed,
                                                  pp, ps, np_, ns, err, dev.stream_ptr()), "ptk_random_rows")
        return [Val(h=gen), Val(d=out)]
