"""CPU suite: the discrete-count and row samplers (poisson, binomial, negative_binomial, geometric, beta_binomial,
categorical, multinomial, dirichlet) lower to device random nodes, and their launch logic runs in trace-only mode; the
samplers without a device implementation stay compile-time errors."""

import numpy as np
import pytest

from helpers import pytensor

import pytensor.tensor as pt
from pytensor.graph.traversal import graph_inputs
from pytensor_b200.precompile import trace_function

R = pt.random

CASES = [
    ("poisson", lambda r: R.poisson(pt.dvector("lam"), size=(4, 3), rng=r), [np.ones(3)], "RandomVariableNode"),
    ("binomial", lambda r: R.binomial(pt.lvector("n"), 0.3, rng=r), [np.arange(5, dtype="int64")], "RandomVariableNode"),
    ("negative_binomial", lambda r: R.negative_binomial(2.5, pt.dvector("p"), rng=r), [np.full(3, 0.4)], "RandomVariableNode"),
    ("geometric", lambda r: R.geometric(0.2, size=(7,), rng=r), [], "RandomVariableNode"),
    ("beta_binomial", lambda r: R.betabinom(10, 2.0, pt.dvector("b"), rng=r), [np.ones(2)], "RandomVariableNode"),
    ("categorical", lambda r: R.categorical(pt.dmatrix("p"), rng=r), [np.full((3, 4), 0.25)], "RandomRowsNode"),
    ("multinomial", lambda r: R.multinomial(pt.lvector("n"), np.full(4, 0.25), rng=r), [np.arange(3, dtype="int64")],
     "RandomRowsNode"),
    ("dirichlet", lambda r: R.dirichlet(pt.dvector("a"), size=(5,), rng=r), [np.ones(4)], "RandomRowsNode"),
]


@pytest.mark.parametrize("name,build,args,node", CASES, ids=[c[0] for c in CASES])
def test_discrete_and_row_samplers_lower_to_device_nodes(name, build, args, node):
    pytensor.config.floatX = "float64"
    rng = pytensor.shared(np.random.default_rng(3), name="rng")
    nr, x = build(rng).owner.outputs
    ins = [v for v in graph_inputs([x]) if isinstance(v, pt.TensorVariable) and not isinstance(v, pt.TensorConstant)]
    f = pytensor.function(ins, x, updates={rng: nr}, mode="CUDA")
    steps = [type(st.impl).__name__ for st in f.vm.executor.program.steps]
    assert node in steps, steps
    trace_function(f, args)


@pytest.mark.parametrize("build", [
    lambda r: R.multivariate_normal(np.zeros(2), np.eye(2), rng=r),
    lambda r: R.hypergeometric(5, 3, 4, rng=r),
    lambda r: R.vonmises(0.0, 1.0, rng=r),
], ids=["multivariate_normal", "hypergeometric", "vonmises"])
def test_samplers_without_a_device_implementation_stay_compile_time_errors(build):
    rng = pytensor.shared(np.random.default_rng(3), name="rng")
    with pytest.raises(NotImplementedError, match="no device sampler"):
        pytensor.function([], build(rng), mode="CUDA")
