"""CPU check of a scheduling rule that a CUDA kernel implements in index arithmetic (a Python mirror of the device
code; the kernel itself is covered by the -m gpu parity tests):

  * the fused Scan kernel's run-based walk of a circular trace buffer (codegen/scan.py) must write step i to slot
    (L + i) % store, like the reference's circular buffers (pytensor/scan/scan_perform.pyx:544-570).
"""

import numpy as np


def _scan_slots(T, store, L):
    """Mirror of the kernel's phase split + run-based walk: list of (step, slot) writes."""
    writes = []
    i0 = max(0, T - store)            # first step whose result survives
    sl = (L + i0) % store
    i = i0
    while i < T:
        run = min(T - i, store - sl)
        for j in range(run):
            writes.append((i + j, sl + j))
        i += run
        sl += run
        if sl == store:
            sl = 0
    return writes


def test_fused_scan_trace_walk_matches_circular_buffer_rule():
    rng = np.random.default_rng(5)
    for _ in range(2000):
        L = int(rng.integers(1, 4))
        T = int(rng.integers(0, 60))
        store = int(rng.integers(L, L + T + 3))
        writes = _scan_slots(T, store, L)
        assert [w[0] for w in writes] == list(range(max(0, T - store), T))
        for i, slot in writes:
            assert slot == (L + i) % store, (T, store, L, i, slot)


def test_stream_plan_orders_readers_before_an_in_place_writer():
    """`Program.plan_streams` (the capture-time multi-stream schedule) must keep every reader of a buffer ahead of the
    step that overwrites it in place, and may separate independent branches — the role `fgraph.orderings()` /
    destroy-handler dependencies play for the reference's VMs (pytensor/link/utils.py:831-847)."""
    from helpers import pytensor

    import pytensor.tensor as pt

    pytensor.config.floatX = "float32"
    x, y = pt.fmatrix("x"), pt.fmatrix("y")
    a = pt.dot(x, y)
    f = pytensor.function([x, y], [a.sum(axis=0), pt.exp(a) * 2, pt.dot(x.T, x).max()], mode="CUDA")
    p = f.vm.executor.program
    p.plan_streams()
    names = [type(st.impl).__name__ for st in p.steps]
    writer = next(i for i, st in enumerate(p.steps) if getattr(st.impl, "destroy", None))
    victim = p.steps[writer].ins[p.steps[writer].impl.destroy[0]]           # the slot overwritten in place
    readers = [i for i, st in enumerate(p.steps) if victim in st.ins and i != writer]
    assert readers, names
    closure, todo = set(), list(p.deps[writer])
    while todo:                                                                # transitive dependencies of the writer
        d = todo.pop()
        if d not in closure:
            closure.add(d)
            todo.extend(p.deps[d])
    assert all(r in closure for r in readers), (names, p.deps)
    # the two matrix products are independent: they land on different streams of the captured graph
    dots = [i for i, n in enumerate(names) if n == "Dot22Node"]
    assert len(dots) == 2 and p.stream_of[dots[0]] != p.stream_of[dots[1]]
    # every true data dependency is present
    producer = {o: i for i, st in enumerate(p.steps) for o in st.outs}
    for i, st in enumerate(p.steps):
        for s in st.ins:
            if s in producer:
                assert producer[s] in p.deps[i]
