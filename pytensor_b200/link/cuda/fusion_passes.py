"""Peephole passes over the lowered step list (see fusion.py)."""

from __future__ import annotations

from pytensor_b200.vm.nodes_blas import Dot22Node, GemmBiasActNode, MlpChainNode
from pytensor_b200.vm.nodes_elemwise import CAReduceNode, ElemwiseNode, ElemwiseReduceNode
from pytensor_b200.vm.vm import Step


def _bias_act_pattern(ew: ElemwiseNode):
    """(dot_input_idx, bias_input_idx, act) if `ew` computes act(i_dot + i_bias) with a (1,N)-broadcast bias."""
    p = ew.prog
    if ew.ndim != 2 or len(p.in_dtypes) != 2 or len(p.out_dtypes) != 1 or len(set(p.in_dtypes + p.out_dtypes)) != 1:
        return None
    ops = [i.op for i in p.insts]
    if ops not in (["Add"], ["Add", "Tanh"]):
        return None
    add = p.insts[0]
    if sorted(add.args) != [("i", 0), ("i", 1)]:
        return None
    if len(ops) == 2 and (p.insts[1].args != [("t", 0)] or p.outputs != [("t", 1)]):
        return None
    if len(ops) == 1 and p.outputs != [("t", 0)]:
        return None
    bc = ew.in_bcast
    if bc[0] == (False, False) and bc[1] == (True, False):
        d, b = 0, 1
    elif bc[1] == (False, False) and bc[0] == (True, False):
        d, b = 1, 0
    else:
        return None
    return d, b, (1 if len(ops) == 2 else 0)


def fuse_gemm_epilogue(steps, output_slots, opts):
    """Dot22 -> Elemwise{act(x + bias)} (the only reader of the product) ==> one GemmBiasActNode step (K5)."""
    readers = {}
    for i, st in enumerate(steps):
        for s in st.ins:
            readers.setdefault(s, []).append(i)
    outset = set(output_slots)
    drop, repl = set(), {}
    for i, st in enumerate(steps):
        if type(st.impl) is not Dot22Node or st.impl.scalar:
            continue
        s = st.outs[0]
        rd = readers.get(s, [])
        if len(rd) != 1 or s in outset:
            continue
        j = rd[0]
        ew = steps[j]
        if type(ew.impl) is not ElemwiseNode:
            continue
        pw = ew.impl.prog
        if (ew.impl.ndim == 2 and len(pw.in_dtypes) == 1 and [q.op for q in pw.insts] == ["Tanh"] and pw.outputs == [("t", 0)]
                and pw.insts[0].args == [("i", 0)] and pw.out_dtypes == [st.impl.dtype] and pw.in_dtypes == [st.impl.dtype]
                and tuple(ew.impl.in_bcast[0]) == (False, False)):
            # tanh(A @ B) without a bias: the same epilogue with a null bias pointer
            node = GemmBiasActNode(st.impl.dtype, st.impl.precision, 1, name=f"{st.impl.name}+{ew.impl.name}[fused epilogue]")
            repl[i] = Step(node, [st.ins[0], st.ins[1]], list(ew.outs), origin=ew.origin)
            drop.add(j)
            continue
        pat = _bias_act_pattern(ew.impl)
        if pat is None or ew.ins[pat[0]] != s or ew.impl.prog.out_dtypes[0] != st.impl.dtype:
            continue
        # the Elemwise must come after the Dot22 and nothing between them may produce the bias later than the Dot22
        bias_slot = ew.ins[pat[1]]
        producers = {o: k for k, t in enumerate(steps) for o in t.outs}
        if producers.get(bias_slot, -1) > i:
            continue
        node = GemmBiasActNode(st.impl.dtype, st.impl.precision, pat[2], name=f"{st.impl.name}+{ew.impl.name}[fused epilogue]")
        repl[i] = Step(node, [st.ins[0], st.ins[1], bias_slot], list(ew.outs), origin=ew.origin)
        drop.add(j)
    if repl:
        steps = [repl.get(i, st) for i, st in enumerate(steps) if i not in drop]
    return mark_bf16_chains(steps)


def mark_bf16_chains(steps):
    """A tensor-core GEMM whose result is the A operand of another tensor-core GEMM also emits it staged as that operand
    (a nodes_blas.Staged carried as `Val.aux`), so the chain re-stages only the weights (SURVEY.md §8d cfg 3)."""
    tc = (Dot22Node, GemmBiasActNode)
    producers = {o: st for st in steps for o in st.outs}
    for st in steps:
        if isinstance(st.impl, tc) and st.impl.dtype == "float32":
            src = producers.get(st.ins[0])
            # bf16 mode: a bf16 copy; fp32-accurate mode: the three-piece split (used when the weights are resident)
            if src is not None and isinstance(src.impl, tc) and src.impl.precision == st.impl.precision \
                    and src.impl.dtype == "float32":
                src.impl.emit_bf16 = True
    return steps


def fuse_elemwise_reduce(steps, output_slots, opts):
    """Elemwise -> CAReduce(trailing axes) of one of its outputs ==> one ElemwiseReduceNode step.

    Safe when: the CAReduce is the ONLY step between the two that touches the Elemwise's outputs or destroys any of
    its inputs (we simply require the CAReduce to be scheduled anywhere later and move it up next to the Elemwise:
    it only reads that one slot), and the reduced slot has no float16/complex dtype issues (same kernels as before).
    """
    readers = {}
    for i, st in enumerate(steps):
        for s in st.ins:
            readers.setdefault(s, []).append(i)
    outset = set(output_slots)
    fused_away = set()
    new_steps = []
    for i, st in enumerate(steps):
        if i in fused_away:
            continue
        impl = st.impl
        if type(impl) is ElemwiseNode:
            cand = None
            for k, s in enumerate(st.outs):
                for j in readers.get(s, []):
                    r = steps[j]
                    if (type(r.impl) is CAReduceNode and j not in fused_away and r.impl.ndim == impl.ndim
                            and impl.ndim > 0 and r.impl.axes
                            and tuple(r.impl.axes) == tuple(range(impl.ndim - len(r.impl.axes), impl.ndim))
                            and r.impl.in_dtype == impl.prog.out_dtypes[k]):
                        cand = (k, s, j)
                        break
                if cand:
                    break
            if cand is not None:
                k, s, j = cand
                others = [x for x in readers.get(s, []) if x != j]
                store = bool(others) or (s in outset)
                node = ElemwiseReduceNode(impl, steps[j].impl, k, store_reduced_input=store)
                new_steps.append(Step(node, st.ins, list(st.outs) + list(steps[j].outs), origin=st.origin))
                fused_away.add(j)
                continue
        new_steps.append(st)
    return new_steps


def fuse_small_mlp_chains(steps, output_slots, opts, min_layers=4):
    """Runs of >= `min_layers` dense layers, each product read only by the next one as its A operand ==> one MlpChainNode
    step at the position of the run's LAST layer (every weight / bias slot is available there).  Whether the chain
    executes as one launch is decided per call from the actual shapes (MlpChainNode)."""
    dense = (Dot22Node, GemmBiasActNode)
    readers, producer = {}, {}
    for i, st in enumerate(steps):
        for s in st.ins:
            readers.setdefault(s, []).append(i)
        for o in st.outs:
            producer[o] = i
    outset = set(output_slots)

    def is_layer(st):
        return type(st.impl) in dense and not getattr(st.impl, "scalar", False) and st.impl.dtype == "float32"

    nxt = {}
    for i, st in enumerate(steps):
        if not is_layer(st):
            continue
        o = st.outs[0]
        rd = readers.get(o, [])
        if o in outset or len(rd) != 1:
            continue
        j = rd[0]
        if j > i and is_layer(steps[j]) and steps[j].ins[0] == o and o not in steps[j].ins[1:]:
            nxt[i] = j
    heads = set(nxt) - set(nxt.values())
    repl, drop = {}, set()
    for hd in sorted(heads):
        chain = [hd]
        while chain[-1] in nxt:
            chain.append(nxt[chain[-1]])
        if len(chain) < min_layers:
            continue
        ins = [steps[chain[0]].ins[0]]
        layers = []
        for i in chain:
            st = steps[i]
            has_bias = type(st.impl) is GemmBiasActNode and len(st.ins) > 2
            ins += [st.ins[1]] + ([st.ins[2]] if has_bias else [])
            layers.append((st.impl, has_bias))
        last = chain[-1]
        # every other input must exist before the first layer's A operand does NOT matter: the fused step sits at `last`,
        # after every constituent step, hence after everything any of them read
        node = MlpChainNode(layers, name=f"MlpChain[{len(chain)} layers]")
        repl[last] = Step(node, ins, list(steps[last].outs), origin=steps[last].origin)
        drop.update(chain[:-1])
    if not repl:
        return steps
    return [repl.get(i, st) for i, st in enumerate(steps) if i not in drop]
