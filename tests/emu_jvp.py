"""Test-only numpy emulation of forward-mode plans (``cotengra_b200/jvp.py``) on top of
``tests/desc_emulator.py`` and ``tests/emu_absorb.py``: the records of a ``JvpPlan`` walked the way
``ctgb_plan_execute_jvp`` runs them -- NaN-filled arenas of exactly the reported bytes, slice digits,
input / tangent / output views, two-term nodes as both products into one C, the primal root skipped
without ``out``.  NOT a fallback: never imported by the product.
"""

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L
from tests import desc_emulator as emu
from tests.emu_absorb import emulate_absorb


def emulate_jvp(plan, arrays, tangents, slice_ids=None, primal=True):
    """``(out, tangent_out)`` of the slices ``slice_ids`` (default all) for ``tangents``, one per input
    in ``plan.wrt``; ``tangent_out`` alone with ``primal=False``."""
    assert not plan.wide, "the emulator sums in the plan dtype"
    dt = np.dtype(plan.dtype)
    es = plan.esize
    assert plan.workspace_bytes % es == 0 and plan.persistent_bytes % es == 0
    persistent = np.full(plan.persistent_bytes // es, np.nan, dtype=dt)
    scratch = np.full(plan.workspace_bytes // es, np.nan, dtype=dt)
    out = np.zeros(max(plan.out_elements, 1), dtype=dt)
    tout = np.zeros(max(plan.out_elements, 1), dtype=dt)
    flats = [np.ascontiguousarray(a, dtype=dt).reshape(-1) for a in arrays]
    tflats = [None] * len(arrays)
    assert len(tangents) == len(plan.wrt)
    for i, t in zip(plan.wrt, tangents):
        tflats[i] = np.ascontiguousarray(t, dtype=dt).reshape(-1)
    ns = len(plan.sliced)
    radix = [s for _i, s, _p in plan.sliced]
    proj = [p for _i, _s, p in plan.sliced]

    def view(t, digits, out_off):
        if t.kind in (X.K_INPUT, X.K_TANGENT):
            off = sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride))
            src = (flats if t.kind == X.K_INPUT else tflats)[t.input_index]
            assert src is not None, "a tangent slot of an input outside wrt"
            return src[off:]
        if t.kind in (X.K_SCRATCH, X.K_PERSISTENT):
            assert t.offset % es == 0
            return (scratch if t.kind == X.K_SCRATCH else persistent)[t.offset // es:]
        assert t.kind in (X.K_OUTPUT, X.K_TOUT), t.kind
        return (out if t.kind == X.K_OUTPUT else tout)[out_off:]

    def run(phase, digits, out_off):
        for nd in plan.nodes:
            if nd["phase"] != phase or (nd.get("root") == 1 and not primal):
                continue
            v = lambda t: view(t, digits, out_off)  # noqa: E731
            c = v(nd["c"])
            if nd["kind"] == 2:
                w = np.asarray(nd["words"])[:L.DESC_WORDS]
                emu.emulate_pair(w, v(nd["a"]), v(nd["b"]), c)
                w2 = w.copy()
                w2[L.W_FLAGS] |= 1
                emu.emulate_pair(w2, v(nd["a2"]), v(nd["b2"]), c)
            elif nd.get("d") is not None:
                emulate_absorb(nd["words"], v(nd["a"]), v(nd["d"]), v(nd["b"]), c)
            elif nd["kind"] == 0:
                emu.emulate_pair(nd["words"], v(nd["a"]), v(nd["b"]), c)
            else:
                emu.emulate_single(nd["words"], v(nd["a"]), c)

    run(X.PHASE_INV_FWD, [0] * ns, 0)
    strides = [1] * ns
    for j in range(ns - 2, -1, -1):
        strides[j] = strides[j + 1] * radix[j + 1]
    for i in range(plan.nslices) if slice_ids is None else slice_ids:
        digits, rem = [0] * ns, i
        for j in range(ns):
            if proj[j] is not None:
                digits[j] = proj[j]
            else:
                digits[j], rem = rem // strides[j], rem % strides[j]
        run(X.PHASE_VAR_FWD, digits, sum(d * s for d, s in zip(digits, plan.slice_out_stride)))
    shape = lambda x: x[: plan.out_elements].reshape(plan.out_shape)  # noqa: E731
    return (shape(out), shape(tout)) if primal else shape(tout)


def jvp_oracle(spec, contractions, arrays, tangents, wrt, slice_ids=None):
    """The exact JVP of a multilinear tree: ``sum_{i in wrt} f(x_1, ..., v_i, ..., x_n)`` through the
    torch-CPU oracle (``oracle/grad_oracle.py``), in the arrays' dtype."""
    import torch

    from oracle import grad_oracle as go

    total = 0
    for i, t in zip(wrt, tangents):
        xs = [torch.tensor(t if j == i else a) for j, a in enumerate(arrays)]
        total = total + go.contract_tree(spec.inputs, spec.output, spec.sliced, contractions, xs,
                                         slice_ids=slice_ids).detach().numpy()
    return np.asarray(total)
