"""Test-only numpy emulation of absorb-root nodes (``VAR_ABSORB_ROOT``, csrc/absorbdot.cuh), on top of
``tests/desc_emulator.py``: the node's word tables walked as the kernel reads them, and the forward
plans that hold such nodes.  NOT a fallback: never imported by the product.
"""

import math

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L
from tests import desc_emulator as emu


def emulate_absorb(W, A, Bs, V, C):
    """C (flat, modified in place) (+)= the absorb-root node ``W`` (``lowering.build_absorb_desc``):
    R[r, n] = sum_{k', c} (sum_k A[r, k', k] Bs[k, ck(r), c]) V[k', c, n] through the word tables."""
    W = np.asarray(W)
    assert W[L.W_MAGIC] == L.DESC_MAGIC and int(W[L.W_VARIANT]) == L.VAR_ABSORB_ROOT
    N, K, CC, CCP, KL, NG = (int(W[i]) for i in (L.AB_N, L.AB_K, L.AB_C, L.AB_CCP, L.AB_KL, L.AB_NG))
    grid = [tuple(int(x) for x in W[L.AB_G + 4 * j:L.AB_G + 4 * j + 4]) for j in range(NG)]
    units = int(W[L.AB_UNITS])
    assert units == math.prod(g[0] for g in grid)
    u = np.arange(units, dtype=np.int64)
    kA = sum((u // g[1]) % g[0] * g[2] for g in grid) + np.zeros(units, dtype=np.int64)
    kV = sum((u // g[1]) % g[0] * g[3] for g in grid) + np.zeros(units, dtype=np.int64)
    kA = (kA[:, None] + np.arange(KL) * int(W[L.AB_KLA])).reshape(-1)  # every k' of the node
    kV = (kV[:, None] + np.arange(KL) * int(W[L.AB_KLV])).reshape(-1)
    ma, mc = W[L.AB_TMA:L.AB_TMA + 32], W[L.AB_TMC:L.AB_TMC + 32]
    nv, nc = W[L.AB_TNV:L.AB_TNV + N], W[L.AB_TNC:L.AB_TNC + N]
    ka, kb = W[L.AB_TKA:L.AB_TKA + K], W[L.AB_TKB:L.AB_TKB + K]
    tcb, cv = W[L.AB_TCB:L.AB_TCB + 128], W[L.AB_TCV:L.AB_TCV + CC]
    Vt = V[kV[:, None, None] + cv[None, :, None] + nv[None, None, :]]  # [k', c, n]
    accumulate = bool(W[L.W_FLAGS] & 1)
    for r in range(32):
        if mc[r] < 0:
            continue
        ck = int(W[L.AB_TBCK + r // 8])
        cols = tcb[ck * CCP:ck * CCP + CC]
        assert (cols >= 0).all()
        a = A[ma[r] + kA[:, None] + ka[None, :]]                     # [k', k]
        x = a @ Bs[kb[:, None] + cols[None, :]]                      # [k', c]
        row = np.einsum("qc,qcn->n", x, Vt)
        dst = mc[r] + nc
        C[dst] = C[dst] + row if accumulate else row


def emulate_plan(plan, arrays, slice_ids=None):
    """``desc_emulator.emulate_plan`` for forward plans that may hold absorb-root nodes (which only
    unstripped forward plans do): the same arenas (NaN-filled, exactly the reported bytes), slice
    digits, views and phases, with the absorb-root node reading its A, Bs and V."""
    if not any(nd.get("d") is not None for nd in plan.nodes):
        return emu.emulate_plan(plan, arrays, slice_ids=slice_ids)
    assert not plan.strip_exponent and not getattr(plan, "wide", False)
    dt = np.dtype(plan.dtype)
    es = plan.esize
    persistent = np.full(plan.persistent_bytes // es, np.nan, dtype=dt)
    scratch = np.full(plan.workspace_bytes // es, np.nan, dtype=dt)
    out = np.zeros(max(plan.out_elements, 1), dtype=dt)
    flats = [np.ascontiguousarray(a, dtype=dt).reshape(-1) for a in arrays]
    ns = len(plan.sliced)
    radix = [s for _i, s, _p in plan.sliced]
    proj = [p for _i, _s, p in plan.sliced]

    def view(t, digits, out_off):
        if t.kind == X.K_INPUT:
            return flats[t.input_index][sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride)):]
        if t.kind in (X.K_SCRATCH, X.K_PERSISTENT):
            assert t.offset % es == 0
            return (scratch if t.kind == X.K_SCRATCH else persistent)[t.offset // es:]
        assert t.kind == X.K_OUTPUT
        return out[out_off:]

    def run(phase, digits, out_off):
        for nd in plan.nodes:
            if nd["phase"] != phase:
                continue
            a, c = view(nd["a"], digits, out_off), view(nd["c"], digits, out_off)
            if nd.get("d") is not None:
                emulate_absorb(nd["words"], a, view(nd["d"], digits, out_off), view(nd["b"], digits, out_off), c)
            elif nd["kind"] == 0:
                emu.emulate_pair(nd["words"], a, view(nd["b"], digits, out_off), c)
            else:
                emu.emulate_single(nd["words"], a, c)

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
    return out[: plan.out_elements].reshape(plan.out_shape)
