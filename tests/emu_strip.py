"""Test-only numpy model of a stripped reverse-mode plan (``VjpPlan(strip_exponent=True,
stripped_grad=True)``) run the way ``ctgb_plan_execute`` runs it, and an emulated device launch for
it (on top of ``tests/emu_device.py``).

The lazy scheme of the plan: one factor slot per tensor slot (1.0 unless a phase 0/1 pairwise node
records max|C| there), the seed slot ``n_tensors`` set per slice after phase 1 to
``10^(e - e'_s)`` (0 for a zero slice or result, NaN for a NaN exponent), and every node's product
divided by its two slots of ``plan.scale_slots`` (1/0 counts as 0).  The descriptors themselves are
walked by ``tests/desc_emulator.py``.  The arenas are exactly the reported bytes and filled with
NaN, as in ``desc_emulator.emulate_plan``.  NOT a fallback: never imported by the product.
"""

import math

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L
from tests import desc_emulator as emu
from tests import emu_device


def emulate_stripped_vjp(plan, arrays, cotangent, exponent, slice_ids=None, grads=None):
    """The gradients of the mantissa for the cotangent ``cotangent`` and the forward's exponent
    ``exponent``, over the slices ``slice_ids`` (default all); ``None`` outside ``plan.wrt``."""
    assert plan.strip_exponent and plan.scale_slots is not None
    dt = np.dtype(plan.dtype)
    es = plan.esize
    persistent = np.full(plan.persistent_bytes // es, np.nan, dtype=dt)
    scratch = np.full(plan.workspace_bytes // es, np.nan, dtype=dt)
    flats = [np.ascontiguousarray(a, dtype=dt).reshape(-1) for a in arrays]
    if grads is None:
        grads = [np.zeros(a.size, dtype=dt) if i in plan.wrt else None for i, a in enumerate(flats)]
    cot = np.ascontiguousarray(cotangent, dtype=dt).reshape(-1)
    if plan.cotangent_offset >= 0:
        o = plan.cotangent_offset // es
        persistent[o:o + cot.size] = np.conj(cot)
        cot = persistent[o:o + cot.size]
    seed = len(plan.tensors)
    factors = np.ones(seed + 2)
    slot_of = {id(t): i for i, t in enumerate(plan.tensors)}
    slot_a, slot_b = plan.scale_slots

    def view(t, digits, out_off):
        if t.kind in (X.K_INPUT, X.K_GRAD):
            off = sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride))
            return (flats if t.kind == X.K_INPUT else grads)[t.input_index][off:]
        if t.kind in (X.K_SCRATCH, X.K_PERSISTENT, X.K_HACC):
            assert t.offset % es == 0
            return (scratch if t.kind == X.K_SCRATCH else persistent)[t.offset // es:]
        assert t.kind == X.K_COT
        return cot[out_off:]

    def inv(k):
        return 1.0 if k < 0 else (0.0 if factors[k] == 0 else 1.0 / factors[k])

    def run(phase, digits, out_off):
        """runs the phase's nodes; returns the sum of log10 of the factors they record"""
        exp = 0.0
        for i, nd in enumerate(plan.nodes):
            if nd["phase"] != phase:
                continue
            c = view(nd["c"], digits, out_off)
            n = nd["c"].nbytes // es
            if nd.get("zero_fill"):
                c[:n] = 0
            a = view(nd["a"], digits, out_off)
            s = inv(slot_a[i]) * inv(slot_b[i]) if slot_a[i] >= 0 else 1.0
            tmp = np.zeros(min(len(c), n), dtype=dt)
            if nd["kind"] == 0:
                emu.emulate_pair(nd["words"], a, view(nd["b"], digits, out_off), tmp)
                acc = int(nd["words"][L.W_FLAGS]) & 1
            else:
                emu.emulate_single(nd["words"], a, tmp)
                acc = int(nd["words"][L.S_FLAGS]) & 1
            if acc:
                c[: len(tmp)] += tmp * s
            else:
                c[: len(tmp)] = tmp * s
            if nd["kind"] == 0 and phase <= X.PHASE_VAR_FWD:
                f = np.max(np.abs(c[: math.prod(nd["c"].shape)]))
                factors[slot_of[id(nd["c"])]] = f
                exp += math.log10(f) if f != 0 else -math.inf
        return exp

    ns = len(plan.sliced)
    radix = [s for _i, s, _p in plan.sliced]
    proj = [p for _i, _s, p in plan.sliced]
    zero = [0] * ns
    inv_exp = run(X.PHASE_INV_FWD, zero, 0)
    for t in plan.tensors:
        if t.kind == X.K_HACC:
            persistent[t.offset // es: (t.offset + t.nbytes) // es] = 0
    strides = [1] * ns
    for j in range(ns - 2, -1, -1):
        strides[j] = strides[j + 1] * radix[j + 1]
    e = float(exponent)
    for sid in range(plan.nslices) if slice_ids is None else slice_ids:
        digits, rem = [0] * ns, sid
        for j in range(ns):
            if proj[j] is not None:
                digits[j] = proj[j]
            else:
                digits[j] = rem // strides[j]
                rem %= strides[j]
        out_off = sum(d * s for d, s in zip(digits, plan.slice_out_stride))
        e_s = inv_exp + run(X.PHASE_VAR_FWD, digits, out_off)
        # the seed divisor (gett_kernels.cuh strip_seed_kernel)
        if math.isnan(e) or math.isnan(e_s):
            factors[seed] = math.nan
        elif e == -math.inf or e_s == -math.inf:
            factors[seed] = 0.0
        else:
            with np.errstate(over="ignore"):
                factors[seed] = np.power(10.0, e - e_s)
        run(X.PHASE_VAR_BWD, digits, out_off)
    run(X.PHASE_INV_BWD, zero, 0)
    res = []
    for i, g in enumerate(grads):
        if g is None or i not in plan.wrt:
            res.append(None)
            continue
        if dt.kind == "c":
            g[:] = np.conj(g)
        res.append(g.reshape(np.shape(arrays[i])))
    return res


def install(monkeypatch):
    """``emu_device.install``, with stripped VJP plans' launches (the forward's exponent read from
    ``exp_ptr``) routed through ``emulate_stripped_vjp``."""
    from cotengra_b200 import vjp

    fake_lib = emu_device.install(monkeypatch)
    plain = vjp.VjpPlan.execute

    def execute(self, input_ptrs, cot_ptr, grad_ptrs, ws_ptr, ws_bytes, begin, step, count, stream=0,
                exp_ptr=None):
        if not self.strip_exponent:
            return plain(self, input_ptrs, cot_ptr, grad_ptrs, ws_ptr, ws_bytes, begin, step, count, stream)
        if ws_bytes < self.total_bytes:
            raise MemoryError("workspace too small")
        assert exp_ptr is not None, "a stripped VJP plan needs the forward's exponent"
        dt = np.dtype(self.dtype)
        arrays, grads = [], []
        for i, (ptr, term) in enumerate(zip(input_ptrs, self.inputs)):
            shape = tuple(self.fwd.size_dict[ix] for ix in term)
            arrays.append(emu_device._view(ptr, dt, math.prod(shape)).reshape(shape))
            gp = grad_ptrs[i]
            grads.append(None if gp is None else emu_device._view(gp, dt, math.prod(shape)))
        cot = emu_device._view(cot_ptr, dt, max(self.out_elements, 1))[: self.out_elements]
        exponent = float(emu_device._view(exp_ptr, np.float64, 1)[0])
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        emulate_stripped_vjp(self, arrays, cot.copy(), exponent, slice_ids=ids, grads=grads)
        emu_device.FakeLib.launches += sum(1 if nd["phase"] in (0, 3) else len(ids) for nd in self.nodes)

    monkeypatch.setattr(vjp.VjpPlan, "execute", execute)
    return fake_lib
