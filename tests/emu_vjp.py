"""Test-only emulation of ``ctgb_vjp_execute``: walks a ``VjpPlan``'s node list phase by phase
with the descriptor emulator (``emulate_pair`` / ``emulate_single``), the way the device loop
does -- arenas, slice digits, input and gradient views, the cotangent's slice view, zero fills,
hoisted H accumulators and the final conjugations.  The arenas are exactly the reported bytes,
so an access outside them raises.  NOT a fallback: it lives under ``tests/``.
"""

import math

import numpy as np

from cotengra_b200 import vjp as V
from tests import desc_emulator as emu
from tests import emu_device


def emulate_vjp(plan, arrays, cotangent, slice_ids=None, grads=None):
    """Gradients (numpy, ``None`` outside ``plan.wrt``) of the slices ``slice_ids`` (default all)."""
    dt = np.dtype(plan.dtype)
    es = plan.esize
    assert plan.workspace_bytes % es == 0 and plan.persistent_bytes % es == 0
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
    ns = len(plan.sliced)
    radix = [s for _i, s, _p in plan.sliced]
    proj = [p for _i, _s, p in plan.sliced]
    out_stride = [int(plan._vd.slice_out_stride[j]) for j in range(ns)]

    def view(t, digits, out_off):
        if t.kind in (V.K_INPUT, V.K_GRAD):
            off = sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride))
            base = flats[t.input_index] if t.kind == V.K_INPUT else grads[t.input_index]
            return base[off:]
        if t.kind == V.K_SCRATCH:
            return scratch[t.offset // es:]
        if t.kind in (V.K_PERSISTENT, V.K_HACC):
            return persistent[t.offset // es:]
        assert t.kind == V.K_COT
        return cot[out_off:]

    def run(phase, digits, out_off):
        for nd in plan.nodes:
            if nd["phase"] != phase:
                continue
            c = view(nd["c"], digits, out_off)
            if nd["zero_fill"]:
                c[: nd["c"].nbytes // es] = 0
            a = view(nd["a"], digits, out_off)
            if nd["kind"] == 0:
                emu.emulate_pair(nd["words"], a, view(nd["b"], digits, out_off), c)
            else:
                emu.emulate_single(nd["words"], a, c)
            emu_device.FakeLib.launches += 1

    zero = [0] * ns
    run(V.PHASE_INV_FWD, zero, 0)
    for t in plan.tensors:
        if t.kind == V.K_HACC:
            persistent[t.offset // es: (t.offset + t.nbytes) // es] = 0
    strides = [1] * ns
    for j in range(ns - 2, -1, -1):
        strides[j] = strides[j + 1] * radix[j + 1]
    for i in (range(plan.nslices) if slice_ids is None else slice_ids):
        digits, rem = [0] * ns, i
        for j in range(ns):
            if proj[j] is not None:
                digits[j] = proj[j]
            else:
                digits[j] = rem // strides[j]
                rem %= strides[j]
        out_off = sum(d * s for d, s in zip(digits, out_stride))
        run(V.PHASE_VAR_FWD, digits, out_off)
        run(V.PHASE_VAR_BWD, digits, out_off)
    run(V.PHASE_INV_BWD, zero, 0)
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
    """``emu_device.install`` plus the VJP plan's device entry points."""
    fake = emu_device.install(monkeypatch)

    def create(self):
        self.handle = "emulated"
        return self

    def execute(self, input_ptrs, cot_ptr, grad_ptrs, ws_ptr, ws_bytes, begin, step, count, stream=0):
        if ws_bytes < self.total_bytes:
            raise MemoryError("workspace too small")
        dt = np.dtype(self.dtype)
        arrays, grads = [], []
        for i, (ptr, term) in enumerate(zip(input_ptrs, self.inputs)):
            shape = tuple(self.fwd.size_dict[ix] for ix in term)
            arrays.append(emu_device._view(ptr, dt, math.prod(shape)).reshape(shape))
            gp = grad_ptrs[i]
            grads.append(None if gp is None else emu_device._view(gp, dt, math.prod(shape)))
        cot = emu_device._view(cot_ptr, dt, max(self.out_elements, 1))[: self.out_elements]
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        emulate_vjp(self, arrays, cot.copy(), slice_ids=ids, grads=grads)

    monkeypatch.setattr(V.VjpPlan, "create", create)
    monkeypatch.setattr(V.VjpPlan, "execute", execute)
    monkeypatch.setattr(V.VjpPlan, "destroy", lambda self: None)
    return fake
