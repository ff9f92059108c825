"""Test-only numpy model of a stripped forward-mode plan (``JvpPlan(strip_exponent=True,
stripped_grad=True)``) run the way ``ctgb_plan_execute_jvp_stripped`` runs it, and an emulated device
launch for it (on top of ``tests/emu_strip.py``).

The lazy scheme of the plan: one factor slot per tensor slot (1.0 unless a primal pairwise record
of phase 0/1 measures max|C| there), every pairwise or two-term record's product divided by its two
slots of ``plan.scale_slots`` (1/0 counts as 0), tangent records (``plan.tangent_marks``) measuring
nothing.  Per slice the exponent ``e_s`` (every factor) and ``e'_s`` (all but the root's), the fold
of the dense raw root into ``(out, E)`` and of the raw tangent root into ``(tout, Et)``, the tangent's
own running exponent, as the rescale / chunk-add kernels do it; after the slices ``tout`` is brought
to ``E`` (``tangent_to_exponent_kernel``).  The descriptors themselves are walked by
``tests/desc_emulator.py``; the arenas are exactly the reported bytes and filled with NaN.  NOT a
fallback: never imported by the product.
"""

import math

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L
from tests import desc_emulator as emu
from tests import emu_device, emu_strip


def _exponent_max(a, b):
    """gett_kernels.cuh exponent_max: NaN if either is"""
    return math.nan if (math.isnan(a) or math.isnan(b)) else max(a, b)


def _pow10(x):
    with np.errstate(over="ignore"):
        return float(np.power(10.0, x))


def emulate_stripped_jvp(plan, arrays, tangents, slice_ids=None, out=None, tout=None, exponent=-math.inf):
    """``(out, E, tout)`` of the slices ``slice_ids`` (default all) for ``tangents``, one per input in
    ``plan.wrt``: the mantissa, its running exponent and the tangent of the mantissa with the exponent
    held constant.  ``out`` / ``tout`` (flat, accumulator dtype, both relative to ``exponent``) and
    ``exponent`` continue an earlier call's sums, as the device buffers do.  ``slice_ids`` is taken in
    the order given."""
    assert plan.strip_exponent and plan.tangent_marks is not None
    dt, adt = np.dtype(plan.dtype), np.dtype(plan.acc_dtype)
    es = plan.esize
    persistent = np.full(plan.persistent_bytes // es, np.nan, dtype=dt)
    scratch = np.full(plan.workspace_bytes // es, np.nan, dtype=dt)
    n_out = max(plan.out_elements, 1)
    out = np.zeros(n_out, dtype=adt) if out is None else out
    tout = np.zeros(n_out, dtype=adt) if tout is None else tout
    flats = [np.ascontiguousarray(a, dtype=dt).reshape(-1) for a in arrays]
    tflats = [None] * len(arrays)
    for i, t in zip(plan.wrt, tangents):
        tflats[i] = np.ascontiguousarray(t, dtype=dt).reshape(-1)
    factors = np.ones(len(plan.tensors) + 2)
    slot_of = {id(t): i for i, t in enumerate(plan.tensors)}
    slot_a, slot_b = plan.scale_slots
    root = next(nd for nd in plan.nodes if nd["root"] == 1)
    troot = [nd for nd in plan.nodes if nd["root"] == 2][-1]

    def view(t, digits):
        if t.kind in (X.K_INPUT, X.K_TANGENT):
            off = sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride))
            src = (flats if t.kind == X.K_INPUT else tflats)[t.input_index]
            assert src is not None, "a tangent slot of an input outside wrt"
            return src[off:]
        assert t.kind in (X.K_SCRATCH, X.K_PERSISTENT), t.kind
        assert t.offset % es == 0
        return (scratch if t.kind == X.K_SCRATCH else persistent)[t.offset // es:]

    def inv(k):
        return 1.0 if k < 0 else (0.0 if factors[k] == 0 else 1.0 / factors[k])

    def run(phase, digits):
        """runs the phase's records; returns the sums of log10 of the factors the primal records
        measure, without and with the root's"""
        exp = exp_root = 0.0
        for i, nd in enumerate(plan.nodes):
            if nd["phase"] != phase:
                continue
            c = view(nd["c"], digits)
            n = nd["c"].nbytes // es
            s = inv(slot_a[i]) * inv(slot_b[i]) if slot_a[i] >= 0 else 1.0
            tmp = np.zeros(min(len(c), n), dtype=dt)
            if nd["kind"] == 2:
                w = np.array(nd["words"][:L.DESC_WORDS], dtype=np.int64)
                w[L.W_FLAGS] &= ~1
                emu.emulate_pair(w, view(nd["a"], digits), view(nd["b"], digits), tmp)
                w[L.W_FLAGS] |= 1
                emu.emulate_pair(w, view(nd["a2"], digits), view(nd["b2"], digits), tmp)
                acc = int(nd["words"][L.W_FLAGS]) & 1
            elif nd["kind"] == 0:
                emu.emulate_pair(nd["words"], view(nd["a"], digits), view(nd["b"], digits), tmp)
                acc = int(nd["words"][L.W_FLAGS]) & 1
            else:
                emu.emulate_single(nd["words"], view(nd["a"], digits), tmp)
                acc = int(nd["words"][L.S_FLAGS]) & 1
            with np.errstate(invalid="ignore", over="ignore"):
                if acc:
                    c[: len(tmp)] += tmp * s
                else:
                    c[: len(tmp)] = tmp * s
            if nd["kind"] == 0 and not plan.tangent_marks[i]:
                f = float(np.max(np.abs(c[: math.prod(nd["c"].shape)])))
                factors[slot_of[id(nd["c"])]] = f
                lg = math.log10(f) if f != 0 else -math.inf
                if nd is root:
                    exp_root = lg
                else:
                    exp += lg
        return exp, exp + exp_root

    ns = len(plan.sliced)
    radix = [s for _i, s, _p in plan.sliced]
    proj = [p for _i, _s, p in plan.sliced]
    inv_exp = run(X.PHASE_INV_FWD, [0] * ns)[1]
    strides = [1] * ns
    for j in range(ns - 2, -1, -1):
        strides[j] = strides[j + 1] * radix[j + 1]
    E = Et = float(exponent)
    for sid in range(plan.nslices) if slice_ids is None else slice_ids:
        digits, rem = [0] * ns, sid
        for j in range(ns):
            if proj[j] is not None:
                digits[j] = proj[j]
            else:
                digits[j] = rem // strides[j]
                rem %= strides[j]
        out_off = sum(d * s for d, s in zip(digits, plan.slice_out_stride))
        e_wo, e_all = run(X.PHASE_VAR_FWD, digits)
        e_t, e_s = inv_exp + e_wo, inv_exp + e_all
        # the fold (rescale_out_kernel / add_chunk_kernel / commit_exponent_kernel)
        e = _exponent_max(E, e_s)
        et = _exponent_max(Et, e_t)
        so = 1.0 if E == e else _pow10(E - e)
        so_t = 1.0 if Et == et else _pow10(Et - et)
        with np.errstate(invalid="ignore"):
            if so != 1.0:
                out *= so
            if so_t != 1.0:
                tout *= so_t
        sn = 1.0 if e_s == e else _pow10(e_s - e)
        if root["kind"] == 0:
            froot = factors[slot_of[id(root["c"])]]
            sn = sn / froot if froot != 0 else 0.0
        st = 0.0 if et == -math.inf else 1.0 if e_t == et else _pow10(e_t - et)
        with np.errstate(invalid="ignore", over="ignore"):
            emu.emulate_single_scaled(plan._chunk_words, view(root["c"], digits), out[out_off:], sn)
            emu.emulate_single_scaled(plan._chunk_words, view(troot["c"], digits), tout[out_off:], st)
        E, Et = e, et
    # tout from Et to E (0 for a zero result, NaN with either exponent NaN)
    if math.isnan(E) or math.isnan(Et):
        tout[:] = math.nan
    elif E == -math.inf:
        tout[:] = 0
    elif Et != E:
        with np.errstate(invalid="ignore", over="ignore"):
            tout *= _pow10(Et - E)
    shape = lambda x: x[: plan.out_elements].reshape(plan.out_shape)  # noqa: E731
    return shape(out), E, shape(tout)


def install(monkeypatch):
    """``emu_strip.install`` (the emulated device with stripped VJP plans), with stripped JVP plans'
    launches routed through ``emulate_stripped_jvp``: the inputs, tangents, mantissa, exponent and
    tangent buffers read from and written to the pointers the product passes."""
    from cotengra_b200 import jvp

    fake_lib = emu_strip.install(monkeypatch)

    def execute(self, input_ptrs, tangent_ptrs, out_ptr, tangent_out_ptr, ws_ptr, ws_bytes, begin, step, count,
                stream=0, exp_ptr=None):
        assert self.strip_exponent, "the emulated device runs stripped JVP plans only"
        if ws_bytes < self.total_bytes:
            raise MemoryError("workspace too small")
        assert out_ptr is not None and exp_ptr is not None
        dt = np.dtype(self.dtype)
        arrays, tangents = [], []
        for i, (ptr, term) in enumerate(zip(input_ptrs, self.inputs)):
            shape = tuple(self.fwd.size_dict[ix] for ix in term)
            arrays.append(emu_device._view(ptr, dt, math.prod(shape)).reshape(shape))
            if i in self.wrt:
                tangents.append(emu_device._view(tangent_ptrs[i], dt, math.prod(shape)).reshape(shape))
        n = max(self.out_elements, 1)
        out = emu_device._view(out_ptr, self.acc_dtype, n)
        tout = emu_device._view(tangent_out_ptr, self.acc_dtype, n)
        exp = emu_device._view(exp_ptr, np.float64, 1)
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        _m, e, _t = emulate_stripped_jvp(self, arrays, tangents, slice_ids=ids, out=out, tout=tout,
                                         exponent=float(exp[0]))
        exp[0] = e
        emu_device.FakeLib.launches += sum(1 if nd["phase"] == 0 else len(ids) for nd in self.nodes)

    monkeypatch.setattr(jvp.JvpPlan, "execute", execute)
    return fake_lib
