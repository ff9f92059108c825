"""Test-only emulation of ``accumulate="double"`` plans, on top of ``tests/desc_emulator.py`` and
``tests/emu_device.py``: the wide-C flag, the wide output and the dense root slot with its fold.

The emulator checks the host's integer work (descriptors, arenas, slice offsets, chunk mapping), not
device rounding, so a wide plan is walked with every value held in its accumulator dtype: the arenas
keep their element counts and offsets (an element of the plan dtype becomes one of the wide dtype),
a flagged dot-stream root adds into the wide output at the slice's offset, and the fold of any other
root (``add_chunk_wide_kernel``) runs as one more single-operand node through the chunk descriptor.
NOT a fallback: never imported by the product.
"""

import copy
import math

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L
from tests import desc_emulator as emu
from tests import emu_device


def check_wide_plan(plan):
    """The invariants of a wide forward plan the library relies on (``ctgb_plan_set_accumulator``)."""
    assert plan.wide and plan.acc_dtype == L.WIDE_DTYPES[plan.dtype]
    flagged = [nd for nd in plan.nodes if nd["kind"] == 0 and int(nd["words"][L.W_FLAGS]) & L.FLAG_WIDE_C]
    root = plan.nodes[-1]
    if plan.strip_exponent:
        # the mantissa slot keeps the plan dtype; only the running mantissa is wide
        assert not flagged and root["c"].kind == X.K_SCRATCH and plan._chunk_words is not None
    elif plan.root_direct:
        assert flagged == [root] and int(root["words"][L.W_VARIANT]) in L.DOTSTREAM_VARIANTS
        assert int(root["words"][L.W_FLAGS]) & 1 and root["c"].kind == X.K_OUTPUT and plan._chunk_words is None
    else:
        assert not flagged and root["c"].kind == X.K_SCRATCH and plan._chunk_words is not None
        flags = int(root["words"][L.W_FLAGS if root["kind"] == 0 else L.S_FLAGS])
        assert not flags & 1, "a dense root slot is stored, not accumulated"


def emulate_plan(plan, arrays, slice_ids=None):
    """``desc_emulator.emulate_plan`` for forward plans of either accumulation mode; a wide plan
    returns its result (or ``(mantissa, exponent)``) in the accumulator dtype."""
    if not getattr(plan, "wide", False):
        return emu.emulate_plan(plan, arrays, slice_ids=slice_ids)
    check_wide_plan(plan)
    wide = copy.copy(plan)
    wide.dtype = plan.acc_dtype  # (esize stays: offsets and sizes count elements of the plan dtype)
    if not plan.strip_exponent and not plan.root_direct:
        fold = np.array(plan._chunk_words, copy=True)
        fold[L.S_FLAGS] |= 1
        out = X._Slot(plan.root_shape, L.row_major_strides(plan.root_shape), X.K_OUTPUT, 0)
        wide.nodes = list(plan.nodes) + [dict(kind=1, a=plan.nodes[-1]["c"], b=None, c=out, words=fold,
                                              phase=X.PHASE_VAR_FWD)]
    res = emu.emulate_plan(wide, [np.asarray(a, dtype=plan.acc_dtype) for a in arrays], slice_ids=slice_ids)
    wide.handle = None
    return res


def install(monkeypatch):
    """``emu_device.install``, with the launches of wide plans routed through ``emulate_plan`` above
    and their output read and written in the accumulator dtype."""
    fake_lib = emu_device.install(monkeypatch)
    plain, plain_host = X.ExecPlan.execute, X.ExecPlan.execute_host

    def execute(self, input_ptrs, out_ptr, exp_ptr, ws_ptr, ws_bytes, begin, step, count, stream=0):
        if not self.wide:
            return plain(self, input_ptrs, out_ptr, exp_ptr, ws_ptr, ws_bytes, begin, step, count, stream)
        dt = np.dtype(self.dtype)
        arrays = []
        for ptr, term in zip(input_ptrs, self.inputs):
            shape = tuple(self.size_dict[ix] for ix in term)
            arrays.append(emu_device._view(ptr, dt, math.prod(shape)).reshape(shape))
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        res = emulate_plan(self, arrays, slice_ids=ids)
        out = emu_device._view(out_ptr, np.dtype(self.acc_dtype), max(self.out_elements, 1))[: self.out_elements]
        emu_device.FakeLib.launches += len(self.nodes)
        if self.strip_exponent:
            assert not np.any(out), "emulated execute: accumulating into a stripped partial sum"
            out[:] = np.asarray(res[0]).reshape(-1)
            emu_device._view(exp_ptr, np.float64, 1)[0] = res[1]
        else:
            out += np.asarray(res).reshape(-1)

    def execute_host(self, host_arrays, host_out, ws_ptr, ws_bytes, begin, step, count, stream=0):
        if not self.wide:
            return plain_host(self, host_arrays, host_out, ws_ptr, ws_bytes, begin, step, count, stream)
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        res = emulate_plan(self, list(host_arrays), slice_ids=ids)
        assert host_out.dtype == np.dtype(self.acc_dtype)
        if self.strip_exponent:
            host_out[...] = np.asarray(res[0]).reshape(host_out.shape)
            return float(res[1])
        host_out[...] = np.asarray(res).reshape(host_out.shape)
        return 0.0

    monkeypatch.setattr(X.ExecPlan, "execute", execute)
    monkeypatch.setattr(X.ExecPlan, "execute_host", execute_host)
    return fake_lib
