"""Test-only stand-in for the GPU *launch*: lets the reference's real control flow
(``ctg.einsum(..., implementation=...)``, ``tree.contract``, ``tree.contract_slice`` after
``cb.install(tree)``) run into the product's host code in the build container, which has the
reference but no GPU.

Everything above the C-ABI call is the product: argument handling, classification, lowering
to descriptors, plan building (arenas, slice offsets, hoisting, stem fusion).  Only the last
step -- ``ctgb_contract_pair`` / ``ctgb_reduce_single`` / ``ctgb_plan_execute`` of forward and
reverse-mode plans -- is replaced by ``tests/desc_emulator.py``, which walks the very descriptors
the kernels would receive.
Host tensors (torch CPU) stand in for device memory.  NOT a fallback: it lives under
``tests/``, is never imported by ``cotengra_b200`` and is installed by monkeypatching only.
"""

import contextlib
import ctypes as C
import math
import types

import numpy as np

from cotengra_b200 import lowering as L
from tests import desc_emulator as emu

_NP = {0: np.float32, 1: np.float64, 2: np.complex64, 3: np.complex128}


def _view(ptr, dtype, count=None):
    """numpy view of raw memory at ``ptr`` (unbounded unless ``count`` is given; nothing is
    touched until indexed)."""
    dtype = np.dtype(dtype)
    n = (1 << 40) if count is None else int(count) * dtype.itemsize
    raw = np.ctypeslib.as_array(C.cast(int(ptr), C.POINTER(C.c_uint8)), shape=(max(n, 1),))
    return raw[: n - n % dtype.itemsize].view(dtype) if count is None else raw[:n].view(dtype)


class FakeLib:
    """The symbols the host code calls, backed by the descriptor emulator."""

    launches = 0

    def ctgb_abi_version(self):
        return 2

    def ctgb_desc_words(self):
        return L.DESC_WORDS

    def ctgb_single_desc_words(self):
        return L.SDESC_WORDS

    def ctgb_last_error(self):
        return b"emulated"

    def ctgb_launch_count(self):
        return FakeLib.launches

    def ctgb_contract_pair(self, words_ptr, pa, pb, pc, stream):
        W = _view(words_ptr, np.int64, L.DESC_WORDS)
        dt = _NP[int(W[L.W_DTYPE])]
        # extent of each operand: 1 + sum (ext - 1) * |stride| over its dims (an upper bound
        # for blocked dims; the surplus is never touched)
        span = [1, 1, 1]  # A, B, C

        def add(off, n, width, cols):
            for i in range(n):
                row = W[off + i * width: off + (i + 1) * width]
                for which, c in cols:
                    span[which] += (int(row[0]) - 1) * abs(int(row[c]))

        add(L.OFF_TM, int(W[L.W_NTM]), 3, ((0, 1), (2, 2)))
        add(L.OFF_TN, int(W[L.W_NTN]), 3, ((1, 1), (2, 2)))
        add(L.OFF_TK, int(W[L.W_NTK]), 3, ((0, 1), (1, 2)))
        add(L.OFF_GM, int(W[L.W_NGM]), 4, ((0, 2), (2, 3)))
        add(L.OFF_GN, int(W[L.W_NGN]), 4, ((1, 2), (2, 3)))
        add(L.OFF_GK, int(W[L.W_NGK]), 4, ((0, 2), (1, 3)))
        add(L.OFF_GB, int(W[L.W_NGB]), 5, ((0, 2), (1, 3), (2, 4)))
        span[2] = max(span[2], int(W[L.W_CELEMS]))
        emu.emulate_pair(W, _view(pa, dt, span[0]), _view(pb, dt, span[1]), _view(pc, dt, span[2]))
        FakeLib.launches += 1
        return 0

    def ctgb_reduce_single(self, words_ptr, px, pout, stream):
        W = _view(words_ptr, np.int64, L.SDESC_WORDS)
        dt = _NP[int(W[L.S_DTYPE])]
        sx = so = 1
        for i in range(int(W[L.S_NO])):
            e, a, b = (int(x) for x in W[L.OFF_SO + 3 * i: L.OFF_SO + 3 * i + 3])
            sx += (e - 1) * abs(a)
            so += (e - 1) * abs(b)
        for i in range(int(W[L.S_NS])):
            e, a = (int(x) for x in W[L.OFF_SS + 2 * i: L.OFF_SS + 2 * i + 2])
            sx += (e - 1) * abs(a)
        emu.emulate_single(W, _view(px, dt, sx), _view(pout, dt, so))
        FakeLib.launches += 1
        return 0


class _FakeCuda:
    def is_available(self):
        return True

    def current_device(self):
        return 0

    def device(self, _d):
        return contextlib.nullcontext()

    def current_stream(self):
        return types.SimpleNamespace(cuda_stream=0)

    def synchronize(self, *_a):
        return None


class _FakeTorch:
    """``torch`` with host memory standing in for the device."""

    def __init__(self):
        import torch

        self._torch = torch
        self.cuda = _FakeCuda()

    def __getattr__(self, name):
        return getattr(self._torch, name)

    def device(self, *_a):
        return self._torch.device("cpu")


def install(monkeypatch):
    """Route the product's launches through the emulator (use from a test with the
    ``monkeypatch`` fixture)."""
    import torch

    from cotengra_b200 import _lib, contract, executor, vjp

    fake_torch = _FakeTorch()
    fake_lib = FakeLib()

    def to_device(x, device=None):
        if isinstance(x, torch.Tensor):
            return x.contiguous(), False
        x = np.asarray(x, order="C")
        L.dtype_name(x.dtype)
        return torch.from_numpy(np.array(x, copy=True)), True

    monkeypatch.setattr(contract, "_torch", lambda: fake_torch)
    monkeypatch.setattr(contract, "_to_device", to_device)
    monkeypatch.setattr(contract, "_stream_ptr", lambda: 0)
    monkeypatch.setattr(_lib, "load", lambda: fake_lib)
    monkeypatch.setattr(_lib, "check", lambda rc: None if not rc else (_ for _ in ()).throw(RuntimeError(rc)))
    monkeypatch.setattr(_lib, "device_info", lambda: {"sm_count": 132, "cc": (9, 0), "smem_optin": 232448})

    def create(self):
        self.handle = "emulated"
        return self

    def execute(self, input_ptrs, out_ptr, exp_ptr, ws_ptr, ws_bytes, begin, step, count, stream=0):
        dt = np.dtype(self.dtype)
        arrays = []
        for ptr, term in zip(input_ptrs, self.inputs):
            shape = tuple(self.size_dict[ix] for ix in term)
            arrays.append(_view(ptr, dt, math.prod(shape)).reshape(shape))
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        res = emu.emulate_plan(self, arrays, slice_ids=ids)
        out = _view(out_ptr, dt, max(self.out_elements, 1))[: self.out_elements]
        FakeLib.launches += len(self.nodes)
        if self.strip_exponent:
            m, e = res
            # fresh accumulators only (what the drop-in tests use)
            assert not np.any(out), "emulated execute: accumulating into a stripped partial sum"
            out[:] = np.asarray(m).reshape(-1)
            _view(exp_ptr, np.float64, 1)[0] = e
        else:
            out += np.asarray(res).reshape(-1)

    def execute_host(self, host_arrays, host_out, ws_ptr, ws_bytes, begin, step, count, stream=0):
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        res = emu.emulate_plan(self, list(host_arrays), slice_ids=ids)
        if self.strip_exponent:
            host_out[...] = np.asarray(res[0]).reshape(host_out.shape)
            return float(res[1])
        host_out[...] = np.asarray(res).reshape(host_out.shape)
        return 0.0

    def execute_vjp(self, input_ptrs, cot_ptr, grad_ptrs, ws_ptr, ws_bytes, begin, step, count, stream=0):
        if ws_bytes < self.total_bytes:
            raise MemoryError("workspace too small")
        dt = np.dtype(self.dtype)
        arrays, grads = [], []
        for i, (ptr, term) in enumerate(zip(input_ptrs, self.inputs)):
            shape = tuple(self.fwd.size_dict[ix] for ix in term)
            arrays.append(_view(ptr, dt, math.prod(shape)).reshape(shape))
            gp = grad_ptrs[i]
            grads.append(None if gp is None else _view(gp, dt, math.prod(shape)))
        cot = _view(cot_ptr, dt, max(self.out_elements, 1))[: self.out_elements]
        ids = range(int(begin), int(begin) + int(step) * int(count), int(step))
        emu.emulate_plan(self, arrays, cot.copy(), slice_ids=ids, grads=grads)
        # phases 0 and 3 run once, phases 1 and 2 once per slice
        FakeLib.launches += sum(1 if nd["phase"] in (0, 3) else len(ids) for nd in self.nodes)

    monkeypatch.setattr(executor._DevicePlan, "create", create)
    monkeypatch.setattr(executor._DevicePlan, "destroy", lambda self: None)
    monkeypatch.setattr(executor.ExecPlan, "execute", execute)
    monkeypatch.setattr(executor.ExecPlan, "execute_host", execute_host)
    monkeypatch.setattr(vjp.VjpPlan, "execute", execute_vjp)
    return fake_lib
