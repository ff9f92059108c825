"""Reference-facing host API: the same names, argument meaning and error
behaviour as cotengra's execution path, backed by the sm_90a kernels.

    einsum(eq, a, b=None) ............ cotengra/contract.py:414
    tensordot(a, b, axes) ............ cotengra/contract.py:521
    implementation() ................. the ``(einsum, tensordot)`` pair accepted by
                                       ``implementation=`` (contract.py:775-776; the
                                       order really is einsum first)
    B200Contractor ................... cotengra/contract.py:654 ``Contractor`` /
                                       :840 ``CuQuantumContractor`` (whole-tree)
    contract_tree(tree, arrays) ...... cotengra/core.py:3943 ``ContractionTree.contract``
    contract_distributed(...) ........ cotengra/core.py:4032 ``contract_mpi`` (NCCL)
    gen_output_chunks(tree, arrays) .. cotengra/core.py:3884 ``gen_output_chunks``
    install(tree) .................... seeds ``tree.contraction_cores`` (core.py:3699)

Arrays may be numpy arrays (copied to the GPU and back: the host path) or torch
CUDA tensors (used in place).  torch is only the carrier of device memory and
streams; all arithmetic happens in ``libctgb200.so``.  There is no CPU
fallback: without a CUDA device these functions raise.
"""

from __future__ import annotations

import ctypes as C
import functools
import math
import warnings

import numpy as np

from . import _lib, lowering
from .executor import ExecPlan, output_chunking
from .lowering import (
    build_pair_desc,
    build_single_desc,
    check_accumulate,
    check_precision,
    check_tensordot_shapes,
    classify_pair,
    classify_single,
    dtype_name,
    split_equation,
    tensordot_terms,
)
from .tree import TreeSpec


def _torch():
    import torch

    if not torch.cuda.is_available():
        raise RuntimeError(
            "cotengra_b200 needs a CUDA device (sm_90a); there is no CPU fallback"
        )
    return torch


def _to_device(x, device=None):
    """numpy / torch -> contiguous torch CUDA tensor; returns (tensor, was_numpy)."""
    torch = _torch()
    if isinstance(x, torch.Tensor):
        if not x.is_cuda:
            x = x.cuda(device)
        return x.contiguous(), False
    x = np.asarray(x, order="C")  # (ascontiguousarray would promote 0-d to 1-d)
    dtype_name(x.dtype)
    return torch.from_numpy(x).cuda(device), True


def _from_device(t, as_numpy):
    return t.cpu().numpy() if as_numpy else t


def _stream_ptr():
    torch = _torch()
    return torch.cuda.current_stream().cuda_stream


def _common_dtype(*ts):
    names = {dtype_name(t.dtype) for t in ts}
    if len(names) != 1:
        raise TypeError(f"operands must share one dtype, got {sorted(names)}")
    return names.pop()


# ---------------------------------------------------------------------------
# single nodes (the tuple interface)
# ---------------------------------------------------------------------------


@functools.lru_cache(4096)
def _pair_words(term_a, shape_a, term_b, shape_b, out, dtype, sm_count, precision="3xtf32"):
    dims = classify_pair(term_a, shape_a, term_b, shape_b, out)
    plan = build_pair_desc(dims, dtype, sm_count=sm_count,
                           c_dense_elems=math.prod(dims.out_shape), precision=precision)
    return plan, dims.out_shape


@functools.lru_cache(4096)
def _single_words(term, shape, out, dtype):
    odims, sdims, oshape = classify_single(term, shape, out)
    return build_single_desc(odims, sdims, dtype), oshape


def _sm_count():
    return _lib.device_info()["sm_count"]


def _run_pair(term_a, a, term_b, b, out, precision="3xtf32"):
    torch = _torch()
    ta, na = _to_device(a)
    tb, nb = _to_device(b, ta.device)
    dtype = _common_dtype(ta, tb)
    plan, oshape = _pair_words(tuple(term_a), tuple(ta.shape), tuple(term_b), tuple(tb.shape),
                               tuple(out), dtype, _sm_count(), precision)
    c = torch.empty(oshape, dtype=ta.dtype, device=ta.device)
    if c.numel():
        pa, pb = (tb, ta) if plan.swapped else (ta, tb)
        with torch.cuda.device(ta.device):
            _lib.check(_lib.load().ctgb_contract_pair(
                plan.words.ctypes.data, pa.data_ptr(), pb.data_ptr(), c.data_ptr(), _stream_ptr()))
    return _from_device(c, na and nb)


def _run_single(term, x, out, precision="3xtf32"):
    torch = _torch()
    tx, nx = _to_device(x)
    dtype = dtype_name(tx.dtype)
    check_precision(precision, dtype)  # (a single-operand node has no tensor-core work to change)
    words, oshape = _single_words(tuple(term), tuple(tx.shape), tuple(out), dtype)
    c = torch.empty(oshape, dtype=tx.dtype, device=tx.device)
    if c.numel():
        with torch.cuda.device(tx.device):
            _lib.check(_lib.load().ctgb_reduce_single(
                words.ctypes.data, tx.data_ptr(), c.data_ptr(), _stream_ptr()))
    return _from_device(c, nx)


def einsum(eq, a, b=None, *, backend=None, precision="3xtf32"):
    """Single or pairwise einsum (cotengra/contract.py:414-459), one kernel.  ``precision="tf32"``
    runs float32 / complex64 tensor-core work in one tf32 pass (``lowering.PRECISIONS``)."""
    check_precision(precision)
    terms, out = split_equation(eq)
    if b is None:
        if len(terms) != 1:
            raise ValueError(f"equation {eq!r} needs {len(terms)} operands, got 1")
        return _run_single(terms[0], a, out, precision)
    if len(terms) != 2:
        raise ValueError(f"equation {eq!r} needs {len(terms)} operands, got 2")
    return _run_pair(terms[0], a, terms[1], b, out, precision)


def tensordot(a, b, axes=2, *, backend=None, precision="3xtf32"):
    """Tensordot (cotengra/contract.py:521-570), one kernel; ``precision`` as for ``einsum``."""
    check_precision(precision)
    na, nb = len(a.shape), len(b.shape)
    try:
        axes = tuple(map(int, axes[0])), tuple(map(int, axes[1]))
    except (IndexError, TypeError):
        n = int(axes)
        axes = tuple(range(na - n, na)), tuple(range(n))
    check_tensordot_shapes(axes, tuple(a.shape), tuple(b.shape))
    ta, tb, to = tensordot_terms(axes, na, nb)
    return _run_pair(ta, a, tb, b, to, precision)


def implementation(precision="3xtf32"):
    """The ``(einsum, tensordot)`` pair for cotengra's ``implementation=`` kwarg
    or ``set_default_implementation`` (contract.py:13-31, 775-776), bound to ``precision``."""
    if check_precision(precision) == "3xtf32":
        return (einsum, tensordot)
    return (functools.partial(einsum, precision=precision), functools.partial(tensordot, precision=precision))


# ---------------------------------------------------------------------------
# whole-tree contractor
# ---------------------------------------------------------------------------


class _Executor:
    """A compiled program ``(contractions, inputs, output, size_dict, sliced)`` on one device: its
    forward ``ExecPlan`` (``plan``), the workspaces, and the forward and reverse-mode entry points over
    a range of its slices.  Every option of a contraction lives here, and every entry point forwards
    its options to the executor it builds:

    ``strip_exponent`` returns results as ``(mantissa, exponent)``.

    ``precision`` is the compute mode of the float32 / complex64 tensor-core nodes of every plan it
    builds (forward, output chunks, reverse mode): ``"3xtf32"`` (default) or ``"tf32"``.

    ``accumulate`` is where the slices are summed: ``"native"`` (default, the plan dtype) or
    ``"double"``, with which a float32 / complex64 program adds every slice to a float64 / complex128
    output in double precision and returns it unrounded (``ExecPlan``); for the double dtypes it is
    ``"native"``.  Gradients through a wide result keep the inputs' dtype: the cotangent is cast to the
    plan dtype and the reverse-mode plans are those of ``"native"``.

    ``vjp_max_bytes`` bounds the workspace of its reverse-mode plans (``vjp_plan``, ``vjp``), which
    then recompute per-slice forward values instead of keeping them (``VjpPlan(max_bytes=...)``).

    ``stripped_grad=True`` (with ``strip_exponent``) differentiates the mantissa ``m`` of a result
    ``(m, e)`` with the exponent held constant, ``dm/dx = 10^-e damp/dx``: exact for every loss that
    depends on the result only through ``m 10^e``.  ``vjp`` then takes the forward's ``exponent``, and
    ``jvp`` returns ``((m, e), dm)`` or, given the forward's ``exponent``, ``dm`` alone.

    ``plan_opts`` go to the forward and reverse-mode plans (``ExecPlan`` / ``VjpPlan`` keywords).

    ``resident`` are device tensors the executor holds for the last plan inputs (folded constants,
    ``TreeExecutor(constants=...)``): every entry point takes only the leading inputs, the
    *variables*, and the executor appends the resident ones.
    """

    _exp_shift = 0.0         # added to every stripped exponent: the exponents of the folded constants
    _constant_result = None  # every input constant: the whole result, formed when the executor is built
    _constant_numpy = False  # ... and whether it is returned as numpy

    def __init__(self, contractions, inputs, output, size_dict, sliced, dtype, strip_exponent=False, device=None,
                 vjp_max_bytes=None, precision="3xtf32", stripped_grad=False, accumulate="native", absorb_root=False,
                 resident=(), **plan_opts):
        torch = _torch()
        self._ir, self._plan_opts = contractions, plan_opts
        # the program without its slicing: the positional head of ``ExecPlan`` and ``VjpPlan``
        self._program, self._sliced = (contractions, inputs, output, size_dict), sliced
        self.device = torch.device("cuda", torch.cuda.current_device() if device is None else device)
        with torch.cuda.device(self.device):
            self.plan = ExecPlan(*self._program, sliced, dtype=dtype, strip_exponent=strip_exponent,
                                 precision=precision, accumulate=accumulate, absorb_root=absorb_root,
                                 **plan_opts).create()
        self.dtype = self.plan.dtype
        self.precision = precision
        self.accumulate = accumulate
        self.out_dtype = self.plan.acc_dtype  # of results: the plan dtype, or its double counterpart
        self.strip_exponent = bool(strip_exponent)
        self.stripped_grad = bool(stripped_grad)
        self.vjp_max_bytes = vjp_max_bytes
        self._resident = list(resident)
        self._shapes = [tuple(size_dict[ix] for ix in term) for term in inputs[:len(inputs) - len(self._resident)]]
        self._ws = None
        self._vjp_plans, self._vjp_ws = {}, None
        self._jvp_plans, self._jvp_ws = {}, None

    @property
    def nslices(self):
        return self.plan.nslices

    def workspace(self, host_staging=False):
        torch = _torch()
        need = self.plan.total_bytes + (self.plan.host_staging_bytes() if host_staging else 0)
        if self._ws is None or self._ws.numel() < need:
            self._ws = None
            self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
        return self._ws

    def _check_inputs(self, arrays):
        shapes = self._shapes
        if len(arrays) != len(shapes):
            what = "variables" if self._resident else "arrays"
            raise ValueError(f"expected {len(shapes)} {what}, got {len(arrays)}")
        for i, (x, s) in enumerate(zip(arrays, shapes)):
            if tuple(x.shape) != tuple(s):
                raise ValueError(f"array {i} has shape {tuple(x.shape)}, expected {tuple(s)}")

    def contract_device(self, tensors, begin=0, step=1, count=None, out=None, exponent=None):
        """Accumulate slices ``begin, begin+step, ...`` (``count`` of them) of
        already-resident CUDA tensors into ``out`` (zeroed here if not given).
        Returns ``out`` or ``(out, exponent_tensor)``; asynchronous."""
        torch = _torch()
        self._check_inputs(tensors)
        begin, step, count = self._check_slice_range(begin, step, count)
        if (self._constant_result is not None and out is None and exponent is None
                and (begin, step, count) == (0, 1, self.nslices)):
            return tuple(t.clone() for t in self._constant_result) if self.strip_exponent \
                else self._constant_result.clone()
        tdt = getattr(torch, self.out_dtype)
        with torch.cuda.device(self.device):
            if out is None:
                out = torch.zeros(self.plan.out_shape, dtype=tdt, device=self.device)
            elif (out.device != self.device or not out.is_contiguous() or out.dtype != tdt
                  or tuple(out.shape) != tuple(self.plan.out_shape)):
                raise ValueError("out must be a contiguous tensor of the plan's output shape, accumulator dtype "
                                 "and device")
            if self.strip_exponent and exponent is None:
                exponent = torch.full((1,), -math.inf, dtype=torch.float64, device=self.device)
            ws = self.workspace()
            ptrs, _keep = self._input_ptrs(tensors)
            if self._exp_shift:
                exponent.sub_(self._exp_shift)  # the plan combines its slices with the exponent it was given
            self.plan.execute(ptrs, out.data_ptr(), exponent.data_ptr() if exponent is not None else None,
                              ws.data_ptr(), ws.numel(), begin, step, count, _stream_ptr())
            if self._exp_shift:
                exponent.add_(self._exp_shift)
        return (out, exponent) if self.strip_exponent else out

    def _input_ptrs(self, tensors):
        """Device pointers of the inputs, then of the resident tensors (plus the contiguous copies
        that must outlive the call)."""
        ptrs, keep = [], []
        for i, t in enumerate(tensors):
            if dtype_name(t.dtype) != self.dtype:
                raise TypeError(f"plan was built for {self.dtype}, got {t.dtype}")
            if t.device != self.device:
                raise ValueError(f"array {i} lives on {t.device}, the plan on {self.device}")
            if not t.is_contiguous():
                # the kernels address row-major storage by the plan's own strides
                t = t.contiguous()
                keep.append(t)
            ptrs.append(t.data_ptr())
        return ptrs + [t.data_ptr() for t in self._resident], keep

    # ------------------------------------------------------------------ gradients
    def vjp_plan(self, wrt=None, max_bytes=None):
        """The (cached) ``VjpPlan`` of the executed program for the inputs ``wrt`` (default all),
        within ``max_bytes`` of workspace (default: the executor's ``vjp_max_bytes``)."""
        from .vjp import VjpPlan

        wrt = tuple(range(len(self._shapes))) if wrt is None else tuple(sorted({int(i) for i in wrt}))
        if self._resident and any(i < 0 or i >= len(self._shapes) for i in wrt):
            raise ValueError(f"wrt {list(wrt)} names inputs outside the {len(self._shapes)} variables")
        max_bytes = self.vjp_max_bytes if max_bytes is None else max_bytes
        key = wrt if max_bytes is None else (wrt, max_bytes)
        plan = self._vjp_plans.get(key)
        if plan is None:
            torch = _torch()
            with torch.cuda.device(self.device):
                plan = VjpPlan(*self._program, self._sliced, dtype=self.dtype, wrt=wrt,
                               strip_exponent=self.strip_exponent, max_bytes=max_bytes, precision=self.precision,
                               stripped_grad=self.stripped_grad, **self._plan_opts).create()
            self._vjp_plans[key] = plan
        return plan

    def vjp(self, tensors, cotangent, begin=0, step=1, count=None, wrt=None, max_bytes=None, exponent=None):
        """Gradients of the sum of slices ``begin, begin+step, ...`` (``count`` of them) for the
        output cotangent ``cotangent`` (the full output's shape): a list with one tensor per input,
        ``None`` for inputs outside ``wrt`` (default: all).  Complex gradients follow torch's
        convention.  Asynchronous on the current stream.  Gradients are linear in the cotangent and
        additive over slices, so one call per rank over ``rank_slices(...)`` followed by an
        all-reduce gives the gradient of the whole tree.  ``max_bytes`` as for ``vjp_plan``.

        With ``strip_exponent`` and ``stripped_grad``, ``cotangent`` is that of the mantissa ``m``
        and ``exponent`` (a float or a one-element tensor) the ``e`` of the forward call over the
        same slices that returned ``(m, e)``; the gradients are those of ``m`` with ``e`` held
        constant."""
        torch = _torch()
        self._check_inputs(tensors)
        begin, step, count = self._check_slice_range(begin, step, count)
        plan = self.vjp_plan(wrt, max_bytes)
        tdt = getattr(torch, self.dtype)
        with torch.cuda.device(self.device):
            ptrs, _keep = self._input_ptrs(tensors)
            if tuple(cotangent.shape) != tuple(plan.out_shape):
                raise ValueError(f"cotangent has shape {tuple(cotangent.shape)}, the output {tuple(plan.out_shape)}")
            exp = None
            if plan.strip_exponent:
                if exponent is None:
                    raise ValueError("a stripped gradient needs the exponent of the forward call (exponent=)")
                exp = torch.as_tensor(exponent, dtype=torch.float64).to(self.device).reshape(1).contiguous()
                if self._exp_shift:
                    exp = exp - self._exp_shift  # the plan's own exponent, without the folded constants'

            cot = cotangent.to(device=self.device, dtype=tdt).contiguous()
            grads = [torch.zeros(tuple(t.shape), dtype=tdt, device=self.device) if i in plan.wrt else None
                     for i, t in enumerate(tensors)]
            if self._vjp_ws is None or self._vjp_ws.numel() < plan.total_bytes:
                self._vjp_ws = None
                self._vjp_ws = torch.empty(max(plan.total_bytes, 1), dtype=torch.uint8, device=self.device)
            ws = self._vjp_ws
            # (only a stripped plan takes the forward's exponent)
            extra = {} if exp is None else {"exp_ptr": exp.data_ptr()}
            gptrs = [g.data_ptr() if g is not None else None for g in grads] + [None] * len(self._resident)
            plan.execute(ptrs, cot.data_ptr(), gptrs,
                         ws.data_ptr(), ws.numel(), begin, step, count, _stream_ptr(), **extra)
        return grads

    def jvp_plan(self, wrt=None, _two_term=True):
        """The (cached) ``JvpPlan`` of the executed program for the inputs ``wrt`` (default all; positions
        among the variables).  ``strip_exponent`` executors without ``stripped_grad`` raise
        ``NotImplementedError``."""
        from .jvp import JvpPlan

        if self.strip_exponent and not self.stripped_grad:
            raise NotImplementedError("forward-mode derivatives of strip_exponent results are only defined with "
                                      "stripped_grad=True (the exponent held constant)")
        wrt = tuple(range(len(self._shapes))) if wrt is None else tuple(sorted({int(i) for i in wrt}))
        if any(i < 0 or i >= len(self._shapes) for i in wrt):
            raise ValueError(f"wrt {list(wrt)} names inputs outside the {len(self._shapes)} variables")
        key = (wrt, bool(_two_term))
        plan = self._jvp_plans.get(key)
        if plan is None:
            torch = _torch()
            with torch.cuda.device(self.device):
                plan = JvpPlan(*self._program, self._sliced, dtype=self.dtype, wrt=wrt, precision=self.precision,
                               accumulate=self.accumulate, absorb_root=self.plan.absorb_root,
                               strip_exponent=self.strip_exponent, stripped_grad=self.stripped_grad,
                               _two_term=_two_term, **self._plan_opts).create()
            self._jvp_plans[key] = plan
        return plan

    def jvp(self, tensors, tangents, begin=0, step=1, count=None, wrt=None, primal=True, exponent=None,
            _two_term=True):
        """Forward mode over slices ``begin, begin+step, ...`` (``count`` of them): the tangent of their
        sum for the input tangents ``tangents``, one tensor per input in ``wrt`` (default: all), each of
        its input's shape.  Returns ``(out, tangent_out)``, or ``tangent_out`` alone with
        ``primal=False``; both have the output's shape and the accumulator dtype.  Asynchronous on the
        current stream.  Tangents are additive over slices, so one call per rank over
        ``rank_slices(...)`` followed by an all-reduce gives the JVP of the whole tree.  Folded
        constants carry no tangent.

        With ``strip_exponent`` and ``stripped_grad`` it returns ``((m, e), dm)``: ``(m, e)`` as
        ``contract_device`` returns it and ``dm = 10^-e d(amp)``, the tangent of the mantissa with the
        exponent held constant.  ``primal=False`` needs ``exponent`` (a float or a one-element tensor),
        the ``e`` of the forward call over the same slices, and returns ``dm`` relative to it: the plan
        runs as with the primal and the tangent is rescaled by ``10^(e_run - exponent)``.  A zero result
        gives a zero ``dm``.  ``exponent`` belongs to that call only: given with ``primal=True``, or to an
        executor without ``strip_exponent``, it raises ``ValueError``.  ``strip_exponent`` executors
        without ``stripped_grad`` raise ``NotImplementedError``."""
        torch = _torch()
        if exponent is not None and (primal or not self.strip_exponent):
            raise ValueError("exponent= is the forward's e for a stripped tangent without the primal "
                             "(strip_exponent executors, primal=False)")
        self._check_inputs(tensors)
        begin, step, count = self._check_slice_range(begin, step, count)
        plan = self.jvp_plan(wrt, _two_term)
        if plan.strip_exponent:
            return self._jvp_stripped(plan, tensors, tangents, begin, step, count, primal, exponent)
        odt = getattr(torch, self.out_dtype)
        with torch.cuda.device(self.device):
            ptrs, _keep = self._input_ptrs(tensors)
            tans, tptrs = self._jvp_tangents(plan, tangents, len(tensors))
            out = torch.zeros(plan.out_shape, dtype=odt, device=self.device) if primal else None
            tout = torch.zeros(plan.out_shape, dtype=odt, device=self.device)
            if not plan.tangent_nodes:  # nothing to differentiate: the tangent is zero
                if primal:
                    self.contract_device(tensors, begin, step, count, out=out)
                return (out, tout) if primal else tout
            if self._jvp_ws is None or self._jvp_ws.numel() < plan.total_bytes:
                self._jvp_ws = None
                self._jvp_ws = torch.empty(max(plan.total_bytes, 1), dtype=torch.uint8, device=self.device)
            ws = self._jvp_ws
            plan.execute(ptrs, tptrs, out.data_ptr() if primal else None, tout.data_ptr(), ws.data_ptr(), ws.numel(),
                         begin, step, count, _stream_ptr())
        return (out, tout) if primal else tout

    def _jvp_stripped(self, plan, tensors, tangents, begin, step, count, primal, exponent):
        torch = _torch()
        if not primal and exponent is None:
            raise ValueError("a stripped tangent without the primal needs the exponent of the forward call "
                             "(exponent=)")
        odt = getattr(torch, self.out_dtype)
        with torch.cuda.device(self.device):
            ptrs, _keep = self._input_ptrs(tensors)
            tans, tptrs = self._jvp_tangents(plan, tangents, len(tensors))
            out = torch.zeros(plan.out_shape, dtype=odt, device=self.device)
            tout = torch.zeros(plan.out_shape, dtype=odt, device=self.device)
            if not plan.tangent_nodes:  # nothing to differentiate: the tangent is zero
                m, e = self.contract_device(tensors, begin, step, count, out=out)
                return ((m, e), tout) if primal else tout
            e = torch.full((1,), -math.inf, dtype=torch.float64, device=self.device)
            if self._jvp_ws is None or self._jvp_ws.numel() < plan.total_bytes:
                self._jvp_ws = None
                self._jvp_ws = torch.empty(max(plan.total_bytes, 1), dtype=torch.uint8, device=self.device)
            ws = self._jvp_ws
            plan.execute(ptrs, tptrs, out.data_ptr(), tout.data_ptr(), ws.data_ptr(), ws.numel(), begin, step,
                         count, _stream_ptr(), exp_ptr=e.data_ptr())
            if self._exp_shift:
                e.add_(self._exp_shift)  # (the folds' exponents scale m and dm alike)
            if primal:
                return (out, e), tout
            # dm relative to the caller's exponent: 10^(e - exponent), 1 where both are -inf
            want = torch.as_tensor(exponent, dtype=torch.float64).to(self.device).reshape(1)
            scale = torch.where(e == want, torch.ones_like(e), torch.pow(10.0, e - want))
            tout.mul_(scale.reshape(()).to(tout.dtype))
        return tout

    def _jvp_tangents(self, plan, tangents, n_ptrs):
        """The tangents of ``plan.wrt`` as contiguous device tensors, and one pointer per plan input
        (``None`` outside ``wrt``)."""
        torch = _torch()
        if len(tangents) != len(plan.wrt):
            raise ValueError(f"expected {len(plan.wrt)} tangents (one per input in wrt), got {len(tangents)}")
        tdt = getattr(torch, self.dtype)
        tans, tptrs = [], [None] * (n_ptrs + len(self._resident))
        for i, t in zip(plan.wrt, tangents):
            if tuple(t.shape) != tuple(self._shapes[i]):
                raise ValueError(f"tangent of input {i} has shape {tuple(t.shape)}, expected {self._shapes[i]}")
            t = t.to(device=self.device, dtype=tdt).contiguous()
            tans.append(t)
            tptrs[i] = t.data_ptr()
        return tans, tptrs

    def _check_slice_range(self, begin, step, count):
        """Slice ids ``begin, begin+step, ...`` must all lie in ``[0, nslices)``: the device
        decodes digits modulo the radices, so an id past the end would silently wrap and
        count a slice twice."""
        begin, step = int(begin), int(step)
        if step < 1 or begin < 0:
            raise ValueError(f"bad slice range begin={begin} step={step}")
        if count is None:
            count = max(0, -(-(self.nslices - begin) // step))
        count = int(count)
        if count < 0 or (count > 0 and begin + (count - 1) * step >= self.nslices):
            raise ValueError(
                f"slice ids {begin}..{begin + (count - 1) * step} (step {step}) exceed the tree's "
                f"{self.nslices} slices")
        return begin, step, count

    def contract_host(self, arrays, begin=0, step=1, count=None):
        """End-to-end with HOST buffers through ``ctgb_plan_execute_host``:
        H2D of the inputs, all slices, D2H of the result, synchronised.  An executor with resident
        tensors copies its variables to the device and runs ``contract_device``."""
        torch = _torch()
        self._check_inputs(arrays)
        begin, step, count = self._check_slice_range(begin, step, count)
        if self._resident:
            res = self.contract_device([_to_device(np.asarray(a, dtype=self.dtype), self.device)[0] for a in arrays],
                                       begin, step, count)
            if self.strip_exponent:
                return _from_device(res[0], True), float(res[1].item())
            return _from_device(res, True)
        host = [np.asarray(a, dtype=self.dtype, order="C") for a in arrays]
        out = np.zeros(self.plan.out_shape, dtype=self.out_dtype)
        with torch.cuda.device(self.device):
            ws = self.workspace(host_staging=True)
            e = self.plan.execute_host(host, out, ws.data_ptr(), ws.numel(), begin, step, count,
                                       _stream_ptr())
        return (out, e) if self.strip_exponent else out


class TreeExecutor(_Executor):
    """A compiled sliced contraction: ``ContractionTree.contract`` on the GPU.

    Built from a ``TreeSpec`` or from a live cotengra tree (captured through
    ``TreeSpec.from_cotengra``).  The slice loop, the node loop, the slice
    accumulation and (optionally) exponent stripping all run inside
    ``ctgb_plan_execute``.  The options are those of ``_Executor``.

    ``constants={position: array}`` fixes the inputs at those positions of ``tree.inputs`` (numpy
    arrays or torch tensors of the input's full shape and the executor's dtype).  Every subtree whose
    leaves are all constant is contracted once, here, within ``fold_max_bytes`` of folded arrays
    (default: the unfolded forward plan's ``workspace_bytes``; 0 folds nothing; ``constants.py``), and
    every entry point then takes only the remaining inputs, the *variables*, in their original order;
    ``wrt`` counts positions among them.  The constants are copied: changing them afterwards has no
    effect, and they get no gradient.  ``folded`` lists the folds (``constants.Fold``: SSA id, term,
    bytes, MACs per call removed) and ``folded_bytes`` their size.  When every input is constant the
    result is formed here and each full call returns a fresh copy of it: numpy if every constant was
    numpy, a torch CUDA tensor otherwise.
    """

    def __init__(self, tree, dtype="complex128", strip_exponent=False, device=None,
                 contractions=None, fuse=True, vjp_max_bytes=None, precision="3xtf32", stripped_grad=False,
                 accumulate="native", constants=None, fold_max_bytes=None, **plan_opts):
        check_precision(precision, dtype)
        check_accumulate(accumulate)
        self.spec = spec = tree if isinstance(tree, TreeSpec) else TreeSpec.from_cotengra(tree)
        # stem fusion (fusion.py): an execution-plan transformation of the tree cotengra found --
        # big stem tensors absorb pre-contracted groups of small tensors in one pass.  ``spec``
        # stays the caller's tree; ``exec_spec`` is what runs.  ``fuse=False`` executes the
        # reference's own node sequence one to one.
        self.exec_spec, self.fusion = spec, {"changed": False}
        if fuse and contractions is None:
            from .fusion import fuse_stems

            # (``fuse`` may be a dict of planner options -- min_big, ratio, min_gain, model -- e.g. to
            # force fusion on small trees in tests)
            opts = fuse if isinstance(fuse, dict) else {}
            self.exec_spec, self.fusion = fuse_stems(spec, dtype_name(dtype), **opts)
        ir = self.exec_spec.contractions() if contractions is None else contractions
        opts = dict(strip_exponent=strip_exponent, device=device, vjp_max_bytes=vjp_max_bytes, precision=precision,
                    stripped_grad=stripped_grad, accumulate=accumulate,
                    absorb_root=bool(fuse) and contractions is None, **plan_opts)
        self.constants, self.folded, self.folded_bytes, self._const_digest = (), [], 0, None
        if constants is None:
            super().__init__(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype, **opts)
        else:
            if contractions is not None:
                raise ValueError("constants are folded on the tree's own program: not with contractions=")
            self._init_folded(ir, dtype_name(dtype), constants, fold_max_bytes, opts)
        self._ref_work = None

    def _init_folded(self, ir, dtype, constants, fold_max_bytes, opts):
        """Fold the constant subtrees (``constants.plan_folds``) on the device and compile what
        remains, with the folded arrays and the unfolded constant leaves as resident inputs."""
        from . import constants as K

        torch = _torch()
        spec = self.spec
        consts = K.check_constants(constants, spec.shapes(), dtype)
        self.constants = tuple(sorted(consts))
        self._const_digest = K.digest(consts, dtype)
        dev = torch.device("cuda", torch.cuda.current_device() if opts["device"] is None else opts["device"])
        # the keywords of the plans that form the folded arrays: F is stored in the plan dtype
        fold_kw = {k: v for k, v in opts.items()
                   if k not in ("device", "vjp_max_bytes", "stripped_grad", "absorb_root", "accumulate")}
        with torch.cuda.device(dev):
            leaves = {}
            for i, x in consts.items():
                t, was_numpy = _to_device(x, dev)
                leaves[i] = t.detach() if was_numpy else t.detach().clone()
            if len(consts) == len(spec.inputs):
                terms, ids, resident, runs = list(spec.inputs), None, [leaves[i] for i in range(len(consts))], []
            else:
                cost = ExecPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype, **fold_kw)
                fp = K.plan_folds(self.exec_spec, ir, consts, dtype, fold_max_bytes, cost)
                runs = [self._fold(f, leaves, dtype, fold_kw, dev) for f in fp.folds]
                resident = [r[0] for r in runs] + [leaves[i] for i in fp.resident_leaves]
                terms, ids, ir = fp.inputs, fp.input_ids, fp.records
                self.folded = fp.folds
                self.folded_bytes = sum(f.bytes for f in fp.folds)
            del leaves
            super().__init__(ir, terms, spec.output, spec.size_dict, spec.sliced, dtype, resident=resident,
                             input_ids=ids, **opts)
            if len(consts) == len(spec.inputs):
                self._constant_result = self.contract_device([])
                self._constant_numpy = all(not isinstance(a, torch.Tensor) for a in consts.values())
            torch.cuda.synchronize(dev)
        # the folds' exponents, read once everything has run
        self._exp_shift = sum(float(r[1].item()) for r in runs if r[1] is not None)

    def _fold(self, f, leaves, dtype, fold_kw, dev):
        """Start forming ``F`` of the fold ``f`` from its constant leaves, in the plan dtype: returns
        ``(F, exponent tensor or None, plan, workspace)``, the last two to be kept until it has run."""
        torch = _torch()
        plan = ExecPlan(f.records, [self.spec.inputs[i] for i in f.leaves], f.term, self.spec.size_dict, f.sliced,
                        dtype=dtype, input_ids=f.leaves, **fold_kw).create()
        out = torch.zeros(plan.out_shape, dtype=getattr(torch, dtype), device=dev)
        exp = torch.full((1,), -math.inf, dtype=torch.float64, device=dev) if plan.strip_exponent else None
        ws = torch.empty(max(plan.total_bytes, 1), dtype=torch.uint8, device=dev)
        plan.execute([leaves[i].data_ptr() for i in f.leaves], out.data_ptr(),
                     exp.data_ptr() if exp is not None else None, ws.data_ptr(), ws.numel(), 0, 1, plan.nslices,
                     _stream_ptr())
        return out, exp, plan, ws

    @property
    def reference_work(self):
        """``(macs_per_slice, macs_invariant, elements_per_slice)`` of the caller's (unfused)
        tree -- the algorithmic work throughput figures are quoted on."""
        if self._ref_work is None:
            if self.fusion.get("changed"):
                from .fusion import tree_work

                self._ref_work = tree_work(self.spec)
            else:
                self._ref_work = (self.plan.macs_per_slice, self.plan.macs_invariant,
                                  self.plan.elements_per_slice)
        return self._ref_work

    def __call__(self, arrays, **kw):
        return contract_tree(self, arrays, **kw)

    def _numpy_out(self, torch, arrays):
        """Whether results of a call on ``arrays`` come back as numpy: numpy variables, or, when every
        input is constant, numpy constants."""
        if not arrays and self.constants:
            return self._constant_numpy
        return all(not isinstance(a, torch.Tensor) for a in arrays)

    # ------------------------------------------------------------------ output chunks
    def _chunk_plan(self):
        """A second plan over the same program whose output is ONE chunk: the output term
        without its sliced indices, so that every sliced index is summed.  Executed over the
        ``stepsize`` consecutive slice ids of a chunk (core.py:3916-3935)."""
        if getattr(self, "_chunk", None) is None:
            torch = _torch()
            spec = self.exec_spec
            chunk_out, _step, _n = output_chunking(spec)
            # (with constants: the folded program, whose last inputs are resident)
            ir, inputs = self._program[:2] if self.constants else (spec.contractions(), spec.inputs)
            with torch.cuda.device(self.device):
                self._chunk = ExecPlan(ir, inputs, chunk_out, spec.size_dict,
                                       spec.sliced, dtype=self.dtype,
                                       strip_exponent=self.strip_exponent, precision=self.precision,
                                       accumulate=self.accumulate,
                                       input_ids=self._plan_opts.get("input_ids")).create()
        return self._chunk

    def gen_output_chunks(self, arrays, with_key=False):
        """``tree.gen_output_chunks(arrays, with_key)`` (cotengra/core.py:3884-3941): yield
        every output chunk -- one per setting of the sliced *output* indices -- after its
        inner slices have been summed on the device, without ever forming the full output.
        Like the reference this needs the sliced indices ordered output-first (the default
        order, core.py:99-104); unlike it, ``strip_exponent`` chunks are summed with the
        exponent-aware adder and come as ``(mantissa, exponent)``.
        numpy in -> numpy chunks; torch CUDA in -> torch CUDA chunks (a fresh tensor each)."""
        torch = _torch()
        self._check_inputs(arrays)
        spec = self.spec
        _chunk_out, stepsize, nchunks = output_chunking(spec)
        plan = self._chunk_plan()
        all_numpy = self._numpy_out(torch, arrays)
        tensors = [_to_device(a, self.device)[0] for a in arrays]
        ptrs = [t.data_ptr() for t in tensors] + [t.data_ptr() for t in self._resident]
        tdt = getattr(torch, self.out_dtype)
        need = plan.total_bytes
        # a buffer of its own, not ``_ws``: the generator yields between launches, and a
        # ``contract_device`` call in between must not overwrite the arena of a pending chunk
        with torch.cuda.device(self.device):
            ws = torch.empty(max(need, 1), dtype=torch.uint8, device=self.device)
        for o in range(nchunks):
            with torch.cuda.device(self.device):
                out = torch.zeros(plan.out_shape, dtype=tdt, device=self.device)
                exp = (torch.full((1,), -math.inf, dtype=torch.float64, device=self.device)
                       if self.strip_exponent else None)
                plan.execute(ptrs, out.data_ptr(), exp.data_ptr() if exp is not None else None,
                             ws.data_ptr(), ws.numel(), o * stepsize, 1, stepsize, _stream_ptr())
            chunk = _from_device(out, all_numpy)
            if self.strip_exponent:
                chunk = (chunk, float(exp.item()) + self._exp_shift)
            if with_key:
                key = {ix: x for ix, x in spec.slice_key(o * stepsize).items() if ix in spec.output}
                yield chunk, key
            else:
                yield chunk


def contract_tree(tree, arrays, strip_exponent=False, check_zero=False, dtype=None,
                  slice_ids=None, vjp_max_bytes=None, precision="3xtf32", stripped_grad=False,
                  accumulate="native", **plan_opts):
    """``tree.contract(arrays)`` (cotengra/core.py:3943): takes the *unsliced*
    arrays, handles slicing, contraction and gathering, returns the output in
    ``tree.output`` order -- or ``(mantissa, exponent)`` with ``strip_exponent``.
    numpy in -> numpy out; torch CUDA in -> torch CUDA out.  The options are the executor's
    (``TreeExecutor``); an executor passed in keeps its own, except that ``vjp_max_bytes``, when
    given, bounds the workspace of this call's backward pass.  With ``stripped_grad`` a stripped
    result records the gradient of its mantissa, the exponent (a float, as without it) held constant."""
    torch = _torch()
    ex = _executor_for(tree, arrays, dtype, strip_exponent=strip_exponent, vjp_max_bytes=vjp_max_bytes,
                       precision=precision, stripped_grad=stripped_grad, accumulate=accumulate, **plan_opts)
    slices = (0, 1, None) if slice_ids is None else slice_ids
    if ex._constant_result is not None and not ex._constant_numpy:
        return _run_device(ex, arrays, [], slices, check_zero)
    if all(not isinstance(a, torch.Tensor) for a in arrays):
        res = ex.contract_host(arrays, *slices)
        return _finish_stripped(*res, check_zero) if ex.strip_exponent else res
    tensors = [_to_device(a, ex.device)[0] for a in arrays]
    return _run_device(ex, arrays, tensors, slices, check_zero, max_bytes=vjp_max_bytes)


def _executor_for(tree, arrays, dtype=None, **opts):
    """``tree`` itself if it is a ``TreeExecutor`` (which keeps its own options), else a ``TreeExecutor``
    built from it with ``opts``, for ``dtype`` or by default that of ``arrays[0]``."""
    if isinstance(tree, TreeExecutor):
        return tree
    return TreeExecutor(tree, dtype=dtype_name(arrays[0].dtype) if dtype is None else dtype, **opts)


def _run_device(ex, arrays, tensors, slices, check_zero=False, max_bytes=None, as_numpy=False):
    """``ex.contract_device`` of the device ``tensors`` (made from the caller's ``arrays``) over the
    slices ``(begin, step, count)``: one torch autograd node when ``_records_grad`` says so or some
    array carries a forward-mode tangent (``_tangent_inputs``), whose backward is ``ex.vjp`` over the
    same slices within ``max_bytes`` and whose forward-mode rule is ``ex.jvp`` over them; a plain run
    otherwise.  The result comes back as numpy with ``as_numpy``, and a stripped one as
    ``(mantissa, float exponent)``."""
    torch = _torch()
    begin, step, count = slices
    dual = _tangent_inputs(torch, arrays, ex.strip_exponent, ex.stripped_grad)
    if _records_grad(torch, arrays, ex.strip_exponent, ex.stripped_grad) or dual:
        jvp = None
        if dual:
            def jvp(ts, tans, e=None):
                return ex.jvp(ts, [tans[i] for i in dual], begin, step, count, wrt=dual, primal=False, exponent=e)
        res = _differentiable(torch, lambda ts: ex.contract_device(ts, begin, step, count),
                              lambda ts, g, wrt, e=None: ex.vjp(ts, g, begin, step, count, wrt=wrt,
                                                                max_bytes=max_bytes, exponent=e), tensors, jvp)
    else:
        res = ex.contract_device(tensors, begin, step, count)
    if ex.strip_exponent:
        m, e = res
        return _finish_stripped(m, float(e.item()), check_zero, as_numpy)
    return _from_device(res, as_numpy)


def _records_grad(torch, arrays, strip_exponent, stripped_grad=False):
    """Whether a call records a torch autograd node: torch tensor inputs, at least one requiring
    grad, grad mode on.  ``strip_exponent`` results get no gradient (a warning says so) unless
    ``stripped_grad`` asks for the mantissa's, with the exponent held constant."""
    if not torch.is_grad_enabled() or not arrays:
        return False
    if not all(isinstance(a, torch.Tensor) for a in arrays) or not any(a.requires_grad for a in arrays):
        return False
    if strip_exponent and not stripped_grad:
        warnings.warn("strip_exponent=True: no gradient is recorded for the (mantissa, exponent) result",
                      UserWarning, stacklevel=4)  # (the caller of contract_tree / B200Contractor, past _run_device)
        return False
    return True


def _tangent_inputs(torch, arrays, strip_exponent, stripped_grad=False):
    """Positions of the arrays that carry a ``torch.autograd.forward_ad`` tangent (all must be torch
    tensors).  ``strip_exponent`` results get no tangent (a warning says so and the list is empty)
    unless ``stripped_grad`` asks for the mantissa's, with the exponent held constant."""
    if not arrays or not all(isinstance(a, torch.Tensor) for a in arrays):
        return []
    from torch.autograd import forward_ad

    dual = [i for i, a in enumerate(arrays) if forward_ad.unpack_dual(a).tangent is not None]
    if dual and strip_exponent and not stripped_grad:
        warnings.warn("strip_exponent=True: no forward-mode tangent is recorded for the (mantissa, exponent) "
                      "result", UserWarning, stacklevel=4)
        return []
    return dual


_GRAD_FN = None


def _differentiable(torch, run, vjp, tensors, jvp=None):
    """``run(tensors)`` as one torch autograd node whose backward is ``vjp(tensors, grad, wrt)``
    (a ``VjpPlan`` on the device; ``wrt`` from ``ctx.needs_input_grad``) and whose forward-mode rule
    is ``jvp(tensors, tangents)`` (a ``JvpPlan``; ``tangents`` has one entry per tensor, zeros where
    torch has none, and ``jvp`` reads those of the inputs it was made for).  A stripped ``run``
    returns ``(m, e)``: ``e`` is not differentiable, the backward is ``vjp(tensors, grad_m, wrt, e)``
    and the forward-mode rule, if any, ``jvp(tensors, tangents, e)``, the tangent of ``m``."""
    global _GRAD_FN
    if _GRAD_FN is None:
        from torch.autograd.function import once_differentiable

        class _Contract(torch.autograd.Function):
            @staticmethod
            def forward(ctx, run, vjp, jvp, *tensors):
                ctx.vjp, ctx.jvp_fn = vjp, jvp
                res = run(list(tensors))
                ctx.stripped = isinstance(res, tuple)
                if ctx.stripped:
                    ctx.mark_non_differentiable(res[1])
                    ctx.save_for_backward(*tensors, res[1])
                    if jvp is not None:
                        ctx.save_for_forward(*tensors, res[1])  # (dm is relative to this e)
                else:
                    ctx.save_for_backward(*tensors)
                    if jvp is not None:
                        ctx.save_for_forward(*tensors)
                return res

            @staticmethod
            @once_differentiable
            def backward(ctx, grad, *_grad_e):
                wrt = [i for i, need in enumerate(ctx.needs_input_grad[3:]) if need]
                saved = list(ctx.saved_tensors)
                if ctx.stripped:
                    grads = ctx.vjp(saved[:-1], grad, wrt, saved[-1])
                else:
                    grads = ctx.vjp(saved, grad, wrt)
                return (None, None, None, *grads)

            @staticmethod
            def jvp(ctx, _run_t, _vjp_t, _jvp_t, *tangents):
                if ctx.jvp_fn is None:
                    return (None, None) if ctx.stripped else None
                saved = list(ctx.saved_tensors)
                if ctx.stripped:
                    return ctx.jvp_fn(saved[:-1], list(tangents), saved[-1]), None
                return ctx.jvp_fn(saved, list(tangents))

        _GRAD_FN = _Contract
    return _GRAD_FN.apply(run, vjp, jvp, *tensors)


def gen_output_chunks(tree, arrays, with_key=False, strip_exponent=False, dtype=None, precision="3xtf32",
                      accumulate="native", **plan_opts):
    """``tree.gen_output_chunks(arrays, with_key=...)`` (cotengra/core.py:3884-3941) on the
    GPU executor; see ``TreeExecutor.gen_output_chunks``."""
    ex = _executor_for(tree, arrays, dtype, strip_exponent=strip_exponent, precision=precision,
                       accumulate=accumulate, **plan_opts)
    yield from ex.gen_output_chunks(arrays, with_key=with_key)


def array_contract_expression(inputs, output=None, size_dict=None, shapes=None, optimize=None, constants=None,
                              strip_exponent=False, dtype=None, **executor_opts):
    """``cotengra.array_contract_expression`` (interface.py:673-768) on the tree executor: a callable
    ``expr(*variables, backend=None)`` that contracts the inputs not in ``constants`` (``{position:
    array}``, folded once, ``TreeExecutor(constants=...)``) along the tree ``optimize``, a
    ``TreeSpec`` or a live cotengra ``ContractionTree`` whose inputs, output and index sizes match
    the arguments (``ValueError`` otherwise; path search stays in cotengra).  ``size_dict`` or
    ``shapes`` give the sizes, default the tree's; ``output`` defaults to the tree's.  ``dtype``
    defaults to the constants' common dtype, or without constants to that of the first call's arrays.
    Results as ``contract_tree``: ``(mantissa, exponent)`` with ``strip_exponent``, numpy for numpy
    variables.  ``executor_opts`` are ``TreeExecutor``'s."""
    if optimize is None:
        raise ValueError("optimize must be a TreeSpec or a cotengra ContractionTree (path search stays in cotengra)")
    try:
        spec = optimize if isinstance(optimize, TreeSpec) else TreeSpec.from_cotengra(optimize)
    except AttributeError:
        raise ValueError(f"optimize must be a TreeSpec or a cotengra ContractionTree, got {type(optimize)}") from None
    inputs = tuple(tuple(t) for t in inputs)
    if shapes is not None:
        if len(shapes) != len(inputs):
            raise ValueError(f"{len(shapes)} shapes for {len(inputs)} inputs")
        size_dict = {}
        for term, shp in zip(inputs, shapes):
            if len(term) != len(shp):
                raise ValueError(f"input {term} has {len(shp)} dimensions")
            for ix, d in zip(term, shp):
                if size_dict.setdefault(ix, int(d)) != int(d):
                    raise ValueError(f"index {ix!r} has two sizes")
    if inputs != spec.inputs:
        raise ValueError("the tree's inputs differ from the expression's")
    if output is not None and tuple(output) != spec.output:
        raise ValueError(f"the tree's output {''.join(map(str, spec.output))!r} differs from the expression's")
    if size_dict is not None and any(int(size_dict.get(ix, -1)) != d for ix, d in spec.size_dict.items()
                                     if any(ix in t for t in inputs)):
        raise ValueError("the tree's index sizes differ from the expression's")
    if constants is not None:
        from .constants import check_constants

        constants = check_constants(constants, spec.shapes())
        if dtype is None and constants:
            names = {dtype_name(a.dtype) for a in constants.values()}
            if len(names) != 1:
                raise TypeError(f"constants of several dtypes {sorted(names)}: give dtype=")
            dtype = names.pop()
    return _Expression(spec, constants, dict(executor_opts, strip_exponent=strip_exponent), dtype)


class _Expression:
    """``expr(*variables, backend=None)`` of ``array_contract_expression``: one ``TreeExecutor``,
    built on the first call when the dtype comes from the arrays."""

    def __init__(self, spec, constants, opts, dtype):
        self.spec, self.constants, self.opts = spec, constants, opts
        self.executor = None if dtype is None else TreeExecutor(spec, dtype=dtype, constants=constants, **opts)

    def __call__(self, *arrays, backend=None):
        if self.executor is None:
            if not arrays:
                raise ValueError("the expression's dtype comes from its arrays: call it with its variables")
            self.executor = TreeExecutor(self.spec, dtype=dtype_name(arrays[0].dtype), constants=self.constants,
                                         **self.opts)
        return contract_tree(self.executor, list(arrays))


def benchmark(tree, dtype="float64", max_time=60, min_reps=3, max_reps=100, warmup=True,
              executor=None, precision="3xtf32", accumulate="native", **plan_opts):
    """``tree.benchmark(dtype, max_time, min_reps, max_reps, warmup)`` (cotengra/core.py:
    4092-4164) on the GPU executor, same protocol and same keys: random inputs, ``warmup``
    untimed slices, then single slices ``i % nslices`` (each one synchronised, as the
    reference's eager numpy calls are) until ``max_time`` seconds or ``max_reps`` repetitions
    are over, but at least ``min_reps``.  Returns ``time_per_slice``, ``est_time_total`` (x
    nslices) and ``est_gigaflops`` with the reference's own flop count
    (``total_flops(dtype)``, core.py:1196-1227: 2 flops per scalar multiply-add for float
    dtypes, 4 for complex ones -- half of the 8-flop convention bench.py reports)."""
    import time

    torch = _torch()
    ex = executor if executor is not None else _executor_for(tree, (), dtype, precision=precision,
                                                             accumulate=accumulate, **plan_opts)
    tdt = getattr(torch, ex.dtype)
    gen = torch.Generator(device=ex.device)
    gen.manual_seed(0)
    tensors = []
    for shp in ex._shapes:  # (the variables of an executor with constants)
        t = torch.empty(tuple(shp), dtype=tdt, device=ex.device)
        (torch.view_as_real(t) if t.is_complex() else t).normal_(generator=gen)
        tensors.append(t / max(1.0, float(t.numel()) ** 0.5))
    nslices = int(ex.nslices)
    out = torch.zeros(ex.plan.out_shape, dtype=getattr(torch, ex.out_dtype), device=ex.device)

    def one(i):
        ex.contract_device(tensors, begin=i % nslices, step=1, count=1, out=out)
        torch.cuda.synchronize(ex.device)

    for i in range(int(warmup)):
        one(i)
    t0 = ti = time.time()
    i = 0
    while (ti - t0 < max_time) or (i < min_reps):
        one(i)
        ti = time.time()
        i += 1
        if i >= max_reps:
            break
    time_per_slice = (ti - t0) / i
    est_time_total = time_per_slice * nslices
    per_mac = 4 if "complex" in ex.dtype else 2
    # tree.total_flops(dtype) counts every node of every slice (core.py:1196-1227), the
    # slice-invariant ones included -- each timed single-slice call re-runs them here too
    macs_v, macs_i, _el = ex.reference_work
    total_flops = per_mac * (macs_v + macs_i) * nslices
    return {
        "time_per_slice": time_per_slice,
        "est_time_total": est_time_total,
        "est_gigaflops": total_flops / (1e9 * est_time_total),
    }


def _combine_stripped(m1, e1, m2, e2):
    """``AdderWithMaybeExponentStripped`` (cotengra/core.py:163-170) for two
    (mantissa, exponent) partial sums."""
    if e1 == -math.inf:
        return m2, e2
    if e2 == -math.inf:
        return m1, e1
    # a NaN exponent stays NaN whichever side it is on (Python's max would keep it on one side only)
    e = math.nan if math.isnan(e1) or math.isnan(e2) else max(e1, e2)
    return m1 * 10.0 ** (e1 - e) + m2 * 10.0 ** (e2 - e), e


def contract_checkpointed(tree, arrays, checkpoint, every=1024, strip_exponent=False, dtype=None,
                          executor=None, on_block=None, precision="3xtf32", accumulate="native", **plan_opts):
    """``tree.contract(arrays)`` for runs too long to lose (SURVEY 8f-4, partial-sum
    checkpointing; the reference has no equivalent -- ``tree.contract`` restarts at
    slice 0): the slices are contracted in blocks of ``every``, and after each block
    the running sum -- ``(mantissa, exponent)`` with ``strip_exponent``, combined as
    core.py:163-170 -- and the next slice id are written to ``checkpoint`` (.npz,
    atomic replace).  A later call with the same tree, dtype and input values finds
    the file and resumes behind the last completed block; a file written for a
    different tree or different inputs is refused (``ValueError``), never silently
    overwritten.  Slices are independent, so the result equals the uninterrupted
    run up to floating-point summation order.  numpy inputs and outputs (host path).
    ``on_block(next_slice, nslices)`` is called after every saved block.  A file written
    under the other ``precision`` is refused too: the two modes give different sums.  With
    ``accumulate="double"`` on a float32 / complex64 tree the stored partial is the float64 /
    complex128 one, and a file of one accumulation mode is refused by the other."""
    import hashlib
    import os

    ex = executor if executor is not None else _executor_for(tree, arrays, dtype, strip_exponent=strip_exponent,
                                                             precision=precision, accumulate=accumulate,
                                                             **plan_opts)
    spec = ex.spec
    host = [np.asarray(a, dtype=ex.dtype, order="C") for a in arrays]
    h = hashlib.sha256()
    h.update(spec.to_json().encode())
    h.update(f"|{ex.dtype}|{int(bool(ex.strip_exponent))}|".encode())
    precision = getattr(ex, "precision", "3xtf32")
    if precision != "3xtf32":  # (the default mode hashes as before: existing checkpoints resume)
        h.update(f"precision={precision}|".encode())
    out_dtype = getattr(ex, "out_dtype", ex.dtype)
    if out_dtype != ex.dtype:  # (as above: the native tag is the one files already carry)
        h.update(f"accumulate={out_dtype}|".encode())
    for a in host:
        h.update(str(a.shape).encode())
        h.update(a.tobytes())
    if getattr(ex, "constants", ()):  # (executors without constants hash as before)
        h.update(f"|constants={list(ex.constants)}|{ex._const_digest}".encode())
    tag = h.hexdigest()
    nslices = int(ex.nslices)
    every = max(1, int(every))

    done, total, exponent = 0, None, -math.inf
    if os.path.exists(checkpoint):
        with np.load(checkpoint, allow_pickle=False) as z:
            if str(z["tag"]) != tag:
                raise ValueError(f"{checkpoint} belongs to a different tree, dtype, precision, accumulator or set of "
                                 f"input values")
            done, total, exponent = int(z["next_slice"]), z["partial"], float(z["exponent"])
    while done < nslices:
        count = min(every, nslices - done)
        res = ex.contract_host(host, done, 1, count)
        if ex.strip_exponent:
            m, e = res
            total, exponent = (m, float(e)) if total is None else _combine_stripped(total, exponent, m, float(e))
        else:
            total = res if total is None else total + res
        done += count
        tmp = f"{checkpoint}.tmp.npz"
        np.savez(tmp, tag=np.array(tag), next_slice=np.int64(done), partial=np.asarray(total),
                 exponent=np.float64(exponent))
        os.replace(tmp, checkpoint)
        if on_block is not None:
            on_block(done, nslices)
    return (total, exponent) if ex.strip_exponent else total


def _finish_stripped(m, e, check_zero, as_numpy=False):
    if check_zero and e == -math.inf:
        # contract.py:819-820
        return 0.0, float("-inf")
    return _from_device(m, as_numpy), e


class B200Contractor:
    """Drop-in for ``cotengra.contract.Contractor`` (contract.py:654-837): built
    from the reference's contraction records, called with the (already sliced)
    arrays of one slice, returns the output array or ``(mantissa, exponent)``.

    Where the reference walks the records in Python and dispatches three array
    ops per node, this compiles them once per (shapes, dtype) into a ``ctgb_plan``
    and runs the whole node loop in one C call.
    """

    __slots__ = ("contractions", "strip_exponent", "check_zero", "implementation", "backend",
                 "progbar", "vjp_max_bytes", "precision", "stripped_grad", "accumulate", "_plans", "__weakref__")

    def __init__(self, contractions, strip_exponent=False, check_zero=False,
                 implementation="b200", backend=None, progbar=False, vjp_max_bytes=None, precision="3xtf32",
                 stripped_grad=False, accumulate="native"):
        self.contractions = tuple(contractions)
        self.accumulate = check_accumulate(accumulate)  # dtype the result is summed and returned in (TreeExecutor)
        # compute mode of the float32 / complex64 tensor-core nodes (TreeExecutor); checked per dtype at call
        self.precision = check_precision(precision)
        self.vjp_max_bytes = vjp_max_bytes  # workspace bound of the backward pass (VjpPlan max_bytes)
        # stripped results record the mantissa's gradient, the exponent held constant (TreeExecutor)
        self.stripped_grad = bool(stripped_grad)
        self.strip_exponent = strip_exponent
        self.check_zero = check_zero
        self.implementation = implementation
        self.backend = backend
        self.progbar = progbar
        self._plans = {}

    @classmethod
    def from_tree(cls, tree, **kw):
        """Build from a cotengra tree or a ``TreeSpec`` (records of one slice)."""
        spec = tree if isinstance(tree, TreeSpec) else TreeSpec.from_cotengra(tree)
        return cls(spec.contractions(), **kw)

    def _executor(self, shapes, dtype, strip):
        key = (shapes, dtype, strip, _torch().cuda.current_device())
        ex = self._plans.get(key)
        if ex is None:
            # synthesise a flat (unsliced) network whose inputs are the given arrays and whose
            # output term is whatever the program produces
            inputs = [tuple((i, k) for k in range(len(s))) for i, s in enumerate(shapes)]
            size_dict = {(i, k): d for i, s in enumerate(shapes) for k, d in enumerate(s)}
            out_shape = _program_output_shape(self.contractions, shapes)
            output = tuple(("o", k) for k in range(len(out_shape)))
            size_dict.update({("o", k): d for k, d in enumerate(out_shape)})
            ex = self._plans[key] = _Executor(self.contractions, inputs, output, size_dict, (), dtype,
                                              strip_exponent=strip, vjp_max_bytes=self.vjp_max_bytes,
                                              precision=self.precision, stripped_grad=self.stripped_grad,
                                              accumulate=self.accumulate)
        return ex

    def __call__(self, *arrays, **kwargs):
        kwargs.pop("backend", None)
        kwargs.pop("progbar", None)
        check_zero = kwargs.pop("check_zero", self.check_zero)
        strip_exponent = kwargs.pop("strip_exponent", self.strip_exponent)
        kwargs.pop("implementation", None)
        if kwargs:
            raise TypeError(f"Unknown keyword arguments: {kwargs}.")
        torch = _torch()
        devs = [_to_device(a) for a in arrays]
        tensors = [d[0] for d in devs]
        dtype = _common_dtype(*tensors)
        with torch.cuda.device(tensors[0].device if tensors else torch.cuda.current_device()):
            ex = self._executor(tuple(tuple(t.shape) for t in tensors), dtype, strip_exponent is not False)
            return _run_device(ex, arrays, [t.to(ex.device) for t in tensors], (0, 1, 1), check_zero,
                               as_numpy=all(d[1] for d in devs))


def _program_output_shape(contractions, shapes):
    """Propagate shapes through the IR (host integer work)."""
    live = {i: tuple(s) for i, s in enumerate(shapes)}
    shp = None
    for p, l, r, tdot, arg, perm in contractions:
        if r is None:
            src = live[p] if l is None else live[l]
            terms, out = split_equation(arg)
            ext = {}
            for ix, d in zip(terms[0], src):
                ext[ix] = d
            shp = tuple(ext[ix] for ix in out)
            live[p] = shp
            continue
        sa, sb = live.pop(l), live.pop(r)
        if tdot:
            axes = (tuple(arg[0]), tuple(arg[1]))
            check_tensordot_shapes(axes, sa, sb)
            ta, tb, to = tensordot_terms(axes, len(sa), len(sb), perm)
        else:
            terms, to = split_equation(arg)
            ta, tb = terms
        shp = classify_pair(ta, sa, tb, sb, to).out_shape
        live[p] = shp
    return shp


def make_contractor(tree, strip_exponent=False, check_zero=False, vjp_max_bytes=None, precision="3xtf32",
                    stripped_grad=False, accumulate="native", **_ignored):
    """``cotengra.contract.make_contractor`` for ``implementation="b200"``
    (contract.py:925-1006): the per-slice callable for ``tree``."""
    return B200Contractor.from_tree(tree, strip_exponent=strip_exponent, check_zero=check_zero,
                                    vjp_max_bytes=vjp_max_bytes, precision=precision, stripped_grad=stripped_grad,
                                    accumulate=accumulate)


def install(tree, strip_exponent=False, check_zero=False, vjp_max_bytes=None, precision="3xtf32",
            stripped_grad=False, accumulate="native"):
    """Route ``tree.contract(...)`` / ``tree.contract_slice(...)`` of a live
    cotengra tree through this package's contractor by seeding its contractor cache
    (core.py:3699-3711).  Key order: ``(autojit, order, prefer_einsum,
    strip_exponent, check_zero, implementation, progbar)``.  Call after the tree
    is final: slicing/reconfiguration clears the cache (core.py:2040, 2087).  ``vjp_max_bytes``
    bounds the workspace of the backward pass of ``tree.contract`` on torch tensors; ``precision``
    is the compute mode of its float32 / complex64 tensor-core nodes (``TreeExecutor``).
    ``stripped_grad`` with ``strip_exponent``: each slice's ``(m_s, e_s)`` records the gradient of
    ``m_s`` with ``e_s`` held constant, so that the reference's slice combiner backpropagates.
    ``accumulate="double"``: every slice of a float32 / complex64 tree comes back as float64 /
    complex128 (a dot-type root summed in double), so that the reference's slice sum runs in double."""
    fn = make_contractor(tree, strip_exponent=strip_exponent, check_zero=check_zero,
                         vjp_max_bytes=vjp_max_bytes, precision=precision, stripped_grad=stripped_grad,
                         accumulate=accumulate)
    key = (False, None, False, bool(strip_exponent), check_zero, None, False)
    tree.contraction_cores[key] = fn
    return fn


# ---------------------------------------------------------------------------
# multi-GPU: slices round-robin over ranks, one reduce at the end
# ---------------------------------------------------------------------------


def contract_distributed(tree, arrays, root=None, group=None, strip_exponent=False,
                         dtype=None, executor=None, precision="3xtf32", accumulate="native", **plan_opts):
    """``tree.contract_mpi(arrays, comm, root)`` (cotengra/core.py:4032-4090)
    over ``torch.distributed`` (NCCL on NVLink): rank ``r`` of ``W`` contracts
    slices ``r, r+W, ...`` (core.py:4070), sums them locally on its GPU, then a
    single all-reduce (``root=None``) or reduce (``root=int``) combines the
    partial results.  Refuses fewer slices than ranks as the reference does
    (core.py:4062-4066).  Sliced *output* indices, which ``contract_mpi`` refuses
    (core.py:4051-4055), are sharded too (SURVEY 8f-4): every rank scatters its
    slices into the chunks of a zeroed full-size output (the executor's root
    strides, core.py:3865-3876), so the same single all-reduce assembles the
    stacked result; only the combination with ``strip_exponent`` stays refused.  With
    ``accumulate="double"`` the ranks' float64 / complex128 partials are what is reduced."""
    import torch.distributed as dist

    torch = _torch()
    spec = executor.spec if executor is not None else (
        tree if isinstance(tree, TreeSpec) else TreeSpec.from_cotengra(tree))
    strip = executor.strip_exponent if executor is not None else strip_exponent
    if strip and not {s[0] for s in spec.sliced}.isdisjoint(spec.output):
        raise NotImplementedError(
            "Sliced and output indices overlap - with stripped exponents only a simple "
            "sum of result slices is supported currently."
        )
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    rank_slices(rank, world, spec.nslices)  # raises like core.py:4062-4066
    if executor is None:
        executor = _executor_for(spec, arrays, dtype, strip_exponent=strip_exponent, precision=precision,
                                 accumulate=accumulate, **plan_opts)
    all_numpy = all(not isinstance(a, torch.Tensor) for a in arrays)
    tensors = [_to_device(a, executor.device)[0] for a in arrays]
    begin, step, count = rank_slices(rank, world, spec.nslices)
    res = executor.contract_device(tensors, begin=begin, step=step, count=count)
    if executor.strip_exponent:
        m, e = reduce_partials(res[0], res[1], root=root, group=group)
        if m is None:
            return None
        return _from_device(m, all_numpy), float(e.item())
    res = reduce_partials(res, None, root=root, group=group)
    if res is None:
        return None
    return _from_device(res, all_numpy)


def rank_slices(rank, world, nslices):
    """Round-robin share of rank ``rank``: slices ``rank, rank+world, ...``
    (core.py:4070) as ``(begin, step, count)``."""
    if nslices < world:
        raise ValueError(
            f"Need to have more slices than MPI processes, but have "
            f"{nslices} and {world} respectively."
        )
    return rank, world, max(0, -(-(nslices - rank) // world))


def reduce_partials(partial, exponent=None, root=None, group=None):
    """Sum the per-rank partial results with ONE collective (core.py:4078-4090):
    all-reduce when ``root is None`` else reduce to ``root`` (other ranks get
    ``None``).  With stripped exponents the pairs are first brought to the
    global maximum exponent (core.py:163-170).  Works on any torch.distributed
    backend (NCCL over NVLink on the GPUs; gloo in the CPU tests)."""
    import torch
    import torch.distributed as dist

    rank = dist.get_rank(group)
    emax = None
    if exponent is not None:
        emax = exponent.clone()
        dist.all_reduce(emax, op=dist.ReduceOp.MAX, group=group)
        scale = torch.where(torch.isneginf(emax), torch.zeros_like(emax),
                            torch.pow(10.0, exponent - emax))
        rdt = partial.real.dtype if partial.is_complex() else partial.dtype
        partial = partial * scale.to(rdt)
    buf = torch.view_as_real(partial) if partial.is_complex() else partial
    if root is None:
        dist.all_reduce(buf, op=dist.ReduceOp.SUM, group=group)
    else:
        dist.reduce(buf, dst=root, op=dist.ReduceOp.SUM, group=group)
        if rank != root:
            return None if exponent is None else (None, None)
    return partial if exponent is None else (partial, emax)
