"""The kernel cases of ``tests/kernel_cases.py`` that run on the float32 / complex64 tensor cores,
built with ``precision="tf32"``, and the numpy model of one tf32 pass they are checked against.

The model: every operand component rounded to nearest (ties away from zero) onto tf32's 10
mantissa bits, as ``round_tf32`` / ``tc05_hi`` (tc05_policy.cuh) and ``cvt.rna`` (tf32_policy.cuh)
do, then the products summed in float64.  What the kernel adds to that is its fp32 accumulation,
which ``kernel_cases.C_SINGLE`` bounds.  No GPU imports here."""

from __future__ import annotations

import math

import numpy as np

from cotengra_b200 import lowering as L
from tests import kernel_cases as KC


def round_tf32(x):
    """``x`` (float32 or complex64) with every component rounded to nearest onto the tf32 grid; a
    finite component that would round past FLT_MAX is truncated instead, inf and NaN stay."""
    x = np.asarray(x)
    comp = x.view(np.float32) if x.dtype == np.complex64 else x.astype(np.float32, copy=False)
    u = comp.view(np.uint32)
    a = u & np.uint32(0x7FFFFFFF)
    h = (u + np.uint32(0x1000)) & np.uint32(0xFFFFE000)
    near_max = (a >= 0x7F7FF000) & (a < 0x7F800000)
    h = np.where(near_max, u & np.uint32(0xFFFFE000), h)
    h = np.where(a >= 0x7F800000, u, h)  # inf, NaN
    out = h.astype(np.uint32).view(np.float32)
    return out.view(np.complex64).reshape(x.shape) if x.dtype == np.complex64 else out.reshape(x.shape)


def build_plan(case, precision):
    ta, tb, out = case.terms()
    dims = L.classify_pair(ta, case.shapes[0], tb, case.shapes[1], out, out_strides=case.out_strides,
                           strides_a=case.strides[0], strides_b=case.strides[1])
    dense = math.prod(case.out_shape()) if case.out_strides is None else 0
    return L.build_pair_desc(dims, case.dtype, accumulate=case.accumulate, sm_count=KC.SM_COUNT,
                             variant=case.variant, c_dense_elems=dense, force_splitk=case.force_splitk,
                             precision=precision)


def tf32_reference(case, lay):
    """(ref, scale) as ``kernel_cases.reference``, with the operands rounded onto tf32 first."""
    wd = KC.wide_dtype(case.dtype)
    a, b = (round_tf32(x).astype(wd) for x in lay.ops)
    ref = np.einsum(case.eq, a, b, optimize=True)
    scale = np.einsum(case.eq, np.abs(a), np.abs(b), optimize=True)
    if case.accumulate:
        ref = ref + lay.c0.astype(wd)
        scale = scale + np.abs(lay.c0.astype(wd))
    return np.asarray(ref), np.asarray(scale)


# every single-precision case whose plan runs on the tensor cores (wgmma and the mma.sync tiles)
CASES = [c for c in KC.CASES if KC.is_single(c.dtype) and KC.build_plan(c).variant in L.TF32_VARIANTS]
