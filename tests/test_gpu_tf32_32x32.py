"""The ``TF32_32x32`` kernel variant (one 32 x 32 3xTF32 mma.sync tile, the contracted range split
over two CTAs per SM, partial sums added atomically) driven directly through
``ctgb_contract_pair``: ``C[m, n] = sum_k A[k, m] B[k, n]`` -- the small-result backward node of a
stem absorption -- against float64, and the dependency cone of a NaN or inf."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import torch  # noqa: E402

from cotengra_b200 import _lib  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402

TDT = {"float32": torch.float32, "complex64": torch.complex64}
HI = {"float32": torch.float64, "complex64": torch.complex128}


def _operands(K, M, N, dtype, seed):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed)

    def one(shape):
        t = torch.empty(shape, dtype=TDT[dtype], device="cuda")
        (torch.view_as_real(t) if t.is_complex() else t).uniform_(-1.0, 1.0, generator=g)
        return t

    return one((K, M)), one((K, N))


def _contract(A, B, dtype):
    K, M = A.shape
    N = B.shape[1]
    dims = L.classify_pair(("k", "m"), (K, M), ("k", "n"), (K, N), ("m", "n"))
    plan = L.build_pair_desc(dims, dtype, variant=L.VAR_TF32_32x32, c_dense_elems=M * N,
                             sm_count=_lib.device_info()["sm_count"])
    assert plan.variant == L.VAR_TF32_32x32 and plan.splitk > 1
    C = torch.full((M, N), float("nan"), dtype=TDT[dtype], device="cuda")
    pa, pb = (B, A) if plan.swapped else (A, B)
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa.data_ptr(), pb.data_ptr(), C.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return C


def _reference(A, B, dtype):
    """float64 / complex128 A^T B, accumulated in chunks of the contracted range"""
    K = A.shape[0]
    C = torch.zeros((A.shape[1], B.shape[1]), dtype=HI[dtype], device="cuda")
    step = 1 << 22
    for k in range(0, K, step):
        C += A[k:k + step].to(HI[dtype]).T @ B[k:k + step].to(HI[dtype])
    return C


def _rel(x, ref):
    return float((x.to(ref.dtype) - ref).abs().max() / ref.abs().max())


MN = [5, 8, 16, 32]
CASES = [(dt, K, M, N) for dt in ("float32", "complex64") for K in (1 << 14, 1 << 20) for M in MN for N in MN]
CASES += [("float32", (1 << 25) + 3, 5, 5), ("float32", (1 << 25) + 3, 8, 32), ("float32", (1 << 25) + 3, 32, 32),
          ("complex64", (1 << 25) + 3, 32, 16)]


@pytest.mark.parametrize("dtype,K,M,N", CASES)
def test_against_float64(dtype, K, M, N):
    A, B = _operands(K, M, N, dtype, seed=K % 1000 + 10 * M + N)
    got = _contract(A, B, dtype)
    ref = _reference(A, B, dtype)
    err = _rel(got, ref)
    assert torch.isfinite(torch.view_as_real(got) if got.is_complex() else got).all()
    # the 3xTF32 mma.sync tiles' bound (BASELINE.json: 1e-5 for single precision)
    assert err < 1e-5, err
    del A, B
    torch.cuda.empty_cache()


@pytest.mark.parametrize("dtype", ["float32", "complex64"])
@pytest.mark.parametrize("where", ["A", "B"])
@pytest.mark.parametrize("value", ["nan", "inf"])
def test_special_value_stays_in_its_cone(dtype, where, value):
    K, M, N = (1 << 20) + 5, 24, 13
    A, B = _operands(K, M, N, dtype, seed=3)
    clean = _contract(A, B, dtype)
    k0, m0, n0 = K - 3, 7, 11
    v = float(value)
    if where == "A":
        A[k0, m0] = v
    else:
        B[k0, n0] = v
    got = _contract(A, B, dtype)
    bad = (~torch.isfinite(torch.view_as_real(got))).any(-1) if got.is_complex() else ~torch.isfinite(got)
    cone = torch.zeros((M, N), dtype=torch.bool, device="cuda")
    if where == "A":
        cone[m0, :] = True
    else:
        cone[:, n0] = True
    assert bool(bad[cone].all())
    assert not bool(bad[~cone].any())
    if value == "nan":
        nan = torch.isnan(torch.view_as_real(got)).any(-1) if got.is_complex() else torch.isnan(got)
        assert bool(nan[cone].all())
    # outside the cone: the clean values (split-K partial sums arrive in any order: dtype tolerance)
    assert _rel(got[~cone], clean[~cone].to(HI[dtype])) < 1e-5
