"""The DMMA stream kernel (csrc/dmmastream.cuh) on the nodes it takes beyond N = 16: 16-row warp blocks
with eight column fragments for 32 < N <= 64 (K <= 32; run when asked for by name, choose_variant keeps
these on DMMA_128x64), 32-row blocks with four for 16 < N <= 32 up to K = 64.

Each case runs once through ``ctgb_contract_pair`` in the sentinel-guarded buffers of
tests/kernel_cases.py (NaN guard bands and stride gaps, an all-NaN C unless accumulating), and every
element must lie within 1e-14 (|A| |B|)_ij (+ |C0|_ij) of a complex128 einsum.  Each asserts that the plan
is the stream kernel's and which instantiation its launcher takes.  The stripped-exponent instantiations
run inside a small tree."""

import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from tests import kernel_cases as KC  # noqa: E402
from tests.helpers import make_arrays, rel_err  # noqa: E402

C128 = "complex128"


def _cases():
    out = []

    def add(family, eq, shapes, nj, rows, **kw):
        out.append((KC._case(L.VAR_DMMASTREAM, C128, family, dict(eq=eq, shapes=shapes, **kw)), nj, rows))

    ta, sa = KC._rows3(200, 32)  # 600 rows: the last 16-row block is 8 rows, a non-power-of-two m extent
    add("n33_k32_row_tail", f"{ta},kc->xac", (sa, (32, 33)), 8, 16, expect={"pair": False, "n_tile": 33,
                                                                             "m_pow2": False})
    add("n48_k32_pair", "ak,kc->ac", ((1024, 32), (32, 48)), 8, 16, expect={"pair": True, "n_tile": 48,
                                                                            "m_pow2": True})
    ta, sa = KC._rows3(200, 24)
    add("n48_k24_permuted", f"{ta},kc->cxa", (sa, (24, 48)), 8, 16, expect={"pair": False, "n_tile": 48})
    ta, sa = KC._rows3(200, 32)
    add("n64_k32_pair", f"{ta},kc->xac", (sa, (32, 64)), 8, 16, expect={"pair": True, "n_tile": 64, "k_tile": 32})
    ta, sa = KC._rows3(200, 13)
    add("n64_k13_accumulate", f"{ta},kc->xac", (sa, (13, 64)), 8, 16, accumulate=True,
        expect={"accumulate": True, "n_tile": 64})
    # N = 17 .. 32 at K = 64: four column fragments, 32-row blocks
    for n in (17, 24, 31, 32):
        ta, sa = KC._rows3(200, 64)  # 600 rows: the last 32-row block is 24 rows
        add(f"n{n}_k64_row_tail", f"{ta},kc->xac", (sa, (64, n)), 4, 32, expect={"n_tile": n, "k_tile": 64,
                                                                                 "pair": n % 2 == 0})
    add("n32_k64_pair", "ak,kc->ac", ((2048, 64), (64, 32)), 4, 32, expect={"pair": True, "m_pow2": True})
    ta, sa = KC._rows3(200, 64)
    add("n24_k64_permuted", f"{ta},kc->cxa", (sa, (64, 24)), 4, 32, expect={"pair": False})
    ta, sa = KC._rows3(200, 40)
    add("n20_k40_accumulate", f"{ta},kc->xac", (sa, (40, 20)), 4, 32, accumulate=True,
        expect={"accumulate": True, "k_tile": 40})
    # non-power-of-two extents in every class: 504 rows in two dims that do not coalesce, one of them
    # blocked into two exact tiles of 7 x 36 rows, decoded by idiv
    add("n36_k30_idiv", "bkc,kef->bcef", ((14, 30, 36), (30, 6, 6)), 8, 16,
        expect={"m_pow2": False, "n_tile": 36, "pgm": True})
    return out


CASES = {c.id: (c, nj, rows) for c, nj, rows in _cases()}


@pytest.mark.parametrize("cid", list(CASES))
def test_wide_stream_case(cid):
    import torch

    from cotengra_b200 import _lib

    case, nj, rows = CASES[cid]
    plan = KC.build_plan(case)
    assert plan.variant == L.VAR_DMMASTREAM
    assert not KC.plan_mismatches(case, plan), KC.plan_mismatches(case, plan)
    info = _lib.device_info()
    launch = _lib.dmmastream_launch_config(plan.words, info["sm_count"])
    assert (launch["nj"], launch["rows"]) == (nj, rows), launch
    lay = KC.make_layout(case, seed=zlib.crc32(cid.encode()))
    dev = [torch.from_numpy(b).cuda() for b in lay.bufs]
    es = np.dtype(case.dtype).itemsize
    ptr = [d.data_ptr() + off * es for d, off in zip(dev, lay.offs)]
    assert ptr[2] % KC.C_ALIGN == 0
    pa, pb = (ptr[1], ptr[0]) if plan.swapped else (ptr[0], ptr[1])
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa, pb, ptr[2], 0))
    torch.cuda.synchronize()
    for d, b in zip(dev[:2], lay.bufs[:2]):
        assert d.cpu().numpy().tobytes() == b.tobytes()  # operands untouched
    got, bad = KC.check_result(case, lay, dev[2].cpu().numpy())
    assert bad.size == 0, f"{bad.size} sentinel components outside C changed, first at {bad[:8]}"
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} described C elements NaN"
    ref, scale = KC.reference(case, lay)
    ratio = KC.error_ratio(got, ref, scale)
    assert ratio <= KC.C_DOUBLE, ratio
    assert rel_err(got, ref) < 1e-12


@pytest.mark.parametrize("M", [1 << 14, 12288])
def test_wide_stream_strip(M):
    """Stripped exponents: m,k x k,n (N = 32, max|C| measured) -> x n,p (N = 64: operand scale applied,
    max|C| measured) -> x p,z (N = 4, K = 64), every node on the stream kernel (asked for by name)."""
    sizes = {"m": M, "k": 16, "n": 32, "p": 64, "z": 4}
    inputs = [("m", "k"), ("k", "n"), ("n", "p"), ("p", "z")]
    arrays = make_arrays([tuple(sizes[i] for i in t) for t in inputs], C128, seed=M % 101)
    arrays[1] = arrays[1] * 1e40  # magnitudes far from 1: the mantissa and the exponent must recombine
    arrays[2] = arrays[2] * 1e-90
    spec = cb.TreeSpec(inputs, ("m", "z"), sizes, [(0, 1), (4, 2), (5, 3)])
    ex = cb.TreeExecutor(spec, dtype=C128, strip_exponent=True, fuse=False, variant=L.VAR_DMMASTREAM)
    from cotengra_b200 import _lib

    sms = _lib.device_info()["sm_count"]
    pairs = [nd for nd in ex.plan.nodes if nd["kind"] == 0]
    assert len(pairs) == 3 and all(int(nd["plan"].variant) == L.VAR_DMMASTREAM for nd in pairs)
    nj = sorted(_lib.dmmastream_launch_config(nd["plan"].words, sms)["nj"] for nd in pairs)
    assert nj == [1, 4, 8]
    m, e = cb.contract_tree(ex, arrays, strip_exponent=True)
    want = ((arrays[0] @ arrays[1]) @ arrays[2]) @ arrays[3]
    got = np.asarray(m) * 10.0 ** float(e)
    assert rel_err(got, want) < 1e-12
