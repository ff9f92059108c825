"""The kernel-path case table (tests/kernel_cases.py) without a GPU.

* every case builds, and its plan takes the path the case exists for (its declared predicates);
* the table covers every (variant, dtype) the dispatcher runs with every family and store mode
  listed here, each cell exactly once -- removing a case, or a lowering change that moves a case
  off its path, fails here;
* every case runs through the descriptor emulator on the same sentinel-guarded buffers as the
  GPU test and must meet the same bounds, with every sentinel intact: a GPU failure then points
  at the kernel, not at the harness or the expected values.
"""

import collections

import numpy as np
import pytest

from cotengra_b200 import lowering as L
from tests import kernel_cases as KC
from tests.desc_emulator import emulate_pair
from tests.helpers import rel_err

CASES = {c.id: c for c in KC.CASES}

_STAGED_FAMILIES = ("ragged", "exact_pow2", "structured", "structured_swapped", "gapped", "accumulate",
                    "splitk2", "splitk3", "splitk_acc", "long_k", "vjp_broadcast", "vjp_diag")
_STAGED_STORES = ("plain", "accumulate", "atomic")


def _required():
    """(cells, store modes): every (variant, dtype, family) the table must hold exactly once, and
    the store modes each (variant, dtype) must reach."""
    all4 = ("float32", "float64", "complex64", "complex128")
    staged = {v: all4 for v in (L.VAR_SIMT_64x64, L.VAR_KRED, L.VAR_DMMA_128x64, L.VAR_DMMA_64x128,
                                L.VAR_DMMA_256x32, L.VAR_DMMA_256x16, L.VAR_ROW_128x8, L.VAR_ROW_256x4)}
    staged.update({L.VAR_DMMA3M_128x32: ("complex128",), L.VAR_DMMA3M_256x16: ("complex128",),
                   L.VAR_DMMA_32x32: ("float64", "complex128"), L.VAR_TF32_32x32: ("float32", "complex64")})
    cells, stores = [], {}
    for v, dtypes in staged.items():
        for d in dtypes:
            fams = list(_STAGED_FAMILIES)
            st = set(_STAGED_STORES)
            if d == "complex128" and v != L.VAR_KRED:
                fams += ["pair_full", "pair_ragged"]
                st |= {"pair_full", "pair_ragged"}
            if v in (L.VAR_ROW_128x8, L.VAR_ROW_256x4):
                fams.append("rows_bcache")
            cells += [(v, d, f) for f in fams]
            stores[(v, d)] = st
    for v, d in [(L.VAR_TF32_32x32, "float64"), (L.VAR_TF32_32x32, "complex128")] + [
            (v3, d) for v3 in (L.VAR_DMMA3M_128x32, L.VAR_DMMA3M_256x16) for d in ("float32", "float64", "complex64")]:
        cells.append((v, d, "remap"))
    rs = ("rs4x4_nonpow2_m", "rs2x8_pow2_m", "rs8x8_quad", "rs8x8_pair8", "rs8x8_accumulate", "rs4x4_gapped")
    for d in all4:
        cells += [(L.VAR_ROWSTREAM, d, f) for f in rs]
        stores[(L.VAR_ROWSTREAM, d)] = {"plain", "accumulate"} | (
            {"quad8", "pair8"} if d in ("float64", "complex64") else {"pair"} if d == "complex128" else set())
        cells += [(L.VAR_DOTSTREAM, d, f) for f in ("dot_blocked_k", "dot_permuted", "dot_accumulate")]
        cells += [(L.VAR_DOTSTREAM4, d, f) for f in ("dot4_permuted_c", "dot4_accumulate")]
        stores[(L.VAR_DOTSTREAM, d)] = stores[(L.VAR_DOTSTREAM4, d)] = {"atomic", "accumulate"}
        cells.append((L.VAR_KRED, d, "kred_small_permuted_c"))
    for d in ("float32", "float64", "complex64"):
        cells += [(L.VAR_ROWSTREAM_K, d, f) for f in ("rsk_k9", "rsk_k64_pow2_m", "rsk_k37_accumulate")]
        stores[(L.VAR_ROWSTREAM_K, d)] = {"plain", "accumulate"} | ({"quad8"} if d != "float32" else set())
    cells += [(L.VAR_DMMASTREAM, "complex128", f) for f in
              ("ds_n9_k32", "ds_n24_k20_pair", "ds_n32_k7_permuted", "ds_n8_k64_pair", "ds_n5_k33_accumulate")]
    stores[(L.VAR_DMMASTREAM, "complex128")] = {"plain", "pair", "accumulate"}
    for v, d in ((L.VAR_DMMA_32x32, "float64"), (L.VAR_DMMA_32x32, "complex128"), (L.VAR_TF32_32x32, "float32"),
                 (L.VAR_TF32_32x32, "complex64")):
        cells.append((v, d, "one_tile_splitk"))
    cells += [(L.VAR_TC05_128x64, "complex64", "tc05_gapped_accumulate"),
              (L.VAR_TC05_128x32, "complex64", "tc05_dense_non_pow2"),
              (L.VAR_TC05_128x16, "complex64", "tc05_splitk_dense")]
    return cells, stores


def test_case_table_coverage():
    cells, stores = _required()
    have = collections.Counter(c.cell for c in KC.CASES)
    dups = sorted(cell for cell, n in have.items() if n > 1)
    assert not dups, f"cells covered more than once: {dups}"
    need = collections.Counter(cells)
    assert not [c for c, n in need.items() if n > 1]
    missing = sorted(set(need) - set(have))
    extra = sorted(set(have) - set(need))
    assert not missing, f"cells without a case: {[(KC.VARIANT_NAMES[v], d, f) for v, d, f in missing]}"
    assert not extra, f"cases outside the coverage list: {[(KC.VARIANT_NAMES[v], d, f) for v, d, f in extra]}"
    # every store mode of every (variant, dtype), as the plans select them
    seen = collections.defaultdict(set)
    for c in KC.CASES:
        seen[(c.variant, c.dtype)].add(KC.store_mode(c, KC.build_plan(c)))
    for key, modes in stores.items():
        lost = modes - seen[key]
        assert not lost, (KC.VARIANT_NAMES[key[0]], key[1], sorted(lost))


@pytest.mark.parametrize("cid", list(CASES))
def test_plan_takes_its_path(cid):
    case = CASES[cid]
    plan = KC.build_plan(case)
    assert not KC.plan_mismatches(case, plan), KC.plan_mismatches(case, plan)
    # the predicates every case pins: no case may quietly run another kernel or split
    keys = dict(case.expect)
    assert "variant" in keys and "splitk" in keys and "swapped" in keys


def _emulate(case, lay, plan):
    a, b = (buf[off:] for buf, off in zip(lay.bufs[:2], lay.offs[:2]))
    cbuf = lay.bufs[2].copy()
    c = cbuf[lay.offs[2]:]
    if plan.swapped:
        a, b = b, a
    emulate_pair(plan.words, a, b, c)
    return cbuf


@pytest.mark.parametrize("cid", list(CASES))
def test_emulated_case_meets_bounds(cid):
    """The harness on the CPU: expected values, per-element bounds and sentinel bookkeeping."""
    case = CASES[cid]
    plan = KC.build_plan(case)
    lay = KC.make_layout(case, seed=7)
    snapshot = [b.copy() for b in lay.bufs]
    with np.errstate(invalid="ignore", over="ignore"):
        cbuf = _emulate(case, lay, plan)
    for before, after in zip(snapshot[:2], lay.bufs[:2]):
        assert before.tobytes() == after.tobytes()  # operands untouched
    got, bad = KC.check_result(case, lay, cbuf)
    assert bad.size == 0, f"{bad.size} sentinel components changed, first at {bad[:8]}"
    assert not np.isnan(got).any(), "a described C element was never written"
    ref, scale = KC.reference(case, lay)
    single = KC.is_single(case.dtype)
    assert KC.error_ratio(got, ref, scale) <= (KC.C_SINGLE if single else KC.C_DOUBLE)
    assert rel_err(got, ref) < (1e-5 if single else 1e-12)
