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
import math

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
_TC05_FAMILIES = ("k4_m64", "pow2_resident", "idiv_ring", "resident_at_fit", "ring_past_fit", "accumulate", "two_chunks_fold", "chunks_accumulate",
                  "nq3_chunks", "nq2", "splitk3_uneven", "splitk3_chunked", "splitk_acc_gapped", "ragged_tile",
                  "gather_odd", "misaligned_a", "bulk_runs", "tmap4", "tmap5", "swapped", "batched",
                  "permuted_gapped", "many_items_resident", "many_items_ring", "same_sign_k256", "same_sign_k4096")
TC05_CASES = {cid: c for cid, c in CASES.items() if c.variant in L.TC05_VARIANTS}


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
    for v in L.TC05_VARIANTS:
        cells += [(v, "complex64", f) for f in _TC05_FAMILIES]
        stores[(v, "complex64")] = set(_STAGED_STORES)
    cells += [(L.VAR_TC05_128x64, "complex64", "same_sign_108x54x12"),
              (L.VAR_TC05_128x64, "complex64", "tc05_gapped_accumulate"),
              (L.VAR_TC05_128x32, "complex64", "tc05_dense_non_pow2"),
              (L.VAR_TC05_128x16, "complex64", "tc05_splitk_dense")]
    for name, eq, shapes, kw, (v, _splitk) in KC.TC05_LEGACY:
        cells += [(v, "complex64", f"legacy_{name}"), (v, "complex64", f"legacy_{name}_a_plus_8_bytes")]
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


_BASE = 1 << 30  # a 256-byte aligned device allocation holding the operand buffers


@pytest.mark.parametrize("cid", list(TC05_CASES))
def test_tc05_launch_facts(cid):
    """The wgmma launch takes the choices its case declares on an H100 SXM (132 SMs) and PCIe (114),
    and a resident B' always comes with a grid that is a multiple of tiles_n (every work item of a CTA
    then has the same B' tiles) -- so a launcher branch that dropped B' residency for grids that are not
    such a multiple could never run."""
    case = TC05_CASES[cid]
    plan = KC.build_plan(case)
    tiles_n = int(plan.words[L.W_TILES_N])
    for sms in KC.H100_SMS:
        f = KC.launch_facts(case, plan, KC.a_operand_addr(case, plan, _BASE), sms, KC.H100_SMEM_OPTIN)
        assert not KC.launch_mismatches(case, f), (sms, KC.launch_mismatches(case, f))
        assert 1 <= f["grid"] <= min(sms, f["work"])
        assert not f["b_stat"] or f["grid"] % tiles_n == 0, (sms, f)
        assert f["sa"] >= 2 and f["smem"] + 1024 <= KC.H100_SMEM_OPTIN
        assert (f["chunks"] - 1) * f["chunk_steps"] < -(-int(plan.words[L.W_STEPS_K]) // plan.splitk)


def _tc05_cells(case, plan, f):
    """The coverage cells of the wgmma table one case (at 132 SMs) hits."""
    p = KC.plan_facts(plan)
    steps, splitk, nq = p["steps_k"], p["splitk"], p["nq"]
    tiles_m, tiles_n, tiles_b = p["tiles"]
    fit = KC.TC05_RESIDENT_STEPS[L.VARIANT_TILES[p["variant"]][1]]
    c = set()
    # A staging
    if f["tm_rank"]:
        c.add(f"tmap_rank{f['tm_rank']}")
    elif f["bulk"]:
        c.add("bulk_runs")
    elif p["bulk_flag"]:
        c.add("gather_misaligned")
    else:
        c.add("gather_odd_strides")
    # B'
    if f["b_stat"]:
        c.add("resident_1_step" if steps == 1 else "resident_steps")
    elif tiles_b > 1:
        c.add("ring_batch")
    elif splitk > 1:
        c.add("ring_splitk")
    elif steps > fit:
        c.add("ring_long_k")
    if f["b_stat"] and steps == fit:
        c.add("resident_at_fit")
    if not f["b_stat"] and steps == fit + 1 and tiles_b == 1 and splitk == 1:
        c.add("ring_at_fit_plus_1")
    # k
    c.add(f"nq{nq}")
    if nq == 1 and steps == 1:
        c.add("nq1_one_step")
    if f["chunks"] == 1:
        c.add("one_chunk")
    elif f["chunks"] == 2 and steps == 17 and f["chunk_steps"] == 9:
        c.add("two_balanced_chunks")
    elif f["chunks"] >= 3:
        c.add("three_or_more_chunks")
    if nq == 3 and steps == 25 and f["chunk_steps"] == 9 and f["chunks"] == 3:
        c.add("nq3_chunks_9_8_8")
    # epilogue
    if splitk > 1:
        c.add("splitk_accumulate_gapped" if p["accumulate"] and case.out_strides else "splitk_atomic")
        if steps == 7 and splitk == 3:
            c.add("splitk_uneven_7_3")
        if f["chunks"] > 1:
            c.add("splitk_chunked")
    elif p["accumulate"]:
        c.add("accumulate_chunks" if f["chunks"] > 1 else "accumulate")
    else:
        c.add("fold_into_nan" if f["chunks"] > 1 else "plain")
    # tiles
    if p["full_tiles"] and p["grid_pow2"]:
        c.add("full_pow2_shift_decode")
    if tiles_m == 3 and not p["grid_pow2"]:
        c.add("idiv_3_m_tiles")
    if p["m_tile"] <= 64:
        c.add("m_tile_le_64")
    elif p["m_tile"] < 128:
        c.add("m_tile_64_128")
    if p["n_tile"] < L.VARIANT_TILES[p["variant"]][1] and p["n_tile"] % 4:
        c.add("n_tile_straddles_quads")
    c.add("lbopad_0" if p["lbopad"] == 0 else "lbopad_nonzero")
    # layout
    if p["swapped"]:
        c.add("swapped")
    if p["batch"]:
        c.add("batch_grid")
    if case.out_strides is not None and case.terms()[2] != "".join(sorted(case.terms()[2])):
        c.add("permuted_gapped_c")
    if case.strides[1] is not None:
        c.add("strided_gapped_b")
    # work
    if f["one_item"] and f["grid"] < 132:
        c.add("one_item_per_cta")
    if f["uneven"] and f["work"] > 2 * f["grid"]:
        c.add("many_uneven_items_resident" if f["b_stat"] else "many_uneven_items_ring")
    # numerics
    if case.dist == "same_sign":
        if steps == 16 and nq == 4 and f["chunks"] == 1:
            c.add("same_sign_k256")
        if steps == 256 and f["chunks"] == 16:
            c.add("same_sign_k4096")
        if (p["m_tile"], p["n_tile"], p["k_tile"]) == (108, 54, 12):
            c.add("same_sign_108x54x12")
    return c


# every cell of the wgmma kernel's code paths and launch choices the table must reach
_TC05_CELLS = {
    "tmap_rank2", "tmap_rank3", "tmap_rank4", "tmap_rank5", "bulk_runs", "gather_odd_strides", "gather_misaligned",
    "resident_1_step", "resident_steps", "ring_batch", "ring_splitk", "ring_long_k", "resident_at_fit",
    "ring_at_fit_plus_1",
    "nq1", "nq2", "nq3", "nq4", "nq1_one_step", "one_chunk", "two_balanced_chunks", "three_or_more_chunks",
    "nq3_chunks_9_8_8",
    "plain", "fold_into_nan", "accumulate", "accumulate_chunks", "splitk_atomic", "splitk_uneven_7_3",
    "splitk_chunked", "splitk_accumulate_gapped",
    "full_pow2_shift_decode", "idiv_3_m_tiles", "m_tile_le_64", "m_tile_64_128", "n_tile_straddles_quads",
    "lbopad_0", "lbopad_nonzero",
    "swapped", "batch_grid", "permuted_gapped_c", "strided_gapped_b",
    "one_item_per_cta", "many_uneven_items_resident", "many_uneven_items_ring",
    "same_sign_k256", "same_sign_k4096", "same_sign_108x54x12",
}


def test_tc05_table_reaches_every_cell():
    hit = collections.defaultdict(set)
    for cid, case in TC05_CASES.items():
        plan = KC.build_plan(case)
        f = KC.launch_facts(case, plan, KC.a_operand_addr(case, plan, _BASE), 132, KC.H100_SMEM_OPTIN)
        for cell in _tc05_cells(case, plan, f):
            hit[cell].add(case.variant)
    assert not _TC05_CELLS - set(hit), sorted(_TC05_CELLS - set(hit))
    # the cells every N tile reaches on its own
    for cell in ("tmap_rank2", "tmap_rank3", "tmap_rank4", "tmap_rank5", "bulk_runs", "gather_odd_strides",
                 "gather_misaligned", "resident_1_step", "resident_steps", "ring_batch", "ring_splitk",
                 "ring_long_k", "resident_at_fit", "ring_at_fit_plus_1", "nq1", "nq2", "nq3", "nq4", "two_balanced_chunks", "nq3_chunks_9_8_8",
                 "fold_into_nan", "accumulate_chunks", "splitk_uneven_7_3", "splitk_chunked",
                 "splitk_accumulate_gapped", "m_tile_le_64", "m_tile_64_128", "n_tile_straddles_quads",
                 "many_uneven_items_resident", "many_uneven_items_ring", "same_sign_k256", "same_sign_k4096"):
        assert hit[cell] == set(L.TC05_VARIANTS), (cell, sorted(KC.VARIANT_NAMES[v] for v in hit[cell]))


def test_legacy_tc05_shapes_are_rows():
    """Every shape the earlier wgmma mode test ran (with A aligned and 8 bytes off) is a row of the
    table, with the variant, split and accumulation the automatic plan for 132 SMs gives it."""
    assert len(KC.TC05_LEGACY) == 12
    rows = {(c.eq, c.shapes, c.offsets, c.accumulate, c.force_splitk): c for c in TC05_CASES.values()}
    for name, eq, shapes, kw, runs in KC.TC05_LEGACY:
        (ta, tb), to = L.split_equation(eq)
        dims = L.classify_pair(ta, shapes[0], tb, shapes[1], to)
        want = L.build_pair_desc(dims, "complex64", sm_count=132, c_dense_elems=math.prod(dims.out_shape), **kw)
        assert (want.variant, want.splitk) == runs, (name, want.variant, want.splitk)
        for off in (0, 1):
            case = rows[(eq, tuple(shapes), (off, 0), bool(kw.get("accumulate")), kw.get("force_splitk"))]
            assert case.family == f"legacy_{name}" + ("_a_plus_8_bytes" if off else "")
            plan = KC.build_plan(case)
            assert plan.variant == want.variant and plan.splitk == want.splitk and not plan.swapped
            assert (plan.words == want.words).all()


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
