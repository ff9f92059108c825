"""Table of pairwise-kernel cases: one case per (kernel variant, dtype, code path).

Each case is a contraction (equation, operand shapes, optional operand and output strides,
element offsets of the operands in their buffers, accumulate, forced split-K), the kernel
variant to force, and the predicates its plan must satisfy, read back from the descriptor
words.  ``tests/test_kernel_paths_cpu.py`` checks the predicates, the coverage of the table and
the harness itself (through the descriptor emulator); ``tests/test_gpu_kernel_paths.py`` runs
every case once on the device.  No GPU imports here.

Buffer layout shared by both tests (``make_layout``):
  * A and B sit at an element offset inside a larger buffer whose every other element (gaps of a
    strided view, guard bands before and after) holds ``SENTINEL`` -- a NaN, so a stray read of
    it poisons the result;
  * C sits 256 bytes (the alignment the executor's arenas give every C) into a buffer whose guard
    bands and stride gaps hold the same sentinel; a non-accumulating launch starts with every
    described element a (plain) NaN, an accumulating one with random C0.
"""

from __future__ import annotations

import math
from dataclasses import dataclass

import numpy as np

from cotengra_b200 import lowering as L

# descriptors are built for the 132 SMs of an H100 SXM; only the automatic split-K choice reads it
SM_COUNT = 132
F32, F64, C64, C128 = "float32", "float64", "complex64", "complex128"
ALL_DTYPES = (F32, F64, C64, C128)

VARIANT_NAMES = {v: k[4:] for k, v in vars(L).items() if k.startswith("VAR_") and isinstance(v, int)}

# staged (warp-specialised gett_kernel) variants and the dtypes the dispatcher runs them for
STAGED = {
    L.VAR_SIMT_64x64: ALL_DTYPES,
    L.VAR_KRED: ALL_DTYPES,
    L.VAR_DMMA_128x64: ALL_DTYPES,   # DmmaPolicy for the double types, Tf32Policy for the single ones
    L.VAR_DMMA_64x128: ALL_DTYPES,
    L.VAR_DMMA_256x32: ALL_DTYPES,
    L.VAR_DMMA_256x16: ALL_DTYPES,
    L.VAR_ROW_128x8: ALL_DTYPES,
    L.VAR_ROW_256x4: ALL_DTYPES,
    L.VAR_DMMA3M_128x32: (C128,),
    L.VAR_DMMA3M_256x16: (C128,),
    L.VAR_DMMA_32x32: (F64, C128),
    L.VAR_TF32_32x32: (F32, C64),
}
# documented dtype remaps of build_pair_desc: (forced variant, dtype) -> the variant that runs
REMAPS = {
    (L.VAR_TF32_32x32, F64): L.VAR_DMMA_32x32,
    (L.VAR_TF32_32x32, C128): L.VAR_DMMA_32x32,
    **{(L.VAR_DMMA3M_128x32, d): L.VAR_DMMA_256x32 for d in (F32, F64, C64)},
    **{(L.VAR_DMMA3M_256x16, d): L.VAR_DMMA_256x16 for d in (F32, F64, C64)},
}
ROW_VARIANTS = (L.VAR_ROW_128x8, L.VAR_ROW_256x4)

SENTINEL_BITS = {np.dtype(np.float64): 0x7FF4C0FFEE5EA1ED, np.dtype(np.float32): 0x7FA5C0DE}
C_ALIGN = 256  # bytes
# per-element bound |got - ref| <= c * (|A| |B|)_ij (+ c |C0|_ij): c for the double and single types.
# Largest ratios measured over the table on an H100 80GB HBM3 (400 W power limit): 6.0e-16 for the
# double types (DMMA_128x64 complex128, a margin above 15x); for the single types 3.6e-7 with uniform
# operands (TC05_128x64; SIMT_64x64 float32 2.6e-7), a margin above 10x, and 2.4e-6 in the wgmma kernel's
# same-sign cases, where its truncating accumulation cannot cancel (seeded inputs, no atomics: the same
# every run), a margin of 1.7x.  A dropped k4 step or swapped output rows measured 2e-2 and more; the
# wgmma kernel without its lo correction terms 1.4e-5 and more.
C_DOUBLE, C_SINGLE = 1e-14, 4e-6


def real_dtype(dtype):
    return np.empty(0, dtype=dtype).real.dtype


def is_single(dtype):
    return real_dtype(dtype).itemsize == 4


def wide_dtype(dtype):
    return np.complex128 if np.dtype(dtype).kind == "c" else np.float64


@dataclass(frozen=True)
class Case:
    variant: int            # the variant forced through build_pair_desc
    dtype: str
    family: str             # the code path this case exists for
    eq: str
    shapes: tuple
    strides: tuple = (None, None)   # element strides of A and B in their buffers (None: dense)
    out_strides: tuple = None       # element strides of C (None: dense, row-major)
    offsets: tuple = (0, 0)         # element offsets of A and B in their buffers
    accumulate: bool = False
    force_splitk: int = 1           # None: the automatic choice
    expect: tuple = ()              # ((predicate, value), ...) the plan (and wgmma launch) must satisfy
    dist: str = "uniform"           # operand values: "uniform" in [-1, 1], or "same_sign" (see _random)

    @property
    def id(self):
        return f"{VARIANT_NAMES[self.variant]}-{self.dtype}-{self.family}"

    @property
    def cell(self):
        return (self.variant, self.dtype, self.family)

    def terms(self):
        lhs, out = self.eq.split("->")
        ta, tb = lhs.split(",")
        return ta, tb, out

    def out_shape(self):
        ta, tb, out = self.terms()
        ext = dict(zip(ta + tb, tuple(self.shapes[0]) + tuple(self.shapes[1])))
        return tuple(ext[ix] for ix in out)


def build_plan(case):
    ta, tb, out = case.terms()
    dims = L.classify_pair(ta, case.shapes[0], tb, case.shapes[1], out, out_strides=case.out_strides,
                           strides_a=case.strides[0], strides_b=case.strides[1])
    dense = math.prod(case.out_shape()) if case.out_strides is None else 0
    return L.build_pair_desc(dims, case.dtype, accumulate=case.accumulate, sm_count=SM_COUNT, variant=case.variant,
                             c_dense_elems=dense, force_splitk=case.force_splitk)


# ---------------------------------------------------------------------------- plan predicates


def plan_facts(plan):
    """Everything a case may assert about its plan, from the descriptor words alone."""
    W = plan.words
    flags = int(W[L.W_FLAGS])
    variant = int(W[L.W_VARIANT])
    MT, NT, _KT = L.VARIANT_TILES[variant]
    steps_k = int(W[L.W_STEPS_K])
    ngm, ngn, ngk, ngb = (int(W[i]) for i in (L.W_NGM, L.W_NGN, L.W_NGK, L.W_NGB))
    ntm, ntn, ntk = (int(W[i]) for i in (L.W_NTM, L.W_NTN, L.W_NTK))
    MTa, NTa = int(W[L.W_MTA]), int(W[L.W_NTA])

    def last_valid(base, tile):
        # valid rows (columns) of the last tile of a class
        pg, full, text, w = (int(W[base + i]) for i in range(4))
        if pg < 0:
            return tile
        return (full - (-(-full // text) - 1) * text) * w

    def full_tiles(base, tile, pol):
        pg, full, text = (int(W[base + i]) for i in range(3))
        return tile == pol and (pg < 0 or full % text == 0)

    def rows(off, n, width):
        return [[int(x) for x in W[off + width * i: off + width * (i + 1)]] for i in range(n)]

    # operand strides of every dim: (ext, sA|sB, sC) m/n tile rows, (ext, sA, sB) k tile rows,
    # (ext, div, sA|sB, sC) m/n grid rows, (ext, div, sA, sB) k grid rows
    op_strides = [r[1] for r in rows(L.OFF_TM, ntm, 3) + rows(L.OFF_TN, ntn, 3)]
    op_strides += [s for r in rows(L.OFF_TK, ntk, 3) for s in r[1:]]
    op_strides += [g[2] for g in rows(L.OFF_GM, ngm, 4) + rows(L.OFF_GN, ngn, 4)]
    op_strides += [s for g in rows(L.OFF_GK, ngk, 4) for s in g[2:]]
    return {
        "variant": variant,
        "swapped": bool(plan.swapped),
        "accumulate": bool(flags & 1),
        "pair": bool(flags & 2),
        "grid_pow2": bool(flags & 4),
        "m_pow2": bool(flags & 8),
        "quad8": bool(flags & 16),
        "pair8": bool(flags & 32),
        "pgm": int(W[L.W_PGM]) >= 0,
        "pgn": int(W[L.W_PGN]) >= 0,
        "pgk": int(W[L.W_PGK]) >= 0,
        "splitk": int(W[L.W_SPLITK]),
        "long_k": steps_k > 128,
        "batch": ngb > 0,
        "b_invariant": steps_k == 1 and ngn == 0 and ngb == 0,
        "multi_m": ntm + ngm >= 2,
        "multi_n": ntn + ngn >= 2,
        "multi_k": ntk + ngk >= 2,
        "odd_tail": last_valid(L.W_PGM, MTa) % 2 == 1,
        "full_tiles": full_tiles(L.W_PGM, MTa, MT) and full_tiles(L.W_PGN, NTa, NT),
        "zero_stride": 0 in op_strides,
        "steps_k": steps_k,
        "m_tile": MTa,
        "n_tile": NTa,
        "k_tile": int(W[L.W_KTA]),
        "nq": int(W[L.W_KTA]) // 4,            # wgmma k8 groups per k-step
        "lbopad": int(W[L.W_LBOPAD]),
        "run_a": int(W[L.W_RUNA]),
        "bulk_flag": bool(flags & 64),
        "tiles": (int(W[L.W_TILES_M]), int(W[L.W_TILES_N]), int(W[L.W_TILES_B])),
    }


# the launch-time choices of the wgmma kernel (ctgb_tc05_launch_config) and what follows from them
LAUNCH_KEYS = ("b_stat", "nb", "sa", "tm_rank", "bulk", "staging", "chunk_steps", "chunks", "one_item", "uneven")
# an H100 SXM and an H100 PCIe: 132 and 114 SMs, 227 KB of opt-in shared memory per block on both
H100_SMS = (132, 114)
H100_SMEM_OPTIN = 232448


def a_operand_addr(case, plan, base):
    """Device address of the plan's A operand when the case's operand buffers start at ``base``
    (a 256-byte aligned allocation): the streamed operand is B when the plan swaps them."""
    which = 1 if plan.swapped else 0
    return base + case.offsets[which] * np.dtype(case.dtype).itemsize


def launch_facts(case, plan, a_addr, sms, smem_optin):
    """The wgmma launch's choices for A at ``a_addr`` on a device with ``sms`` SMs."""
    from cotengra_b200 import _lib

    f = _lib.tc05_launch_config(plan.words, a_addr, sms, smem_optin)
    W = plan.words
    work = int(W[L.W_TILES_M]) * int(W[L.W_TILES_N]) * int(W[L.W_TILES_B]) * int(W[L.W_SPLITK])
    f["staging"] = "tmap" if f["tm_rank"] else ("bulk" if f["bulk"] else "gather")
    f["work"] = work
    f["one_item"] = f["grid"] == work
    f["uneven"] = work % f["grid"] != 0
    return f


def plan_mismatches(case, plan):
    facts = plan_facts(plan)
    return {k: (v, facts[k]) for k, v in case.expect if k not in LAUNCH_KEYS and facts[k] != v}


def launch_mismatches(case, facts):
    return {k: (v, facts[k]) for k, v in case.expect if k in LAUNCH_KEYS and facts[k] != v}


def store_mode(case, plan):
    """The epilogue store path the kernel takes for this plan (gett_ws.cuh, rowstream.cuh,
    dmmastream.cuh, dotstream.cuh)."""
    f = plan_facts(plan)
    v = f["variant"]
    c128 = case.dtype == C128
    eight = np.dtype(case.dtype).itemsize == 8
    if v in (L.VAR_DOTSTREAM, L.VAR_DOTSTREAM4):
        return "accumulate" if f["accumulate"] else "atomic"
    if v in (L.VAR_ROWSTREAM, L.VAR_ROWSTREAM_K, L.VAR_DMMASTREAM):
        if f["accumulate"]:
            return "accumulate"
        if eight and f["quad8"] and v != L.VAR_DMMASTREAM:
            return "quad8"
        if eight and f["pair8"] and v == L.VAR_ROWSTREAM:
            return "pair8"
        if c128 and f["pair"] and v != L.VAR_ROWSTREAM_K:
            return "pair"
        return "plain"
    if v in L.TC05_VARIANTS:
        return "atomic" if f["splitk"] > 1 else ("accumulate" if f["accumulate"] else "plain")
    if f["splitk"] > 1:
        return "atomic"
    if f["accumulate"]:
        return "accumulate"
    if c128 and f["pair"]:
        return "pair_full" if f["full_tiles"] else "pair_ragged"
    return "plain"


# ---------------------------------------------------------------------------- staged families
# Each family maps a policy tile (MT, NT, KT) to the keyword arguments of one Case.


def _gemm(M, N, K, **kw):
    return dict(eq="ab,bc->ac", shapes=((M, K), (K, N)), **kw)


def fam_ragged(MT, NT, KT):
    # partial m (last tile: 5 rows, odd), n and k together; 3 m tiles: a non-power-of-two grid
    exp = {"pgk": True, "grid_pow2": False}
    if MT > 1:
        exp.update(pgm=True, pgn=True, odd_tail=True)
    return _gemm(2 * MT + 5, NT + 3, 2 * KT + 3, expect=exp)


def fam_exact_pow2(MT, NT, KT):
    # every class made of whole dims -- a tile-sized one and a binary one that cannot coalesce with
    # it -- so no blocked dim anywhere: exactA/exactB tables and shift/mask grid decoding
    p = max(2, 2 * NT // MT)
    return dict(eq="prca,rqcb->paqb", shapes=((p, 2, KT, MT), (2, 2, KT, NT)),
                expect={"pgm": False, "pgn": False, "pgk": False, "grid_pow2": True, "m_pow2": True})


def _structured(MT, NT, KT):
    ma, nb, kc = max(3, MT // 2 + 3), max(3, NT // 2 + 1), max(3, KT // 2 + 1)
    # binary i, j (m), u (n), v (k), a batch of 3, interleaved; C's order matches neither operand
    return ("aixcjv", (ma, 2, 3, kc, 2, 2)), ("vbxcu", (2, nb, 3, kc, 2)), "ujxbia"


def fam_structured(MT, NT, KT):
    (ta, sa), (tb, sb), out = _structured(MT, NT, KT)
    return dict(eq=f"{ta},{tb}->{out}", shapes=(sa, sb),
                expect={"batch": True, "multi_m": True, "multi_n": True, "multi_k": True, "swapped": False})


def fam_structured_swapped(MT, NT, KT):
    (ta, sa), (tb, sb), out = _structured(MT, NT, KT)
    return dict(eq=f"{tb},{ta}->{out}", shapes=(sb, sa),
                expect={"batch": True, "multi_m": True, "multi_n": True, "multi_k": True, "swapped": True})


def _gapped_c(N):
    return (2 * N + 7, 2)  # every other element a gap, and 7 more after each row


def fam_gapped(MT, NT, KT):
    # A with row gaps, B column-major with gaps, C with gaps between every element
    M, N, K = 2 * MT + 5, NT + 3, 2 * KT + 3
    return _gemm(M, N, K, strides=((K + 3, 1), (1, K + 2)), out_strides=_gapped_c(N), offsets=(5, 3),
                 accumulate=True, expect={"pgk": True, "pair": False})


def fam_accumulate(MT, NT, KT):
    return _gemm(2 * MT + 5, NT + 3, 2 * KT + 3, accumulate=True, expect={"accumulate": True, "pgk": True})


def _splitk_shape(MT, NT, KT):
    return max(MT, NT) + 5, max(2, NT - 1), 6 * KT + KT // 2  # 7 k-steps, the last one half


def fam_splitk2(MT, NT, KT):
    M, N, K = _splitk_shape(MT, NT, KT)
    return _gemm(M, N, K, force_splitk=2, expect={"splitk": 2, "steps_k": 7})


def fam_splitk3(MT, NT, KT):
    M, N, K = _splitk_shape(MT, NT, KT)
    return _gemm(M, N, K, force_splitk=3, expect={"splitk": 3, "steps_k": 7})  # ranges of 3, 3 and 1 steps


def fam_splitk_acc(MT, NT, KT):
    M, N, K = _splitk_shape(MT, NT, KT)
    return _gemm(M, N, K, force_splitk=2, accumulate=True, out_strides=_gapped_c(N),
                 expect={"splitk": 2, "accumulate": True})


def fam_long_k(MT, NT, KT):
    # 300 k-steps (windowed k table), split in two ranges of 150 that each cross a 128-step window
    return _gemm(max(MT, NT), NT, 300 * KT - 3, force_splitk=2,
                 expect={"long_k": True, "splitk": 2, "steps_k": 300, "pgk": True})


def fam_vjp_broadcast(MT, NT, KT):
    # an output-only index of a VJP: stride 0 in A
    ma = max(MT, NT) // 2 + 3
    K = KT + 5
    return dict(eq="abk,kc->bac", shapes=((ma, 3, K), (K, NT + 3)), strides=((K, 0, 1), None), offsets=(2, 1),
                expect={"zero_stride": True})


def fam_vjp_diag(MT, NT, KT):
    # a diagonal operand: the repeated index i is one dim with summed strides
    ma = max(MT, NT) // 2 + 3
    K = KT + 5
    return dict(eq="iaki,kc->aic", shapes=((3, ma, K, 3), (K, NT + 3)), offsets=(1, 0), expect={"multi_m": True})


def fam_pair_full(MT, NT, KT):
    return _gemm(2 * max(MT, NT), NT, 2 * KT, expect={"pair": True, "full_tiles": True})


def fam_pair_ragged(MT, NT, KT):
    return _gemm(2 * max(MT, NT) + 5, NT - 2, KT + 3, expect={"pair": True, "full_tiles": False, "odd_tail": True})


def fam_rows_bcache(MT, NT, KT):
    # one k-step, no n or batch grid: the row policy keeps B in registers (b_invariant)
    return _gemm(2 * MT + 37, NT - 1, 3, expect={"b_invariant": True, "pgm": True})


STAGED_FAMILIES = {
    "ragged": fam_ragged,
    "exact_pow2": fam_exact_pow2,
    "structured": fam_structured,
    "structured_swapped": fam_structured_swapped,
    "gapped": fam_gapped,
    "accumulate": fam_accumulate,
    "splitk2": fam_splitk2,
    "splitk3": fam_splitk3,
    "splitk_acc": fam_splitk_acc,
    "long_k": fam_long_k,
    "vjp_broadcast": fam_vjp_broadcast,
    "vjp_diag": fam_vjp_diag,
}
PAIR_FAMILIES = {"pair_full": fam_pair_full, "pair_ragged": fam_pair_ragged}


def _case(variant, dtype, family, kw, runs=None):
    kw = dict(kw)
    exp = dict(kw.pop("expect", {}))
    exp.setdefault("variant", variant if runs is None else runs)
    exp.setdefault("splitk", kw.get("force_splitk", 1) or 1)
    if "swapped" not in exp:
        exp["swapped"] = False
    return Case(variant, dtype, family, expect=tuple(sorted(exp.items())), **kw)


def staged_cases():
    out = []
    for v, dtypes in STAGED.items():
        MT, NT, KT = L.VARIANT_TILES[v]
        for d in dtypes:
            fams = dict(STAGED_FAMILIES)
            if d == C128 and v != L.VAR_KRED:
                fams.update(PAIR_FAMILIES)
            if v in ROW_VARIANTS:
                fams["rows_bcache"] = fam_rows_bcache
            for name, fam in fams.items():
                kw = fam(MT, NT, KT)
                if v in ROW_VARIANTS and name == "ragged":
                    kw["expect"] = dict(kw["expect"], b_invariant=False)
                out.append(_case(v, d, name, kw))
    for (v, d), runs in REMAPS.items():
        MT, NT, KT = L.VARIANT_TILES[runs]
        out.append(_case(v, d, "remap", fam_ragged(MT, NT, KT), runs=runs))
    return out


# ---------------------------------------------------------------------------- stream kernels


def _rows3(M0, K):
    # M = 3 * M0 rows as two dims that never coalesce (the tile takes the M0 one whole): A stored k-major
    return "xka", (3, K, M0)


def stream_cases():
    out = []

    def add(v, d, family, eq, shapes, **kw):
        out.append(_case(v, d, family, dict(eq=eq, shapes=shapes, **kw)))

    # ---- ROWSTREAM: the 4x4, 2x8 and 8x8 instantiations, every store of each element type
    for d in ALL_DTYPES:
        eight, c128 = np.dtype(d).itemsize == 8, d == C128
        ta, sa = _rows3(200, 4)
        add(L.VAR_ROWSTREAM, d, "rs4x4_nonpow2_m", f"{ta},kc->xac", (sa, (4, 3)),
            expect={"m_pow2": False, "pair": False, "quad8": False, "pair8": False})
        add(L.VAR_ROWSTREAM, d, "rs2x8_pow2_m", "ak,kc->ac", ((1024, 7), (7, 2)),
            expect={"m_pow2": True, "pair8": eight, "pair": c128, "n_tile": 2, "k_tile": 7})
        add(L.VAR_ROWSTREAM, d, "rs8x8_quad", "ak,kc->ac", ((768, 8), (8, 8)),
            expect={"m_pow2": False, "quad8": eight, "pair": c128, "grid_pow2": False})
        ta, sa = _rows3(200, 5)
        add(L.VAR_ROWSTREAM, d, "rs8x8_pair8", f"{ta},kc->xac", (sa, (5, 6)),
            expect={"quad8": False, "pair8": eight, "pair": c128})
        ta, sa = _rows3(200, 6)
        add(L.VAR_ROWSTREAM, d, "rs8x8_accumulate", f"{ta},kc->xac", (sa, (6, 5)), accumulate=True,
            expect={"accumulate": True})
        add(L.VAR_ROWSTREAM, d, "rs4x4_gapped", "ak,kc->ac", ((512, 3), (3, 4)), strides=((5, 1), None),
            out_strides=_gapped_c(4), offsets=(3, 1), accumulate=True, expect={"accumulate": True})
    # ---- ROWSTREAM_K: K from 9 to 64 (8-byte and narrower types)
    for d in (F32, F64, C64):
        eight = np.dtype(d).itemsize == 8
        ta, sa = _rows3(200, 9)
        add(L.VAR_ROWSTREAM_K, d, "rsk_k9", f"{ta},kc->xac", (sa, (9, 8)), expect={"quad8": eight, "k_tile": 9})
        add(L.VAR_ROWSTREAM_K, d, "rsk_k64_pow2_m", "ak,kc->ac", ((1024, 64), (64, 3)),
            expect={"m_pow2": True, "k_tile": 64})
        ta, sa = _rows3(200, 37)
        add(L.VAR_ROWSTREAM_K, d, "rsk_k37_accumulate", f"{ta},kc->xac", (sa, (37, 6)), accumulate=True,
            expect={"accumulate": True, "k_tile": 37})
    # ---- DMMASTREAM (complex128): 9 <= N <= 32 with K <= 32, N <= 8 with 8 < K <= 64, masked row tails
    ta, sa = _rows3(200, 32)  # 600 rows: the last 32-row block is 24 rows
    add(L.VAR_DMMASTREAM, C128, "ds_n9_k32", f"{ta},kc->xac", (sa, (32, 9)), expect={"pair": False, "n_tile": 9})
    add(L.VAR_DMMASTREAM, C128, "ds_n24_k20_pair", "ak,kc->ac", ((1024, 20), (20, 24)),
        expect={"pair": True, "n_tile": 24})
    ta, sa = _rows3(200, 7)
    add(L.VAR_DMMASTREAM, C128, "ds_n32_k7_permuted", f"{ta},kc->cxa", (sa, (7, 32)),
        expect={"pair": False, "n_tile": 32})
    ta, sa = _rows3(200, 64)
    add(L.VAR_DMMASTREAM, C128, "ds_n8_k64_pair", f"{ta},kc->xac", (sa, (64, 8)), expect={"pair": True, "k_tile": 64})
    ta, sa = _rows3(200, 33)
    add(L.VAR_DMMASTREAM, C128, "ds_n5_k33_accumulate", f"{ta},kc->xac", (sa, (33, 5)), accumulate=True,
        expect={"accumulate": True})
    # ---- DOTSTREAM (M = N = 1), DOTSTREAM4 (M, N <= 4), KRED: blocked or partial k, permuted dense C
    for d in ALL_DTYPES:
        add(L.VAR_DOTSTREAM, d, "dot_blocked_k", "k,k->", ((6144,), (6144,)), expect={"pgk": True, "steps_k": 3})
        add(L.VAR_DOTSTREAM, d, "dot_permuted", "abc,cba->", ((16, 8, 32), (32, 8, 16)), expect={"multi_k": True})
        add(L.VAR_DOTSTREAM, d, "dot_accumulate", "ab,ba->", ((64, 96), (96, 64)), accumulate=True,
            expect={"accumulate": True})
        add(L.VAR_DOTSTREAM4, d, "dot4_permuted_c", "km,kn->nm", ((6144, 4), (6144, 3)), expect={"pgk": True})
        add(L.VAR_DOTSTREAM4, d, "dot4_accumulate", "akm,kan->mn", ((32, 64, 3), (64, 32, 2)), accumulate=True,
            expect={"accumulate": True, "multi_k": True})
        add(L.VAR_KRED, d, "kred_small_permuted_c", "km,kn->nm", ((1500, 4), (1500, 2)), force_splitk=None,
            expect={"pgk": True, "splitk": 3})
    # ---- DMMA_32x32 / TF32_32x32: odd M, N <= 32, one tile, split-K over 2 x SMs
    for v, d in ((L.VAR_DMMA_32x32, F64), (L.VAR_DMMA_32x32, C128), (L.VAR_TF32_32x32, F32),
                 (L.VAR_TF32_32x32, C64)):
        add(v, d, "one_tile_splitk", "ab,bc->ac", ((31, 4219), (4219, 27)), force_splitk=None,
            expect={"splitk": 2 * SM_COUNT, "steps_k": 264})
    return out


# ---------------------------------------------------------------------------- wgmma (complex64)
# Each family maps the N tile NT of a wgmma variant to the keyword arguments of one Case.  Its
# expectations cover the plan (tile shape, k8 groups, flags) and the launch (ctgb_tc05_launch_config:
# resident B' or ring, A staging, chunking), and hold on 132 and 114 SMs alike.  A's offset is even
# (16-byte aligned tiles) except in the cases that exist for a misaligned A.

# k-steps of B' that stay resident next to three A stages in 227 KB (32, 16 and 8 KB per k-step),
# at most Tc05Cfg::NB_MAX = 8
TC05_RESIDENT_STEPS = {64: 3, 32: 6, 16: 8}
# A staging depth (16 KB stages) left beside that many resident k-steps
_SA_AT_FIT = {64: 3, 32: 3, 16: 5}
# NTa < NT with NTa % 4 != 0: the column quads of the last lanes straddle the tile's edge
_NT_RAGGED = {64: 54, 32: 27, 16: 13}


def _resident(NT, steps):
    return {"b_stat": int(steps <= TC05_RESIDENT_STEPS[NT]), "nb": steps if steps <= TC05_RESIDENT_STEPS[NT] else 3}


def tc_k4_m64(NT):
    # ONE 4-wide k-step (nq 1) of a 64-row tile: consumer warpgroup 1 stores nothing.  Three work items,
    # one per CTA; A's 256-element tile is one contiguous box dim: a rank-2 tensor map
    return dict(eq="xak,kc->xac", shapes=((3, 64, 4), (4, NT)), strides=((300, 4, 1), None), offsets=(2, 0),
                expect={"m_tile": 64, "k_tile": 4, "nq": 1, "steps_k": 1, "tiles": (3, 1, 1), "grid_pow2": False,
                        "tm_rank": 2, "one_item": True, "chunks": 1, **_resident(NT, 1)})


def tc_pow2_resident(NT):
    # full 128 x NT x 16 tiles on a power-of-two grid (shift decode), two k-steps of resident B'
    return _gemm(512, 2 * NT, 32, expect={"full_tiles": True, "grid_pow2": True, "m_pow2": True, "nq": 4,
                                             "tiles": (4, 2, 1), "steps_k": 2, "tm_rank": 3, "lbopad": 1,
                                             "one_item": True, "chunks": 1, **_resident(NT, 2)})


def tc_idiv_ring(NT):
    # three m tiles (idiv decode) and nine k-steps: more than fit, so B' streams through the ring
    return _gemm(384, NT, 144, expect={"grid_pow2": False, "tiles": (3, 1, 1), "steps_k": 9, "chunk_steps": 9,
                                          "chunks": 1, "tm_rank": 3, **_resident(NT, 9)})


def tc_resident_at_fit(NT):
    # the most k-steps whose B' stays resident next to three A stages: the most B' slots and barriers, and
    # the least shared memory left for A
    s = TC05_RESIDENT_STEPS[NT]
    return _gemm(256, NT, 16 * s, expect={"steps_k": s, "b_stat": 1, "nb": s, "sa": _SA_AT_FIT[NT], "chunks": 1})


def tc_ring_past_fit(NT):
    # one k-step more: B' streams through the 3-slot ring
    s = TC05_RESIDENT_STEPS[NT] + 1
    return _gemm(256, NT, 16 * s, expect={"steps_k": s, "b_stat": 0, "nb": 3, "chunks": 1})


def tc_accumulate(NT):
    return _gemm(256, NT, 32, accumulate=True, expect={"accumulate": True, "chunks": 1, "steps_k": 2})


def tc_two_chunks_fold(NT):
    # 17 k-steps: two balanced chunks (9 + 8), the second folded into what the first stored (C starts NaN)
    return _gemm(256, NT, 272, expect={"steps_k": 17, "chunk_steps": 9, "chunks": 2, "accumulate": False,
                                          "b_stat": 0})


def tc_chunks_accumulate(NT):
    # 50 k-steps in four chunks (13, 13, 12, 12), every one added to C0
    return _gemm(128, NT, 800, accumulate=True, expect={"steps_k": 50, "chunk_steps": 13, "chunks": 4,
                                                           "accumulate": True})


def tc_nq3_chunks(NT):
    # 12-wide k-steps (6^n extents: nq 3): 25 steps in chunks of at most 36 k8 accumulations: 9, 8, 8
    return _gemm(256, NT, 300, expect={"k_tile": 12, "nq": 3, "steps_k": 25, "chunk_steps": 9, "chunks": 3})


def tc_nq2(NT):
    return _gemm(256, NT, 40, expect={"k_tile": 8, "nq": 2, "steps_k": 5, "chunks": 1, **_resident(NT, 5)})


def tc_splitk3_uneven(NT):
    # 7 k-steps over three CTAs: ranges of 3, 3 and 1, added with atomics after the memset
    return _gemm(256, NT, 112, force_splitk=3, expect={"splitk": 3, "steps_k": 7, "b_stat": 0, "chunks": 1})


def tc_splitk3_chunked(NT):
    # 50 k-steps over three CTAs: ranges of 17, 17 and 16, each in two chunks
    return _gemm(128, NT, 800, force_splitk=3, expect={"splitk": 3, "steps_k": 50, "chunk_steps": 9, "chunks": 2})


def tc_splitk_acc_gapped(NT):
    return _gemm(256, NT, 112, force_splitk=2, accumulate=True, out_strides=_gapped_c(NT),
                    expect={"splitk": 2, "accumulate": True, "b_stat": 0})


def tc_ragged_tile(NT):
    # 108 x NTa x 12 tiles (64 < MTa < 128, NTa % 4 != 0): the bond-6 PEPS shape of each N tile
    R = _NT_RAGGED[NT]
    return _gemm(216, 2 * R, 24, expect={"m_tile": 108, "n_tile": R, "k_tile": 12, "nq": 3, "tiles": (2, 2, 1),
                                            "steps_k": 2, "full_tiles": False, **_resident(NT, 2)})


def tc_gather_odd(NT):
    # A rows 17 elements apart: runs of 16 at odd offsets -- no tensor map, no bulk copies
    return _gemm(256, NT, 16, strides=((17, 1), None), offsets=(2, 0),
                    expect={"bulk_flag": False, "staging": "gather", "tm_rank": 0, **_resident(NT, 1)})


def tc_misaligned_a(NT):
    # bulk runs in the descriptor, but A 8 bytes off 16-byte alignment: the launch gathers
    return _gemm(256, NT, 32, offsets=(1, 0), expect={"bulk_flag": True, "staging": "gather", "tm_rank": 0})


def tc_bulk_runs(NT):
    # five box dims (k and four m dims that never coalesce): no tensor map; runs of 16 elements
    return dict(eq="abcdk,kn->abcdn", shapes=((32, 2, 2, 2, 16), (16, NT)), strides=((160, 78, 38, 18, 1), None),
                offsets=(4, 0), expect={"bulk_flag": True, "run_a": 16, "staging": "bulk", "tm_rank": 0,
                                        "tiles": (2, 1, 1)})


def tc_tmap4(NT):
    # three box dims of A (k, then two m dims with gaps): a rank-4 tensor map
    return dict(eq="abk,kc->abc", shapes=((32, 8, 16), (16, NT)), strides=((164, 20, 1), None), offsets=(2, 0),
                expect={"tm_rank": 4, "tiles": (2, 1, 1)})


def tc_tmap5(NT):
    # four box dims: a rank-5 tensor map
    return dict(eq="abck,kn->abcn", shapes=((16, 4, 4, 16), (16, NT)), strides=((310, 76, 18, 1), None),
                offsets=(6, 0), expect={"tm_rank": 5, "tiles": (2, 1, 1)})


def tc_swapped(NT):
    # the larger operand second: the plan swaps them, so the launch streams B's buffer as A
    return dict(eq="kc,ak->ac", shapes=((16, NT), (256, 16)), offsets=(0, 2), expect={"swapped": True})


def tc_batched(NT):
    # a batch grid of 3: B' changes between work items of a CTA, so it streams through the ring
    return dict(eq="xab,xbc->xac", shapes=((3, 256, 32), (3, 32, NT)),
                expect={"batch": True, "tiles": (2, 1, 3), "b_stat": 0, "nb": 3})


def tc_permuted_gapped(NT):
    # C transposed with gaps, B column-major with gaps (bprime_kernel reads past sentinels)
    return dict(eq="ab,bc->ca", shapes=((256, 32), (32, NT)), strides=(None, (1, 34)), out_strides=(519, 2),
                offsets=(0, 3), expect={"swapped": False})


def tc_many_items_resident(NT):
    # 512 work items over the CTAs, unevenly, with B' resident (one k-step)
    return _gemm(65536, NT, 16, expect={"tiles": (512, 1, 1), "uneven": True, **_resident(NT, 1)})


def tc_many_items_ring(NT):
    # the same number of items in two batches: B' streamed
    return dict(eq="xab,xbc->xac", shapes=((2, 32768, 16), (2, 16, NT)),
                expect={"tiles": (256, 1, 2), "uneven": True, "b_stat": 0})


def tc_same_sign_k256(NT):
    # no cancellation: 16 k-steps = 64 truncating wgmma accumulations in one chunk
    return _gemm(256, NT, 256, dist="same_sign", expect={"nq": 4, "steps_k": 16, "chunk_steps": 16, "chunks": 1})


def tc_same_sign_k4096(NT):
    # ... and 256 k-steps: 16 such chunks folded with round-to-nearest adds
    return _gemm(128, NT, 4096, dist="same_sign", expect={"steps_k": 256, "chunk_steps": 16, "chunks": 16})


TC05_FAMILIES = {
    "k4_m64": tc_k4_m64,
    "pow2_resident": tc_pow2_resident,
    "idiv_ring": tc_idiv_ring,
    "resident_at_fit": tc_resident_at_fit,
    "ring_past_fit": tc_ring_past_fit,
    "accumulate": tc_accumulate,
    "two_chunks_fold": tc_two_chunks_fold,
    "chunks_accumulate": tc_chunks_accumulate,
    "nq3_chunks": tc_nq3_chunks,
    "nq2": tc_nq2,
    "splitk3_uneven": tc_splitk3_uneven,
    "splitk3_chunked": tc_splitk3_chunked,
    "splitk_acc_gapped": tc_splitk_acc_gapped,
    "ragged_tile": tc_ragged_tile,
    "gather_odd": tc_gather_odd,
    "misaligned_a": tc_misaligned_a,
    "bulk_runs": tc_bulk_runs,
    "tmap4": tc_tmap4,
    "tmap5": tc_tmap5,
    "swapped": tc_swapped,
    "batched": tc_batched,
    "permuted_gapped": tc_permuted_gapped,
    "many_items_resident": tc_many_items_resident,
    "many_items_ring": tc_many_items_ring,
    "same_sign_k256": tc_same_sign_k256,
    "same_sign_k4096": tc_same_sign_k4096,
}

# The shapes the wgmma kernel's first mode tests used (name, eq, shapes, build_pair_desc kwargs, and the
# (variant, split-K) the plan must take), each run with A aligned and with A 8 bytes further on.  Without
# a forced variant or split the plan takes the automatic choice for 132 SMs.
_T64, _T32, _T16 = L.VAR_TC05_128x64, L.VAR_TC05_128x32, L.VAR_TC05_128x16
TC05_LEGACY = [
    ("ring_b_long_k", "ab,bc->ac", ((1024, 256), (256, 64)), {"force_splitk": 1}, (_T64, 1)),  # 16 k-steps: a ring
    ("m_fastest", "ba,bc->ac", ((64, 512), (64, 128)), {"force_splitk": 1}, (_T64, 1)),  # A k-major: runs of 128
    ("batched", "xab,xbc->xac", ((3, 256, 32), (3, 32, 64)), {"variant": _T64}, (_T64, 1)),
    ("gather_odd_strides", "abx,bcx->acx", ((256, 32, 3), (32, 32, 3)), {"variant": _T32}, (_T32, 1)),
    ("split_k", "ab,bc->ac", ((128, 256), (256, 64)), {"force_splitk": 4}, (_T64, 4)),
    ("accumulate", "ab,bc->ac", ((512, 64), (64, 64)), {"accumulate": True, "force_splitk": 1}, (_T64, 1)),
    ("accumulate_split", "ab,bc->ac", ((512, 64), (64, 64)), {"accumulate": True, "force_splitk": 2}, (_T64, 2)),
    ("non_pow2_grid", "ab,bc->ac", ((384, 48), (48, 32)), {"variant": _T32, "force_splitk": 1}, (_T32, 1)),
    ("permuted_out", "aibj,ijc->cba", ((16, 4, 16, 8), (4, 8, 64)), {"variant": _T64}, (_T64, 1)),
    ("wide_n", "ab,bc->ac", ((1024, 64), (64, 512)), {"force_splitk": 1}, (_T64, 1)),
    ("narrow_n16", "ab,cb->ac", ((4096, 32), (16, 32)), {}, (_T16, 1)),
    ("narrow_n16_batched", "xab,xbc->xca", ((2, 512, 64), (2, 64, 16)), {"variant": _T16}, (_T16, 4)),
]

def tc05_cases():
    out = []
    for v in L.TC05_VARIANTS:
        NT = L.VARIANT_TILES[v][1]
        for name, fam in TC05_FAMILIES.items():
            out.append(_case(v, C64, name, fam(NT)))
    # guard bands around a gapped A and C (accumulating), a dense non-power-of-two grid, dense split-K
    out.append(_case(_T64, C64, "tc05_gapped_accumulate", _gemm(
        256, 64, 32, strides=((36, 1), None), out_strides=_gapped_c(64), offsets=(4, 0), accumulate=True,
        expect={"accumulate": True, "staging": "tmap", "b_stat": 1, "nb": 2})))
    out.append(_case(_T32, C64, "tc05_dense_non_pow2", _gemm(
        384, 32, 48, expect={"grid_pow2": False, "tiles": (3, 1, 1), "b_stat": 1, "nb": 3})))
    out.append(_case(_T16, C64, "tc05_splitk_dense", _gemm(
        256, 16, 64, force_splitk=2, expect={"splitk": 2, "b_stat": 0})))
    # the bond-6 PEPS tile with same-sign operands: 18 k-steps of 12 in two chunks (9 + 9)
    out.append(_case(_T64, C64, "same_sign_108x54x12", _gemm(
        1296, 216, 216, dist="same_sign",
        expect={"m_tile": 108, "n_tile": 54, "k_tile": 12, "steps_k": 18, "chunk_steps": 9, "chunks": 2})))
    for name, eq, shapes, kw, (v, want_splitk) in TC05_LEGACY:
        kw = dict(kw)
        splitk = kw.pop("force_splitk", None)
        kw.pop("variant", None)
        exp = {"bulk_flag": name != "gather_odd_strides", "splitk": want_splitk}
        for suffix, off, staging in (("", 0, None), ("_a_plus_8_bytes", 1, "gather")):
            e = dict(exp, **({"staging": staging} if staging else {}))
            out.append(_case(v, C64, f"legacy_{name}{suffix}", dict(eq=eq, shapes=shapes, offsets=(off, 0),
                                                                    force_splitk=splitk, expect=e, **kw)))
    return out


CASES = staged_cases() + stream_cases() + tc05_cases()


# ---------------------------------------------------------------------------- buffers


def _reach(shape, strides):
    off = np.zeros((), dtype=np.int64)
    for d, s in zip(shape, strides):
        off = np.add.outer(off, np.arange(d, dtype=np.int64) * int(s))
    return off


def sentinel_fill(n, dtype):
    """``n`` elements of ``dtype`` whose every real component holds the sentinel NaN."""
    rd = real_dtype(dtype)
    comp = 2 if np.dtype(dtype).kind == "c" else 1
    bits = np.full(n * comp, SENTINEL_BITS[rd], dtype=np.uint64 if rd.itemsize == 8 else np.uint32)
    return bits.view(rd).view(dtype)


def _random(rng, shape, dtype, dist="uniform", which=0):
    """Operand ``which`` (0: A, 1: B, 2: C0).  "same_sign": A real in [0.5, 1], B with real and
    imaginary parts in [0.5, 1] -- every product of the contraction has positive real and imaginary
    parts, so nothing cancels and a truncating accumulation shows its bias."""
    if dist == "same_sign" and which < 2:
        x = rng.uniform(0.5, 1.0, size=shape)
        if which == 1:
            x = x + 1j * rng.uniform(0.5, 1.0, size=shape)
        return x.astype(dtype)
    x = rng.uniform(-1.0, 1.0, size=shape)
    if np.dtype(dtype).kind == "c":
        x = x + 1j * rng.uniform(-1.0, 1.0, size=shape)
    return x.astype(dtype)


@dataclass
class Layout:
    bufs: list          # host buffers of A, B, C (initial contents)
    offs: list          # element offsets of A, B, C in them
    ops: list           # A and B as described (numpy arrays, values as the kernel sees them)
    c_reach: np.ndarray  # element offset (from C's origin) of every described C element, out_shape
    c0: np.ndarray      # initial described C (random when accumulating, NaN otherwise)


def make_layout(case, seed=0):
    rng = np.random.default_rng(seed)
    dt = np.dtype(case.dtype)
    guard = max(32, C_ALIGN // dt.itemsize)
    bufs, offs, ops = [], [], []
    ta, tb, _ = case.terms()
    for which, (shape, strides, off) in enumerate(zip(case.shapes, case.strides, case.offsets)):
        strides = L.row_major_strides(shape) if strides is None else strides
        reach = _reach(shape, strides)
        buf = sentinel_fill(off + int(reach.max()) + 1 + guard, dt)
        # (repeated offsets -- stride 0, diagonals: the last write wins)
        buf[off + reach] = _random(rng, reach.shape, dt, case.dist, which)
        bufs.append(buf)
        offs.append(off)
        ops.append(buf[off + reach])
    out_shape = case.out_shape()
    cs = L.row_major_strides(out_shape) if case.out_strides is None else case.out_strides
    c_reach = _reach(out_shape, cs)
    assert np.unique(c_reach).size == c_reach.size, "C elements overlap"
    c_off = C_ALIGN // dt.itemsize
    cbuf = sentinel_fill(c_off + int(c_reach.max()) + 1 + guard, dt)
    c0 = _random(rng, out_shape, dt) if case.accumulate else np.full(out_shape, np.nan, dtype=dt)
    cbuf[c_off + c_reach] = c0
    bufs.append(cbuf)
    offs.append(c_off)
    return Layout(bufs, offs, ops, c_reach, c0)


def reference(case, lay):
    """(ref, scale): the contraction in float64/complex128 (+ C0), and the same contraction over
    absolute values (+ |C0|) -- the per-element error scale."""
    wd = wide_dtype(case.dtype)
    a, b = (x.astype(wd) for x in lay.ops)
    ref = np.einsum(case.eq, a, b, optimize=True)
    scale = np.einsum(case.eq, np.abs(a), np.abs(b), optimize=True)
    if case.accumulate:
        ref = ref + lay.c0.astype(wd)
        scale = scale + np.abs(lay.c0.astype(wd))
    return np.asarray(ref), np.asarray(scale)


def check_result(case, lay, cbuf_after):
    """Sentinels bit-identical, no described C element NaN; returns (got, bad_sentinels)."""
    c_off = lay.offs[2]
    rd = real_dtype(case.dtype)
    ui = np.uint64 if rd.itemsize == 8 else np.uint32
    before = lay.bufs[2].view(rd).view(ui)
    after = np.asarray(cbuf_after).view(rd).view(ui)
    described = np.zeros(lay.bufs[2].size, dtype=bool)
    described[c_off + lay.c_reach.reshape(-1)] = True
    comp = 2 if np.dtype(case.dtype).kind == "c" else 1
    mask = np.repeat(~described, comp)
    bad = np.flatnonzero(mask & (before != after))
    got = np.asarray(cbuf_after)[c_off + lay.c_reach]
    return got, bad


def error_ratio(got, ref, scale):
    """max_ij |got - ref| / scale (inf where scale is 0 and got != ref)."""
    err = np.abs(got.astype(ref.dtype) - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(scale > 0, err / np.where(scale > 0, scale, 1.0), np.where(err > 0, np.inf, 0.0))
    return float(np.max(r)) if r.size else 0.0
