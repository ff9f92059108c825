"""Host-side lowering of one contraction-tree node to a kernel descriptor.

The reference lowers a pairwise node to ``transpose -> reshape(copy) -> matmul
-> reshape/transpose`` (cotengra/contract.py:167-329 plans it, :364-411 runs
it).  Here the same index classification is done once on the host --

    bat_inds  (on A, B and the output)      contract.py:226-237
    con_inds  (on A and B, not the output)  contract.py:226-237
    a_keep    (on A and the output)         contract.py:238-239
    b_keep    (on B and the output)         contract.py:241-243

-- but instead of permuting data each class becomes a list of *dims with
strides* in A, B and C.  Repeated indices (diagonals) add their strides,
size-1 dims drop out, broadcast dims get stride 0, indices summed on a single
operand become contracted dims with stride 0 on the other operand
(contract.py:193-216, 256-274).  Adjacent dims that stay adjacent in every
operand are coalesced, each class is split into CTA-tile dims and grid dims,
and everything is packed into the int64 word layout of ``csrc/gett_desc.h``.

All of this is integer work and is tested bit-exactly against the reference's
own planners (tests/test_lowering.py).
"""

from __future__ import annotations

import math
from collections import Counter, namedtuple
from dataclasses import dataclass, field

import numpy as np

# ---- word layout: mirror of csrc/gett_desc.h (checked against the built
# library in _lib.py through ctgb_desc_words()) -----------------------------
MAX_T, MAX_G, MAX_GB, MAX_LD = 12, 40, 12, 24
(W_MAGIC, W_DTYPE, W_NTM, W_NTN, W_NTK, W_NGM, W_NGN, W_NGK, W_NGB, W_MTA,
 W_NTA, W_KTA, W_TILES_M, W_TILES_N, W_TILES_B, W_STEPS_K, W_SPLITK, W_PGM,
 W_MFULL, W_MTEXT, W_MW, W_PGN, W_NFULL, W_NTEXT, W_NW, W_PGK, W_KFULL,
 W_KTEXT, W_KW, W_NLDA, W_NLDB, W_FLAGS, W_VARIANT, W_CELEMS, W_RUNA, W_LBOPAD) = range(36)
# fused strip_exponent: device addresses of doubles (0 = off) -- the factors fA and fB the product
# is divided by, and the slot that receives max|product| of the launch (patched in by ctgb_plan_create)
W_SCALE_A, W_SCALE_B, W_FACTOR_C = 36, 37, 38
W_HDR = 40
OFF_TM = W_HDR
OFF_TN = OFF_TM + MAX_T * 3
OFF_TK = OFF_TN + MAX_T * 3
OFF_GM = OFF_TK + MAX_T * 3
OFF_GN = OFF_GM + MAX_G * 4
OFF_GK = OFF_GN + MAX_G * 4
OFF_GB = OFF_GK + MAX_G * 4
OFF_LDA = OFF_GB + MAX_GB * 5
OFF_LDB = OFF_LDA + MAX_LD * 4
DESC_WORDS = OFF_LDB + MAX_LD * 4
DESC_MAGIC = 0x4354474232303031

MAX_S = 40
S_MAGIC, S_DTYPE, S_NO, S_NS, S_OUT_ELEMS, S_SUM_ELEMS, S_FLAGS = range(7)
S_HDR = 8
OFF_SO = S_HDR
OFF_SS = OFF_SO + MAX_S * 3
SDESC_WORDS = OFF_SS + MAX_S * 2
SDESC_MAGIC = 0x4354474253303031

VAR_SIMT_64x64, VAR_KRED, VAR_DMMA_128x64, VAR_DMMA_64x128, VAR_DMMA_256x32 = 0, 1, 2, 3, 4
VAR_DMMA_256x16, VAR_ROW_128x8, VAR_ROW_256x4, VAR_ROWSTREAM = 5, 6, 7, 8
VAR_TC05_128x64, VAR_TC05_128x32, VAR_TC05_128x16 = 9, 10, 11
VAR_DMMA3M_128x32, VAR_DMMA3M_256x16, VAR_DMMASTREAM, VAR_DOTSTREAM, VAR_DOTSTREAM4 = 12, 13, 14, 15, 16
VAR_DMMA_32x32, VAR_ROWSTREAM_K, VAR_TF32_32x32 = 18, 19, 20
VAR_ABSORB_ROOT = 21
# the DMMA stream kernel (csrc/dmmastream.cuh) takes N <= 32 with K <= 64 (32-row warp blocks) and
# 32 < N <= 64 with K <= 32 (16-row warp blocks)
DMMASTREAM_KMAX, DMMASTREAM_WIDE_N, DMMASTREAM_WIDE_KMAX = 64, 64, 32


def dmmastream_fits(N, K):
    return (N <= 32 and K <= DMMASTREAM_KMAX) or (N <= DMMASTREAM_WIDE_N and K <= DMMASTREAM_WIDE_KMAX)


# choose_variant sends it the complex128 nodes with N <= 32, K <= 64.  One Sycamore-m20 slice on an H100
# 80GB HBM3 (700 W), per node against the staged tiles (DESIGN.md 6a): N = 32 ran at 2.4-2.8 TB/s against
# 2.0-2.4 (2^25 x 32 x 32: 12.25 vs 15.71 ms; 2^24 x 32 x 64: 9.26 vs 12.66 ms), but the 16-row N = 64
# blocks were not faster than DMMA_128x64 (2^24 x 64 x 32: 11.3-11.8 vs 10.8 ms), so N > 32 stays staged.
DMMASTREAM_MAX_N = 32


TC05_VARIANTS = (VAR_TC05_128x64, VAR_TC05_128x32, VAR_TC05_128x16)
TC05_MAX_K = 16384       # 1024 k-steps (the kernel's k table); beyond 256 in chunks of 256
TC05_CHUNK_STEPS = 16    # full k-steps accumulated in one register accumulation before a round-to-nearest fold (tc05_chunk_steps in
                         # csrc/tc05_kernel.cuh balances the chunks and shortens them for tiles with fewer than 16 k)
# (MT, NT, KT) of every kernel variant -- must match ctg_b200.cu's dispatch
VARIANT_TILES = {
    VAR_SIMT_64x64: (64, 64, 8),
    VAR_KRED: (1, 1, 512),
    VAR_DMMA_128x64: (128, 64, 16),
    VAR_DMMA_64x128: (64, 128, 16),
    VAR_DMMA_256x32: (256, 32, 8),
    VAR_DMMA_256x16: (256, 16, 8),
    VAR_ROW_128x8: (256, 8, 4),
    VAR_ROW_256x4: (256, 4, 4),
    VAR_ROWSTREAM: (256, 8, 8),
    VAR_TC05_128x64: (128, 64, 16),
    VAR_TC05_128x32: (128, 32, 16),
    VAR_TC05_128x16: (128, 16, 16),
    VAR_DMMA3M_128x32: (128, 32, 16),
    VAR_DMMA3M_256x16: (256, 16, 8),
    VAR_DMMASTREAM: (256, 64, 64),
    VAR_DOTSTREAM: (1, 1, 2048),
    VAR_DOTSTREAM4: (4, 4, 1024),
    VAR_DMMA_32x32: (32, 32, 16),
    VAR_ROWSTREAM_K: (256, 8, 64),
    VAR_TF32_32x32: (32, 32, 16),
}

# compute modes of the float32 / complex64 tensor-core variants: "3xtf32" (the default, fp32 accuracy:
# hi*hi + hi*lo + lo*hi) or "tf32" (ONE round-to-nearest tf32 pass, fp32 accumulation: about 1e-3
# relative error per product).  "tf32" sets descriptor flags bit7 on exactly these variants.
PRECISIONS = ("3xtf32", "tf32")
FLAG_TF32_ONE_PASS = 128
TF32_VARIANTS = (VAR_DMMA_128x64, VAR_DMMA_64x128, VAR_DMMA_256x32, VAR_DMMA_256x16, VAR_TF32_32x32) + TC05_VARIANTS

# where the slices of a tree are summed: "native" (the plan dtype) or "double" (float64 / complex128
# for float32 / complex64 trees; the same as "native" for the double dtypes).  A "double" plan sets
# descriptor flags bit8, "C is the wide type", on its dot-stream root and on nothing else.
ACCUMULATORS = ("native", "double")
FLAG_WIDE_C = 256
WIDE_DTYPES = {"float32": "float64", "complex64": "complex128"}
DOTSTREAM_VARIANTS = (VAR_DOTSTREAM, VAR_DOTSTREAM4)

DTYPE_CODES = {"float32": 0, "float64": 1, "complex64": 2, "complex128": 3}
DTYPE_SIZES = {"float32": 4, "float64": 8, "complex64": 8, "complex128": 16}


def dtype_name(dtype) -> str:
    if isinstance(dtype, str):
        name = dtype
    elif str(dtype).startswith("torch."):
        name = str(dtype)[len("torch."):]
    else:
        name = str(np.dtype(dtype))
    if name not in DTYPE_CODES:
        raise TypeError(f"unsupported dtype {dtype!r}")
    return name


def check_precision(precision, dtype=None):
    """``precision`` if it is one of ``PRECISIONS`` (and, with ``dtype``, one that dtype has), else
    ``ValueError``: there is no TF32 path for float64 / complex128."""
    if not isinstance(precision, str) or precision not in PRECISIONS:
        raise ValueError(f"precision must be one of {PRECISIONS}, got {precision!r}")
    if precision == "tf32" and dtype is not None and dtype_name(dtype) in ("float64", "complex128"):
        raise ValueError(f"precision='tf32' applies to float32 and complex64, not {dtype_name(dtype)}")
    return precision


def check_accumulate(accumulate):
    """``accumulate`` if it is one of ``ACCUMULATORS``, else ``ValueError``."""
    if not isinstance(accumulate, str) or accumulate not in ACCUMULATORS:
        raise ValueError(f"accumulate must be one of {ACCUMULATORS}, got {accumulate!r}")
    return accumulate


def accumulator_dtype(dtype, accumulate="native"):
    """The dtype a tree of ``dtype`` sums its slices in, and returns, under ``accumulate``."""
    dtype = dtype_name(dtype)
    return WIDE_DTYPES.get(dtype, dtype) if check_accumulate(accumulate) == "double" else dtype


def row_major_strides(shape):
    strides, acc = [0] * len(shape), 1
    for i in range(len(shape) - 1, -1, -1):
        strides[i] = acc
        acc *= int(shape[i])
    return strides


# ---------------------------------------------------------------------------
# classification
# ---------------------------------------------------------------------------


@dataclass
class PairDims:
    """Index classes of one pairwise node; every dim is ``[ext, sA, sB, sC]``
    (strides in elements, 0 where the operand does not carry the index)."""

    batch: list = field(default_factory=list)
    m: list = field(default_factory=list)
    n: list = field(default_factory=list)
    k: list = field(default_factory=list)
    out_shape: tuple = ()

    def sizes(self):
        pr = lambda ds: math.prod(d[0] for d in ds)  # noqa: E731
        return pr(self.batch), pr(self.m), pr(self.n), pr(self.k)


def classify_pair(term_a, shape_a, term_b, shape_b, out, out_strides=None,
                  strides_a=None, strides_b=None):
    """Classify the indices of ``term_a,term_b->out``.

    ``term_*`` / ``out`` are sequences of hashable labels.  Raises the same
    ``ValueError`` conditions as contract.py:183-186, 200-204, 218-222.
    """
    term_a, term_b, out = tuple(term_a), tuple(term_b), tuple(out)
    shape_a, shape_b = tuple(map(int, shape_a)), tuple(map(int, shape_b))
    if len(term_a) != len(shape_a):
        raise ValueError(f"Term '{term_a}' does not match shape {shape_a}.")
    if len(term_b) != len(shape_b):
        raise ValueError(f"Term '{term_b}' does not match shape {shape_b}.")
    sa = row_major_strides(shape_a) if strides_a is None else list(strides_a)
    sb = row_major_strides(shape_b) if strides_b is None else list(strides_b)

    ext, st_a, st_b = {}, {}, {}
    order = []
    for term, shape, strides, acc in ((term_a, shape_a, sa, st_a),
                                      (term_b, shape_b, sb, st_b)):
        for ix, d, s in zip(term, shape, strides):
            if ix not in ext and ix not in order:
                order.append(ix)
            if d == 1:
                continue
            if ext.setdefault(ix, d) != d:
                raise ValueError(
                    f"Index {ix} has mismatched sizes {ext[ix]} and {d}."
                )
            acc[ix] = acc.get(ix, 0) + s
    for ix in out:
        if ix not in order:
            raise ValueError(f"Output index {ix} does not appear in the inputs.")

    out_shape = tuple(ext.get(ix, 1) for ix in out)
    sc_list = row_major_strides(out_shape) if out_strides is None else list(out_strides)
    st_c = {}
    for ix, s in zip(out, sc_list):
        st_c[ix] = st_c.get(ix, 0) + s

    dims = PairDims(out_shape=out_shape)
    for ix in order:
        if ix not in ext:
            continue  # extent 1 everywhere: no loop at all
        rec = [ext[ix], st_a.get(ix, 0), st_b.get(ix, 0), st_c.get(ix, 0)]
        on_a, on_b = ix in st_a, ix in st_b
        if ix in st_c:
            if on_a and on_b:
                dims.batch.append(rec)
            elif on_a:
                dims.m.append(rec)
            else:
                dims.n.append(rec)
        else:
            dims.k.append(rec)
    return dims


def tensordot_terms(axes, ndim_a, ndim_b, perm=None):
    """Integer labels equivalent to ``tensordot(a, b, axes)`` followed by
    ``transpose(perm)`` (contract.py:472-518 builds the same equation out of
    characters; contract.py:811-812 applies the permutation)."""
    ax_a, ax_b = axes
    if len(ax_a) != len(ax_b):
        raise ValueError(
            f"Axes should have the same length, got {ax_a} and {ax_b}."
        )
    term_a = list(range(ndim_a))
    term_b, out = [], list(term_a)
    nxt = ndim_a
    for j in range(ndim_b):
        if j in ax_b:
            ix = term_a[ax_a[ax_b.index(j)]]
            out.remove(ix)
        else:
            ix = nxt
            nxt += 1
            out.append(ix)
        term_b.append(ix)
    if perm is not None:
        out = [out[p] for p in perm]
    return term_a, term_b, out


def check_tensordot_shapes(axes, shape_a, shape_b):
    for i, j in zip(*axes):
        if shape_a[i] != shape_b[j]:
            raise ValueError(
                f"Dimension mismatch between axes {i} of {tuple(shape_a)} and "
                f"{j} of {tuple(shape_b)}: {shape_a[i]} != {shape_b[j]}."
            )


# ---------------------------------------------------------------------------
# coalescing and tiling
# ---------------------------------------------------------------------------


def coalesce(dims):
    """Merge dims that are adjacent (outer stride == inner stride * inner
    extent) in *every* operand: a rank-30 all-dims-2 Sycamore tensor drops to a
    handful of super-dims (SURVEY.md Appx D.5)."""
    dims = [list(d) for d in dims if d[0] != 1]
    changed = True
    while changed:
        changed = False
        for i in range(len(dims)):
            for j in range(len(dims)):
                if i == j:
                    continue
                inner, outer = dims[i], dims[j]
                if all(outer[t] == inner[t] * inner[0] for t in range(1, len(inner))):
                    inner[0] *= outer[0]
                    del dims[j]
                    changed = True
                    break
            if changed:
                break
    return dims


def _min_stride(d, cols):
    vals = [abs(d[c]) for c in cols if d[c] != 0]
    return min(vals) if vals else 0


def _largest_divisor(n, cap, prod=1, multiple=1):
    """Largest divisor t of n, 2 <= t <= cap, with prod * t a multiple of ``multiple`` (1 if none)."""
    for t in range(min(n, cap), 1, -1):
        if n % t == 0 and (prod * t) % multiple == 0:
            return t
    return 1


def split_tile(dims, cols, limit, order_col, exact=False, multiple=1):
    """Pick the tile dims of one class.

    Greedy by smallest stride in any operand carrying the dim (those are the
    dims whose inclusion makes global accesses contiguous); at most one dim is
    taken partially (blocked).  Returns ``(tile, grid, partial)`` with

      tile : [[text, *strides]]           local order, partial dim last
      grid : [[count, *strides_per_step]] remaining loops (block dim included)
      partial : (grid_index, full_ext, text, weight) or None

    ``exact``: the blocked dim is cut into equal blocks (the largest divisor of its extent
    that fits), so that every tile has the same shape -- for kernels without ragged tiles;
    ``multiple``: ... among the divisors that make the tile's extent a multiple of this (the k of a
    wgmma tile is whole wgmma k8 groups of complex numbers: 4).
    """
    cand = sorted(range(len(dims)), key=lambda i: (_min_stride(dims[i], cols), i))
    tile, used, prod, partial_src = [], set(), 1, None
    for i in cand:
        e = dims[i][0]
        if len(tile) >= MAX_T - 1:
            break
        if prod * e <= limit:
            tile.append(list(dims[i]))
            used.add(i)
            prod *= e
        else:
            t = limit // prod
            if exact:
                t = _largest_divisor(e, t, prod, multiple)
            if t >= 2:
                rec = list(dims[i])
                rec[0] = t
                partial_src = (i, rec)
                used.add(i)
                prod *= t
            break
    tile.sort(key=lambda d: (abs(d[order_col]) if d[order_col] else 1 << 62))
    grid = [list(dims[i]) for i in range(len(dims)) if i not in used]
    partial = None
    if partial_src is not None:
        i, rec = partial_src
        full, t = dims[i][0], rec[0]
        weight = math.prod(d[0] for d in tile)
        tile.append(rec)
        blocks = -(-full // t)
        grid.append([blocks] + [s * t for s in dims[i][1:]])
        partial = [len(grid) - 1, full, t, weight]
    return tile, grid, partial


def _order_grid(grid, partial, key_col):
    """Fastest-varying grid dim first = smallest stride of the streamed operand
    (consecutive tiles touch neighbouring memory)."""
    idx = sorted(range(len(grid)),
                 key=lambda i: (abs(grid[i][key_col]) if grid[i][key_col] else 1 << 62, i))
    new = [grid[i] for i in idx]
    if partial is not None:
        partial = [idx.index(partial[0])] + partial[1:]
    return new, partial


def _with_divs(grid):
    out, div = [], 1
    for g in grid:
        out.append([g[0], div] + list(g[1:]))
        div *= g[0]
    return out, div


@dataclass
class PairPlan:
    words: np.ndarray
    variant: int
    sizes: tuple  # (B, M, N, K)
    swapped: bool
    tiles: int
    splitk: int


def choose_variant(dtype, B, M, N, K, allow_dmma=True, allow_stream=True, allow_tc05=True, allow_3m=False):
    if M == 1 and N == 1 and B == 1 and K >= 1 << 20 and allow_stream:
        return VAR_DOTSTREAM
    if M <= 4 and N <= 4 and B == 1 and K >= 1 << 20 and allow_stream:
        return VAR_DOTSTREAM4  # a stem tail peeled over the final inner product (fusion.py)
    if (dtype in ("complex128", "float64") and allow_dmma and M <= 32 and N <= 32 and M * N >= 4 and B == 1
            and K >= 1 << 14):
        # the same with a few more peeled tensors (fusion.py): ONE 32 x 32 fp64 tensor-core tile,
        # the contracted range split over two CTAs per SM
        return VAR_DMMA_32x32
    if M == 1 and N == 1 and B == 1 and K >= 8192:
        return VAR_KRED
    if N <= 8 and K <= 8 and B == 1 and 64 <= M < 1 << 32 and allow_stream:
        return VAR_ROWSTREAM
    # narrow complex128 nodes: DMMA fragments streamed from global memory, no staging
    # (N <= 8 with a contracted space too long for the row-stream kernel included)
    if (allow_dmma and allow_stream and dtype == "complex128" and B == 1 and 4096 <= M < 1 << 32
            and N <= DMMASTREAM_MAX_N and K <= DMMASTREAM_KMAX):
        return VAR_DMMASTREAM
    # ... and the narrower element types: the row stream walked in chunks of 8 k
    if (allow_stream and DTYPE_SIZES[dtype] <= 8 and N <= 8 and 8 < K <= 64 and B == 1
            and 4096 <= M < 1 << 32):
        return VAR_ROWSTREAM_K
    if N <= 8 and M >= 64:
        return VAR_ROW_256x4 if N <= 4 else VAR_ROW_128x8
    # complex64 dense nodes with exact power-of-two tiles: wgmma (tf32 x3, register accumulators)
    # (K > 256 runs in chunks of 256 inside the kernel: every chunk accumulates from zero
    # and the epilogue folds it into C with round-to-nearest adds -- the tensor core's own
    # accumulation truncates, which is why a single accumulation stops at K = 256)
    if (allow_dmma and allow_tc05 and dtype == "complex64" and M >= 128 and K >= 4 and N >= 12
            and K <= TC05_MAX_K and M * N * K >= 1 << 20):
        # (extents need not be powers of two: build_pair_desc cuts every class into EQUAL tiles by
        # divisors -- 108 x 54 x 12 for the bond-6 PEPS GEMMs -- and falls back to the mma.sync
        # policy when that leaves the tensor-core tile too empty)
        if N >= 48:
            return VAR_TC05_128x64
        if N >= 24:
            return VAR_TC05_128x32
        return VAR_TC05_128x16
    # tensor-core tiles: fp64 DMMA for float64/complex128, 3xTF32 for float32/complex64
    if allow_dmma and M * N * K >= 1 << 15 and M * N >= 1024:
        if dtype == "complex128" and allow_3m and N >= 64 and K >= 64:
            # 3M complex product (opt-in): 25 % fewer DMMAs but narrower tiles (accumulator
            # registers): faster on long k, slower on short k (per-tile epilogue dominates) and no
            # gain on the whole Sycamore slice, so the default stays the 4-DMMA product.
            return VAR_DMMA3M_128x32
        if N >= 96:
            return VAR_DMMA_64x128
        if N >= 48:
            return VAR_DMMA_128x64
        if N >= 24:
            return VAR_DMMA_256x32
        return VAR_DMMA_256x16
    return VAR_SIMT_64x64


# a blocked dim (split_tile's ``partial``), if any, is cut into whole blocks
_whole = lambda partial: partial is None or partial[1] % partial[2] == 0  # noqa: E731
# what the hand-over rules read of a node besides its tiling (sizes after the swap)
_Node = namedtuple("_Node", "dtype B M N K allow_dmma accumulate c_dense_elems")
# one variant's split of a node: tile dims, grid dims (with their divisors), the blocked dim of each class
# (split_tile's ``partial``), the tile's extents, the tile dims' local weights and the operand load orders
_Tiling = namedtuple("_Tiling", "variant tm tn tk gm gn gk gb pm pn pk tiles_m tiles_n tiles_b tiles steps_k "
                                "MTa NTa KTa wm wn wk lda ldb")
# How a specialised variant is admitted, and what runs when it is not: ``fits(node)`` is checked on dtype
# and sizes before tiling (``unfit(node)`` runs if it fails), ``admits(node, tiling)`` on the variant's
# finished tiling (``to(node)`` runs if it fails).  Variants without an entry in HANDOVER take any node.
Handover = namedtuple("Handover", "fits unfit admits to", defaults=(lambda nd: True, None, lambda nd, t: True, None))


_row_tile = lambda nd: VAR_ROW_256x4 if nd.N <= 4 else VAR_ROW_128x8  # noqa: E731


def _rowstream_k_admits(nd, t):
    # exact tiles, and the k offsets must decompose as chunk_base[k // 8] + in_chunk[k % 8]
    koff = lambda e: sum((e // w) % d[0] * d[1] for d, w in zip(t.tk, t.wk))  # noqa: E731
    return (t.pn is None and t.pk is None and _whole(t.pm) and DTYPE_SIZES[nd.dtype] <= 8 and nd.N <= 8
            and nd.K <= 64 and nd.B == 1 and nd.M < 1 << 32
            and all(koff(e) == koff(e - e % 8) + koff(e % 8) for e in range(t.KTa)))


def _tc05_admits(nd, t):
    # the wgmma kernel takes tiles of ONE shape: its native 128 x NT x 16, or smaller with
    # the rest of the tensor-core tile as padding (KTa in steps of 4: whole wgmma k8 groups);
    # below 40 % occupancy the mma.sync policy is the better choice
    # (k padding is free -- the wgmmas of missing k8 groups are not issued -- so only rows and columns count)
    MT, NT, KT = VARIANT_TILES[t.variant]
    return (t.MTa <= MT and t.NTa <= NT and t.KTa <= KT and t.KTa % 4 == 0 and nd.dtype == "complex64"
            and (t.MTa * t.NTa) / float(MT * NT) >= 0.4 and t.steps_k <= 1024
            and (t.KTa >= 8 or t.steps_k == 1)  # many 4-wide k-steps: per-step overhead, mma.sync is better
            and _whole(t.pm) and _whole(t.pn) and _whole(t.pk))


HANDOVER = {
    # a ragged blocked m dim: the staged row policy
    VAR_ROWSTREAM: Handover(fits=lambda nd: nd.N <= 8 and nd.K <= 8 and nd.B == 1 and nd.M < 1 << 32,
                            unfit=_row_tile, admits=lambda nd, t: _whole(t.pm), to=_row_tile),
    VAR_ROWSTREAM_K: Handover(admits=_rowstream_k_admits, to=_row_tile),
    # ragged, or more dims than one tile holds: the staged tile choose_variant picks without the
    # stream kernel (N <= 16: 256x16, as before N = 17..32 streamed)
    VAR_DMMASTREAM: Handover(
        fits=lambda nd: nd.dtype == "complex128" and dmmastream_fits(nd.N, nd.K) and nd.B == 1 and nd.M < 1 << 32,
        unfit=lambda nd: VAR_DMMA_256x16,
        admits=lambda nd, t: t.pn is None and t.pk is None and _whole(t.pm) and t.tiles_n == 1 and t.steps_k == 1,
        to=lambda nd: (VAR_DMMA_256x16 if nd.N <= 16 else
                       choose_variant(nd.dtype, nd.B, nd.M, nd.N, nd.K, nd.allow_dmma, allow_stream=False))),
    VAR_DOTSTREAM: Handover(
        admits=lambda nd, t: nd.M == 1 and nd.N == 1 and nd.B == 1 and t.steps_k < 1 << 31 and _whole(t.pk),
        to=lambda nd: VAR_KRED),
    VAR_DOTSTREAM4: Handover(
        admits=lambda nd, t: (nd.M <= 4 and nd.N <= 4 and nd.B == 1 and t.steps_k < 1 << 31
                              and t.pm is None and t.pn is None and _whole(t.pk)
                              and (nd.accumulate or nd.c_dense_elems == nd.M * nd.N)),
        to=lambda nd: VAR_SIMT_64x64),
    **{v: Handover(admits=_tc05_admits,
                   to=lambda nd: choose_variant(nd.dtype, nd.B, nd.M, nd.N, nd.K, nd.allow_dmma, allow_tc05=False))
       for v in TC05_VARIANTS},
    # the same tile on the fp64 tensor cores
    VAR_TF32_32x32: Handover(fits=lambda nd: nd.dtype not in ("float64", "complex128"),
                             unfit=lambda nd: VAR_DMMA_32x32),
    # the 3M identity is a complex128 kernel: other dtypes take the plain tensor-core tiles
    VAR_DMMA3M_128x32: Handover(fits=lambda nd: nd.dtype == "complex128", unfit=lambda nd: VAR_DMMA_256x32),
    VAR_DMMA3M_256x16: Handover(fits=lambda nd: nd.dtype == "complex128", unfit=lambda nd: VAR_DMMA_256x16),
}
STAGED = Handover()


def build_pair_desc(dims: PairDims, dtype, accumulate=False, sm_count=132,
                    variant=None, allow_dmma=True, c_dense_elems=0,
                    force_splitk=None, precision="3xtf32", wide_c=False) -> PairPlan:
    """Pack a classified node into descriptor words.  ``variant`` (default: ``choose_variant``'s pick)
    is the kernel to run; a specialised one the node does not suit hands over as ``HANDOVER`` says.
    ``precision`` (``PRECISIONS``) selects the compute mode of the float32 / complex64 tensor-core
    variants; it changes no other word.  ``wide_c`` sets flags bit8 (C has ``WIDE_DTYPES[dtype]`` and
    the kernel sums in it): only the dot-stream kernels have it, so a node that lowers to any other
    variant raises ``ValueError``."""
    dtype = dtype_name(dtype)
    check_precision(precision, dtype)
    if wide_c and dtype not in WIDE_DTYPES:
        raise ValueError(f"a wide C applies to float32 and complex64, not {dtype}")
    m = coalesce([[d[0], d[1], d[3]] for d in dims.m])          # ext, sA, sC
    n = coalesce([[d[0], d[2], d[3]] for d in dims.n])          # ext, sB, sC
    k = coalesce([[d[0], d[1], d[2]] for d in dims.k])          # ext, sA, sB
    b = coalesce([list(d) for d in dims.batch])                 # ext, sA, sB, sC
    B, M, N, K = dims.sizes()

    # the streamed (large) operand is "A": swap roles when B's kept space is larger
    swapped = N > M
    if swapped:
        m, n = n, m
        k = [[d[0], d[2], d[1]] for d in k]
        b = [[d[0], d[2], d[1], d[3]] for d in b]
        M, N = N, M

    nd = _Node(dtype, B, M, N, K, allow_dmma, accumulate, c_dense_elems)
    if variant is None:
        variant = choose_variant(dtype, B, M, N, K, allow_dmma)
    while True:
        h = HANDOVER.get(variant, STAGED)
        if not h.fits(nd):
            variant = h.unfit(nd)
            continue
        if wide_c and variant not in DOTSTREAM_VARIANTS:
            raise ValueError(f"a wide C needs a dot-stream node, this one lowers to variant {variant}")
        t = _tile(variant, dtype, m, n, k, b)
        splitk = _splitk(t, sm_count, force_splitk)  # (a node of 2^31 tiles raises before it hands over)
        if h.admits(nd, t):
            break
        variant = h.to(nd)

    run_a, bulk_a, lbopad = _wgmma_words(t) if variant in TC05_VARIANTS else (1, False, 0)
    flags = ((1 if accumulate else 0) | _layout_flags(dtype, t) | (64 if bulk_a else 0)
             | (FLAG_TF32_ONE_PASS if precision == "tf32" and variant in TF32_VARIANTS else 0)
             | (FLAG_WIDE_C if wide_c else 0))
    words = _pack(dtype, t, splitk, flags, run_a, lbopad, c_dense_elems)
    return PairPlan(words, variant, (B, M, N, K), swapped, t.tiles, splitk)


def _tile(variant, dtype, m, n, k, b):
    """Split the coalesced classes into the tile and grid dims of ``variant``."""
    MT, NT, KT = VARIANT_TILES[variant]
    if variant == VAR_DOTSTREAM4 and DTYPE_SIZES[dtype] < 16:
        KT = 2048  # 8 k per thread for the narrower element types (csrc/dotstream.cuh dot4_u)
    if variant in TC05_VARIANTS:
        # wgmma: the epilogue addresses every row through its own offset, so the rows of a tile need
        # not be neighbours in C -- pick them for the longest contiguous runs of A instead
        # (and B is re-packed by bprime_kernel anyway: only A's strides matter for k too)
        tm, gm, pm = split_tile(m, (1,), MT, order_col=1, exact=True)
        tk, gk, pk = split_tile(k, (1,), KT, order_col=1, exact=True, multiple=4)
        tn, gn, pn = split_tile(n, (1, 2), NT, order_col=2, exact=True)
    else:
        tm, gm, pm = split_tile(m, (1, 2), MT, order_col=2)
        tk, gk, pk = split_tile(k, (1, 2), KT, order_col=1)
        tn, gn, pn = split_tile(n, (1, 2), NT, order_col=2)
    gm, pm = _order_grid(gm, pm, 1)
    gn, pn = _order_grid(gn, pn, 1)
    gk, pk = _order_grid(gk, pk, 1)
    gb = list(b)
    for name, lst, cap in (("m", gm, MAX_G), ("n", gn, MAX_G), ("k", gk, MAX_G), ("batch", gb, MAX_GB)):
        if len(lst) > cap:
            raise NotImplementedError(f"{len(lst)} non-coalescable {name} dims exceed the descriptor capacity {cap}")
    (gm, tiles_m), (gn, tiles_n), (gk, steps_k), (gb, tiles_b) = map(_with_divs, (gm, gn, gk, gb))

    # local weights (dim 0 fastest; partial dim is last by construction)
    (wm, MTa), (wn, NTa), (wk, KTa) = (_weights(ts) for ts in (tm, tn, tk))
    # operand load orders: ascending stride in that operand (coalesced gathers)
    lda = [[d[0], d[1], w, 0] for d, w in zip(tm, wm)] + [[d[0], d[1], 0, w] for d, w in zip(tk, wk)]
    ldb = [[d[0], d[2], w, 0] for d, w in zip(tk, wk)] + [[d[0], d[1], 0, w] for d, w in zip(tn, wn)]
    key = lambda r: (abs(r[1]) if r[1] else 1 << 62)  # noqa: E731
    lda.sort(key=key)
    ldb.sort(key=key)
    return _Tiling(variant, tm, tn, tk, gm, gn, gk, gb, pm, pn, pk, tiles_m, tiles_n, tiles_b, tiles_m * tiles_n * tiles_b,
                   steps_k, MTa, NTa, KTa, wm, wn, wk, lda, ldb)


def _weights(tile):
    """The local weight of every tile dim (the product of the extents before it), and the tile's size."""
    w, acc = [], 1
    for d in tile:
        w.append(acc)
        acc *= d[0]
    return w, acc


def _splitk(t, sm_count, force_splitk):
    if force_splitk is not None:
        splitk = max(1, min(int(force_splitk), t.steps_k))
    else:
        splitk = 1
        if t.tiles < sm_count and t.steps_k >= 4:
            splitk = min(t.steps_k, -(-2 * sm_count // t.tiles))
        if t.variant == VAR_KRED:
            splitk = min(t.steps_k, 4 * sm_count)
        if t.variant in (VAR_DMMA_32x32, VAR_TF32_32x32) and t.tiles == 1:
            splitk = min(t.steps_k, 2 * sm_count)  # two resident CTAs per SM
    if splitk > 1:
        per = -(-t.steps_k // splitk)
        splitk = -(-t.steps_k // per)
    if t.tiles * splitk >= 1 << 31:
        raise NotImplementedError("node needs more than 2^31 tiles")
    return splitk


def _layout_flags(dtype, t):
    """Flags bits 1-5: what the tiling's layout lets the kernels assume."""
    # bit1: columns (2q, 2q+1) of every tile row are adjacent in C and 32-byte
    # aligned -> the kernels may use 256-bit stores (complex128 only)
    dense_n = all(d[2] == w for d, w in zip(t.tn, t.wn))
    # (tile rows and the grid steps of m, n and batch move C by multiples of g elements)
    aligned = lambda g: (all(d[2] % g == 0 for d in t.tm) and all(x[3] % g == 0 for x in t.gm + t.gn)  # noqa: E731
                         and all(x[4] % g == 0 for x in t.gb))
    pair_ok = dtype == "complex128" and dense_n and t.pn is None and t.NTa >= 2 and t.NTa % 2 == 0 and aligned(2)
    # bit2: all tile-grid extents are powers of two (Sycamore: always) -> the
    # producers decode tile indices with shifts/masks instead of idiv
    is_p2 = lambda e: e > 0 and (e & (e - 1)) == 0  # noqa: E731
    grid_pow2 = all(is_p2(g[0]) for g in t.gm + t.gn + t.gb)
    m_pow2 = all(is_p2(d[0]) for d in t.tm) and all(is_p2(g[0]) for g in t.gm)

    # 8-byte element types: groups of 4 (bit4) / 2 (bit5) columns adjacent in C and
    # 32- / 16-byte aligned -> vector row stores in the streaming row kernel
    def cols_ok(g):
        if t.variant in TC05_VARIANTS:
            # exact tiles: only the leading columns of a tile row have to be adjacent
            run = next((w for d, w in zip(t.tn, t.wn) if d[2] != w), t.NTa)
            dense = run % g == 0
        else:
            dense = dense_n and t.pn is None
        return DTYPE_SIZES[dtype] == 8 and dense and t.NTa % g == 0 and aligned(g)

    return (2 if pair_ok else 0) | (4 if grid_pow2 else 0) | (8 if m_pow2 else 0) | (16 if cols_ok(4) else 0) \
        | (32 if cols_ok(2) else 0)


def _wgmma_words(t):
    """``(RUNA, bit6, LBOPAD)`` of a wgmma node."""
    # if the A tile is made of long contiguous runs (dense prefix of the load order),
    # the producers fetch whole runs with TMA bulk copies (bit6)
    run_a = 1
    for r_ in t.lda:
        if r_[1] != run_a:
            break
        run_a *= r_[0]
    rest = [r_[1] for r_ in t.lda if r_[1] >= run_a] + [g[2] for g in t.gm + t.gk + t.gb]
    # (cp.async.bulk: 16-byte aligned source, size a multiple of 16 bytes; one run per
    # producer thread -> at most 128 runs of >= 128 bytes)
    bulk_a = (run_a >= 16 and run_a % 2 == 0 and (t.MTa * t.KTa) % run_a == 0
              and all(x % 2 == 0 for x in rest))
    # chunk-stride padding of the A' images (x16 B): 16 consecutive elements of A's memory
    # order -- the lanes of a half warp in the scatter pass -- should hit 16 different
    # 8-byte bank pairs.  Element (r, kk) sits at (kk//2)*LBO + r*16 + (kk%2)*8 bytes.
    pos = []
    for x in range(32):
        r_ = kk_ = 0
        for ext, _s, wr, wk_ in t.lda:
            r_, kk_, x = r_ + (x % ext) * wr, kk_ + (x % ext) * wk_, x // ext
        pos.append((r_, kk_))

    def conflicts(pad):
        lbo = VARIANT_TILES[t.variant][0] * 16 + 16 * pad
        slots = [(((kk_ // 2) * lbo + r_ * 16 + (kk_ % 2) * 8) >> 3) & 15 for r_, kk_ in pos]
        return sum(max(Counter(slots[h:h + 16]).values()) for h in (0, 16))
    return run_a, bulk_a, min((0, 1, 2, 4), key=conflicts)


def _pack(dtype, t, splitk, flags, run_a, lbopad, c_dense_elems):
    W = np.zeros(DESC_WORDS, dtype=np.int64)
    W[W_MAGIC] = DESC_MAGIC
    W[W_DTYPE] = DTYPE_CODES[dtype]
    W[W_NTM], W[W_NTN], W[W_NTK] = len(t.tm), len(t.tn), len(t.tk)
    W[W_NGM], W[W_NGN], W[W_NGK], W[W_NGB] = len(t.gm), len(t.gn), len(t.gk), len(t.gb)
    W[W_MTA], W[W_NTA], W[W_KTA] = t.MTa, t.NTa, t.KTa
    W[W_TILES_M], W[W_TILES_N], W[W_TILES_B], W[W_STEPS_K] = t.tiles_m, t.tiles_n, t.tiles_b, t.steps_k
    W[W_SPLITK] = splitk
    for base, p in ((W_PGM, t.pm), (W_PGN, t.pn), (W_PGK, t.pk)):
        W[base:base + 4] = (-1, 0, 0, 0) if p is None else p
    W[W_NLDA], W[W_NLDB] = len(t.lda), len(t.ldb)
    W[W_FLAGS], W[W_VARIANT], W[W_CELEMS], W[W_RUNA], W[W_LBOPAD] = flags, t.variant, int(c_dense_elems), run_a, lbopad
    for off, rows, width in ((OFF_TM, t.tm, 3), (OFF_TN, t.tn, 3), (OFF_TK, t.tk, 3), (OFF_GM, t.gm, 4),
                             (OFF_GN, t.gn, 4), (OFF_GK, t.gk, 4), (OFF_GB, t.gb, 5), (OFF_LDA, t.lda, 4),
                             (OFF_LDB, t.ldb, 4)):
        for i, r in enumerate(rows):
            W[off + i * width: off + (i + 1) * width] = r
    return W


# ---------------------------------------------------------------------------
# single-operand nodes  (contract.py:61-119, 332-361)
# ---------------------------------------------------------------------------


# ---------------------------------------------------------------------------
# absorb-root nodes (csrc/absorbdot.cuh; word layout in csrc/gett_desc.h)
# ---------------------------------------------------------------------------
AB_M, AB_N, AB_K, AB_C, AB_KL, AB_NG, AB_UNITS, AB_KLA, AB_KLV, AB_GRID, AB_BS_SLOT, AB_CCP = range(2, 14)
AB_MAXG = 32
AB_TMA = W_HDR
AB_TMC, AB_TNV, AB_TNC = AB_TMA + 32, AB_TMA + 64, AB_TMA + 96
AB_TKA = AB_TMA + 128
AB_TKB = AB_TKA + 16
AB_TCB = AB_TKB + 16
AB_TCV = AB_TCB + 128
AB_G = AB_TCV + 128
AB_TBCK = AB_G + AB_MAXG * 4


@dataclass
class AbsorbPlan:
    """An absorb-root node: ``words`` and what the executor needs to wire its operands.
    ``small_is_a``: the absorption's small operand is its term A (else B)."""

    words: np.ndarray
    small_is_a: bool
    sizes: tuple
    macs: int
    variant: int = VAR_ABSORB_ROOT
    swapped: bool = False
    splitk: int = 1
    tiles: int = 1


def _enum(dims, cols):
    """Offsets (one list per column of ``cols``) of every point of ``dims`` (first dim fastest)."""
    out = [[0] for _ in cols]
    for d in dims:
        out = [[o + i * d[c] for i in range(d[0]) for o in lst] for lst, c in zip(out, cols)]
    return out


def build_absorb_desc(dp: PairDims, dr: PairDims, x_is_a, accumulate=False, sm_count=132, c_dense_elems=0):
    """Fold the absorption ``X = P`` (dims ``dp``) into the product ``R`` that reads it (dims ``dr``;
    X is R's operand A if ``x_is_a``), or None when the absorb-root kernel does not take the pair.
    One side of P is the small operand Bs: its kept dims are each contracted in R (cc) or kept by R
    (ck); the other side's kept dims are kept by R (rows) or contracted (k').  The kernel takes
    N <= 32, K <= 16, 32 * ceil(CC / 32) * CK <= 128 and either CK = 1 with up to 32 rows or CK <= 4
    with up to 8; no batch, and the dims of P and R must match one to one by their X stride."""
    if dp.batch or dr.batch:
        return None
    xi = 1 if x_is_a else 2  # X's stride column in R's dims
    vi = 3 - xi
    r_keep = {d[xi]: (d[0], d[3]) for d in (dr.m if x_is_a else dr.n)}  # X stride -> (ext, sC)
    v_keep = [[d[0], d[vi], d[3]] for d in (dr.n if x_is_a else dr.m)]
    r_con = {d[xi]: (d[0], d[vi]) for d in dr.k}  # X stride -> (ext, sV)
    if len(r_con) != len(dr.k) or len(r_keep) != len(dr.m if x_is_a else dr.n):
        return None
    for small_is_a in (False, True):
        small = dp.m if small_is_a else dp.n   # [ext, sA, sB, sC]: P's side of Bs
        big = dp.n if small_is_a else dp.m
        bi, si = (2, 1) if small_is_a else (1, 2)  # columns of the big and the small operand in P
        xdims = {d[3]: d for d in small + big}
        if not small or len(xdims) != len(small) + len(big) or set(xdims) != set(r_keep) | set(r_con):
            continue
        if any(xdims[x][0] != (r_keep.get(x) or r_con[x])[0] for x in xdims):
            continue
        small_x = {d[3] for d in small}
        rows = [[d[0], d[bi], r_keep[d[3]][1]] for d in big if d[3] in r_keep]
        ck = [[d[0], d[si], r_keep[d[3]][1]] for d in small if d[3] in r_keep]
        cc = sorted(([d[0], d[si], r_con[d[3]][1]] for d in small if d[3] in r_con), key=lambda d: d[2])
        kprime = [[d[0], d[bi], r_con[d[3]][1]] for d in big if d[3] in r_con]
        MX, CK = math.prod(d[0] for d in rows), math.prod(d[0] for d in ck)
        N, K, CC = math.prod(d[0] for d in v_keep), math.prod(d[0] for d in dp.k), math.prod(d[0] for d in cc)
        CCP = -(-CC // 32) * 32
        rows_per = 8 if CK > 1 else 32
        if MX > rows_per or CK * rows_per > 32 or N > 32 or K > 16 or CK * CCP > 128 or not small_x:
            return None
        kl = min(kprime, key=lambda d: d[2], default=None)
        if kl is not None and kl[0] == 2:
            kprime.remove(kl)
        else:
            kl = [1, 0, 0]
        grid = sorted(kprime, key=lambda d: (d[1], d[2]))  # unit u + 1 reads the other half of A's sectors
        if len(grid) > AB_MAXG:
            return None
        units = math.prod(d[0] for d in grid)
        w = np.zeros(DESC_WORDS, dtype=np.int64)
        w[0], w[1] = DESC_MAGIC, DTYPE_CODES["complex128"]
        w[AB_M], w[AB_N], w[AB_K], w[AB_C], w[AB_CCP], w[AB_KL] = CK * rows_per if CK > 1 else MX, N, K, CC, CCP, kl[0]
        w[AB_NG], w[AB_UNITS], w[AB_KLA], w[AB_KLV] = len(grid), units, kl[1], kl[2]
        w[AB_GRID] = min(units, sm_count)
        w[AB_BS_SLOT] = -1
        w[W_FLAGS] = int(bool(accumulate))
        w[W_VARIANT] = VAR_ABSORB_ROOT
        w[W_CELEMS] = c_dense_elems
        ra, rc = _enum(rows, (1, 2))
        ckb, ckc = _enum(ck, (1, 2))
        ma, mc = [-1] * 32, [-1] * 32
        for j, (ob, oc) in enumerate(zip(ckb, ckc)):
            for r, (a, c) in enumerate(zip(ra, rc)):
                ma[j * rows_per + r], mc[j * rows_per + r] = a, c + oc
        tbck = [min(mb * 8 // rows_per, CK - 1) for mb in range(4)]
        nv, nc = _enum(v_keep, (1, 2))
        ka, kb = _enum([[d[0], d[bi], d[si]] for d in dp.k], (1, 2))
        cb, cv = _enum(cc, (1, 2))
        tcb = [-1] * 128
        for j, ob in enumerate(ckb):
            tcb[j * CCP:j * CCP + CC] = [ob + o for o in cb]
        for off, vals in ((AB_TMA, ma), (AB_TMC, mc), (AB_TNV, nv), (AB_TNC, nc), (AB_TKA, ka), (AB_TKB, kb),
                          (AB_TCB, tcb), (AB_TCV, cv), (AB_TBCK, tbck)):
            w[off:off + len(vals)] = vals
        div = 1
        for j, (e, sa, sv) in enumerate(grid):
            w[AB_G + 4 * j:AB_G + 4 * j + 4] = (e, div, sa, sv)
            div *= e
        kp = units * kl[0]
        M = MX * CK
        return AbsorbPlan(w, small_is_a, (1, M, N, kp * CC), MX * kp * K * CC * CK + M * N * kp * CC)
    return None


def classify_single(term, shape, out, out_strides=None, strides_x=None):
    """``out[o] = sum_s X[...]``: output dims ``[ext, sX, sOut]`` and summed
    dims ``[ext, sX]``; repeated labels (diagonals/traces) add their strides."""
    term, out = tuple(term), tuple(out)
    shape = tuple(map(int, shape))
    if len(term) != len(shape):
        raise ValueError(f"Term '{term}' does not match shape {shape}.")
    sx = row_major_strides(shape) if strides_x is None else list(strides_x)
    ext, st_x, order = {}, {}, []
    for ix, d, s in zip(term, shape, sx):
        if ix not in order:
            order.append(ix)
        if ext.setdefault(ix, d) != d:
            raise ValueError(f"Index {ix} has mismatched sizes {ext[ix]} and {d}.")
        st_x[ix] = st_x.get(ix, 0) + s
    for ix in out:
        if ix not in ext:
            raise ValueError(f"Output index {ix} does not appear in the input.")
    out_shape = tuple(ext[ix] for ix in out)
    so = row_major_strides(out_shape) if out_strides is None else list(out_strides)
    odims = [[ext[ix], st_x[ix], s] for ix, s in zip(out, so) if ext[ix] != 1]
    sdims = [[ext[ix], st_x[ix]] for ix in order if ix not in out and ext[ix] != 1]
    return odims, sdims, out_shape


def build_single_desc(odims, sdims, dtype, accumulate=False) -> np.ndarray:
    dtype = dtype_name(dtype)
    odims = coalesce(odims)
    sdims = coalesce(sdims)
    # fastest output dim = smallest output stride (coalesced stores)
    odims.sort(key=lambda d: abs(d[2]) if d[2] else 1 << 62)
    sdims.sort(key=lambda d: abs(d[1]) if d[1] else 1 << 62)
    if len(odims) > MAX_S or len(sdims) > MAX_S:
        raise NotImplementedError("too many dims for a single-operand node")
    W = np.zeros(SDESC_WORDS, dtype=np.int64)
    W[S_MAGIC] = SDESC_MAGIC
    W[S_DTYPE] = DTYPE_CODES[dtype]
    W[S_NO], W[S_NS] = len(odims), len(sdims)
    W[S_OUT_ELEMS] = math.prod(d[0] for d in odims)
    W[S_SUM_ELEMS] = math.prod(d[0] for d in sdims)
    W[S_FLAGS] = 1 if accumulate else 0
    for i, d in enumerate(odims):
        W[OFF_SO + 3 * i: OFF_SO + 3 * i + 3] = d
    for i, d in enumerate(sdims):
        W[OFF_SS + 2 * i: OFF_SS + 2 * i + 2] = d
    return W


def split_equation(eq):
    """``(lhs_terms, out)`` of an explicit or implicit einsum equation
    (contract.py:34-58)."""
    eq = eq.replace(" ", "")
    if "..." in eq:
        raise NotImplementedError("Ellipsis not supported.")
    if "->" in eq:
        lhs, out = eq.split("->")
    else:
        lhs = eq
        flat = lhs.replace(",", "")
        out = "".join(c for c in sorted(set(flat)) if flat.count(c) == 1)
    return lhs.split(","), out
