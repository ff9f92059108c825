"""Special values and power-of-two scaling through every kernel.

The parity tests feed every kernel finite, well-scaled operands.  These tests put NaN (every
encoding that occurs in practice, as explicit bit patterns: a numpy NaN alone is 0x7FC00000 and
misses the encodings GPU arithmetic produces), +-inf, values at the ends of the float range and
power-of-two-rescaled operands through each kernel variant, and check:

* the dependency cone: a non-finite input element makes exactly the output elements that share its
  kept indices non-finite, and every other element is bitwise what a clean run of the same plan
  gives (a kernel that multiplies padding or garbage by zero, or drops a NaN, fails this);
* coverage: a non-accumulating launch into a NaN-filled C leaves no NaN behind;
* scaling by 2^j is exact in floating point, so every kernel must return 2^j x the unscaled
  result, bit for bit, while the values stay normal;
* whole trees: NaN positions match the numpy oracle, with and without strip_exponent, and the
  strip_exponent mantissa / exponent pair is right separately (max|m| == 1, e == log10 max|value|).
"""

import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from oracle import ctg_oracle as orc  # noqa: E402
from tests.helpers import load_json, make_arrays, rel_err, tree_spec  # noqa: E402

# bit patterns: quiet NaN as numpy makes it, the NaN GPU arithmetic makes (inf - inf, 0 * inf), the
# negative NaN, a signalling NaN, and +-inf
NAN32 = {"qnan": 0x7FC00000, "nan_ones": 0x7FFFFFFF, "nan_neg": 0xFFFFFFFF, "snan": 0x7F800001}
NAN64 = {"qnan": 0x7FF8000000000000, "nan_ones": 0x7FFFFFFFFFFFFFFF, "nan_neg": 0xFFFFFFFFFFFFFFFF,
         "snan": 0x7FF0000000000001}
INF32 = {"inf": 0x7F800000, "neg_inf": 0xFF800000}
INF64 = {"inf": 0x7FF0000000000000, "neg_inf": 0xFFF0000000000000}
DOTS = (L.VAR_DOTSTREAM, L.VAR_DOTSTREAM4, L.VAR_KRED)
ALL = ("complex128", "float64", "complex64", "float32")
SINGLE = ("complex64", "float32")


def _single(dtype):
    return np.dtype(dtype) in (np.float32, np.complex64)


def _uint(dtype):
    return np.uint32 if _single(dtype) else np.uint64


def _encodings(dtype):
    nan, inf = (NAN32, INF32) if _single(dtype) else (NAN64, INF64)
    return [(k, v, True) for k, v in nan.items()] + [(k, v, False) for k, v in inf.items()]


def _poke(x, flat, bits, part=0):
    """Write a raw bit pattern into component ``part`` (0 real, 1 imaginary) of element ``flat``."""
    per = 2 if x.dtype.kind == "c" else 1
    x.reshape(-1).view(_uint(x.dtype))[flat * per + part] = bits


def _nan_fill(shape, dtype):
    c = np.zeros(shape, dtype=dtype)
    c.reshape(-1).view(_uint(dtype))[:] = 0x7FFFFFFF if _single(dtype) else 0x7FFFFFFFFFFFFFFF
    return c


# (variant, eq, shape_a, shape_b, build_pair_desc kwargs, dtypes, note)
_T64, _T32, _T16 = L.VAR_TC05_128x64, L.VAR_TC05_128x32, L.VAR_TC05_128x16
CASES = [
    (L.VAR_SIMT_64x64, "ab,bc->ac", (130, 19), (19, 70), {}, ALL, "ragged"),
    (L.VAR_KRED, "k,k->", (50001,), (50001,), {}, ALL, "dot"),
    (L.VAR_DMMA_128x64, "ab,bc->ac", (300, 40), (40, 100), {}, ALL, "ragged"),
    (L.VAR_DMMA_64x128, "ab,bc->ac", (300, 40), (40, 150), {}, ALL, "ragged"),
    (L.VAR_DMMA_256x32, "ab,bc->ac", (300, 40), (40, 50), {}, ALL, "ragged"),
    (L.VAR_DMMA_256x16, "ab,bc->ac", (300, 40), (40, 20), {}, ALL, "ragged"),
    (L.VAR_ROW_128x8, "ab,bc->ac", (300, 19), (19, 7), {}, ALL, "ragged"),
    (L.VAR_ROW_256x4, "ab,bc->ac", (300, 19), (19, 3), {}, ALL, "ragged"),
    (L.VAR_ROWSTREAM, "ab,bc->ac", (1024, 5), (5, 7), {}, ALL, "ragged_n"),
    (L.VAR_DMMA3M_128x32, "ab,bc->ac", (300, 72), (72, 100), {}, ("complex128",), "ragged"),
    (L.VAR_DMMA3M_256x16, "ab,bc->ac", (300, 40), (40, 20), {}, ("complex128",), "ragged"),
    (L.VAR_DMMASTREAM, "ab,bc->ac", (4096, 20), (20, 12), {}, ("complex128",), "ragged_n"),
    (L.VAR_DOTSTREAM, "k,k->", (1 << 20,), (1 << 20,), {}, ALL, "dot"),
    (L.VAR_DOTSTREAM4, "mk,kn->mn", (3, 1 << 20), (1 << 20, 2), {}, ALL, "dot"),
    (L.VAR_DMMA_32x32, "mk,kn->mn", (20, 1 << 14), (1 << 14, 24), {}, ("complex128", "float64"), "split"),
    (L.VAR_ROWSTREAM_K, "ab,bc->ac", (4096, 40), (40, 7), {}, ("float64", "complex64", "float32"), "ragged_n"),
    # the wgmma complex64 kernel: every N tile, every A staging mode, split-K, the non-power-of-two exact
    # tiles, and shapes whose B' the launcher keeps resident or streams through its ring (both asserted:
    # _RESIDENT_B)
    (_T64, "ab,bc->ac", (512, 64), (64, 64), {"force_splitk": 1}, SINGLE[:1], "tmap,few_k"),
    (_T32, "ab,bc->ac", (512, 64), (64, 32), {"force_splitk": 1}, SINGLE[:1], "tmap,few_k"),
    (_T16, "ab,bc->ac", (512, 64), (64, 16), {"variant": _T16, "force_splitk": 1}, SINGLE[:1], "tmap,few_k"),
    (_T64, "ab,bc->ac", (256, 256), (256, 64), {"force_splitk": 1}, SINGLE[:1], "tmap,long_k"),
    (_T64, "xab,xbc->xac", (3, 256, 32), (3, 32, 64), {"variant": _T64}, SINGLE[:1], "tmap,batched"),
    (_T32, "abx,bcx->acx", (256, 32, 3), (32, 32, 3), {"variant": _T32}, SINGLE[:1], "gather"),
    # (five separated box dims: no tensor map, runs of 128 elements: TMA bulk copies)
    (_T64, "fqepdrcobka,kopqrn->abcdefn", (2, 2, 2, 2, 2, 2, 2, 2, 2, 16, 4), (16, 2, 2, 2, 2, 64),
     {"force_splitk": 1}, SINGLE[:1], "bulk,long_k"),
    (_T64, "ab,bc->ac", (1296, 216), (216, 216), {"force_splitk": 1}, SINGLE[:1], "tmap,exact108x54x12"),
    (_T64, "ab,bc->ac", (128, 256), (256, 64), {"force_splitk": 4}, SINGLE[:1], "tmap,split"),
]
# wgmma rows whose B' stays resident: four k-steps fit next to three A stages for N tiles of 32 and 16,
# not for 64 (three at most); long k, a batch or split-K always stream it through the ring
_RESIDENT_B = {(_T32, "tmap,few_k"), (_T16, "tmap,few_k")}
PARAMS = [pytest.param(c, dt, id=f"v{c[0]}-{dt}-{c[6]}-{'x'.join(map(str, c[2]))}")
          for c in CASES for dt in c[5]]


def _operands(case, dtype, seed=0):
    _v, eq, sa, sb, _kw, _d, _n = case
    a, b = make_arrays([sa, sb], "complex128", seed=seed)
    if np.dtype(dtype).kind != "c":
        a, b = a.real, b.real
    return np.ascontiguousarray(a.astype(dtype)), np.ascontiguousarray(b.astype(dtype))


def _launch(eq, a, b, dtype, c0=None, accumulate=False, **kw):
    """One ctgb_contract_pair launch.  C starts as ``c0`` (NaN-filled if not given).
    Returns (C, plan, staging mode of a wgmma launch)."""
    import torch

    from cotengra_b200 import _lib

    (ta, tb), to = L.split_equation(eq)
    dims = L.classify_pair(ta, a.shape, tb, b.shape, to)
    out_shape = tuple(dims.out_shape)
    plan = L.build_pair_desc(dims, dtype, accumulate=accumulate, c_dense_elems=max(1, math.prod(out_shape)),
                             sm_count=_lib.device_info()["sm_count"], **kw)
    if c0 is None:
        c0 = _nan_fill(out_shape, dtype)
    da = torch.from_numpy(np.ascontiguousarray(a)).cuda()
    db = torch.from_numpy(np.ascontiguousarray(b)).cuda()
    dc = torch.from_numpy(np.array(c0, dtype=dtype).reshape(out_shape).copy()).cuda()
    pa, pb = (db, da) if plan.swapped else (da, db)
    before = _lib.tensor_map_launches()
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa.data_ptr(), pb.data_ptr(),
                                              dc.data_ptr(), 0))
    torch.cuda.synchronize()
    mode = None
    if plan.variant in L.TC05_VARIANTS:
        if _lib.tensor_map_launches() > before:
            mode = "tmap"
        else:
            mode = "bulk" if plan.words[L.W_FLAGS] & 64 else "gather"
    return dc.cpu().numpy(), plan, mode


def _deterministic(plan):
    return plan.splitk == 1 and plan.variant not in DOTS


def _cone(eq, which, shape, flat, out_shape):
    """Output elements that share the kept (and batch) indices of element ``flat`` of operand ``which``."""
    terms, out = L.split_equation(eq)
    fixed = dict(zip(terms[which], np.unravel_index(flat, shape)))
    mask = np.zeros(out_shape, dtype=bool)
    mask[tuple(int(fixed[ix]) if ix in fixed else slice(None) for ix in out)] = True
    return mask


def _positions(case, which, shape):
    """Flat positions to poison: the first element (first element of the first tile), the last one
    (last k-step, inside the ragged or last tile), the last row / column of the first tile, and an
    interior element."""
    v = case[0]
    mt, nt, _kt = L.VARIANT_TILES[v]
    idx = [tuple(0 for _ in shape), tuple(d - 1 for d in shape)]
    if len(shape) == 2:
        edge = (mt - 1) if which == 0 else (nt - 1)
        axis = 0 if which == 0 else 1
        e = [0, 0]
        e[axis] = min(edge, shape[axis] - 1)
        e[1 - axis] = shape[1 - axis] - 1
        idx.append(tuple(e))
    rng = np.random.default_rng(len(shape) + which)
    idx.append(tuple(int(rng.integers(d)) for d in shape))
    return sorted({int(np.ravel_multi_index(i, shape)) for i in idx})


def _tol(dtype):
    return 1e-5 if _single(dtype) else 1e-12


def _expect_variant(case, plan, mode):
    v, eq, sa, sb, kw, _d, note = case
    assert plan.variant == v, (note, plan.variant)
    if "force_splitk" in kw:
        assert plan.splitk == kw["force_splitk"], (note, plan.splitk)
    if v in L.TC05_VARIANTS:
        want_mode = note.split(",")[0]
        assert mode == want_mode, (note, mode)
        if "exact" in note:
            assert (int(plan.words[L.W_MTA]), int(plan.words[L.W_NTA]), int(plan.words[L.W_KTA])) == (108, 54, 12)
        from cotengra_b200 import _lib

        info = _lib.device_info()
        launch = _lib.tc05_launch_config(plan.words, 0, info["sm_count"], info["smem_optin"])
        assert launch["b_stat"] == ((v, note) in _RESIDENT_B), (note, launch)


@pytest.mark.parametrize("case,dtype", PARAMS)
def test_nonfinite_dependency_cone(case, dtype):
    v, eq, sa, sb, kw, _d, note = case
    kw = dict(kw)
    kw.setdefault("variant", v)
    a, b = _operands(case, dtype)
    clean, plan, mode = _launch(eq, a, b, dtype, **kw)
    _expect_variant(case, plan, mode)
    print(f"variant={plan.variant} dtype={dtype} mode={mode} splitk={plan.splitk} case={note}")
    # every element written: C started NaN-filled
    assert not np.isnan(clean).any(), "a non-accumulating launch left elements of C unwritten"
    cplx = np.dtype(dtype).kind == "c"
    for which, shape in ((0, sa), (1, sb)):
        positions = _positions(case, which, shape)
        for name, bits, is_nan in _encodings(dtype):
            # real part at every position; imaginary part only at the last one
            for flat, part in [(p, 0) for p in positions] + ([(positions[-1], 1)] if cplx else []):
                x = [a.copy(), b.copy()]
                _poke(x[which], flat, bits, part)
                got, plan2, _ = _launch(eq, x[0], x[1], dtype, **kw)
                assert plan2.variant == plan.variant
                cone = _cone(eq, which, shape, flat, got.shape)
                where = (which, name, np.unravel_index(flat, shape), part)
                if is_nan:
                    inside = got[cone]
                    ok = (np.isnan(inside.real) & np.isnan(inside.imag)) if cplx else np.isnan(inside)
                    assert ok.all(), ("NaN lost in the cone", where, inside[~ok][:4])
                else:
                    assert not np.isfinite(got[cone]).any(), ("inf lost in the cone", where)
                out = got[~cone]
                if out.size == 0:
                    continue
                if _deterministic(plan):
                    same = out.reshape(-1).view(_uint(dtype)) == clean[~cone].reshape(-1).view(_uint(dtype))
                    assert same.all(), ("value outside the cone changed", where)
                else:
                    assert np.isfinite(out).all(), ("non-finite outside the cone", where)
                    assert rel_err(out, clean[~cone]) < _tol(dtype) * 10, where


@pytest.mark.parametrize("case,dtype", PARAMS)
def test_accumulate_keeps_exactly_one_nan(case, dtype):
    """An accumulating launch adds into C: one NaN in C0 stays NaN, no other element becomes NaN."""
    v, eq, sa, sb, kw, _d, note = case
    kw = dict(kw)
    kw.setdefault("variant", v)
    a, b = _operands(case, dtype, seed=1)
    (ta, tb), to = L.split_equation(eq)
    out_shape = tuple(L.classify_pair(ta, sa, tb, sb, to).out_shape)
    c0 = make_arrays([out_shape], "complex128", seed=5)[0]
    c0 = np.ascontiguousarray((c0 if np.dtype(dtype).kind == "c" else c0.real).astype(dtype))
    flat = c0.size - 1 if c0.size > 1 else 0
    _poke(c0, flat, NAN32["nan_ones"] if _single(dtype) else NAN64["nan_ones"])
    got, plan, _ = _launch(eq, a, b, dtype, c0=c0, accumulate=True, **kw)
    assert plan.variant == v, plan.variant
    nan = np.isnan(got).reshape(-1)
    assert nan[flat] and nan.sum() == 1, np.flatnonzero(nan)[:8]


@pytest.mark.parametrize("dtype", ALL)
@pytest.mark.parametrize("eq,shape", [("ab->a", (300, 70)), ("abc->b", (7, 3000, 5)), ("ab->", (300, 70)),
                                      ("aab->b", (40, 40, 9))])
def test_reduce_single_cone(eq, shape, dtype):
    """ctgb_reduce_single (thread-per-output and block-per-output kernels): a poisoned element reaches
    exactly its own output element; the rest is bitwise unchanged."""
    (x,) = make_arrays([shape], "complex128", seed=3)
    x = np.ascontiguousarray((x if np.dtype(dtype).kind == "c" else x.real).astype(dtype))
    clean = np.asarray(cb.einsum(eq, x))
    (term,), out = L.split_equation(eq)
    for name, bits, is_nan in _encodings(dtype):
        for flat in (0, x.size - 1, x.size // 2 + 1):
            y = x.copy()
            _poke(y, flat, bits)
            got = np.asarray(cb.einsum(eq, y))
            digits = {}
            for ix, dgt in zip(term, np.unravel_index(flat, shape)):
                digits.setdefault(ix, set()).add(int(dgt))
            cone = np.zeros(got.shape, dtype=bool)
            if all(len(s) == 1 for s in digits.values()):  # (off a repeated index's diagonal: never read)
                cone[tuple(next(iter(digits[ix])) for ix in out)] = True
            if is_nan:
                assert np.isnan(got[cone]).all(), (eq, name, flat)
            else:
                assert not np.isfinite(got[cone]).any(), (eq, name, flat)
            assert (got[~cone].reshape(-1).view(_uint(dtype)) == clean[~cone].reshape(-1).view(_uint(dtype))).all()


# ------------------------------------------------------------------ power-of-two scaling
@pytest.mark.parametrize("case,dtype", PARAMS)
def test_power_of_two_scaling_is_exact(case, dtype):
    """2^j A B == 2^j (A B) bit for bit (global 2^j on A or B, per-row 2^j_i on A, per-column 2^j_c on
    B, j in -40..40); split-K and atomic plans to the dtype tolerance."""
    v, eq, sa, sb, kw, _d, note = case
    kw = dict(kw)
    kw.setdefault("variant", v)
    a, b = _operands(case, dtype, seed=2)
    base, plan, _ = _launch(eq, a, b, dtype, **kw)
    assert plan.variant == v
    terms, out = L.split_equation(eq)
    rng = np.random.default_rng(7)
    trials = [("A", 0, None, 37), ("B", 1, None, -40)]
    for which in (0, 1):
        kept = [ix for ix in terms[which] if ix in out and ix not in terms[1 - which]]
        if kept:
            trials.append(("row" if which == 0 else "col", which, kept[0], None))
    real = a.real.dtype
    for label, which, ix, j in trials:
        x = [a.copy(), b.copy()]
        if ix is None:
            x[which] = x[which] * np.asarray(2.0**j, dtype=real)
            fo = np.asarray(2.0**j, dtype=real)
        else:
            ax = terms[which].index(ix)
            f = np.ldexp(1.0, rng.integers(-40, 41, size=x[which].shape[ax])).astype(real)
            shp = [1] * x[which].ndim
            shp[ax] = -1
            x[which] = x[which] * f.reshape(shp)
            oshp = [1] * base.ndim
            oshp[out.index(ix)] = -1
            fo = f.reshape(oshp)
        got, _p, _ = _launch(eq, x[0], x[1], dtype, **kw)
        if _deterministic(plan):
            expect = np.ascontiguousarray(base * fo)
            assert (got.reshape(-1).view(_uint(dtype)) == expect.reshape(-1).view(_uint(dtype))).all(), label
        else:
            assert rel_err(got / fo, base) < _tol(dtype) * 10, label


SINGLE_PARAMS = [p for p in PARAMS if p.values[1] in SINGLE]


@pytest.mark.parametrize("case,dtype", SINGLE_PARAMS)
def test_near_flt_max_operands(case, dtype):
    """Entries within 2^-11 of FLT_MAX (the tf32 rounding of the 3xTF32 split would carry into the
    exponent there) with |B| small enough that the exact result stays finite."""
    v, eq, sa, sb, kw, _d, note = case
    kw = dict(kw)
    kw.setdefault("variant", v)
    terms, _out = L.split_equation(eq)
    k = math.prod(d for ix, d in zip(terms[0], sa) if ix in terms[1])
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    rng = np.random.default_rng(1)
    for big in (0, 1):  # the streamed operand (A: scatter) and the packed one (B: bprime_kernel)
        x = list(_operands(case, dtype, seed=4))
        n = x[big].size * (2 if np.dtype(dtype).kind == "c" else 1)
        bits = rng.integers(0x7F7FF000, 0x7F800000, size=n, dtype=np.uint64).astype(np.uint32)
        bits |= rng.integers(0, 2, size=n, dtype=np.uint64).astype(np.uint32) << np.uint32(31)
        x[big].reshape(-1).view(np.uint32)[:] = bits
        x[1 - big] = (x[1 - big] / np.asarray(4 * k, dtype=x[1 - big].real.dtype)).astype(dtype)
        got, plan, _ = _launch(eq, x[0], x[1], dtype, **kw)
        assert plan.variant == v
        want = np.einsum(eq, x[0].astype(wide), x[1].astype(wide))
        bound = np.einsum(eq, np.abs(x[0].astype(wide)), np.abs(x[1].astype(wide)))
        assert np.isfinite(got).all(), ("finite operands near FLT_MAX gave a non-finite product", big)
        assert np.max(np.abs(got - want) / bound) < 1e-5, big


# Products near the bottom of the float range, where the lo terms of a 3xTF32 split become denormal.
# Measured on H100 (DESIGN.md, "Special values"), componentwise error against the float64 product: the
# wgmma path, the FMA kernel, the 128x64 / 64x128 mma.sync tiles and the row-stream kernels keep < 1e-6
# down to products of 2^-126; KRED and the dot streams keep 1e-5 down to 2^-120; the 256x32 / 256x16
# mma.sync tiles and the staged row kernels lose the lo terms below ~2^-110 (1e-5 near 2^-114, 1e-3 at
# 2^-120).  Split-K plans add their partial sums with float atomics, which flush denormals.  Each kernel
# is pinned to 1e-5 down to its measured floor.
SINGLE_FLOOR = {L.VAR_SIMT_64x64: -126, L.VAR_DMMA_128x64: -126, L.VAR_DMMA_64x128: -126, L.VAR_ROWSTREAM: -126,
                L.VAR_ROWSTREAM_K: -126, L.VAR_KRED: -120, L.VAR_DOTSTREAM: -120, L.VAR_DOTSTREAM4: -120,
                L.VAR_DMMA_256x32: -110, L.VAR_DMMA_256x16: -110, L.VAR_ROW_128x8: -110, L.VAR_ROW_256x4: -110,
                _T64: -126, _T32: -126, _T16: -126}
DOUBLE_PARAMS = [p for p in PARAMS if p.values[1] not in SINGLE]


def _floor_errors(case, dtype, powers):
    v, eq, sa, sb, kw, _d, note = case
    kw = dict(kw)
    kw.setdefault("variant", v)
    a, b = _operands(case, dtype, seed=6)
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    report, plan = [], None
    for p in powers:
        x = (a * np.asarray(2.0 ** (p // 2), dtype=a.real.dtype)).astype(dtype)
        y = (b * np.asarray(2.0 ** (p - p // 2), dtype=a.real.dtype)).astype(dtype)
        got, plan, _ = _launch(eq, x, y, dtype, **kw)
        assert np.isfinite(got).all()
        # (the reference product in float64 for single precision; for double precision the bound is
        # formed from exactly rescaled operands, so that it does not underflow itself)
        if _single(dtype):
            want = np.einsum(eq, x.astype(wide), y.astype(wide))
            bound = np.einsum(eq, np.abs(x.astype(wide)), np.abs(y.astype(wide)))
            err = float(np.max(np.abs(got - want) / np.maximum(bound, 1e-300)))
        else:
            up = 2.0 ** -p
            want = np.einsum(eq, a, b)
            bound = np.einsum(eq, np.abs(a), np.abs(b))
            err = float(np.max(np.abs(got * up - want) / bound))
        report.append((p, err))
    print(f"small-magnitude floor variant={v} dtype={dtype} {note}: " +
          " ".join(f"2^{p}:{e:.1e}" for p, e in report))
    return report, plan


@pytest.mark.parametrize("case,dtype", SINGLE_PARAMS)
def test_small_magnitude_floor(case, dtype):
    v = case[0]
    report, plan = _floor_errors(case, dtype, (-100, -110, -114, -120, -126))
    floor = SINGLE_FLOOR[v] if plan.splitk == 1 else -100
    for p, err in report:
        if p >= floor:
            assert err < 1e-5, (p, err, floor)


@pytest.mark.parametrize("case,dtype", DOUBLE_PARAMS)
def test_small_magnitude_floor_double(case, dtype):
    """float64 / complex128 products down to 2^-1022 (DMMA, FMA, stream and dot kernels): measured on H100,
    every kernel keeps <= 2e-15 of the exactly rescaled product; pinned at 1e-12."""
    report, _plan = _floor_errors(case, dtype, (-1000, -1010, -1016, -1020, -1022))
    for p, err in report:
        assert err < 1e-12, (p, err)


# ------------------------------------------------------------------ whole trees
def _chain_spec(shapes, inds, path, output):
    size = {}
    for t, s in zip(inds, shapes):
        size.update(zip(t, s))
    return cb.TreeSpec([tuple(t) for t in inds], tuple(output), size, path)


def _tree_arrays(spec, dtype, seed):
    arrays = make_arrays(spec.shapes(), "complex128", seed=seed)
    return [np.ascontiguousarray(x.astype(dtype)) for x in arrays]


def _nan_mask(x):
    x = np.asarray(x)
    return np.isnan(x.real) | np.isnan(x.imag) if x.dtype.kind == "c" else np.isnan(x)


TREE_NAMES = ["config1_rand10", "rand_r2_o0_hi0_ho1_root_s666", "lattice4x4", "peps8x8_d2",
              "rand_r3_o1_hi1_ho2_root_s42"]


@pytest.mark.parametrize("single", [False, True], ids=["stored_dtype", "single_precision"])
@pytest.mark.parametrize("name", TREE_NAMES)
def test_nan_through_golden_trees(name, single):
    """The golden trees in their stored dtype (complex128 / float64) and cast to complex64 / float32,
    with the 0x7FFF... NaN of that width in one input."""
    rec = next(r for r in load_json("trees.json") if r["name"] == name)
    spec = tree_spec(rec)
    dtype = rec["dtype"]
    if single:
        dtype = "complex64" if np.dtype(dtype).kind == "c" else "float32"
    arrays = [np.ascontiguousarray(x.astype(dtype)) for x in make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])]
    _poke(arrays[0], arrays[0].size - 1, NAN32["nan_ones"] if single else NAN64["nan_ones"])
    contr = spec.contractions()
    inputs = [tuple(t) for t in spec.inputs]
    want = orc.contract_tree(inputs, spec.output, spec.sliced, contr, arrays)
    got = cb.contract_tree(spec, arrays)
    assert _nan_mask(want).any()
    assert (_nan_mask(got) == _nan_mask(want)).all()
    assert rel_err(np.where(_nan_mask(want), 0, got), np.where(_nan_mask(want), 0, want)) < (1e-4 if single else 1e-10)
    # strip_exponent: the first normalisation divides everything by a NaN factor
    m, e = cb.contract_tree(spec, arrays, strip_exponent=True)
    assert math.isnan(e) and _nan_mask(m).all()
    if not spec.sliced:
        wm, we = orc.run_contractions(contr, arrays, strip_exponent=True)
        assert math.isnan(we) and _nan_mask(wm).all()


def _overflow_chain():
    # node 0: X0 (256 x 64) row 0 = 1e38, times all-ones -> row 0 of C0 overflows to +inf
    # node 1: C0 x X2 (mixed signs)       -> row 0 = inf - inf = NaN, made by the GPU (0x7FFFFFFF)
    # node 2: C1 x X3, a wgmma node        -> must keep the NaN
    spec = _chain_spec([(256, 64), (64, 64), (64, 64), (64, 64)], ["ab", "bc", "cd", "de"],
                       [(0, 1), (4, 2), (5, 3)], "ae")
    x = _tree_arrays(spec, "complex64", seed=8)
    x[0][0, :] = 1e38
    x[1][:] = 1.0
    return spec, x


@pytest.mark.parametrize("strip", [False, True])
def test_overflow_then_inf_minus_inf_through_wgmma(strip):
    spec, x = _overflow_chain()
    ex = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=strip, fuse=False)
    variants = [nd["plan"].variant for nd in ex.plan.nodes if "plan" in nd]
    assert variants[-1] in L.TC05_VARIANTS, variants
    want = orc.contract_tree([tuple(t) for t in spec.inputs], spec.output, [], spec.contractions(), x)
    assert _nan_mask(want)[0].all() and not _nan_mask(want)[1:].any()
    res = cb.contract_tree(ex, x)
    if strip:
        m, e = res
        assert math.isnan(e) and _nan_mask(m).all()
    else:
        got = np.asarray(res)
        assert (_nan_mask(got) == _nan_mask(want)).all(), np.flatnonzero(_nan_mask(got) != _nan_mask(want))[:8]
        assert np.isfinite(got[1:]).all()


@pytest.mark.parametrize("name", ["nan_ones", "nan_neg", "snan", "qnan"])
def test_nan_input_through_wgmma_tree(name):
    """complex64 chain whose nodes run on wgmma: a NaN input element reaches the oracle's NaN positions."""
    spec = _chain_spec([(256, 64), (64, 64), (64, 64)], ["ab", "bc", "cd"], [(0, 1), (3, 2)], "ad")
    x = _tree_arrays(spec, "complex64", seed=9)
    _poke(x[0], 5 * 64 + 63, NAN32[name], part=1)
    ex = cb.TreeExecutor(spec, dtype="complex64", fuse=False)
    assert all(nd["plan"].variant in L.TC05_VARIANTS for nd in ex.plan.nodes if "plan" in nd)
    want = orc.contract_tree([tuple(t) for t in spec.inputs], spec.output, [], spec.contractions(), x)
    got = np.asarray(cb.contract_tree(ex, x))
    assert (_nan_mask(got) == _nan_mask(want)).all()
    assert _nan_mask(got)[5].all() and not _nan_mask(got)[:5].any()


@pytest.mark.parametrize("name", ["rand_r2_o0_hi0_ho1_root_s666_sliced", "rand_r3_o1_hi1_ho1_root_s42_sliced"])
def test_one_nan_slice_makes_the_sum_nan(name):
    """A NaN in one slice only: the summed value is NaN where the oracle's is, and with strip_exponent
    the exponent and the whole mantissa are NaN (a NaN exponent is kept, not dropped by a max)."""
    rec = next(r for r in load_json("trees.json") if r["name"] == name)
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    sliced_ix = [s[0] for s in spec.sliced]
    c = next(i for i, t in enumerate(spec.inputs) if any(ix in sliced_ix for ix in t))
    term = spec.inputs[c]
    idx = tuple(1 if ix in sliced_ix else 0 for ix in term)   # belongs to slices with that digit = 1
    arrays[c] = arrays[c].copy()
    _poke(arrays[c], int(np.ravel_multi_index(idx, arrays[c].shape)), NAN64["nan_ones"])
    inputs = [tuple(t) for t in spec.inputs]
    want = orc.contract_tree(inputs, spec.output, spec.sliced, spec.contractions(), arrays)
    got = cb.contract_tree(spec, arrays)
    assert _nan_mask(want).any()
    assert (_nan_mask(got) == _nan_mask(want)).all()
    m, e = cb.contract_tree(spec, arrays, strip_exponent=True)
    assert math.isnan(e) and _nan_mask(m).all()


# ------------------------------------------------------------------ strip_exponent: m and e separately
# Trees for the strip_exponent checks, with the node whose strip handling each one is there for:
#   big          the join of two 24-50 MB intermediates: its small operand is above the 16 MiB under which
#                a scaled copy is made first, so the kernel's epilogue multiplies by 1/(fA fB) (StripCtx)
#   wgmma_k512   a K = 512 complex64 wgmma node, folded chunk by chunk: max|C| measured after the launch
#   splitk       a one-tile node with K = 4096: split-K, measured after the launch
#   dot          an inner product over 2^20 elements (dot stream), measured after the launch
STRIP_TREES = {
    "big": ([(2048, 16), (16, 1536), (1536, 16), (16, 2048)], ["ab", "bc", "cd", "de"], [(0, 1), (2, 3), (4, 5)], "ae", 2),
    "wgmma_k512": ([(256, 512), (512, 64), (64, 16), (16, 32)], ["ab", "bc", "cd", "de"], [(0, 1), (2, 3), (4, 5)], "ae", 0),
    "splitk": ([(128, 16), (16, 4096), (4096, 64)], ["ab", "bc", "cd"], [(0, 1), (3, 2)], "ad", 1),
    "dot": ([(1024, 16), (16, 1024), (1024, 1024)], ["ab", "bc", "ac"], [(0, 1), (3, 2)], "", 1),
}


def _strip_executor(kind, dtype):
    shapes, inds, path, out, node = STRIP_TREES[kind]
    spec = _chain_spec(shapes, inds, path, out)
    ex = cb.TreeExecutor(spec, dtype=dtype, strip_exponent=True, fuse=False)
    nd = ex.plan.nodes[node]
    prescale, after = ex.plan.strip_modes()[node]
    if kind == "big":
        assert prescale == 0, "the join must scale in its epilogue"
    elif kind == "wgmma_k512":
        assert dtype != "complex64" or (nd["plan"].variant in L.TC05_VARIANTS and after == 1)
    elif kind == "splitk":
        assert nd["plan"].splitk > 1 and after == 1, (nd["plan"].variant, nd["plan"].splitk)
    else:
        assert nd["plan"].variant == L.VAR_DOTSTREAM and after == 1, nd["plan"].variant
    return spec, ex


@pytest.mark.parametrize("dtype", ["complex128", "complex64"])
@pytest.mark.parametrize("kind", list(STRIP_TREES))
def test_strip_mantissa_and_exponent_separately(kind, dtype):
    """max|m| == 1 to an ulp, and e == log10 max|value| (the reference's exponent)."""
    spec, ex = _strip_executor(kind, dtype)
    x = _tree_arrays(spec, dtype, seed=12)
    m, e = cb.contract_tree(ex, x)
    wide = [a.astype(np.complex128) for a in x]
    wm, we = orc.run_contractions(spec.contractions(), wide, strip_exponent=True)
    eps = np.finfo(np.asarray(m).real.dtype).eps
    assert abs(np.max(np.abs(m)) - 1.0) <= 2 * eps
    assert abs(e - we) < (1e-12 if dtype == "complex128" else 1e-6) * max(1.0, abs(we))
    assert rel_err(np.asarray(m).astype(np.complex128), wm) < (1e-10 if dtype == "complex128" else 1e-5)


# (tree, dtype, (j0, j2): inputs 0 and 2 scaled by 2^j, how the scaled node applies 1/(fA fB) or measures
# its factor, whether the unscaled run does the same)
STRIP_SCALINGS = [
    ("big", "complex64", (20, -7), "float multiply sf", True),
    ("big", "complex64", (-60, -60), "double fallback: 1/(fA fB) ~ 1e34", False),
    ("big", "complex128", (20, -7), "double multiply", True),
    # the join multiplies the RAW intermediates (~2^-597 each) before applying 1/(fA fB): their product
    # underflows to 0 before the two-factor route can rescale it, and the exponent comes out -inf where the
    # reference, which divides each intermediate by its factor first, is finite.  A known limitation of
    # the lazy scaling (DESIGN.md, "Special values"), kept here as an expected failure.
    pytest.param("big", "complex128", (-600, -600), "two factors: 1/(fA fB) ~ 2^1194", False,
                 marks=pytest.mark.xfail(strict=True, reason="raw product of two unnormalised intermediates "
                                         "underflows before the two-factor scaling")),
    ("big", "complex128", (-1000, 0), "hypot: |C|^2 below 1e-280", False),
    ("big", "complex128", (700, 300), "hypot: |C|^2 above 1e300", False),
    ("wgmma_k512", "complex64", (20, 0), "measured after", True),
    ("splitk", "complex64", (20, 0), "measured after", True),
    ("splitk", "complex128", (20, 0), "measured after", True),
    ("dot", "complex64", (20, 0), "measured after", True),
    ("dot", "complex128", (-600, 0), "measured after, hypot", False),
]


def _strip_id(p):
    k, d, j, _b, _s = p.values if hasattr(p, "values") else p
    return f"{k}-{d}-{j[0]}_{j[1]}"


@pytest.mark.parametrize("kind,dtype,js,branch,same", STRIP_SCALINGS, ids=[_strip_id(p) for p in STRIP_SCALINGS])
def test_strip_exponent_shifts_by_scaling(kind, dtype, js, branch, same):
    """Scaling inputs by 2^j shifts the exponent by j log10(2) and leaves the mantissa unchanged.  The
    node products scale exactly (test_power_of_two_scaling_is_exact), but a factor max|C| that comes
    from hypot (the measure-after pass, and the epilogue for squares outside 1e-280..1e300) is not
    always exactly 2^j times the unscaled one, and the mantissa is divided by it.  Measured on H100 with
    both runs on the same route: up to 4.3 ulps (complex64 split-K), 5.6 ulps (complex128 split-K), ~3e-8
    in a complex64 exponent.  So the mantissa is allowed 8 ulps whichever route is taken; ``same`` only
    records whether the scaled run takes the unscaled run's route."""
    spec, ex = _strip_executor(kind, dtype)
    x = _tree_arrays(spec, dtype, seed=12)
    m0, e0 = cb.contract_tree(ex, x)
    y = list(x)
    y[0] = (x[0] * np.ldexp(1.0, js[0])).astype(dtype)
    y[2] = (x[2] * np.ldexp(1.0, js[1])).astype(dtype)
    wide = [a.astype(np.complex128) for a in y]
    assert all(np.isfinite(a).all() and (np.abs(a) > 0).all() for a in wide)
    m, e = cb.contract_tree(ex, y)
    shift = (js[0] + js[1]) * math.log10(2.0)
    assert abs((e - e0) - shift) < (1e-12 if dtype == "complex128" else 2e-7) * max(1.0, abs(e))
    m, m0 = np.asarray(m), np.asarray(m0)
    eps = np.finfo(m.real.dtype).eps
    assert np.max(np.abs(m - m0)) <= 8 * eps, (branch, same)
    wm, we = orc.run_contractions(spec.contractions(), wide, strip_exponent=True)
    assert abs(e - we) < (1e-12 if dtype == "complex128" else 1e-6) * max(1.0, abs(we))
    assert rel_err(m.astype(np.complex128), wm) < (1e-10 if dtype == "complex128" else 1e-5)
