"""The fused strip_exponent epilogue of every pairwise kernel, launch by launch: the numpy model of
what it stores and measures, which launches measure in it, which kernel instantiation runs, and the
cases and rank-one operands the device tests drive it with.  No GPU imports here.

With ``strip_exponent`` a pairwise launch reads three descriptor words (gett_desc.h), each the
device address of a double or 0:
  * ``W_SCALE_A`` / ``W_SCALE_B``: factors fA, fB; the epilogue multiplies the product by
    1/(fA fB) (``strip_begin`` / ``strip_mul``, gett_kernels.cuh);
  * ``W_FACTOR_C``: a slot that receives max|product| of the launch, as scaled, by an atomicMax of
    the double's bits (``strip_track`` / ``strip_end``).
A plan measures a launch afterwards instead (``measure_after``, ctg_b200.cu) when its epilogue sees
partial sums: split-K, the dot streams, KRED and wgmma launches that fold the contracted range into
C chunk by chunk.  Such launches are only ever scaled.
"""

from __future__ import annotations

import numpy as np

from cotengra_b200 import lowering as L
from tests import kernel_cases as KC
from tests import precision_cases as PC

# the factors of the sweep's scale mode: 1/(3 * 0.7) is no power of two
FA, FB = 3.0, 0.7
_DBL_MAX_PROD = 1.7e308
QNAN_BITS = 0x7FF8000000000000

# ---------------------------------------------------------------------------- the scale model


def strip_factors(fA, fB):
    """``(s, sb, sf, two)`` as ``strip_begin`` forms them from the factors fA and fB."""
    fA, fB = np.float64(fA), np.float64(fB)
    with np.errstate(over="ignore", under="ignore", divide="ignore"):
        sa = np.float64(1.0) / fA if fA != 0 else np.float64(0.0)
        sb = np.float64(1.0) / fB if fB != 0 else np.float64(0.0)
        prod = sa * sb
    two = bool(sa != 0 and sb != 0 and (prod == 0 or prod > _DBL_MAX_PROD))
    ap = abs(prod)
    sf = np.float32(prod) if (not two and (ap == 0 or 1e-30 < ap < 1e30)) else np.float32(0.0)
    return (sa if two else prod), (sb if two else np.float64(1.0)), sf, two


def strip_route(fA, fB, dtype):
    """How the epilogue scales a ``dtype`` value: "zero" (a factor is 0: s = 0), "two" (1/fA and
    1/fB one after the other: their product leaves the double range), "float" (single types: one
    float multiply by (float)s) or "double" (one double multiply; for the single types the
    fallback when |s| lies outside 1e-30..1e30)."""
    s, _sb, sf, two = strip_factors(fA, fB)
    if s == 0:
        return "zero"
    if two:
        return "two"
    return "float" if KC.is_single(dtype) and sf != 0 else "double"


def strip_expect(plain_c, fA, fB, dtype):
    """What a scaling epilogue stores for the unscaled values ``plain_c``: ``strip_mul`` applied to
    every real component separately."""
    dt = np.dtype(dtype)
    rd = KC.real_dtype(dt)
    s, sb, sf, two = strip_factors(fA, fB)
    x = np.ascontiguousarray(plain_c, dtype=dt)
    comp = x.reshape(-1).view(rd)
    with np.errstate(all="ignore"):
        if rd == np.float64:
            out = comp * s
            if two:
                out = out * sb
        elif sf != 0 or s == 0:
            out = comp * sf
        else:
            d = comp.astype(np.float64) * s
            if two:
                d = d * sb
            out = d.astype(np.float32)
    return np.ascontiguousarray(out, dtype=rd).view(dt).reshape(x.shape)


def max_abs(c):
    """max |c| in float64, hypot for complex values (0 for an empty array)."""
    c = np.asarray(c).reshape(-1)
    if c.size == 0:
        return 0.0
    if c.dtype.kind == "c":
        return float(np.max(np.hypot(c.real.astype(np.float64), c.imag.astype(np.float64))))
    return float(np.max(np.abs(c.astype(np.float64))))


# ---------------------------------------------------------------------------- launch classes


def _variant(plan):
    return int(plan.words[L.W_VARIANT])


def wgmma_facts(plan, a_addr=0, sms=KC.SM_COUNT):
    """The wgmma launch's choices (``KC.launch_facts``); chunking depends on the descriptor alone."""
    from cotengra_b200 import _lib

    return _lib.tc05_launch_config(plan.words, a_addr, sms, KC.H100_SMEM_OPTIN)


def measures_in_epilogue(case, plan, launch_facts=None):
    """Does a plan let this launch measure max|C| in its own epilogue?  The mirror of the
    ``measure_after`` rule of ``ctgb_plan_create``: not with split-K, the dot streams, KRED, or a
    wgmma launch whose contracted range is folded into C in chunks (``launch_facts["chunks"]``)."""
    v = _variant(plan)
    if int(plan.words[L.W_SPLITK]) > 1 or v in L.DOTSTREAM_VARIANTS or v == L.VAR_KRED:
        return False
    if v in L.TC05_VARIANTS:
        facts = launch_facts if launch_facts is not None else wgmma_facts(plan)
        return facts["chunks"] <= 1
    return True


def deterministic(case, plan, launch_facts=None):
    """One rounding per stored value, independent of scheduling: no atomics, no partial sums."""
    v = _variant(plan)
    return int(plan.words[L.W_SPLITK]) == 1 and v not in L.DOTSTREAM_VARIANTS and v != L.VAR_KRED and (
        v not in L.TC05_VARIANTS or measures_in_epilogue(case, plan, launch_facts))


def _one_pass(plan):
    return bool(int(plan.words[L.W_FLAGS]) & L.FLAG_TF32_ONE_PASS)


def instantiation(case, plan, scale=True):
    """The kernel instantiation (and, for the staged kernel, the epilogue path) a stripped launch
    runs: ``scale`` says whether the launch scales (W_SCALE_A set).  The staged epilogue scans the
    tile before its ordinary stores when it only measures, and scales and measures in the stores
    (``strip_store``) otherwise -- always for KRED, whose epilogue runs once."""
    from cotengra_b200 import _lib

    v, d, W = _variant(plan), case.dtype, plan.words
    if v == L.VAR_ROWSTREAM:
        N, K = int(W[L.W_NTA]), int(W[L.W_KTA])
        # launch_rowstream: N, K <= 4; else N <= 2 (K <= 8); else N, K <= 8
        return ("rowstream", "4x4" if N <= 4 and K <= 4 else "2x8" if N <= 2 else "8x8", d)
    if v == L.VAR_ROWSTREAM_K:
        return ("rowstream_k", d)
    if v == L.VAR_DMMASTREAM:
        return ("dmmastream", _lib.dmmastream_launch_config(W, KC.SM_COUNT)["nj"])
    if v in L.DOTSTREAM_VARIANTS:
        return ("dot", KC.VARIANT_NAMES[v], d)
    prec = "tf32" if _one_pass(plan) else "3xtf32"
    if v in L.TC05_VARIANTS:
        chunked = wgmma_facts(plan)["chunks"] > 1
        return ("wgmma", L.VARIANT_TILES[v][1], prec, "chunked" if chunked else "whole")
    path = "strip_store" if scale or v == L.VAR_KRED else "scan"
    return ("staged", KC.VARIANT_NAMES[v], d, prec if KC.is_single(d) and v in L.TF32_VARIANTS else "", path)


def required_keys():
    """Every instantiation a stripped launch can run, from the dispatch of ``launch_gett_typed``."""
    keys = set()
    for d in KC.ALL_DTYPES:
        keys |= {("rowstream", s, d) for s in ("4x4", "2x8", "8x8")}
        keys |= {("dot", KC.VARIANT_NAMES[v], d) for v in L.DOTSTREAM_VARIANTS}
    keys |= {("rowstream_k", d) for d in (KC.F32, KC.F64, KC.C64)}
    keys |= {("dmmastream", nj) for nj in (1, 2, 4, 8)}
    for v in L.TC05_VARIANTS:
        keys |= {("wgmma", L.VARIANT_TILES[v][1], p, c) for p in L.PRECISIONS for c in ("chunked", "whole")}
    for v, dtypes in KC.STAGED.items():
        for d in dtypes:
            precs = L.PRECISIONS if KC.is_single(d) and v in L.TF32_VARIANTS else ("",)
            paths = ("strip_store",) if v == L.VAR_KRED else ("scan", "strip_store")
            keys |= {("staged", KC.VARIANT_NAMES[v], d, p, path) for p in precs for path in paths}
    return keys


def key_id(key):
    """A test id for an instantiation key."""
    return "-".join(str(x) for x in key if x != "")


def stream_keys():
    """The 19 instantiations compiled only for strip_exponent (``STRIP = true``)."""
    return {k for k in required_keys() if k[0] in ("rowstream", "rowstream_k", "dmmastream")}


# ---------------------------------------------------------------------------- the sweep


# the DMMA stream kernel's 16-row warp blocks (nj = 8: 32 < N <= 64, K <= 32), which no case of the
# kernel-path table takes: 600 rows end in a half block, adjacent column pairs in C
EXTRA_CASES = [
    KC._case(L.VAR_DMMASTREAM, KC.C128, "ds_n40_k24_pair", dict(eq="xka,kc->xac", shapes=((3, 24, 200), (24, 40)),
                                                                  expect={"pair": True, "n_tile": 40})),
]


class Entry:
    """One sweep case: a kernel-path case and the precision its plan is built with."""

    def __init__(self, case, precision="3xtf32"):
        self.case, self.precision = case, precision
        self.id = case.id if precision == "3xtf32" else f"{precision}-{case.id}"

    def plan(self):
        return PC.build_plan(self.case, self.precision)


SWEEP = [Entry(c) for c in KC.CASES + EXTRA_CASES] + [Entry(c, "tf32") for c in PC.CASES]


def sweep_modes(entry, plan, launch_facts=None):
    """The stripped launches the sweep makes of a case after its plain one: always "scale"; "measure"
    and "both" where a plan could measure the launch in its epilogue and C0 is not added."""
    if measures_in_epilogue(entry.case, plan, launch_facts) and not entry.case.accumulate:
        return ("scale", "measure", "both")
    return ("scale",)


def sweep_keys(entry, plan):
    """The instantiations the sweep's stripped launches of one case run."""
    modes = sweep_modes(entry, plan)
    keys = {instantiation(entry.case, plan, scale=True)}
    if "measure" in modes:
        keys.add(instantiation(entry.case, plan, scale=False))
    return keys


# ---------------------------------------------------------------------------- targeted cases


def index_classes(case):
    """(contracted, kept in A, kept in B, batch) indices of a case's equation."""
    ta, tb, out = case.terms()
    con = [ix for ix in ta if ix in tb and ix not in out]
    keep_a = [ix for ix in ta if ix not in tb]
    keep_b = [ix for ix in tb if ix not in ta]
    batch = [ix for ix in ta if ix in tb and ix in out]
    return con, keep_a, keep_b, batch


def rank_one_ok(case):
    """Cases the rank-one operands are built for: no repeated index in a term, no zero stride, no
    index summed in one operand alone, no swap (the kernel's rows are then A's kept indices)."""
    ta, tb, out = case.terms()
    if len(set(ta)) != len(ta) or len(set(tb)) != len(tb) or any(ix not in ta + tb for ix in out):
        return False
    if any(ix not in out and not (ix in ta and ix in tb) for ix in ta + tb):
        return False
    if any(s is not None and 0 in s for s in case.strides):
        return False
    return not KC.build_plan(case).swapped


def _score(entry, plan):
    """Lower is better: a non-accumulating launch that measures (if the key can), one index of
    columns, a ragged last tile, small."""
    case = entry.case
    f = KC.plan_facts(plan)
    _con, keep_a, keep_b, batch = index_classes(case)
    cols = keep_a if plan.swapped else keep_b
    return (
        case.accumulate,
        not measures_in_epilogue(case, plan),
        plan.swapped,
        len(cols) != 1,
        bool(batch),
        case.out_strides is not None,
        not (f["pgm"] or f["odd_tail"] or not f["full_tiles"]),
        int(np.prod(case.out_shape())) * int(np.prod(case.shapes[0])),
        entry.id,
    )


def targeted_entries():
    """One sweep case per instantiation key, the best fit for rank-one operands."""
    best = {}
    for e in SWEEP:
        if not rank_one_ok(e.case):
            continue
        plan = e.plan()
        for key in sweep_keys(e, plan):
            sc = _score(e, plan)
            if key not in best or sc < best[key][0]:
                best[key] = (sc, e)
    return {key: e for key, (_sc, e) in sorted(best.items(), key=lambda kv: str(kv[0]))}


def measure_modes(key, entry, plan):
    """The modes the targeted measurements of ``key`` run in: the staged scan measures without
    scaling, its store path measures while scaling, a stream or wgmma kernel does both; launches a
    plan never measures in their epilogue get none."""
    if entry.case.accumulate or not measures_in_epilogue(entry.case, plan):
        return ()
    if key[0] == "staged":
        return ("measure",) if key[-1] == "scan" else ("both",)
    return ("measure", "both")


def scales(key):
    return not (key[0] == "staged" and key[-1] == "scan")


# the scale routes of the targeted tests: (name, fA, fB, exponent of 2 operand A and B are scaled by)
ROUTES_SINGLE = (
    ("float", FA, FB, 0, 0),
    ("double_above", 1e-16, 1e-16, -53, -53),   # s = 1e32: (float)((double)v * s)
    ("double_below", 1e16, 1e16, 53, 53),       # s = 1e-32
    ("zero", 0.0, FB, 0, 0),
)
ROUTES_DOUBLE = (
    ("double", FA, FB, 0, 0),
    ("two_overflow", 1.1 * 2.0 ** -512, 1.3 * 2.0 ** -513, -512, -513),  # (1/fA)(1/fB) > DBL_MAX
    ("two_underflow", 1.1 * 2.0 ** 540, 1.1 * 2.0 ** 540, 500, 500),     # (1/fA)(1/fB) == 0
    ("zero", 0.0, FB, 0, 0),
)


def routes(dtype):
    return ROUTES_SINGLE if KC.is_single(dtype) else ROUTES_DOUBLE


class RankOne:
    """Operands A = u x onehot(k0), B = w x onehot(k0) over a case's index classes, so that
    C = u (x) w over the kept indices (per batch index) and every product is exact: u and w hold
    small multiples of 1/16 (4 significant bits), which every kernel -- tf32 passes included --
    multiplies and sums without rounding."""

    def __init__(self, case, seed=0):
        self.case = case
        ta, tb, out = case.terms()
        self.ta, self.tb, self.out = ta, tb, out
        self.ext = dict(zip(ta + tb, tuple(case.shapes[0]) + tuple(case.shapes[1])))
        self.con, self.keep_a, self.keep_b, self.batch = index_classes(case)
        self.ua = [ix for ix in ta if ix not in self.con]   # axes of u (A's order)
        self.wb = [ix for ix in tb if ix not in self.con]   # axes of w (B's order)
        self.k0 = {ix: self.ext[ix] - 1 for ix in self.con}  # the last contracted element
        self.cplx = np.dtype(case.dtype).kind == "c"
        rng = np.random.default_rng(seed)
        self.u = self._background(rng, [self.ext[ix] for ix in self.ua])
        self.w = self._background(rng, [self.ext[ix] for ix in self.wb])
        self.nan_at = None

    def _background(self, rng, shape):
        def part():
            return rng.integers(1, 16, size=shape) / 16.0 * rng.choice([-1.0, 1.0], size=shape)
        x = part() + (1j * part() if self.cplx else 0)
        return np.asarray(x, dtype=np.complex128 if self.cplx else np.float64)

    # positions of C as {index: value}
    def rows(self):
        """The kernel's rows: A's kept and batch indices in C's order (fastest last)."""
        return [ix for ix in self.out if ix in self.ua]

    def cols(self):
        return [ix for ix in self.out if ix in self.keep_b]

    def at(self, row, col):
        """C position of flat row ``row`` and flat column ``col`` (C's index order, negatives from
        the end)."""
        pos = {}
        for names, flat in ((self.rows(), row), (self.cols(), col)):
            shape = [self.ext[ix] for ix in names]
            n = int(np.prod(shape))
            flat = flat % n
            pos.update(zip(names, np.unravel_index(flat, shape) if shape else ()))
        return {k: int(v) for k, v in pos.items()}

    def n_rows(self):
        return int(np.prod([self.ext[ix] for ix in self.rows()]))

    def n_cols(self):
        return int(np.prod([self.ext[ix] for ix in self.cols()]))

    def set_u(self, pos, value):
        self.u[tuple(pos[ix] for ix in self.ua)] = value

    def set_w(self, pos, value):
        self.w[tuple(pos[ix] for ix in self.wb)] = value

    def dominant(self, pos, value=4.0):
        """C[pos] = value^2, unique: every other element stays below 4 * 1.5 * value / 4."""
        self.set_u(pos, value)
        self.set_w(pos, value)

    def operands(self, scale_a=1.0, scale_b=1.0):
        dt = np.dtype(self.case.dtype)
        a = np.zeros([self.ext[ix] for ix in self.ta], dtype=self.u.dtype)
        b = np.zeros([self.ext[ix] for ix in self.tb], dtype=self.w.dtype)
        a[tuple(self.k0[ix] if ix in self.k0 else slice(None) for ix in self.ta)] = self.u * scale_a
        b[tuple(self.k0[ix] if ix in self.k0 else slice(None) for ix in self.tb)] = self.w * scale_b
        if self.nan_at is not None:
            a[self.nan_at] = np.nan
        return a.astype(dt), b.astype(dt)

    def poison(self):
        """One NaN in A inside the contracted range (not at k0, where B is 0): its C elements
        become NaN."""
        first = self.con[0] if self.con else None
        self.nan_at = tuple(0 if ix == first or ix not in self.k0 else self.k0[ix] for ix in self.ta)


def fill_layout(lay, case, a, b):
    """Writes operands ``a``, ``b`` into the described elements of a ``KC.make_layout`` layout."""
    out = []
    for which, x in ((0, a), (1, b)):
        strides = case.strides[which]
        strides = L.row_major_strides(case.shapes[which]) if strides is None else strides
        reach = KC._reach(case.shapes[which], strides)
        buf = lay.bufs[which]
        buf[lay.offs[which] + reach] = x
        out.append(buf[lay.offs[which] + reach])
    lay.ops = out
    return lay
