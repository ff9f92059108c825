"""The fused strip_exponent epilogue of every pairwise kernel, launch by launch, through
``ctgb_contract_pair`` with the descriptor words ``W_SCALE_A`` / ``W_SCALE_B`` pointing at device
doubles fA, fB and ``W_FACTOR_C`` at a factor slot (tests/strip_epilogue.py has the model).

* Sweep: every case of tests/kernel_cases.py (and its tensor-core cases with ``precision="tf32"``)
  in the same sentinel-guarded buffers as test_gpu_kernel_paths.py, launched plain and then
    - scaled by 1/(3.0 * 0.7): bit for bit the model applied to the plain result where one launch
      rounds each value once and adds no C0, else within the kernel-path bounds of s * product + C0;
    - measuring (where a plan measures the launch in its epilogue and C0 is not added): C bit for bit
      the plain result, the slot max|C| -- exactly for real types (sqrt of a correctly rounded square
      is |x|), within 2 ulps for complex ones;
    - both: the scaled C, and the slot its max.
  Sentinels stay bit-identical, operands untouched, no described element NaN.
* Targeted, one case per kernel instantiation: rank-one operands (C = u (x) w exactly, so the
  competing magnitudes are known) with a unique dominant element at the first, last, ragged-edge and
  second / fifth column positions; complex elements whose magnitude beats the running maximum while
  neither component does, in both processing orders; double outputs whose squares leave the double
  range; every scale route; zero factors and zero outputs; preloaded slots above and below max|C|;
  a NaN operand element.
* The measure-after rule of ``ctgb_plan_create`` agrees with ``measures_in_epilogue``.
"""

import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from cotengra_b200 import lowering as L  # noqa: E402
from tests import kernel_cases as KC  # noqa: E402
from tests import precision_cases as PC  # noqa: E402
from tests import strip_epilogue as S  # noqa: E402

SWEEP = {e.id: e for e in S.SWEEP}
TARGETS = S.targeted_entries()


def _launch(case, plan, lay, factors=None, slot=None):
    """One launch on fresh copies of the layout's buffers; returns (described C, slot bits or None)."""
    import torch

    from cotengra_b200 import _lib

    dev = [torch.from_numpy(b).cuda() for b in lay.bufs]
    es = np.dtype(case.dtype).itemsize
    ptr = [d.data_ptr() + off * es for d, off in zip(dev, lay.offs)]
    pa, pb = (ptr[1], ptr[0]) if plan.swapped else (ptr[0], ptr[1])
    words = plan.words.copy()
    fac = sl = None
    if factors is not None:
        # (strip_begin reads both factors whenever W_SCALE_A is set: always the two together)
        fac = torch.tensor(list(factors), dtype=torch.float64, device="cuda")
        words[L.W_SCALE_A], words[L.W_SCALE_B] = fac.data_ptr(), fac.data_ptr() + 8
    if slot is not None:
        sl = torch.tensor([slot], dtype=torch.float64, device="cuda")
        words[L.W_FACTOR_C] = sl.data_ptr()
    _lib.check(_lib.load().ctgb_contract_pair(words.ctypes.data, pa, pb, ptr[2], 0))
    torch.cuda.synchronize()
    for d, b in zip(dev[:2], lay.bufs[:2]):
        assert d.cpu().numpy().tobytes() == b.tobytes(), "operands changed"
    got, bad = KC.check_result(case, lay, dev[2].cpu().numpy())
    assert bad.size == 0, f"{bad.size} sentinel components outside C changed, first at {bad[:8]}"
    bits = None if sl is None else int(sl.cpu().numpy().view(np.uint64)[0])
    return got, bits


def _as_double(bits):
    return float(np.array([bits], dtype=np.uint64).view(np.float64)[0])


def _same_bits(got, want, what):
    got, want = np.ascontiguousarray(got), np.ascontiguousarray(want, dtype=got.dtype)
    rd = KC.real_dtype(got.dtype)
    ui = np.uint64 if rd.itemsize == 8 else np.uint32
    g, w = got.reshape(-1).view(rd).view(ui), want.reshape(-1).view(rd).view(ui)
    bad = np.flatnonzero(g != w)
    assert bad.size == 0, (f"{what}: {bad.size} of {g.size} components differ, first at {bad[:4]}: "
                           f"{g.view(rd)[bad[:4]]} vs {w.view(rd)[bad[:4]]}")


def _check_slot(bits, stored, what):
    """The slot holds max|stored| (0 for nothing stored): exactly for real values, within 2 ulps of
    hypot for complex ones."""
    slot, want = _as_double(bits), S.max_abs(stored)
    if np.asarray(stored).dtype.kind == "c":
        assert abs(slot - want) <= 2 * np.spacing(want), (what, slot, want)
    else:
        assert slot == want, (what, slot, want)


def _no_nan(got, what):
    assert not np.isnan(got).any(), f"{what}: {int(np.isnan(got).sum())} described C elements NaN"


def _product(case, lay, precision):
    """The product alone (no C0) in float64 / complex128, and the same over absolute values."""
    wd = KC.wide_dtype(case.dtype)
    a, b = ((PC.round_tf32(x) if precision == "tf32" else x).astype(wd) for x in lay.ops)
    return (np.asarray(np.einsum(case.eq, a, b, optimize=True)),
            np.asarray(np.einsum(case.eq, np.abs(a), np.abs(b), optimize=True)))


# ---------------------------------------------------------------------------- sweep


@pytest.mark.parametrize("eid", list(SWEEP))
def test_strip_sweep(eid):
    e = SWEEP[eid]
    case, plan = e.case, e.plan()
    dt = case.dtype
    lay = KC.make_layout(case, seed=zlib.crc32(case.id.encode()))
    plain, _ = _launch(case, plan, lay)
    _no_nan(plain, "plain")
    modes = S.sweep_modes(e, plan)

    got, _ = _launch(case, plan, lay, factors=(S.FA, S.FB))
    _no_nan(got, "scale")
    if S.deterministic(case, plan) and not case.accumulate:
        _same_bits(got, S.strip_expect(plain, S.FA, S.FB, dt), "scale")
    else:
        s = float(S.strip_factors(S.FA, S.FB)[0])
        p, absp = _product(case, lay, e.precision)
        wd = KC.wide_dtype(dt)
        c0 = lay.c0.astype(wd) if case.accumulate else np.zeros((), wd)
        ratio = KC.error_ratio(got, s * p + c0, s * absp + np.abs(c0))
        assert ratio <= (KC.C_SINGLE if KC.is_single(dt) else KC.C_DOUBLE), ratio

    if "measure" in modes:
        got, bits = _launch(case, plan, lay, slot=0.0)
        _same_bits(got, plain, "measure")
        _check_slot(bits, got, "measure")
    if "both" in modes:
        got, bits = _launch(case, plan, lay, factors=(S.FA, S.FB), slot=0.0)
        _same_bits(got, S.strip_expect(plain, S.FA, S.FB, dt), "both")
        _check_slot(bits, got, "both")


# ---------------------------------------------------------------------------- targeted


class _Target:
    def __init__(self, key):
        self.key, self.entry = key, TARGETS[key]
        self.case, self.plan = self.entry.case, self.entry.plan()
        self.dt = self.case.dtype
        self.seed = zlib.crc32(str(key).encode())
        self.cplx = np.dtype(self.dt).kind == "c"

    def rank_one(self):
        return S.RankOne(self.case, seed=self.seed)

    def expect(self, r1, mode, factors=(S.FA, S.FB), exps=(0, 0)):
        """The operands of ``r1`` (scaled by 2^exps) and what ``mode`` stores for them: the exact
        product, scaled in "scale" and "both"."""
        a, b = r1.operands(2.0 ** exps[0], 2.0 ** exps[1])
        wd = KC.wide_dtype(self.dt)
        with np.errstate(invalid="ignore"):
            exact = np.asarray(np.einsum(self.case.eq, a.astype(wd), b.astype(wd))).astype(self.dt)
        return a, b, (S.strip_expect(exact, *factors, self.dt) if mode in ("scale", "both") else exact)

    def run(self, r1, mode, factors=(S.FA, S.FB), exps=(0, 0), slot=0.0):
        """Launch rank-one operands in ``mode`` ("scale", "measure", "both"); returns (stored C,
        expected C, slot bits)."""
        a, b, want = self.expect(r1, mode, factors, exps)
        lay = S.fill_layout(KC.make_layout(self.case, seed=self.seed), self.case, a, b)
        scaled = mode in ("scale", "both")
        got, bits = _launch(self.case, self.plan, lay, factors=factors if scaled else None,
                            slot=slot if mode != "scale" else None)
        return got, want, bits


@pytest.mark.parametrize("key", list(TARGETS), ids=S.key_id)
def test_strip_targeted(key):
    t = _Target(key)
    modes = S.measure_modes(key, t.entry, t.plan)
    probe = t.rank_one()
    nr, nc = probe.n_rows(), probe.n_cols()

    for mode in modes:
        # a unique dominant element: first, last, last row at the second column (the second of a
        # pair / quad store), first row at the last column (the last column chunk), last row at the
        # first column, a middle row at the fifth column (c0 = 4 of the 16-byte row stream)
        for row, col in dict.fromkeys([(0, 0), (-1, -1), (-1, 1), (0, -1), (-1, 0), (nr // 2, min(4, nc - 1))]):
            r1 = t.rank_one()
            r1.dominant(r1.at(row, col))
            got, want, bits = t.run(r1, mode)
            what = f"{mode} dominant at row {row}, column {col}"
            _same_bits(got, want, what)
            _check_slot(bits, got, what)
            assert S.max_abs(got) == S.max_abs(got[tuple(r1.at(row, col)[ix] for ix in r1.out)]), what

        if t.cplx:
            # X = 16 (real) and Y = 13 (1 + i): |Y| > |X| although neither component of Y reaches 16,
            # the same thread's elements for one of the partner offsets, Y after X and before it
            for axis, d in (("col", 1), ("col", 4), ("col", 16), ("row", 1)):
                if (nc if axis == "col" else nr) <= d:
                    continue
                for order in (0, 1):
                    r1 = t.rank_one()
                    px, py = (0, d) if order == 0 else (d, 0)
                    if axis == "col":
                        x, y = r1.at(0, px), r1.at(0, py)
                        r1.set_u(x, 4.0)
                        r1.set_w(x, 4.0)
                        r1.set_w(y, 3.25 + 3.25j)
                    else:
                        x, y = r1.at(px, 0), r1.at(py, 0)
                        r1.set_w(x, 4.0)
                        r1.set_u(x, 4.0)
                        r1.set_u(y, 3.25 + 3.25j)
                    got, want, bits = t.run(r1, mode)
                    what = f"{mode} complex magnitude, {axis} partner {d}, order {order}"
                    _same_bits(got, want, what)
                    _check_slot(bits, got, what)

        if not KC.is_single(t.dt):
            # squares outside 1e-280..1e300: the hypot branch and its own maximum
            for e in (-240, 250):
                r1 = t.rank_one()
                r1.dominant(r1.at(-1, -1))
                got, want, bits = t.run(r1, mode, exps=(e, e))
                _same_bits(got, want, f"{mode} 2^{2 * e}")
                _check_slot(bits, got, f"{mode} 2^{2 * e}")

        # an all-zero output leaves a preloaded slot alone
        r1 = t.rank_one()
        r1.u[...] = 0
        got, want, bits = t.run(r1, mode, slot=0.5)
        _same_bits(got, want, f"{mode} zero output")
        assert _as_double(bits) == 0.5, (mode, "zero output", _as_double(bits))

        # a preloaded slot above max|C| stays, one below it is raised to max|C|
        for f in (2.0, 0.5):
            r1 = t.rank_one()
            r1.dominant(r1.at(-1, -1))
            want_max = S.max_abs(t.expect(r1, mode)[2])
            got, _want, bits = t.run(r1, mode, slot=f * want_max)
            if f > 1:
                assert _as_double(bits) == f * want_max, (mode, "slot above", _as_double(bits), want_max)
            else:
                _check_slot(bits, got, f"{mode} slot below")

        # one NaN operand element inside the contracted range: the slot reads the canonical NaN
        r1 = t.rank_one()
        r1.poison()
        got, want, bits = t.run(r1, mode)
        assert np.isnan(got).any(), (mode, "NaN operand")
        assert bits == S.QNAN_BITS, (mode, "NaN operand", hex(bits))
        keep = ~np.isnan(want)
        _same_bits(got[keep], want[keep], f"{mode} NaN operand, other elements")

    if S.scales(key):
        # every scale route, bit for bit: the operands carry the factors' magnitudes, so the scaled
        # values are normal numbers
        for name, fa, fb, ea, eb in S.routes(t.dt):
            assert S.strip_route(fa, fb, t.dt) == name.split("_")[0], name
            r1 = t.rank_one()
            r1.dominant(r1.at(-1, -1))
            got, want, _ = t.run(r1, "scale", factors=(fa, fb), exps=(ea, eb))
            if name == "zero":
                # (a launch that adds scaled partial sums -- to a memset C, or a chunk to the one
                # before -- turns -0 into +0: only the sign of one stored zero is the model's)
                if S.deterministic(t.case, t.plan):
                    _same_bits(got, want, f"scale route {name}")
                assert not np.any(got), "a zero factor leaves a nonzero value"
            else:
                _same_bits(got, want, f"scale route {name}")
                _no_nan(got, name)
                assert np.all(np.isfinite(got)) and S.max_abs(got) > 1e-30, (name, S.max_abs(got))


# ---------------------------------------------------------------------------- the plan's rule


_RULE_CASES = {
    # name: (equation, shapes, dtype, forced variant, measured in the epilogue)
    "epilogue": ("ab,bc->ac", ((2053, 24), (24, 67)), "float64", L.VAR_SIMT_64x64, True),
    "splitk": ("ab,bc->ac", ((31, 4219), (4219, 27)), "float64", L.VAR_DMMA_32x32, False),
    "dotstream": ("k,k->", ((6144,), (6144,)), "complex128", L.VAR_DOTSTREAM, False),
    "dotstream4": ("km,kn->nm", ((6144, 4), (6144, 3)), "float32", L.VAR_DOTSTREAM4, False),
    "kred": ("km,kn->nm", ((1500, 4), (1500, 2)), "complex64", L.VAR_KRED, False),
    "wgmma_chunked": ("ab,bc->ac", ((256, 272), (272, 64)), "complex64", L.VAR_TC05_128x64, False),
    "wgmma_whole": ("ab,bc->ac", ((256, 32), (32, 64)), "complex64", L.VAR_TC05_128x64, True),
}


@pytest.mark.parametrize("name", list(_RULE_CASES))
def test_measure_after_rule(name):
    import cotengra_b200 as cb

    eq, shapes, dtype, variant, epilogue = _RULE_CASES[name]
    (ta, tb), out = eq.split("->")[0].split(","), eq.split("->")[1]
    size = dict(zip(ta + tb, shapes[0] + shapes[1]))
    plan = cb.ExecPlan(((2, 0, 1, False, eq, None),), [tuple(ta), tuple(tb)], tuple(out), size,
                       dtype=dtype, strip_exponent=True, variant=variant)
    node = plan.nodes[0]["plan"]
    assert node.variant == variant
    case = KC.Case(variant, dtype, name, eq, shapes)
    assert S.measures_in_epilogue(case, node) == epilogue
    try:
        plan.create()
        (_prescale, measure_after), = plan.strip_modes()
    finally:
        plan.destroy()
    assert bool(measure_after) == (not epilogue)
