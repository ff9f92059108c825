"""The strip_exponent epilogue model and case selection of tests/strip_epilogue.py without a GPU.

* ``strip_expect`` takes the route ``strip_begin`` takes, on both sides of every threshold: a zero
  factor, the single types' float multiply inside 1e-30..1e30 and the double fallback outside, the
  ``two`` route where (1/fA)(1/fB) leaves the double range (above 1.7e308, or 0);
* the sweep of test_gpu_strip_epilogue.py reaches every kernel instantiation a stripped launch can
  run -- the 19 stream instantiations compiled for strip_exponent alone among them -- and the
  targeted tests have a rank-one case for each;
* the rank-one operands give a unique, exactly known dominant element.
"""

import collections

import numpy as np
import pytest

from cotengra_b200 import lowering as L
from tests import kernel_cases as KC
from tests import precision_cases as PC
from tests import strip_epilogue as S

# (fA, fB, dtype, route), derived by hand from strip_begin
ROUTES = [
    (3.0, 0.7, KC.F32, "float"),
    (3.0, 0.7, KC.F64, "double"),
    (3.0, 0.7, KC.C64, "float"),
    (3.0, 0.7, KC.C128, "double"),
    # |s| around 1e30 and 1e-30: the single types' float multiply inside, the double one outside
    (1e-15, 1.001e-15, KC.F32, "float"),      # s = 0.999e30
    (1e-15, 0.999e-15, KC.F32, "double"),     # s = 1.001e30
    (1e15, 0.999e15, KC.C64, "float"),        # s = 1.001e-30
    (1e15, 1.001e15, KC.C64, "double"),       # s = 0.999e-30
    (1e-15, 0.999e-15, KC.F64, "double"),     # (the double types always multiply by s)
    # (1/fA)(1/fB) against 1.7e308: below it one multiply, above it (finite or not) two
    (1.0, 1 / 1.65e308, KC.F64, "double"),
    (1.0, 1 / 1.75e308, KC.F64, "two"),
    (2.0 ** -511, 2.0 ** -512, KC.C128, "double"),   # 2^1023
    (2.0 ** -512, 2.0 ** -512, KC.C128, "two"),      # 2^1024: overflows
    (2.0 ** -512, 2.0 ** -512, KC.F32, "two"),
    # ... and against 0: 2^-1074 is the least subnormal, 2^-1080 rounds to 0
    (2.0 ** 537, 2.0 ** 537, KC.F64, "double"),
    (2.0 ** 540, 2.0 ** 540, KC.F64, "two"),
    (2.0 ** 540, 2.0 ** 540, KC.C64, "two"),
    # a zero factor: s = 0, whatever the other one is
    (0.0, 0.7, KC.F32, "zero"),
    (3.0, 0.0, KC.C128, "zero"),
    (0.0, 2.0 ** -600, KC.F64, "zero"),
]


@pytest.mark.parametrize("fa,fb,dtype,route", ROUTES)
def test_strip_route(fa, fb, dtype, route):
    assert S.strip_route(fa, fb, dtype) == route


def test_strip_expect_values():
    # the float route: one float multiply by (float)((1/3)(1/0.7)), components separately
    s = (1.0 / 3.0) * (1.0 / 0.7)
    x = np.array([1.5 - 0.25j, -3.0 + 7.0j], dtype=np.complex64)
    got = S.strip_expect(x, 3.0, 0.7, KC.C64)
    want = (x.view(np.float32) * np.float32(s)).view(np.complex64)
    assert got.tobytes() == want.tobytes()
    # the double fallback rounds once from double: not the same as the float multiply
    x = np.array([1.0000001, 3.3333333], dtype=np.float32)
    s2 = (1.0 / 1e-15) * (1.0 / 0.999e-15)
    got = S.strip_expect(x, 1e-15, 0.999e-15, KC.F32)
    assert got.tobytes() == (x.astype(np.float64) * s2).astype(np.float32).tobytes()
    # the two route multiplies by 1/fA, then by 1/fB: 2^-1030 * 2^512 * 2^520 = 4 (one multiply
    # by 2^1032 would overflow first)
    got = S.strip_expect(np.array([2.0 ** -1030]), 2.0 ** -512, 2.0 ** -520, KC.F64)
    assert got[0] == 4.0
    # a zero factor stores signed zeros; inf and NaN stay NaN
    got = S.strip_expect(np.array([-2.0, 5.0, np.inf], dtype=np.float32), 0.0, 1.0, KC.F32)
    assert got[0] == 0 and np.signbit(got[0]) and got[1] == 0 and not np.signbit(got[1]) and np.isnan(got[2])


def test_max_abs():
    assert S.max_abs(np.array([3 + 4j, -1j], dtype=np.complex64)) == 5.0
    assert S.max_abs(np.array([-7.0, 2.0])) == 7.0
    assert S.max_abs(np.zeros(0)) == 0.0


def test_sweep_reaches_every_instantiation():
    need = S.required_keys()
    assert len(S.stream_keys()) == 19  # 12 row-stream, 3 long-k, 4 DMMA-stream STRIP instantiations
    seen = collections.Counter()
    for e in S.SWEEP:
        for key in S.sweep_keys(e, e.plan()):
            seen[key] += 1
    missing = sorted(need - set(seen), key=str)
    assert not missing, f"instantiations the sweep never runs: {missing}"
    assert set(seen) <= need, sorted(set(seen) - need, key=str)


def test_targeted_cases_cover_every_instantiation():
    targets = S.targeted_entries()
    assert set(targets) == S.required_keys(), sorted(S.required_keys() ^ set(targets), key=str)
    for key, e in targets.items():
        plan = e.plan()
        assert key in S.sweep_keys(e, plan)
        assert not e.case.accumulate and S.rank_one_ok(e.case), key
        # a launch a plan measures in its epilogue is measured (the staged store path while scaling)
        if S.measures_in_epilogue(e.case, plan):
            assert S.measure_modes(key, e, plan), key


def test_sweep_has_every_measure_after_class():
    """The launches a plan measures afterwards are swept (scaled only): split-K, the two dot streams,
    KRED and chunked wgmma launches."""
    classes = collections.Counter()
    for e in S.SWEEP:
        plan = e.plan()
        if S.measures_in_epilogue(e.case, plan):
            assert S.deterministic(e.case, plan)
            continue
        assert S.sweep_modes(e, plan) == ("scale",)
        v = plan.variant
        if plan.splitk > 1:
            classes["splitk"] += 1
        if v in L.DOTSTREAM_VARIANTS or v == L.VAR_KRED:
            classes[KC.VARIANT_NAMES[v]] += 1
        if v in L.TC05_VARIANTS and plan.splitk == 1:
            classes["wgmma_chunked"] += 1
    assert set(classes) == {"splitk", "DOTSTREAM", "DOTSTREAM4", "KRED", "wgmma_chunked"}, classes


@pytest.mark.parametrize("key", list(S.targeted_entries()), ids=S.key_id)
def test_rank_one_operands(key):
    """C = u (x) w exactly, with the dominant element unique and at its position, and every operand
    value exact on the tf32 grid (so no tensor-core pass rounds it)."""
    e = S.targeted_entries()[key]
    case = e.case
    r1 = S.RankOne(case, seed=1)
    pos = r1.at(-1, 1 if r1.n_cols() > 1 else 0)
    r1.dominant(pos)
    a, b = r1.operands()
    if KC.is_single(case.dtype):
        assert PC.round_tf32(a).tobytes() == a.tobytes() and PC.round_tf32(b).tobytes() == b.tobytes()
    wd = KC.wide_dtype(case.dtype)
    c = np.einsum(case.eq, a.astype(wd), b.astype(wd))
    at = tuple(pos[ix] for ix in r1.out)
    assert c[at] == 16.0
    mags = np.abs(c).reshape(-1)
    assert np.sum(mags == 16.0) == 1 and (mags.size == 1 or np.sort(mags)[-2] < 8.0)
    assert np.array_equal(c.astype(case.dtype).astype(wd), c)  # representable: the kernels form it exactly
    r1.poison()
    a, _b = r1.operands()
    assert np.isnan(a).sum() == 1
