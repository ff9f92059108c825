"""The absorb-root kernel (csrc/absorbdot.cuh) on the GPU: R = (A . Bs) . V without forming A . Bs.

Every case runs through ``ctgb_absorb_root`` in guarded buffers (NaN sentinels before and after each
operand and around C) against a complex128 einsum, within 1e-14 |A| |Bs| |V| per element; the fused
Sycamore-m20 slice is checked against its golden amplitude."""

import string

import numpy as np
import pytest

from cotengra_b200 import lowering as L

pytestmark = pytest.mark.gpu

GUARD = 64


def _case(seed, groups, ext=2):
    """Random index orders for A[rows, k', k], Bs[k, cc, ck], V[k', cc, n] and the two outputs."""
    rng = np.random.default_rng(seed)
    letters = iter(string.ascii_letters)
    names = {g: [next(letters) for _ in range(len(sz))] for g, sz in groups.items()}
    size = {ix: s for g, sz in groups.items() for ix, s in zip(names[g], sz)}

    def shuf(*gs):
        t = [ix for g in gs for ix in names[g]]
        rng.shuffle(t)
        return "".join(t)

    ta, tb, tv = shuf("rows", "kp", "k"), shuf("k", "cc", "ck"), shuf("kp", "cc", "n")
    tx, tr = shuf("rows", "kp", "cc", "ck"), shuf("n", "rows", "ck")

    def cr(t):
        s = tuple(size[ix] for ix in t)
        return rng.standard_normal(s) + 1j * rng.standard_normal(s)

    return (ta, tb, tv, tx, tr), cr(ta), cr(tb), cr(tv)


def _guarded(torch, x):
    n = x.size
    buf = torch.full((n + 2 * GUARD,), complex(float("nan"), float("nan")), dtype=torch.complex128, device="cuda")
    if n:
        buf[GUARD:GUARD + n] = torch.from_numpy(np.ascontiguousarray(x).reshape(-1)).cuda()
    return buf


def _run(terms, A, Bs, V, x_is_a, accumulate=False):
    import torch

    from cotengra_b200 import _lib

    ta, tb, tv, tx, tr = terms
    X = np.einsum(f"{ta},{tb}->{tx}", A, Bs)
    want = np.einsum(f"{tv},{tx}->{tr}", V, X) if not x_is_a else np.einsum(f"{tx},{tv}->{tr}", X, V)
    want = want.reshape(-1)
    dp = L.classify_pair(ta, A.shape, tb, Bs.shape, tx)
    if x_is_a:
        dr = L.classify_pair(tx, X.shape, tv, V.shape, tr)
    else:
        dr = L.classify_pair(tv, V.shape, tx, X.shape, tr)
    ab = L.build_absorb_desc(dp, dr, x_is_a, accumulate=accumulate, c_dense_elems=want.size)
    assert ab is not None
    ga, gb, gv = (_guarded(torch, x) for x in (A, Bs, V))
    c0 = np.arange(want.size) * (1 + 1j) if accumulate else np.zeros(want.size)
    gc = _guarded(torch, c0)
    ptr = lambda b: b.data_ptr() + GUARD * 16  # noqa: E731
    _lib.check(_lib.load().ctgb_absorb_root(ab.words.ctypes.data, ptr(ga), ptr(gb), ptr(gv), ptr(gc), None))
    torch.cuda.synchronize()
    got = gc.cpu().numpy()
    assert np.isnan(got[:GUARD]).all() and np.isnan(got[GUARD + want.size:]).all()
    got = got[GUARD:GUARD + want.size] - c0
    for g, x in ((ga, A), (gb, Bs), (gv, V)):
        h = g.cpu().numpy()
        assert np.isnan(h[:GUARD]).all() and np.isnan(h[GUARD + x.size:]).all()
    scale = np.abs(A).max() * np.abs(Bs).max() * np.abs(V).max() * (X.size // max(want.size, 1) + 1) * 16
    err = np.abs(got - want).max()
    assert err <= 1e-14 * scale, (err, scale, ab.words[L.AB_M:L.AB_CCP + 1])
    return ab


@pytest.mark.parametrize("seed,x_is_a", [(1, False), (2, True), (3, False)])
def test_binary_dims_with_kept_bs_columns(seed, x_is_a):
    """All extents 2, as on the Sycamore stems: 3 row dims, 2 kept and 5 contracted Bs columns."""
    groups = {"rows": (2,) * 3, "ck": (2,) * 2, "cc": (2,) * 5, "kp": (2,) * 9, "k": (2,) * 4, "n": (2,) * 5}
    terms, A, Bs, V = _case(seed, groups)
    ab = _run(terms, A, Bs, V, x_is_a)
    assert int(ab.words[L.AB_KL]) == 2


@pytest.mark.parametrize("kp", [(1000,), (37, 3), (2, 129)])
def test_ragged_units(kp):
    """k' ranges that split unevenly over the CTAs, rows without kept Bs columns, C < 32."""
    groups = {"rows": (20,), "ck": (), "cc": (24,), "kp": kp, "k": (12,), "n": (30,)}
    terms, A, Bs, V = _case(7, groups)
    _run(terms, A, Bs, V, False)


def test_exact_units_accumulate():
    groups = {"rows": (4, 2), "ck": (2, 2), "cc": (32,), "kp": (2,) * 10, "k": (16,), "n": (32,)}
    terms, A, Bs, V = _case(11, groups)
    _run(terms, A, Bs, V, True, accumulate=True)


@pytest.mark.parametrize("key", ["appxB_w30_slice0", "appxB_w28_slice0"])
def test_fused_m20_slice_matches_golden(key):
    """The fused Sycamore-m20 complex128 slice, whose plan has one absorb-root node, against the
    oracle's value in big_slices.json."""
    import torch

    import cotengra_b200 as cb
    from tests.helpers import load_json, make_arrays
    from tests.slicing_util import appxB_at_width

    g = load_json("big_slices.json")[key]
    spec = appxB_at_width(g["width_log2"])
    ex = cb.TreeExecutor(spec, dtype="complex128")
    assert sum(1 for nd in ex.plan.nodes if nd.get("d") is not None) == 1
    arrays = make_arrays(spec.shapes(), "complex128", seed=g["seed"], scale=g["scale"])
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    got = complex(ex.contract_device(dev, begin=g["slice_id"], step=1, count=1).cpu().numpy().reshape(-1)[0])
    want = complex(g["re"], g["im"])
    assert abs(got - want) / abs(want) < 1e-10, (got, want)
    del ex, dev
    torch.cuda.empty_cache()
