"""Host-side lowering (classification, coalescing, tiling, descriptor packing)
checked on the CPU through ``tests/desc_emulator.py`` against the golden values
of the unmodified reference and against numpy.einsum."""

import numpy as np
import pytest

from cotengra_b200 import lowering as L
from tests.desc_emulator import emulate_pair, emulate_single
from tests.helpers import load_json, load_npz, make_arrays, rel_err

PARSERS = load_json("parsers.json")
PVALS = load_npz("parsers_values.npz")
VARIANTS = [L.VAR_SIMT_64x64, L.VAR_DMMA_128x64, L.VAR_DMMA_64x128, L.VAR_DMMA_256x32,
            L.VAR_DMMA_256x16, L.VAR_ROW_128x8, L.VAR_ROW_256x4, L.VAR_ROWSTREAM, L.VAR_TC05_128x64, L.VAR_TC05_128x32, L.VAR_TC05_128x16,
            L.VAR_DMMA3M_128x32, L.VAR_DMMA3M_256x16, L.VAR_DMMASTREAM, L.VAR_DOTSTREAM]


def run_pair(eq, a, b, variant=None, splitk=None, sm_count=132):
    terms, out = L.split_equation(eq)
    dims = L.classify_pair(terms[0], a.shape, terms[1], b.shape, out)
    n_out = int(np.prod(dims.out_shape)) if dims.out_shape else 1
    plan = L.build_pair_desc(dims, str(a.dtype), sm_count=sm_count, variant=variant,
                             c_dense_elems=n_out, force_splitk=splitk)
    C = np.full(max(n_out, 1), np.nan, dtype=a.dtype)
    A, B = a.reshape(-1), b.reshape(-1)
    if plan.swapped:
        A, B = B, A
    if n_out:
        emulate_pair(plan.words, A, B, C)
    return C[:n_out].reshape(dims.out_shape), plan


def test_golden_pair_cases_all_variants():
    checked = 0
    for n, rec in enumerate(PARSERS["pair"]):
        sa, sb = tuple(rec["shape_a"]), tuple(rec["shape_b"])
        terms, out = L.split_equation(rec["eq"])
        if "error" in rec:
            with pytest.raises(ValueError):
                L.classify_pair(terms[0], sa, terms[1], sb, out)
            continue
        key = f"pair_{n}"
        if key not in PVALS:
            continue
        a, b = make_arrays([sa, sb], "complex128", seed=n)
        variant = VARIANTS[n % len(VARIANTS)]
        got, _ = run_pair(rec["eq"], a, b, variant=variant)
        want = PVALS[key]
        assert got.shape == want.shape, rec
        assert rel_err(got, want) < 1e-12, (rec, variant)
        checked += 1
    assert checked > 300


def _rand_eq(rng, dmax=7):
    letters = "abcdefghijkl"
    n_ix = int(rng.integers(2, 9))
    pool = list(rng.choice(list(letters), n_ix, replace=False))
    sizes = {c: int(rng.integers(1, dmax + 1)) for c in pool}
    ta = list(rng.permutation(pool)[: rng.integers(1, min(6, n_ix) + 1)])
    tb = list(rng.permutation(pool)[: rng.integers(1, min(6, n_ix) + 1)])
    present = list(dict.fromkeys(ta + tb))
    out = [c for c in present if rng.random() < 0.55]
    out = list(rng.permutation(out)) if out else []
    eq = f"{''.join(ta)},{''.join(tb)}->{''.join(out)}"
    return eq, tuple(sizes[c] for c in ta), tuple(sizes[c] for c in tb)


@pytest.mark.parametrize("seed", range(6))
def test_random_equations_vs_numpy(seed):
    rng = np.random.default_rng(seed)
    for trial in range(25):
        eq, sa, sb = _rand_eq(rng)
        a, b = make_arrays([sa, sb], "float64", seed=seed * 100 + trial)
        want = np.einsum(eq, a, b)
        for variant in (None, VARIANTS[trial % len(VARIANTS)]):
            for splitk in (None, 3):
                got, plan = run_pair(eq, a, b, variant=variant, splitk=splitk, sm_count=4)
                assert got.shape == want.shape
                assert rel_err(got, want) < 1e-12, (eq, sa, sb, variant, splitk)


def test_partial_tiles_and_large_dims():
    # extents that do not divide the tile: ragged last blocks in m, n and k
    for (m, n, k) in [(130, 70, 19), (257, 3, 33), (5, 300, 9), (64, 64, 8), (1, 1, 2500)]:
        a, b = make_arrays([(m, k), (k, n)], "complex128", seed=m + n + k)
        want = a @ b
        for variant in VARIANTS:
            got, plan = run_pair("ab,bc->ac", a, b, variant=variant)
            assert rel_err(got, want) < 1e-12, (m, n, k, variant)
    # dot product goes to the k-reduction variant with split-K
    a, b = make_arrays([(40, 300), (300, 40)], "complex128", seed=3)
    got, plan = run_pair("ab,ba->", a, b)
    assert plan.variant == L.VAR_KRED and plan.splitk > 1
    assert rel_err(got, np.einsum("ab,ba->", a, b)) < 1e-12


def test_rank30_permuted_operand_coalesces():
    # Sycamore-like: all dims 2, scattered contracted indices
    rng = np.random.default_rng(0)
    ixs = [chr(ord("a") + i) for i in range(14)]
    ta = list(rng.permutation(ixs))
    con = list(rng.choice(ixs, 4, replace=False))
    extra = ["A", "B", "C"]
    tb = list(rng.permutation(con + extra))
    out = [c for c in ta if c not in con] + [c for c in tb if c not in con]
    eq = f"{''.join(ta)},{''.join(tb)}->{''.join(out)}"
    a, b = make_arrays([(2,) * len(ta), (2,) * len(tb)], "complex128", seed=1)
    want = np.einsum(eq, a, b)
    for variant in VARIANTS:
        got, plan = run_pair(eq, a, b, variant=variant)
        assert rel_err(got, want) < 1e-12


def test_tensordot_terms_match_numpy():
    rng = np.random.default_rng(4)
    for trial in range(60):
        na, nb = int(rng.integers(0, 5)), int(rng.integers(0, 5))
        nc = int(rng.integers(0, min(na, nb) + 1))
        ax_a = tuple(int(x) for x in rng.choice(na, nc, replace=False)) if nc else ()
        ax_b = tuple(int(x) for x in rng.choice(nb, nc, replace=False)) if nc else ()
        sa = [int(rng.integers(1, 4)) for _ in range(na)]
        sb = [int(rng.integers(1, 4)) for _ in range(nb)]
        for i, j in zip(ax_a, ax_b):
            sb[j] = sa[i]
        a, b = make_arrays([sa, sb], "float64", seed=trial)
        want = np.tensordot(a, b, (ax_a, ax_b))
        perm = tuple(int(x) for x in rng.permutation(want.ndim)) if want.ndim else None
        ta, tb, to = L.tensordot_terms((ax_a, ax_b), na, nb, perm)
        dims = L.classify_pair(ta, a.shape, tb, b.shape, to)
        plan = L.build_pair_desc(dims, "float64", c_dense_elems=max(want.size, 1))
        C = np.zeros(max(want.size, 1))
        A, B = (b.reshape(-1), a.reshape(-1)) if plan.swapped else (a.reshape(-1), b.reshape(-1))
        emulate_pair(plan.words, A, B, C)
        if perm is not None:
            want = np.transpose(want, perm)
        assert dims.out_shape == want.shape
        assert rel_err(C[: want.size].reshape(want.shape), want) < 1e-12
    with pytest.raises(ValueError):
        L.check_tensordot_shapes(((0,), (0,)), (2, 3), (3, 2))
    with pytest.raises(ValueError):
        L.tensordot_terms(((0, 1), (0,)), 2, 2)


def test_single_operand_cases():
    for n, rec in enumerate(PARSERS["single"]):
        shape = tuple(rec["shape"])
        (x,) = make_arrays([shape], "complex128", seed=1000 + n)
        terms, out = L.split_equation(rec["eq"])
        odims, sdims, oshape = L.classify_single(terms[0], shape, out)
        W = L.build_single_desc(odims, sdims, "complex128")
        want = PVALS[f"single_{n}"]
        res = np.zeros(max(want.size, 1), dtype=np.complex128)
        emulate_single(W, x.reshape(-1), res)
        assert tuple(oshape) == want.shape
        assert rel_err(res[: want.size].reshape(want.shape), want) < 1e-12, rec


def test_errors_match_reference():
    with pytest.raises(ValueError):
        L.classify_pair("ab", (2, 3), "bc", (4, 2), "ac")  # mismatched b
    with pytest.raises(ValueError):
        L.classify_pair("ab", (2,), "bc", (2, 2), "ac")  # term vs shape
    with pytest.raises(NotImplementedError):
        L.split_equation("a...,b->")
    with pytest.raises(TypeError):
        L.dtype_name("int32")


def test_tcgen05_descriptor_properties():
    """Host side of the tcgen05 complex64 kernel (tc05_kernel.cuh): exact tiles, TMA run
    flag, chunk-stride padding -- on permuted power-of-two layouts like the Sycamore nodes,
    with the data path checked through the emulator."""
    rng = np.random.default_rng(5)
    seen_bulk = seen_gather = 0
    for trial in range(40):
        nm, nk, nn = int(rng.integers(10, 13)), int(rng.integers(4, 7)), int(rng.integers(4, 8))
        m_ix = [chr(ord("a") + i) for i in range(nm)]
        k_ix = [chr(ord("A") + i) for i in range(nk)]
        n_ix = [chr(ord("n") + i) for i in range(nn)]
        ta = list(rng.permutation(m_ix + k_ix))
        tb = list(rng.permutation(k_ix + n_ix))
        out = list(rng.permutation(m_ix + n_ix))
        if trial % 5 == 4:
            ta = ta + ["z"]  # a trailing batch index of extent 3: odd strides, no TMA runs
            tb = tb + ["z"]
            out = out + ["z"]
        sizes = {c: 2 for c in m_ix + k_ix + n_ix}
        sizes["z"] = 3
        sa, sb = tuple(sizes[c] for c in ta), tuple(sizes[c] for c in tb)
        dims = L.classify_pair("".join(ta), sa, "".join(tb), sb, "".join(out))
        plan = L.build_pair_desc(dims, "complex64", sm_count=132, c_dense_elems=1, force_splitk=1)
        W = plan.words
        if plan.variant not in L.TC05_VARIANTS:
            continue
        MT, NT, KT = L.VARIANT_TILES[plan.variant]
        assert (W[L.W_MTA], W[L.W_NTA], W[L.W_KTA]) == (MT, NT, KT)
        run_a, pad, bulk = int(W[34]), int(W[35]), bool(W[L.W_FLAGS] & 64)
        assert pad in (0, 1, 2, 4)
        n_lda = int(W[L.W_NLDA])
        lda = [tuple(int(x) for x in W[L.OFF_LDA + 4 * i:L.OFF_LDA + 4 * i + 4]) for i in range(n_lda)]
        # the run is the dense prefix of A's load order
        prod = 1
        for ext, stride, _wr, _wk in lda:
            if stride != prod:
                break
            prod *= ext
        assert prod == run_a
        if bulk:
            seen_bulk += 1
            assert run_a >= 16 and run_a % 2 == 0 and (MT * KT) % run_a == 0
            assert all(s % 2 == 0 for _e, s, _r, _k in lda if s >= run_a)
        else:
            seen_gather += 1
        # every (row, k) position of the tile is hit exactly once by the load order
        pos = set()
        for e in range(MT * KT):
            r = kk = 0
            x = e
            for ext, _s, wr, wk in lda:
                r += (x % ext) * wr
                kk += (x % ext) * wk
                x //= ext
            pos.add((r, kk))
        assert len(pos) == MT * KT and max(p[0] for p in pos) == MT - 1 and max(p[1] for p in pos) == KT - 1
        if trial % 8 == 3:  # the data path of a few of them (emulator)
            a, b = make_arrays([sa, sb], "complex128", seed=trial)
            got, _ = run_pair("".join(ta) + "," + "".join(tb) + "->" + "".join(out), a.astype(np.complex64),
                              b.astype(np.complex64), variant=plan.variant, splitk=1)
            want = np.einsum("".join(ta) + "," + "".join(tb) + "->" + "".join(out), a, b)
            assert rel_err(got, want) < 1e-5
    assert seen_bulk >= 10 and seen_gather >= 3, (seen_bulk, seen_gather)


@pytest.mark.parametrize("variant,dtype,mn", [
    (L.VAR_DOTSTREAM4, "complex128", (4, 3)), (L.VAR_DOTSTREAM4, "complex64", (2, 4)),
    (L.VAR_DMMA_32x32, "complex128", (32, 20)), (L.VAR_DMMA_32x32, "complex128", (32, 32)),
    (L.VAR_DMMA_32x32, "float64", (24, 32)),
])
def test_small_result_long_k_descriptors(variant, dtype, mn):
    """The dot-type variants stem fusion produces (a small kept space on both operands over a
    long, permuted contracted space): descriptor addressing through the emulator vs einsum."""
    from tests.desc_emulator import emulate_pair

    M, N = mn
    shape_a = (4, 16, M, 2, 64)        # a, b, m, c, d     K = 4*16*2*64 = 8192
    shape_b = (64, N, 2, 4, 16)        # d, n, c, a, b
    a, b = make_arrays([shape_a, shape_b], dtype, seed=2)
    dims = L.classify_pair("abmcd", shape_a, "dncab", shape_b, "mn")
    plan = L.build_pair_desc(dims, dtype, c_dense_elems=M * N, variant=variant, force_splitk=4 if variant == L.VAR_DMMA_32x32 else None)
    assert plan.variant == variant
    x, y = (b, a) if plan.swapped else (a, b)
    out = np.full(M * N, 7, dtype=dtype)
    emulate_pair(plan.words, x.reshape(-1), y.reshape(-1), out)
    want = np.einsum("abmcd,dncab->mn", a, b)
    assert rel_err(out.reshape(M, N), want) < (1e-12 if "128" in dtype or dtype == "float64" else 1e-5)


@pytest.mark.parametrize("eq,sa,sb", [
    ("abcdefgh,bdfgxy->acehxy", (6, 6, 6, 6, 6, 6, 6, 36), (6, 6, 6, 6, 6, 36)),   # the PEPS top-node pattern
    ("mk,kn->mn", (1296, 216), (216, 216)),
    ("km,kn->mn", (72, 1296), (72, 54)),
    ("amb,bna->mn", (3, 640, 12), (12, 96, 3)),                                      # mixed 2^a 3^b 5 extents
    ("mk,kn->mn", (2560, 40), (40, 96)),
])
def test_tcgen05_tiles_on_extents_that_are_not_powers_of_two(eq, sa, sb):
    """complex64 nodes on 6^n-like extents go to the tcgen05 kernel with EQUAL tiles (divisors of the
    index classes) inside the 128 x NT x 16 tensor-core tile: the tiles cover the node exactly, fill at
    least 40 % of the tensor-core tile in M x N, k is a multiple of 4 (whole UMMA k8 groups), and the
    descriptor addresses the right elements (emulator against einsum)."""
    a, b = make_arrays([sa, sb], "complex128", seed=3)
    terms, out = L.split_equation(eq)
    dims = L.classify_pair(terms[0], sa, terms[1], sb, out)
    n_out = int(np.prod(dims.out_shape))
    plan = L.build_pair_desc(dims, "complex64", sm_count=132, c_dense_elems=n_out)
    assert plan.variant in L.TC05_VARIANTS, plan.variant
    W = plan.words
    MT, NT, KT = L.VARIANT_TILES[plan.variant]
    Bn, M, N, K = plan.sizes
    MTa, NTa, KTa = int(W[L.W_MTA]), int(W[L.W_NTA]), int(W[L.W_KTA])
    assert MTa <= MT and NTa <= NT and KTa <= KT and KTa % 4 == 0
    assert MTa * int(W[L.W_TILES_M]) == M and NTa * int(W[L.W_TILES_N]) == N and KTa * int(W[L.W_STEPS_K]) == K
    assert MTa * NTa >= 0.4 * MT * NT
    assert int(W[L.W_STEPS_K]) <= 1024
    got, _ = run_pair(eq, a.astype(np.complex64), b.astype(np.complex64))
    assert rel_err(got, np.einsum(eq, a, b)) < 1e-5


def test_tcgen05_refuses_what_it_cannot_tile():
    """Extents without a usable divisor (primes), too few rows or columns, or a contracted range beyond
    the 1024 tabulated k-steps stay on the staged mma.sync / FMA kernels."""
    for eq, sa, sb in [("mk,kn->mn", (127 * 4, 64), (64, 64)),       # M = 4 * 127: largest divisor <= 128 is 127 -> ragged k? no: 127 rows ok
                       ("mk,kn->mn", (1024, 64), (64, 7)),            # N = 7 < 12
                       ("mk,kn->mn", (64, 64), (64, 64)),             # M < 128
                       ("mk,kn->mn", (1024, 13), (13, 64)),           # K = 13: no multiple of 4 divides it
                       ("mk,kn->mn", (256, 32768), (32768, 64))]:     # K > 16384
        terms, out = L.split_equation(eq)
        dims = L.classify_pair(terms[0], sa, terms[1], sb, out)
        plan = L.build_pair_desc(dims, "complex64", sm_count=132, c_dense_elems=int(np.prod(dims.out_shape)))
        if plan.variant in L.TC05_VARIANTS:
            # whatever it accepted must still be an exact, sufficiently full tiling
            W = plan.words
            MT, NT, _KT = L.VARIANT_TILES[plan.variant]
            Bn, M, N, K = plan.sizes
            assert int(W[L.W_MTA]) * int(W[L.W_TILES_M]) == M and int(W[L.W_NTA]) * int(W[L.W_TILES_N]) == N
            assert int(W[L.W_KTA]) * int(W[L.W_STEPS_K]) == K and int(W[L.W_KTA]) % 4 == 0
            assert int(W[L.W_MTA]) * int(W[L.W_NTA]) >= 0.4 * MT * NT and int(W[L.W_STEPS_K]) <= 1024
            assert (eq, sa) == ("mk,kn->mn", (127 * 4, 64)), (eq, sa, sb)


def test_tcgen05_random_layouts_on_mixed_radix_extents():
    """Random permuted layouts with extents drawn from {2, 3, 4, 6, 12}: whenever the lowering hands a
    complex64 node to the tcgen05 kernel the tiles are exact, every (row, k) position of the real tile is
    hit exactly once by A's load order, and the emulated data path agrees with einsum."""
    rng = np.random.default_rng(17)
    taken = checked = 0
    for trial in range(60):
        nm, nk, nn = int(rng.integers(3, 6)), int(rng.integers(1, 4)), int(rng.integers(1, 4))
        m_ix = [chr(ord("a") + i) for i in range(nm)]
        k_ix = [chr(ord("A") + i) for i in range(nk)]
        n_ix = [chr(ord("n") + i) for i in range(nn)]
        sizes = {c: int(rng.choice([2, 3, 4, 6, 12])) for c in m_ix + k_ix + n_ix}
        M = int(np.prod([sizes[c] for c in m_ix]))
        if M < 128 or M > 20000:
            continue
        ta = list(rng.permutation(m_ix + k_ix))
        tb = list(rng.permutation(k_ix + n_ix))
        out = list(rng.permutation(m_ix + n_ix))
        sa, sb = tuple(sizes[c] for c in ta), tuple(sizes[c] for c in tb)
        eq = "".join(ta) + "," + "".join(tb) + "->" + "".join(out)
        dims = L.classify_pair("".join(ta), sa, "".join(tb), sb, "".join(out))
        n_out = int(np.prod(dims.out_shape))
        plan = L.build_pair_desc(dims, "complex64", sm_count=132, c_dense_elems=n_out)
        if plan.variant not in L.TC05_VARIANTS:
            continue
        taken += 1
        W = plan.words
        MT, NT, KT = L.VARIANT_TILES[plan.variant]
        Bn, Mp, Np, Kp = plan.sizes
        MTa, NTa, KTa = int(W[L.W_MTA]), int(W[L.W_NTA]), int(W[L.W_KTA])
        assert MTa * int(W[L.W_TILES_M]) == Mp and NTa * int(W[L.W_TILES_N]) == Np and KTa * int(W[L.W_STEPS_K]) == Kp
        assert KTa % 4 == 0 and MTa <= MT and NTa <= NT and KTa <= KT and MTa * NTa >= 0.4 * MT * NT
        n_lda = int(W[L.W_NLDA])
        lda = [tuple(int(x) for x in W[L.OFF_LDA + 4 * i:L.OFF_LDA + 4 * i + 4]) for i in range(n_lda)]
        pos = set()
        for e in range(MTa * KTa):
            r = kk = 0
            x = e
            for ext, _s, wr, wk in lda:
                r += (x % ext) * wr
                kk += (x % ext) * wk
                x //= ext
            pos.add((r, kk))
        assert len(pos) == MTa * KTa and max(p[0] for p in pos) == MTa - 1 and max(p[1] for p in pos) == KTa - 1
        if checked < 12:
            checked += 1
            a, b = make_arrays([sa, sb], "complex128", seed=trial)
            got, _ = run_pair(eq, a.astype(np.complex64), b.astype(np.complex64))
            assert rel_err(got, np.einsum(eq, a, b)) < 1e-5, eq
    assert taken >= 8 and checked >= 8, (taken, checked)
