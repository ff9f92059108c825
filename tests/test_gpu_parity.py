"""GPU parity tests proper: the sm_90a kernels, called through the C-ABI,
against (a) the golden vectors of the unmodified reference, (b) the numpy oracle
on the same seeded inputs, and (c) size-independent properties at large sizes.

Tolerances (BASELINE.json north_star): complex128/float64 <= 1e-10 relative,
complex64/float32 <= 1e-5 relative (judged against the float64-class result),
integer index work bit-exact (covered by the CPU suite)."""

import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from oracle import ctg_oracle as orc  # noqa: E402
from tests.helpers import (  # noqa: E402
    decode_ir,
    decode_sliced,
    load_json,
    load_npz,
    make_arrays,
    rel_err,
)

TOL = {"float32": 1e-5, "complex64": 1e-5, "float64": 1e-10, "complex128": 1e-10}
PARSERS = load_json("parsers.json")
PVALS = load_npz("parsers_values.npz")
TREES = load_json("trees.json")
TVALS = load_npz("trees_values.npz")


def _cast(x, dtype):
    dtype = np.dtype(dtype)
    if dtype.kind != "c":
        x = np.real(x)
    return np.asarray(x, order="C").astype(dtype)


def test_native_library_is_loaded_and_launches():
    from cotengra_b200 import _lib

    info = _lib.device_info()
    assert info["sm_count"] > 0
    before = _lib.launch_count()
    a, b = make_arrays([(8, 8), (8, 8)], "complex128", seed=1)
    got = cb.einsum("ab,bc->ac", a, b)
    assert _lib.launch_count() > before
    assert rel_err(got, a @ b) < 1e-12


@pytest.mark.parametrize("dtype", ["complex128", "complex64", "float64", "float32"])
def test_pair_cases_golden(dtype):
    n_ok = 0
    for n, rec in enumerate(PARSERS["pair"]):
        key = f"pair_{n}"
        if key not in PVALS:
            continue
        a, b = make_arrays([rec["shape_a"], rec["shape_b"]], "complex128", seed=n)
        if np.dtype(dtype).kind != "c":
            a, b = a.real, b.real
            want = orc.einsum(rec["eq"], a, b)
        else:
            want = PVALS[key]
        got = cb.einsum(rec["eq"], _cast(a, dtype), _cast(b, dtype))
        assert got.dtype == np.dtype(dtype)
        assert got.shape == np.shape(want), rec
        assert rel_err(got, want) < TOL[dtype] * 10, rec
        n_ok += 1
    assert n_ok > 300


def test_pair_errors_match_reference():
    for rec in PARSERS["pair"]:
        if "error" in rec:
            a = np.zeros(rec["shape_a"])
            b = np.zeros(rec["shape_b"])
            with pytest.raises(ValueError):
                cb.einsum(rec["eq"], a, b)
    with pytest.raises(ValueError):
        cb.tensordot(np.zeros((2, 3)), np.zeros((2, 3)), ((1,), (0,)))
    with pytest.raises(NotImplementedError):
        cb.einsum("a...,a->", np.zeros(2), np.zeros(2))


def test_single_cases_golden():
    for n, rec in enumerate(PARSERS["single"]):
        (x,) = make_arrays([rec["shape"]], "complex128", seed=1000 + n)
        got = cb.einsum(rec["eq"], x)
        want = PVALS[f"single_{n}"]
        assert got.shape == want.shape
        assert rel_err(got, want) < 1e-12


def test_tensordot_golden_shapes():
    for n, rec in enumerate(PARSERS["tdot"]):
        a, b = make_arrays([rec["shape_a"], rec["shape_b"]], "complex128", seed=n)
        axes = (tuple(rec["axes"][0]), tuple(rec["axes"][1]))
        got = cb.tensordot(a, b, axes)
        want = np.tensordot(a, b, axes)
        assert got.shape == want.shape
        assert rel_err(got, want) < 1e-12


_RAGGED_GEMMS = [(130, 70, 19), (257, 3, 33), (5, 300, 9), (512, 128, 64), (1000, 96, 40)]
# (m, n, k) that each non-staged variant accepts as it is (build_pair_desc falls back otherwise)
_GEMMS_ACCEPTED = {
    L.VAR_ROWSTREAM: [(200, 3, 4), (512, 2, 7), (768, 8, 8), (1024, 6, 5), (256, 5, 2)],
    L.VAR_DMMASTREAM: [(4096, 16, 16), (1024, 9, 32), (768, 32, 7), (512, 8, 64), (200, 24, 20)],
    L.VAR_DOTSTREAM: [(1, 1, 6144), (1, 1, 2048), (1, 1, 1000), (1, 1, 10240), (1, 1, 4096)],
    **{v: [(256, 64, 32), (384, 64, 48), (128, 48, 16), (512, 96, 64), (1000, 64, 40)] for v in L.TC05_VARIANTS},
}


def _variant_that_runs(variant, dtype, m, n, k):
    """The forced variant, or what build_pair_desc documents for a dtype the kernel does not take."""
    if variant in (L.VAR_DMMA3M_128x32, L.VAR_DMMA3M_256x16) and dtype != "complex128":
        return L.VAR_DMMA_256x32 if variant == L.VAR_DMMA3M_128x32 else L.VAR_DMMA_256x16
    if variant == L.VAR_DMMASTREAM and dtype != "complex128":
        return L.VAR_DMMA_256x16
    if variant in L.TC05_VARIANTS and dtype != "complex64":
        # the mma.sync policy the heuristic picks without the wgmma kernel
        return L.choose_variant(dtype, 1, max(m, n), min(m, n), k, allow_tc05=False)
    return variant


@pytest.mark.parametrize("variant", [L.VAR_SIMT_64x64, L.VAR_DMMA_128x64, L.VAR_DMMA_64x128,
                                     L.VAR_DMMA_256x32, L.VAR_DMMA_256x16, L.VAR_ROW_128x8, L.VAR_ROW_256x4, L.VAR_ROWSTREAM, L.VAR_TC05_128x64, L.VAR_TC05_128x32, L.VAR_TC05_128x16,
                                     L.VAR_DMMA3M_128x32, L.VAR_DMMA3M_256x16, L.VAR_DMMASTREAM, L.VAR_DOTSTREAM])
@pytest.mark.parametrize("dtype", ["complex128", "float64", "complex64", "float32"])
def test_every_kernel_variant_ragged_gemm(variant, dtype):
    """Each variant on GEMMs it runs as forced (the plan's variant is asserted), into a NaN-filled C.
    The staged variants take ragged shapes; the stream and wgmma variants shapes they accept.
    tests/test_gpu_kernel_paths.py covers each kernel's code paths one by one."""
    import torch

    from cotengra_b200 import _lib

    for (m, n, k) in _GEMMS_ACCEPTED.get(variant, _RAGGED_GEMMS):
        a, b = make_arrays([(m, k), (k, n)], dtype, seed=m + n + k + 1000 * variant)
        dims = L.classify_pair("ab", a.shape, "bc", b.shape, "ac")
        plan = L.build_pair_desc(dims, dtype, variant=variant, c_dense_elems=m * n,
                                 sm_count=_lib.device_info()["sm_count"])
        assert plan.variant == _variant_that_runs(variant, dtype, m, n, k), (m, n, k, variant, dtype, plan.variant)
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        c = torch.full((m, n), float("nan"), dtype=ta.dtype, device="cuda")
        pa, pb = (tb, ta) if plan.swapped else (ta, tb)
        _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa.data_ptr(),
                                                  pb.data_ptr(), c.data_ptr(), 0))
        torch.cuda.synchronize()
        want = a.astype(np.complex128 if np.dtype(dtype).kind == "c" else np.float64) @ b
        assert rel_err(c.cpu().numpy(), want) < (1e-12 if dtype in ("complex128", "float64") else 1e-5), \
            (m, n, k, variant, dtype)


DSTREAM_CASES = [
    ("n16_k16", "ab,bc->ac", [(8192, 16), (16, 16)], {}),
    ("ragged_rows_cols", "xyzb,bc->zyxc", [(8, 27, 19, 7), (7, 11)], {}),   # 4104 rows (masked tail), odd N, K % 4 != 0
    ("n32_k32", "ab,bc->ac", [(4096, 32), (32, 32)], {}),                 # four column fragments
    ("n24_k20", "bxy,cb->cyx", [(20, 72, 72), (24, 20)], {}),              # transposed operands and output
    ("permuted", "aibjc,ijd->dcba", [(8, 4, 8, 4, 8), (4, 4, 16)], {}),   # multi-dim rows, strided C
    ("accumulate", "ab,bc->ac", [(4096, 16), (16, 16)], {"accumulate": True}),
]


@pytest.mark.parametrize("case", DSTREAM_CASES, ids=[c[0] for c in DSTREAM_CASES])
def test_dmma_stream_kernel(case):
    """dmmastream.cuh: DMMA fragments loaded straight from global memory (narrow complex128 nodes)."""
    import torch

    from cotengra_b200 import _lib

    name, eq, shapes, kw = case
    lhs, out = eq.split("->")
    ta_, tb_ = lhs.split(",")
    a, b = make_arrays(shapes, "complex128", seed=len(name))
    dims = L.classify_pair(ta_, a.shape, tb_, b.shape, out)
    out_shape = tuple(dict(zip(ta_ + tb_, a.shape + b.shape))[ix] for ix in out)
    plan = L.build_pair_desc(dims, "complex128", c_dense_elems=math.prod(out_shape), variant=L.VAR_DMMASTREAM,
                             sm_count=_lib.device_info()["sm_count"], **kw)
    assert plan.variant == L.VAR_DMMASTREAM, (name, plan.variant)
    da, db = torch.from_numpy(np.ascontiguousarray(a)).cuda(), torch.from_numpy(np.ascontiguousarray(b)).cuda()
    c0 = make_arrays([out_shape], "complex128", seed=78)[0]
    dc = torch.from_numpy(np.ascontiguousarray(c0)).cuda()
    pa, pb = (db, da) if plan.swapped else (da, db)
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa.data_ptr(), pb.data_ptr(), dc.data_ptr(), 0))
    torch.cuda.synchronize()
    want = np.einsum(eq, a, b)
    if kw.get("accumulate"):
        want = want + c0
    assert rel_err(dc.cpu().numpy().reshape(out_shape), want) < 1e-12, name


@pytest.mark.parametrize("dtype", ["complex128", "complex64", "float64", "float32"])
@pytest.mark.parametrize("case", ["pow2_permuted", "odd_extents", "accumulate"])
def test_dot_stream_kernel(case, dtype):
    """dotstream.cuh: M = N = 1 inner products with differently ordered operands."""
    import torch

    from cotengra_b200 import _lib

    if case == "odd_extents":
        ta_, tb_, shape = "abcd", "dbca", {"a": 32, "b": 27, "c": 25, "d": 49}
    else:
        ta_ = "abcdefghijklmnopqrstu"
        tb_ = "utsrqpjihgfedcbaonmlk"
        shape = {c: 2 for c in ta_}
    sa, sb = tuple(shape[c] for c in ta_), tuple(shape[c] for c in tb_)
    a, b = make_arrays([sa, sb], dtype, seed=11)
    dims = L.classify_pair(ta_, sa, tb_, sb, "")
    acc = case == "accumulate"
    plan = L.build_pair_desc(dims, dtype, c_dense_elems=1, accumulate=acc, sm_count=_lib.device_info()["sm_count"])
    assert plan.variant == L.VAR_DOTSTREAM, plan.variant
    da, db = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
    c0 = make_arrays([(1,)], dtype, seed=3)[0]
    dc = torch.from_numpy(c0.copy()).cuda()
    pa, pb = (db, da) if plan.swapped else (da, db)
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa.data_ptr(), pb.data_ptr(), dc.data_ptr(), 0))
    torch.cuda.synchronize()
    wide = np.complex128 if np.dtype(dtype).kind == "c" else np.float64
    want = np.einsum(ta_ + "," + tb_ + "->", a.astype(wide), b.astype(wide))
    scale = np.sqrt(a.size)  # sum of ~N(0,1) terms: compare against the natural magnitude
    if acc:
        want = want + c0[0]
    tol = 1e-12 if dtype in ("complex128", "float64") else 2e-5
    assert abs(dc.cpu().numpy()[0] - want) / scale < tol, (case, dtype)


def test_equations_through_contractor():
    recs = load_json("equations.json")
    vals = load_npz("equations_values.npz")
    for rec in recs:
        arrays = make_arrays(rec["shapes"], "complex128", seed=rec["seed"])
        n = len(arrays)
        # a left-to-right chain tree over the operands of the equation
        terms, out = L.split_equation(rec["eq"])
        inputs = [tuple(t) for t in terms]
        size_dict = {}
        for t, s in zip(inputs, rec["shapes"]):
            for ix, d in zip(t, s):
                size_dict[ix] = max(size_dict.get(ix, 1), d)
        if any(size_dict[ix] != d for t, s in zip(inputs, rec["shapes"]) for ix, d in zip(t, s)):
            continue  # broadcast equations have no single size_dict: covered by pair cases
        path, cur = [], 0
        for i in range(1, n):
            path.append((cur, i))
            cur = n + i - 1
        spec = cb.TreeSpec(inputs, tuple(out), size_dict, path)
        got = cb.contract_tree(spec, arrays)
        want = vals[rec["key"]]
        assert got.shape == want.shape, rec
        assert rel_err(got, want) < 1e-11, rec
        m, e = cb.contract_tree(spec, arrays, strip_exponent=True)
        assert rel_err(m * 10.0**e, want) < 1e-10, rec


def _spec(rec):
    n_in = len(rec["inputs"])
    node_inds = {int(k): v for k, v in rec["inds"].items() if int(k) >= n_in}
    return cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"],
                       decode_sliced(rec["sliced"]), node_inds)


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_trees_golden(rec):
    if rec["name"] not in TVALS:
        pytest.skip("no full value recorded")
    spec = _spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    want = TVALS[rec["name"]]
    got = cb.contract_tree(spec, arrays)
    assert got.shape == want.shape
    assert rel_err(got, want) < 1e-10
    if rec["strip_exponent"]:
        m, e = cb.contract_tree(spec, arrays, strip_exponent=True)
        assert rel_err(m * 10.0**e, want) < 1e-10
        wm, we = TVALS[rec["name"] + "_m"], float(TVALS[rec["name"] + "_e"])
        assert rel_err(m * 10.0 ** (e - we), wm) < 1e-10
    # single precision: as close to the double-precision reference value as the reference's own
    # numpy single-precision path is (within 3x), and within 1e-5 wherever that path is -- any fp32
    # evaluation of a whole tree loses digits with depth and cancellation (per node: 1e-5, above)
    lo = "complex64" if np.dtype(rec["dtype"]).kind == "c" else "float32"
    lo_arrays = [_cast(a, lo) for a in arrays]
    got32 = cb.contract_tree(spec, lo_arrays)
    assert got32.dtype == np.dtype(lo)
    ref32 = orc.contract_tree([tuple(t) for t in spec.inputs], spec.output, spec.sliced,
                              spec.contractions(), lo_arrays)
    assert rel_err(got32, want) < max(1e-5, 3.0 * rel_err(ref32, want))


@pytest.mark.parametrize("strip", [False, True])
def test_checkpointed_run_resumes(strip, tmp_path):
    """contract_checkpointed (SURVEY 8f-4) on the real executor: an interrupted run resumes
    behind its last saved block and ends at the golden value of the reference."""
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    n_in = len(rec["inputs"])
    node_inds = {int(k): v for k, v in rec["inds"].items() if int(k) >= n_in}
    spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]),
                       node_inds)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    ck = str(tmp_path / "ck.npz")
    every = max(1, spec.nslices // 4)

    class Stop(Exception):
        pass

    def stop(done, n):
        raise Stop

    with pytest.raises(Stop):
        cb.contract_checkpointed(spec, arrays, ck, every=every, strip_exponent=strip, on_block=stop)
    blocks = []
    res = cb.contract_checkpointed(spec, arrays, ck, every=every, strip_exponent=strip,
                                   on_block=lambda d, n: blocks.append(d))
    assert blocks[0] == 2 * every and blocks[-1] == spec.nslices
    got = res[0] * 10.0 ** res[1] if strip else res
    assert rel_err(got, TVALS[rec["name"]]) < 1e-10


def test_benchmark_protocol_matches_reference_keys():
    """cb.benchmark == tree.benchmark (core.py:4092-4164): keys, repetition bounds, flop convention."""
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    n_in = len(rec["inputs"])
    node_inds = {int(k): v for k, v in rec["inds"].items() if int(k) >= n_in}
    spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]),
                       node_inds)
    res = cb.benchmark(spec, dtype="complex64", max_time=0.0, min_reps=3, max_reps=5)
    assert set(res) == {"time_per_slice", "est_time_total", "est_gigaflops"}
    assert res["time_per_slice"] > 0 and res["est_gigaflops"] > 0
    assert math.isclose(res["est_time_total"], res["time_per_slice"] * spec.nslices, rel_tol=1e-12)
    ex = cb.TreeExecutor(spec, dtype="float64")
    res2 = cb.benchmark(None, executor=ex, max_time=0.0, min_reps=2, max_reps=2)
    macs_v, macs_i, _el = ex.reference_work  # tree.total_flops counts the hoisted nodes too
    flops = 2 * (macs_v + macs_i) * spec.nslices
    assert math.isclose(res2["est_gigaflops"], flops / (1e9 * res2["est_time_total"]), rel_tol=1e-12)


def test_contractor_dropin_signature():
    rec = next(r for r in TREES if r["name"] == "lattice4x4_sliced")
    spec = _spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    fn = cb.B200Contractor(spec.contractions(), strip_exponent=False)
    inputs = [tuple(t) for t in rec["inputs"]]
    sliced = decode_sliced(rec["sliced"])
    total = 0
    for i in range(spec.nslices):
        sl = orc.slice_arrays(inputs, sliced, arrays, i)
        total = total + fn(*sl)
        m, e = fn(*sl, strip_exponent=True)
        assert rel_err(m * 10.0**e, fn(*sl)) < 1e-10
    assert rel_err(total, TVALS[rec["name"]]) < 1e-10
    with pytest.raises(TypeError):
        fn(*sl, bogus=1)


def test_sycamore_slices_vs_reference_and_oracle():
    recs = {r["name"]: r for r in load_json("sycamore_m20.json")}
    vals = load_npz("sycamore_m20_values.npz")
    rec = recs["sycamore_m20_small"]
    spec = _spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    ex = cb.TreeExecutor(spec, dtype="complex128")
    import torch

    dev = [torch.from_numpy(a).cuda() for a in arrays]
    for i in list(rec["slice_keys"])[:3]:
        if int(i) >= 2**62:
            continue
        got = ex.contract_device(dev, begin=int(i), step=1, count=1).cpu().numpy()
        assert rel_err(got, vals[f"sycamore_m20_small_slice{i}"]) < 1e-10
    # medium: W = 2^22 per slice, with exponent stripping
    rec = recs["sycamore_m20_medium"]
    spec = _spec(rec)
    exs = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True)
    for i in list(rec["slice_keys"])[:1]:
        m, e = exs.contract_device(dev, begin=int(i), step=1, count=1)
        wm = vals[f"sycamore_m20_medium_slice{i}_m"]
        we = float(vals[f"sycamore_m20_medium_slice{i}_e"])
        got = m.cpu().numpy() * 10.0 ** (float(e.item()) - we)
        assert rel_err(got, wm) < 1e-10
        # and against the oracle run live on the same inputs
        inputs = [tuple(t) for t in rec["inputs"]]
        om, oe = orc.run_contractions(
            decode_ir(rec["contractions"]),
            orc.slice_arrays(inputs, decode_sliced(rec["sliced"]), arrays, int(i)),
            strip_exponent=True,
        )
        assert rel_err(got, om * 10.0 ** (oe - we)) < 1e-10
    # complex64 against the complex128 result (strip_exponent keeps it in range)
    ex32 = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True)
    dev32 = [torch.from_numpy(a.astype(np.complex64)).cuda() for a in arrays]
    m32, e32 = ex32.contract_device(dev32, begin=0, step=1, count=1)
    got32 = m32.cpu().numpy() * 10.0 ** (float(e32.item()) - we)
    # judged against the reference's own numpy complex64 path on the same slice (see test_trees_golden)
    rm, re_ = orc.run_contractions(
        decode_ir(rec["contractions"]),
        orc.slice_arrays(inputs, decode_sliced(rec["sliced"]), [a.astype(np.complex64) for a in arrays], 0),
        strip_exponent=True,
    )
    e_ref = rel_err(rm.astype(np.complex128) * 10.0 ** (float(re_) - we), wm)
    e_gpu = rel_err(got32, wm)
    print(f"sycamore_m20_medium c64: gpu {e_gpu:.2e}, numpy c64 {e_ref:.2e}")
    assert e_gpu < max(1e-5, 3.0 * e_ref)


def test_large_slice_properties():
    """Size-independent properties at a width the CPU cannot check directly
    (W = 2^26): (1) a slice equals the sum of its two half-slices when one more
    index is sliced; (2) linearity in one input; (3) DMMA and FMA kernels agree."""
    import torch

    recs = {r["name"]: r for r in load_json("sycamore_m20.json")}
    rec = recs["sycamore_m20_appxB"]
    base = _spec(rec)
    # slice further, greedily on the largest intermediates, down to 2^26
    from tests.slicing_util import slice_to_width

    spec = slice_to_width(base, 2**26)
    arrays = make_arrays(spec.shapes(), "complex128", seed=7, scale=1.0)
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    ex = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True)
    m, e = ex.contract_device(dev, begin=0, step=1, count=1)
    val = m.cpu().numpy() * 10.0 ** float(e.item())
    # (1) slicing one more index: the children of slice 0 sum to slice 0
    from tests.slicing_util import slice_id, slice_one_more

    spec2, extra = slice_one_more(spec)
    ex2 = cb.TreeExecutor(spec2, dtype="complex128", strip_exponent=True)
    tot = 0
    for d in range(spec2.size_dict[extra]):
        key = dict(spec.slice_key(0))
        key[extra] = d
        m2, e2 = ex2.contract_device(dev, begin=slice_id(spec2, key), step=1, count=1)
        tot = tot + m2.cpu().numpy() * 10.0 ** float(e2.item())
    assert rel_err(tot, val) < 1e-9
    # (2) linearity: scaling one sliced-invariant input scales the result
    dev_s = list(dev)
    dev_s[0] = dev[0] * (0.5 - 0.25j)
    m3, e3 = ex.contract_device(dev_s, begin=0, step=1, count=1)
    assert rel_err(m3.cpu().numpy() * 10.0 ** float(e3.item()), val * (0.5 - 0.25j)) < 1e-10
    # (3) tensor-core vs FMA kernels
    ex4 = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True, allow_dmma=False)
    m4, e4 = ex4.contract_device(dev, begin=0, step=1, count=1)
    assert rel_err(m4.cpu().numpy() * 10.0 ** float(e4.item()), val) < 1e-10
