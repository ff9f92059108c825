"""Forward mode on the device: the two-term stream kernels through ``ctgb_contract_pair2`` in
guarded buffers, ``TreeExecutor.jvp`` against the exact multilinear oracle (``tests/helpers.py``),
the dot-product identity with reverse mode, and ``torch.autograd.forward_ad`` through every entry
point that records the autograd node."""

import json
import os
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import torch  # noqa: E402
import torch.autograd.forward_ad as fwAD  # noqa: E402

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import _lib  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from tests.helpers import jvp_oracle  # noqa: E402
from tests.helpers import GOLDEN_DIR, load_json, make_arrays, tree_spec  # noqa: E402

TREES = load_json("trees.json")
GUARD = 64  # elements of NaN guard band around every operand and C


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _wide(dt):
    return "complex128" if "complex" in dt else "float64"


# ------------------------------------------------------------------ ctgb_contract_pair2
# (variant, dtype, M, N, K): every row-stream instantiation (4x4, 2x8, 8x8; long k), every DMMA stream
# one (N <= 8, 16, 32, 64) at its two-term k limit; N and K ragged (M in whole row blocks: a ragged
# blocked m dim hands the node over to a staged tile)
PAIR2 = ([(L.VAR_ROWSTREAM, dt, m, n, k) for dt in ("float32", "float64", "complex64", "complex128")
          for m, n, k in ((1536, 3, 4), (2560, 2, 7), (3072, 8, 8), (1024, 5, 6))]
         + [(L.VAR_ROWSTREAM_K, dt, 2560, n, k) for dt in ("float32", "float64", "complex64")
            for n, k in ((8, 64), (3, 24))]
         + [(L.VAR_DMMASTREAM, "complex128", m, n, k)
            for m, n, k in ((1536, 8, 40), (2560, 16, 64), (3072, 24, 32), (1024, 40, 16), (4096, 64, 16))])


def _pair_words(variant, dtype, M, N, K, accumulate):
    dims = L.classify_pair("mk", (M, K), "kn", (K, N), "mn")
    plan = L.build_pair_desc(dims, dtype, accumulate=accumulate, sm_count=_lib.device_info()["sm_count"],
                             c_dense_elems=0 if accumulate else M * N, variant=variant)
    assert plan.variant == variant and not plan.swapped, (plan.variant, variant)
    return plan.words


def _guarded(x):
    """x inside a NaN-filled buffer: (device buffer, device pointer of x, host copy of the buffer)"""
    buf = np.full(x.size + 2 * GUARD, np.nan, dtype=x.dtype)
    buf[GUARD:GUARD + x.size] = x.reshape(-1)
    d = torch.from_numpy(buf).cuda()
    return d, d.data_ptr() + GUARD * x.itemsize, buf


@pytest.mark.parametrize("variant,dtype,M,N,K", PAIR2)
@pytest.mark.parametrize("accumulate", [False, True])
def test_contract_pair2(variant, dtype, M, N, K, accumulate):
    hi = _wide(dtype)
    A, B, A2, B2, C0 = make_arrays([(M, K), (K, N), (M, K), (K, N), (M, N)], hi, seed=M + N + K)
    ops = [x.astype(dtype) for x in (A, B, A2, B2)]
    words = _pair_words(variant, dtype, M, N, K, accumulate)
    c0 = C0.astype(dtype) if accumulate else np.full((M, N), np.nan, dtype=dtype)
    bufs = [_guarded(x) for x in ops + [c0]]
    pa, pb, pa2, pb2, pc = (b[1] for b in bufs)
    _lib.check(_lib.load().ctgb_contract_pair2(words.ctypes.data, pa, pb, pa2, pb2, pc, 0))
    torch.cuda.synchronize()
    for d, _p, host in bufs[:4]:
        assert d.cpu().numpy().tobytes() == host.tobytes()  # operands untouched
    got = bufs[4][0].cpu().numpy()
    assert np.isnan(got[:GUARD]).all() and np.isnan(got[GUARD + M * N:]).all()  # guard bands untouched
    got = got[GUARD:GUARD + M * N].reshape(M, N)
    a, b, a2, b2 = (x.astype(hi) for x in ops)
    want = a @ b + a2 @ b2 + (c0.astype(hi) if accumulate else 0)
    assert not np.isnan(got).any()
    assert nrel(got, want) <= (1e-12 if dtype == hi else 1e-5)
    # the wide-C bit belongs to the dot-stream kernels: the two-term form refuses it
    w = words.copy()
    w[L.W_FLAGS] |= L.FLAG_WIDE_C
    with pytest.raises(ValueError):
        _lib.check(_lib.load().ctgb_contract_pair2(w.ctypes.data, pa, pb, pa2, pb2, pc, 0))


def test_contract_pair2_refuses_other_variants():
    words = _pair_words(L.VAR_DMMA_256x16, "complex128", 4096, 16, 16, False)
    x = torch.zeros(4096 * 16, dtype=torch.complex128, device="cuda")
    before = _lib.launch_count()
    with pytest.raises(ValueError):
        _lib.check(_lib.load().ctgb_contract_pair2(words.ctypes.data, *([x.data_ptr()] * 5), 0))
    assert _lib.launch_count() == before


# ------------------------------------------------------------------ ex.jvp
def _jvp(ex, arrays, tans, wrt=None, **kw):
    dev = [torch.tensor(np.asarray(a)).cuda() for a in arrays]
    res = ex.jvp(dev, [torch.tensor(np.asarray(t)).cuda() for t in tans], wrt=wrt, **kw)
    torch.cuda.synchronize()
    return tuple(x.cpu().numpy() for x in res) if isinstance(res, tuple) else res.cpu().numpy()


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_device_jvp_matches_oracle(rec):
    spec = tree_spec(rec)
    hi = rec["dtype"]
    lo = "complex64" if hi == "complex128" else "float32"
    arrays = make_arrays(spec.shapes(), hi, seed=rec["seed"])
    n = len(arrays)
    ir = spec.contractions()
    rng = np.random.default_rng(rec["seed"])
    for wrt in ([int(rng.integers(n))], list(range(n))):
        tans = make_arrays([arrays[i].shape for i in wrt], hi, seed=rec["seed"] + 3)
        want = jvp_oracle(spec, ir, arrays, tans, wrt)
        ex = cb.TreeExecutor(spec, dtype=hi)
        out, tout = _jvp(ex, arrays, tans, wrt)
        assert nrel(tout, want) <= 1e-10
        assert nrel(out, ex(arrays)) <= 1e-10
        # single precision against the double oracle: max(1e-5, 3 x the oracle's own single-precision error)
        a32, t32 = [a.astype(lo) for a in arrays], [t.astype(lo) for t in tans]
        ref32 = jvp_oracle(spec, ir, a32, t32, wrt)
        for opts in ({}, {"precision": "tf32"}, {"accumulate": "double"}):
            ex32 = cb.TreeExecutor(spec, dtype=lo, **opts)
            got = _jvp(ex32, a32, t32, wrt, primal=False)
            tol = max(1e-5, 3.0 * nrel(ref32, want))
            if opts.get("precision") == "tf32":
                tol = max(tol, 3e-3)  # one tf32 pass: 10-bit mantissas
            assert nrel(got, want) <= tol, (opts, nrel(got, want), tol)
    if ex.nslices > 1:
        # slice ranges that sum to the whole
        tans = make_arrays(spec.shapes(), hi, seed=rec["seed"] + 4)
        full = _jvp(ex, arrays, tans, primal=False)
        h = ex.nslices // 2
        parts = _jvp(ex, arrays, tans, primal=False, begin=0, count=h) + \
            _jvp(ex, arrays, tans, primal=False, begin=h, count=ex.nslices - h)
        assert nrel(parts, full) <= 1e-12


def test_two_term_and_two_launch_forms_agree():
    """The stem of a tree whose absorptions run on the stream kernels, both forms, complex128."""
    inputs = [("m", "k"), ("k", "n"), ("n", "o"), ("o",)]
    spec = cb.TreeSpec(inputs, ("m",), {"m": 1 << 18, "k": 8, "n": 8, "o": 4}, [(0, 1), (4, 2), (5, 3)])
    arrays = make_arrays(spec.shapes(), "complex128", seed=2)
    tans = make_arrays(spec.shapes(), "complex128", seed=3)
    ex = cb.TreeExecutor(spec, dtype="complex128", fuse=False)
    assert ex.jvp_plan().two_term_nodes >= 1
    one = _jvp(ex, arrays, tans, primal=False)
    two = _jvp(ex, arrays, tans, primal=False, _two_term=False)
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, range(4))
    assert nrel(one, want) <= 1e-12 and nrel(two, want) <= 1e-12


def test_constants_carry_no_tangent():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=9)
    n = len(arrays)
    consts = {i: arrays[i] for i in range(0, n, 2)}
    var = [i for i in range(n) if i not in consts]
    tans = make_arrays([arrays[i].shape for i in var], "complex128", seed=10)
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, var)
    for fold in (None, 0):
        ex = cb.TreeExecutor(spec, dtype="complex128", constants=consts, fold_max_bytes=fold)
        got = _jvp(ex, [arrays[i] for i in var], tans, primal=False)
        assert nrel(got, want) <= 1e-10
        # wrt counts among the variables
        got1 = _jvp(ex, [arrays[i] for i in var], tans[:1], wrt=[0], primal=False)
        assert nrel(got1, jvp_oracle(spec, spec.contractions(), arrays, tans[:1], var[:1])) <= 1e-10
        assert all(t.kind != 7 or t.input_index < len(var) for t in ex.jvp_plan().tensors)


def _vdot(a, b):
    return np.vdot(np.asarray(a).reshape(-1), np.asarray(b).reshape(-1))


def _dot_identity(ex, arrays, wrt, count=None):
    """<g, J v> = <J^T g, v> in torch's complex convention (grad = g conj(d out / dx))"""
    tans = make_arrays([arrays[i].shape for i in wrt], "complex128", seed=21)
    jv = _jvp(ex, arrays, tans, wrt, primal=False, count=count)
    g = make_arrays([jv.shape], "complex128", seed=22)[0]
    dev = [torch.tensor(a).cuda() for a in arrays]
    grads = ex.vjp(dev, torch.tensor(g).cuda(), wrt=wrt, count=count)
    lhs = _vdot(g, jv)
    rhs = sum(_vdot(grads[i].cpu().numpy(), t) for i, t in zip(wrt, tans))
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), 1e-300), (lhs, rhs)


def test_dot_product_with_reverse_mode_peps8x8_config2():
    rec = next(r for r in TREES if r["name"] == "peps8x8_d2")
    spec = cb.TreeSpec(rec["inputs"], rec["output"], {ix: 6 for ix in rec["size_dict"]}, rec["path"])
    arrays = make_arrays(spec.shapes(), "complex128", seed=11, scale=0.35)
    _dot_identity(cb.TreeExecutor(spec, dtype="complex128"), arrays, list(range(len(arrays))))


def test_dot_product_with_reverse_mode_sycamore_m10():
    rec = json.load(open(os.path.join(GOLDEN_DIR, "circuits.json")))["m10"]
    flat = np.load(os.path.join(GOLDEN_DIR, "circuits_arrays.npz"))["m10_arrays_flat"]
    small = cb.TreeSpec.from_dict(rec["small_spec"])
    arrays, off = [], 0
    for shape in small.shapes():
        k = int(np.prod(shape))
        arrays.append(flat[off:off + k].reshape(shape).astype(np.complex128))
        off += k
    ex = cb.TreeExecutor(small, dtype="complex128")
    gate = min(range(len(arrays)), key=lambda i: (arrays[i].size != 16, i))  # a two-qubit gate
    _dot_identity(ex, arrays, [gate], count=2)


# ------------------------------------------------------------------ torch forward AD
def test_forward_ad_entry_points():
    rec = next(r for r in TREES if r["name"] == "lattice4x4_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=31)
    n = len(arrays)
    wrt = [0, n // 2]
    tans = make_arrays([arrays[i].shape for i in wrt], "complex128", seed=32)
    dev = [torch.tensor(a).cuda() for a in arrays]
    tdev = [torch.tensor(t).cuda() for t in tans]
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, wrt)
    ex = cb.TreeExecutor(spec, dtype="complex128")
    ref = ex.jvp(dev, tdev, wrt=wrt, primal=False)
    with fwAD.dual_level():
        xs = [fwAD.make_dual(t, tdev[wrt.index(i)]) if i in wrt else t for i, t in enumerate(dev)]
        out = cb.contract_tree(ex, xs)
        p, t = fwAD.unpack_dual(out)
        assert torch.allclose(t, ref, rtol=1e-12, atol=0)
        assert torch.allclose(p, ex.contract_device(dev), rtol=1e-12, atol=0)
        # the installed per-slice contractor (one slice here: an unsliced program)
        fn = cb.B200Contractor(spec.contractions())
        unsliced = cb.TreeSpec(spec.inputs, spec.output, spec.size_dict, rec["path"])
        want_u = jvp_oracle(unsliced, spec.contractions(), arrays, tans, wrt)
        assert nrel(fwAD.unpack_dual(fn(*xs)).tangent.cpu().numpy(), want_u) <= 1e-10
        # array_contract_expression with constants: tangents of the variables only
        consts = {i: arrays[i] for i in range(n) if i not in wrt and i % 3 == 1}
        var = [i for i in range(n) if i not in consts]
        expr = cb.array_contract_expression(spec.inputs, spec.output, optimize=spec, constants=consts)
        t_e = fwAD.unpack_dual(expr(*[xs[i] for i in var])).tangent
        assert nrel(t_e.cpu().numpy(), want) <= 1e-10
    # reverse mode in the same call is unaffected
    ys = [t.clone().requires_grad_() for t in dev]
    with fwAD.dual_level():
        zs = [fwAD.make_dual(y, tdev[wrt.index(i)]) if i in wrt else y for i, y in enumerate(ys)]
        out = cb.contract_tree(ex, zs)
        assert nrel(fwAD.unpack_dual(out).tangent.detach().cpu().numpy(), want) <= 1e-10
        fwAD.unpack_dual(out).primal.real.sum().backward()
    assert all(y.grad is not None for y in ys)


def test_small_workspace_is_refused_before_any_launch():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=1)
    ex = cb.TreeExecutor(spec, dtype=rec["dtype"])
    plan = ex.jvp_plan()
    dev = [torch.tensor(a).cuda() for a in arrays]
    tout = torch.zeros(plan.out_shape, dtype=dev[0].dtype, device="cuda")
    ws = torch.empty(plan.total_bytes - 1, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    before = _lib.launch_count()
    with pytest.raises(MemoryError):
        plan.execute([t.data_ptr() for t in dev], [t.data_ptr() for t in dev], None, tout.data_ptr(),
                     ws.data_ptr(), ws.numel(), 0, 1, plan.nslices, torch.cuda.current_stream().cuda_stream)
    assert _lib.launch_count() == before


def test_strip_exponent_refuses_jvp():
    rec = next(r for r in TREES if r["name"] == "lattice4x4_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=1)
    ex = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True)
    dev = [torch.tensor(a).cuda() for a in arrays]
    with pytest.raises(NotImplementedError):
        ex.jvp(dev, dev)
    with fwAD.dual_level():
        xs = [fwAD.make_dual(dev[0], dev[0])] + dev[1:]
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            m, _e = cb.contract_tree(ex, xs)
        assert any("tangent" in str(x.message) for x in w)
        assert fwAD.unpack_dual(m).tangent is None
