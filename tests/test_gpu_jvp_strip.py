"""Forward-mode derivatives of strip_exponent results on the device (``stripped_grad=True``): the
two-term stream kernels with scale-only descriptors in guarded buffers, the stripped tangent
``dm = 10^-e d(amp)`` against the unstripped device JVP under the executor's options, the m20 slice in
complex64 with untuned inputs (whose unstripped amplitude overflows or underflows), the dot-product
identity with the stripped VJP, an 8x8 PEPS scaled until complex64 overflows, and forward AD through
every entry point."""

import math
import warnings

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import torch  # noqa: E402
import torch.autograd.forward_ad as fwAD  # noqa: E402

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import _lib  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from cotengra_b200.jvp import JvpPlan  # noqa: E402
from tests.helpers import load_json, make_arrays, tree_spec  # noqa: E402
from tests.slicing_util import appxB_at_width  # noqa: E402
from tests.test_gpu_jvp import GUARD, PAIR2, _guarded, _pair_words, _wide  # noqa: E402

TREES = load_json("trees.json")
GIB = 1 << 30


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _dev(arrays):
    return [torch.tensor(np.asarray(a)).cuda() for a in arrays]


# ------------------------------------------------------------------ ctgb_contract_pair2, scaled
@pytest.mark.parametrize("variant,dtype,M,N,K", PAIR2)
@pytest.mark.parametrize("accumulate", [False, True])
def test_contract_pair2_scaled(variant, dtype, M, N, K, accumulate):
    """scale words alone: C (+)= (A.B + A'.B') / (fA fB), B and B' scaled as they are staged; the factor
    slots are read, never written (a sentinel slot beside them keeps its value)"""
    hi = _wide(dtype)
    A, B, A2, B2, C0 = make_arrays([(M, K), (K, N), (M, K), (K, N), (M, N)], hi, seed=M + N + K + 1)
    ops = [x.astype(dtype) for x in (A, B, A2, B2)]
    words = _pair_words(variant, dtype, M, N, K, accumulate).copy()
    slots = torch.tensor([2.5, 0.125, -7.0], dtype=torch.float64, device="cuda")  # fA, fB, sentinel
    words[L.W_SCALE_A] = slots.data_ptr()
    words[L.W_SCALE_B] = slots.data_ptr() + 8
    c0 = C0.astype(dtype) if accumulate else np.full((M, N), np.nan, dtype=dtype)
    bufs = [_guarded(x) for x in ops + [c0]]
    pa, pb, pa2, pb2, pc = (b[1] for b in bufs)
    _lib.check(_lib.load().ctgb_contract_pair2(words.ctypes.data, pa, pb, pa2, pb2, pc, 0))
    torch.cuda.synchronize()
    for d, _p, host in bufs[:4]:
        assert d.cpu().numpy().tobytes() == host.tobytes()
    assert slots.cpu().tolist() == [2.5, 0.125, -7.0]
    got = bufs[4][0].cpu().numpy()
    assert np.isnan(got[:GUARD]).all() and np.isnan(got[GUARD + M * N:]).all()
    got = got[GUARD:GUARD + M * N].reshape(M, N)
    a, b, a2, b2 = (x.astype(hi) for x in ops)
    want = (a @ b + a2 @ b2) / (2.5 * 0.125) + (c0.astype(hi) if accumulate else 0)
    assert not np.isnan(got).any()
    assert nrel(got, want) <= (1e-12 if dtype == hi else 1e-5)
    # a factor slot of C, or one scale word alone, is refused before any launch
    x = torch.zeros(8, dtype=torch.float64, device="cuda")
    bad_c = words.copy()
    bad_c[L.W_FACTOR_C] = x.data_ptr()
    bad_b = words.copy()
    bad_b[L.W_SCALE_B] = 0
    for w in (bad_c, bad_b):
        before = _lib.launch_count()
        with pytest.raises(ValueError):
            _lib.check(_lib.load().ctgb_contract_pair2(w.ctypes.data, pa, pb, pa2, pb2, pc, 0))
        assert _lib.launch_count() == before
    assert float(x.abs().sum().item()) == 0.0


def test_contract_pair2_zero_factor_scales_by_zero():
    words = _pair_words(L.VAR_ROWSTREAM, "complex128", 1536, 3, 4, False).copy()
    slots = torch.tensor([0.0, 3.0], dtype=torch.float64, device="cuda")
    words[L.W_SCALE_A], words[L.W_SCALE_B] = slots.data_ptr(), slots.data_ptr() + 8
    A, B = make_arrays([(1536, 4), (4, 3)], "complex128", seed=1)
    a, b = torch.tensor(A).cuda(), torch.tensor(B).cuda()
    c = torch.full((1536, 3), float("nan"), dtype=torch.complex128, device="cuda")
    _lib.check(_lib.load().ctgb_contract_pair2(words.ctypes.data, a.data_ptr(), b.data_ptr(), a.data_ptr(),
                                               b.data_ptr(), c.data_ptr(), 0))
    assert torch.all(c == 0)


# ------------------------------------------------------------------ ex.jvp, stripped
def _sjvp(ex, arrays, tans, **kw):
    res = ex.jvp(_dev(arrays), _dev(tans), **kw)
    torch.cuda.synchronize()
    if isinstance(res, tuple):
        (m, e), dm = res
        return m.cpu().numpy(), float(e.item()), dm.cpu().numpy()
    return res.cpu().numpy()


OPTIONS = [{}, {"accumulate": "double"}, {"precision": "tf32"}]


@pytest.mark.parametrize("rec", [r for r in TREES if r["dtype"] == "complex128"], ids=lambda r: r["name"])
def test_complex128_stripped_tangent_equals_unstripped(rec):
    """dm 10^e against the unstripped ex.jvp tangent, over all slices and a slice range, both primal modes"""
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=6.0)
    n = len(arrays)
    tans = make_arrays(spec.shapes(), "complex128", seed=rec["seed"] + 1)
    plain = cb.TreeExecutor(spec, dtype="complex128")
    ex = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True, stripped_grad=True)
    for wrt in ([n - 1], None):
        t = tans if wrt is None else [tans[i] for i in wrt]
        ranges = [(0, None)] + ([(1, ex.nslices - 1)] if ex.nslices > 1 else [])
        for begin, count in ranges:
            _o, want = (x.cpu().numpy() for x in plain.jvp(_dev(arrays), _dev(t), begin, 1, count, wrt=wrt))
            m, e, dm = _sjvp(ex, arrays, t, begin=begin, count=count, wrt=wrt)
            m0, e0 = ex.contract_device(_dev(arrays), begin, 1, count)
            # (the same records; split-K and dot-stream nodes sum in a run-dependent order)
            assert abs(e - float(e0.item())) <= 1e-12 and nrel(m, m0.cpu().numpy()) <= 1e-13
            assert nrel(dm * 10.0 ** e, want) <= 1e-12, (wrt, begin, nrel(dm * 10.0 ** e, want))
            dm2 = _sjvp(ex, arrays, t, begin=begin, count=count, wrt=wrt, primal=False, exponent=e)
            assert nrel(dm2, dm) <= 1e-13


@pytest.mark.parametrize("name", ["lattice6x6_d3_sliced", "rand_r3_o1_hi1_ho1_None_s42_sliced_out", "peps8x8_d2"])
@pytest.mark.parametrize("opts", OPTIONS, ids=lambda o: "-".join(f"{k}={v}" for k, v in o.items()) or "default")
def test_single_precision_options(name, opts):
    """complex64 with accumulate="double" (a wide running mantissa and tangent) or tf32, against the
    complex128 unstripped tangent; sliced outputs ride the chunk descriptor"""
    rec = next(r for r in TREES if r["name"] == name)
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=4.0)
    tans = make_arrays(spec.shapes(), "complex128", seed=rec["seed"] + 2)
    _o, want = (x.cpu().numpy() for x in cb.TreeExecutor(spec, dtype="complex128").jvp(_dev(arrays), _dev(tans)))
    ex = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True, stripped_grad=True, **opts)
    lo = [a.astype("complex64") for a in arrays]
    m, e, dm = _sjvp(ex, lo, [t.astype("complex64") for t in tans])
    if opts.get("accumulate") == "double":
        assert dm.dtype == np.complex128 and m.dtype == np.complex128
    tol = 2e-3 if opts.get("precision") == "tf32" else 1e-4
    got = dm.astype(np.complex128) * 10.0 ** e
    assert nrel(got, want) <= tol, nrel(got, want)


def test_constants_and_stripped_plan_structure():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=5.0)
    tans = make_arrays(spec.shapes(), "complex128", seed=3)
    n = len(arrays)
    const = {i: arrays[i] for i in range(1, n, 3)}
    var = [i for i in range(n) if i not in const]
    _o, want = (x.cpu().numpy() for x in cb.TreeExecutor(spec, dtype="complex128").jvp(
        _dev(arrays), _dev([tans[i] for i in var]), wrt=var))
    ex = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True, stripped_grad=True, constants=const)
    m, e, dm = _sjvp(ex, [arrays[i] for i in var], [tans[i] for i in var])
    assert nrel(dm * 10.0 ** e, want) <= 1e-12
    # every tangent record measures nothing; a one-term record after its primal reuses its scaled copy
    plan = ex.jvp_plan()
    modes = plan.strip_modes()
    assert all(after == 0 for (pre, after), t in zip(modes, plan.tangent_marks) if t)
    print(f"lattice6x6 stripped JVP: {plan.two_term_nodes} two-term nodes, "
          f"{plan.launches_per_slice()} launches per slice")


# ------------------------------------------------------------------ m20 slice, complex64, untuned
def _m20_euler(width, scale):
    spec = appxB_at_width(width)
    arrays = make_arrays(spec.shapes(), "complex64", seed=0, scale=scale)
    ex = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True, stripped_grad=True)
    dev = _dev(arrays)
    n = len(dev)
    (m, e), dm_all = ex.jvp(dev, dev, 0, 1, 1)
    m = m.to(torch.complex128)
    (m1, e1), dm_one = ex.jvp(dev, [dev[n // 2]], 0, 1, 1, wrt=[n // 2])
    torch.cuda.synchronize()
    e, e1 = float(e.item()), float(e1.item())
    dm_one = dm_one.to(torch.complex128) * 10.0 ** (e1 - e)  # (relative to the first call's e)
    # multilinear: along x_i = x_i the tangent is m for one input and n m for all of them
    err_one = float((dm_one.to(torch.complex128) - m).abs().max() / m.abs().max())
    err_all = float((dm_all.to(torch.complex128) / n - m).abs().max() / m.abs().max())
    print(f"m20 W=2^{width} complex64 stripped JVP, scale {scale}: e {e:.4f}, one input {err_one:.2e}, "
          f"all {n} inputs {err_all:.2e}")
    assert math.isfinite(e) and abs(e - e1) <= 1e-5 and float(m.abs().max()) > 0
    assert err_one <= 1e-5 and err_all <= 1e-5
    return ex, dev, e


@pytest.mark.parametrize("scale", [1.0, 0.4])
def test_m20_w26_complex64_euler_identity(scale):
    """inputs without a tuning scale: at 1 the unstripped amplitude overflows, at 0.4 it underflows"""
    spec = appxB_at_width(26)
    arrays = make_arrays(spec.shapes(), "complex64", seed=0, scale=scale)
    amp = cb.TreeExecutor(spec, dtype="complex64").contract_device(_dev(arrays), 0, 1, 1).cpu().numpy()
    assert (not np.isfinite(amp).all()) if scale == 1.0 else np.all(amp == 0)
    torch.cuda.empty_cache()
    ex, dev, e = _m20_euler(26, scale)
    if scale == 1.0:
        # dot-product identity with the stripped VJP on the same e: <g, v> = <1, dm> for v = x
        (m, _e), dm = ex.jvp(dev, [dev[0]], 0, 1, 1, wrt=[0])
        g = ex.vjp(dev, torch.ones(ex.plan.out_shape, dtype=dev[0].dtype, device="cuda"), 0, 1, 1, wrt=[0],
                   exponent=e)[0]
        lhs = complex(torch.sum(dev[0].to(torch.complex128) * g.to(torch.complex128).conj()).item())
        rhs = complex(dm.to(torch.complex128).sum().item())
        assert abs(lhs - rhs) <= 1e-5 * max(abs(rhs), 1e-30), (lhs, rhs)


def test_m20_w30_stripped_jvp_plan_bytes():
    spec = appxB_at_width(30)
    ir = spec.contractions()
    plan = JvpPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype="complex64",
                   strip_exponent=True, stripped_grad=True)
    free = torch.cuda.mem_get_info()[0]
    print(f"m20 W=2^30 complex64 stripped JVP plan: {plan.total_bytes} bytes ({plan.total_bytes / GIB:.2f} GiB), "
          f"{free / GIB:.2f} GiB free")
    if plan.total_bytes + (4 << 30) > free:
        pytest.skip(f"the stripped JVP plan needs {plan.total_bytes} bytes, {free} free")
    del plan
    _m20_euler(30, 1.0)


# ------------------------------------------------------------------ peps8x8, complex64 overflow
def test_peps8x8_log_amplitude_tangent():
    import bench

    spec, arrays, _desc = bench.load_workload("peps8x8", "complex128")
    ex128 = cb.TreeExecutor(spec, dtype="complex128")
    amp0 = complex(ex128.contract_device(_dev(arrays)).cpu().numpy().reshape(-1)[0])
    s = (1e45 / abs(amp0)) ** (1.0 / len(arrays))
    arrays = [a * s for a in arrays]
    tans = make_arrays([a.shape for a in arrays], "complex128", seed=4)
    tans = [t * s for t in tans]
    amp, damp = (complex(x.cpu().numpy().reshape(-1)[0]) for x in ex128.jvp(_dev(arrays), _dev(tans)))
    want = (np.conj(amp) * damp).real / abs(amp) ** 2
    a64 = [a.astype("complex64") for a in arrays]
    t64 = [t.astype("complex64") for t in tans]
    assert not np.isfinite(cb.TreeExecutor(spec, dtype="complex64").contract_device(_dev(a64)).cpu().numpy()).all()
    ex = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True, stripped_grad=True)
    m, e, dm = _sjvp(ex, a64, t64)
    m0, dm0 = complex(m.reshape(-1)[0]), complex(dm.reshape(-1)[0])
    got = (np.conj(m0) * dm0).real / abs(m0) ** 2
    print(f"peps8x8 complex64 stripped JVP: e {e:.4f}, d log|amp| {got:.6e} against {want:.6e}")
    assert abs(got - want) <= 1e-3 * max(1.0, abs(want))


# ------------------------------------------------------------------ forward AD
def test_forward_ad_entry_points():
    rec = next(r for r in TREES if r["name"] == "rand_r3_o1_hi1_ho1_None_s42_sliced_out")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=8.0)
    tans = make_arrays(spec.shapes(), "complex128", seed=9)
    _o, want = (x.cpu().numpy() for x in cb.TreeExecutor(spec, dtype="complex128").jvp(_dev(arrays), _dev(tans)))
    ex = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True, stripped_grad=True)
    with fwAD.dual_level():
        xs = [fwAD.make_dual(x, t) for x, t in zip(_dev(arrays), _dev(tans))]
        with warnings.catch_warnings():
            warnings.simplefilter("error", UserWarning)
            m, e = cb.contract_tree(ex, xs)
            assert isinstance(e, float)
            dm = fwAD.unpack_dual(m).tangent
            assert nrel(dm.cpu().numpy() * 10.0 ** e, want) <= 1e-12
            m2, e2 = cb.contract_tree(spec, xs, strip_exponent=True, stripped_grad=True)
            assert abs(e2 - e) <= 1e-12 and nrel(fwAD.unpack_dual(m2).tangent.cpu().numpy() * 10.0 ** e2, want) <= 1e-12
        # check_zero on a zero result: (0.0, -inf) and no tangent; without it a zero tangent
        zs = [fwAD.make_dual(torch.zeros_like(x), t) for x, t in zip(_dev(arrays), _dev(tans))]
        assert cb.contract_tree(ex, zs, check_zero=True) == (0.0, -math.inf)
        mz, ez = cb.contract_tree(ex, zs)
        assert ez == -math.inf and torch.all(fwAD.unpack_dual(mz).tangent == 0)
        # the per-slice contractor and make_contractor on one slice's flat records
        from oracle import grad_oracle as go

        sl = [np.ascontiguousarray(a) for a in go.slice_arrays(spec.inputs, spec.sliced, arrays, 0)]
        tsl = [np.ascontiguousarray(a) for a in go.slice_arrays(spec.inputs, spec.sliced, tans, 0)]
        flat = cb.B200Contractor.from_tree(spec)
        for con in (cb.B200Contractor.from_tree(spec, strip_exponent=True, stripped_grad=True),
                    cb.make_contractor(spec, strip_exponent=True, stripped_grad=True)):
            ms, es = con(*[fwAD.make_dual(x, t) for x, t in zip(_dev(sl), _dev(tsl))])
            assert isinstance(es, float)
            ref = flat(*[fwAD.make_dual(x, t) for x, t in zip(_dev(sl), _dev(tsl))])
            assert nrel(fwAD.unpack_dual(ms).tangent.cpu().numpy() * 10.0 ** es,
                        fwAD.unpack_dual(ref).tangent.cpu().numpy()) <= 1e-12


# ------------------------------------------------------------------ zero-amplitude slice, installed path, expression
@pytest.mark.parametrize("zero_slice", [0, 1], ids=["zero_slice_first", "zero_slice_second"])
def test_zero_amplitude_slice_keeps_its_tangent(zero_slice):
    """a slice whose root product is exactly zero while its lower factors are not keeps its tangent,
    folded first or second, on the device as in the emulator (tests/test_jvp_strip_cpu.py)"""
    from tests.test_jvp_strip_cpu import zero_amplitude_case

    spec, arrays, tans = zero_amplitude_case(zero_slice)
    _o, want = (x.cpu().numpy() for x in cb.TreeExecutor(spec, dtype="float64").jvp(_dev(arrays), _dev(tans)))
    ex = cb.TreeExecutor(spec, dtype="float64", strip_exponent=True, stripped_grad=True)
    m, e, dm = _sjvp(ex, arrays, tans)
    assert math.isfinite(e)
    assert nrel(dm * 10.0 ** e, want) <= 1e-13, nrel(dm * 10.0 ** e, want)
    # the zero slice alone: a zero result, and a zero tangent
    _m0, e0, dm0 = _sjvp(ex, arrays, tans, begin=zero_slice, count=1)
    assert e0 == -math.inf and np.all(dm0 == 0)


def test_forward_ad_through_array_contract_expression():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=5.0)
    tans = make_arrays(spec.shapes(), "complex128", seed=12)
    n = len(arrays)
    consts = {i: arrays[i] for i in range(0, n, 4)}
    var = [i for i in range(n) if i not in consts]
    _o, want = (x.cpu().numpy() for x in cb.TreeExecutor(spec, dtype="complex128").jvp(
        _dev(arrays), _dev([tans[i] for i in var]), wrt=var))
    expr = cb.array_contract_expression(spec.inputs, spec.output, optimize=spec, constants=consts,
                                        strip_exponent=True, stripped_grad=True)
    with fwAD.dual_level():
        xs = [fwAD.make_dual(x, t) for x, t in zip(_dev([arrays[i] for i in var]), _dev([tans[i] for i in var]))]
        m, e = expr(*xs)
        assert isinstance(e, float)
        dm = fwAD.unpack_dual(m).tangent
    assert nrel(dm.cpu().numpy() * 10.0 ** e, want) <= 1e-12


@pytest.fixture()
def ctg_device(monkeypatch):
    """cotengra from oracle/_ref/ with its numpy-only autoray stand-in dispatching torch tensors to
    torch (the slice sum of gather_slices), launches on the device (the CPU suite's ``ctg`` fixture
    without its emulator)"""
    import os
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(root, "oracle", "refshim"), os.path.join(root, "oracle", "_ref")]
    try:
        import autoray
        import cotengra

        np_do = autoray.do

        def do(fn, *args, like=None, **kwargs):
            first = args[0] if args else None
            if isinstance(first, (list, tuple)) and first:
                first = first[0]
            if isinstance(first, torch.Tensor):
                if fn == "stack":
                    return torch.stack(args[0], *args[1:], **kwargs)
                return getattr(torch, fn)(*args, **kwargs)
            return np_do(fn, *args, like=like, **kwargs)

        monkeypatch.setattr(autoray, "do", do)
        for mod in list(sys.modules.values()):
            if getattr(mod, "__name__", "").startswith("cotengra.") and getattr(mod, "do", None) is np_do:
                monkeypatch.setattr(mod, "do", do)
        yield cotengra
    finally:
        del sys.path[:2]


@pytest.mark.reference
def test_forward_ad_through_installed_tree_contract(ctg_device):
    ctg = ctg_device
    """``cb.install(tree, strip_exponent=True, stripped_grad=True)`` on CUDA tensors: cotengra's own
    stripped slice combiner carries the slices' tangents"""
    con = ctg.utils.lattice_equation([3, 3], d_min=2, d_max=3, seed=1)
    tree = ctg.array_contract_tree(con.inputs, con.output, con.size_dict, optimize="greedy")
    tree.slice_(target_slices=4)
    assert tree.nslices > 1
    arrays = ctg.utils.make_arrays_from_inputs(con.inputs, con.size_dict, seed=0, dtype="complex128")
    arrays = [np.asarray(a) * 30.0 for a in arrays]
    tans = make_arrays([a.shape for a in arrays], "complex128", seed=2)
    spec = cb.TreeSpec.from_cotengra(tree)
    _o, want = (x.cpu().numpy() for x in cb.TreeExecutor(spec, dtype="complex128").jvp(_dev(arrays), _dev(tans)))
    cb.install(tree, strip_exponent=True, stripped_grad=True)
    with fwAD.dual_level():
        xs = [fwAD.make_dual(x, t) for x, t in zip(_dev(arrays), _dev(tans))]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m, e = tree.contract(xs, strip_exponent=True)
        e = float(e)
        dm = fwAD.unpack_dual(m).tangent
    assert e > 5 and dm.is_cuda
    assert nrel(dm.cpu().numpy() * 10.0 ** e, np.asarray(want).reshape(dm.shape)) <= 1e-12
