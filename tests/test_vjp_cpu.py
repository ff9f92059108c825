"""Reverse mode (``cotengra_b200/vjp.py``) on the CPU: the VJP plans' descriptors walked by the
descriptor emulator (``tests/desc_emulator.py``) against the torch-CPU gradient oracle
(``oracle/grad_oracle.py``), finite differences, planner properties, and the autograd paths of
the public interface with the device launch emulated."""

import gc
import os
import sys
import warnings

import numpy as np
import pytest
import torch

import cotengra_b200 as cb
from cotengra_b200 import VjpPlan
from cotengra_b200.fusion import fuse_stems
from oracle import grad_oracle as go
from tests import emu_device
from tests.desc_emulator import emulate_plan
from tests.helpers import load_json, make_arrays, tree_spec

TREES = load_json("trees.json")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(autouse=True)
def _collect_while_emulated(monkeypatch):
    """Autograd graphs hold executors in reference cycles: free them while the emulator's
    ``destroy`` is still installed (teardown runs before monkeypatch's)."""
    yield
    gc.collect()


def _bytes_only(dtype, B, M, N, K, elems):
    """A model that always prefers fewer bytes: forces stem fusion on small test trees."""
    return 1e-9 * elems + 1e-12 * B * M * N * K


def _plan(spec, dtype, **kw):
    return VjpPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced,
                   dtype=dtype, sm_count=8, **kw)


def nrel(got, want):
    """norm-wise relative error of one gradient"""
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _check(got, want, wrt, tol):
    for i, (g, w) in enumerate(zip(got, want)):
        if i in wrt:
            assert g is not None and nrel(g, w) <= tol, (i, nrel(g, w))
        else:
            assert g is None and w is None


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_gradients_match_oracle(rec):
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    n = len(arrays)
    base = _plan(spec, dt)
    cot = make_arrays([base.out_shape], dt, seed=rec["seed"] + 1)[0]
    ir = spec.contractions()
    rng = np.random.default_rng(rec["seed"])
    subsets = [None] + [sorted(rng.choice(n, size=max(1, n // k), replace=False).tolist()) for k in (2, 3)]
    for wrt in subsets:
        want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, arrays, cot, wrt=wrt)
        w = set(range(n)) if wrt is None else set(wrt)
        plan = base if wrt is None else _plan(spec, dt, wrt=wrt)
        _check(emulate_plan(plan, arrays, cotangent=cot), want, w, 1e-10)
        if wrt is None:
            # hoisting off, and stem fusion forced on (the fused program is differentiated as it runs)
            _check(emulate_plan(_plan(spec, dt, hoist=False), arrays, cotangent=cot), want, w, 1e-10)
            fused, _info = fuse_stems(spec, dt, min_big=2, ratio=1.0, min_gain=-1.0, model=_bytes_only)
            fplan = VjpPlan(fused.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced,
                            dtype=dt, sm_count=8)
            _check(emulate_plan(fplan, arrays, cotangent=cot), want, w, 1e-10)
    if base.nslices > 1:
        # a slice range split into two calls adds up to the full call
        h = base.nslices // 2
        g1 = emulate_plan(base, arrays, cotangent=cot, slice_ids=range(0, h))
        g2 = emulate_plan(base, arrays, cotangent=cot, slice_ids=range(h, base.nslices))
        want1 = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, arrays, cot,
                                  slice_ids=range(0, h))
        _check(g1, want1, set(range(n)), 1e-10)
        full = emulate_plan(base, arrays, cotangent=cot)
        for a, b, c in zip(g1, g2, full):
            assert nrel(a + b, c) < 1e-12


FD_TREES = ["lattice4x4_sliced", "pre_diag_sliced", "pre_sum", "rand_r3_o1_hi1_ho1_None_s42_sliced_out"]


@pytest.mark.parametrize("name", [n for n in FD_TREES if any(r["name"] == n for r in TREES)])
def test_central_differences(name):
    """d<c, f(x)>/dx against central differences, in float64 (no complex convention involved)."""
    rec = next(r for r in TREES if r["name"] == name)
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "float64", seed=rec["seed"])
    plan = _plan(spec, "float64")
    fwd = plan.fwd
    cot = make_arrays([plan.out_shape], "float64", seed=3)[0]
    grads = emulate_plan(plan, arrays, cotangent=cot)

    def loss(xs):
        return float(np.sum(cot * emulate_plan(fwd, xs)))

    rng = np.random.default_rng(0)
    eps = 1e-6
    for i in rng.choice(len(arrays), size=min(4, len(arrays)), replace=False):
        for flat in rng.choice(arrays[i].size, size=min(3, arrays[i].size), replace=False):
            xp = [a.copy() for a in arrays]
            xm = [a.copy() for a in arrays]
            xp[i].reshape(-1)[flat] += eps
            xm[i].reshape(-1)[flat] -= eps
            fd = (loss(xp) - loss(xm)) / (2 * eps)
            assert abs(fd - grads[i].reshape(-1)[flat]) <= 1e-6 * max(1.0, abs(fd)), (i, flat)


def test_complex_tree_against_torch_autograd_directly():
    """config1_rand10 (complex128, unsliced) as ONE torch.einsum of the whole network."""
    rec = next(r for r in TREES if r["name"] == "config1_rand10")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    plan = _plan(spec, "complex128")
    cot = make_arrays([plan.out_shape], "complex128", seed=9)[0]
    labels = {}
    sym = lambda ix: labels.setdefault(ix, "abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ"[len(labels)])  # noqa: E731
    eq = ",".join("".join(sym(ix) for ix in t) for t in spec.inputs) + "->" + "".join(sym(ix) for ix in spec.output)
    ts = [torch.tensor(a, requires_grad=True) for a in arrays]
    out = torch.einsum(eq, *ts)
    want = torch.autograd.grad(out, ts, grad_outputs=torch.tensor(cot).reshape(out.shape))
    for g, w in zip(emulate_plan(plan, arrays, cotangent=cot), want):
        assert nrel(g, w.numpy()) < 1e-12


def test_pruned_subtrees_emit_no_backward_nodes():
    rec = next(r for r in TREES if r["name"] == "peps8x8_d2")
    spec = tree_spec(rec)
    full = _plan(spec, rec["dtype"])
    one = _plan(spec, rec["dtype"], wrt=[0])
    # every pairwise node with a wrt input below it forms at most two H, and only those nodes are differentiated
    n_nodes = len(full.fwd.nodes)
    assert full.n_backward_nodes == 2 * (n_nodes - sum(1 for nd in full.fwd.nodes if nd["kind"] == 1)) \
        + sum(1 for nd in full.fwd.nodes if nd["kind"] == 1)
    # with one input: one H per node on the path from the root to input 0, nothing else
    path, t = set(), None
    for i, nd in enumerate(full.fwd.nodes):
        srcs = [nd["a"]] + ([nd["b"]] if nd["b"] is not None else [])
        if any(s.kind == 0 and s.input_index == 0 for s in srcs) or any(id(s) == t for s in srcs):
            path.add(i)
            t = id(nd["c"])
    assert one.differentiated == sorted(path)
    assert one.n_backward_nodes == len(path)
    assert one.vjp_macs(1) < full.vjp_macs(1)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    cot = make_arrays([one.out_shape], rec["dtype"], seed=2)[0]
    g = emulate_plan(one, arrays, cotangent=cot)
    assert g[0] is not None and all(x is None for x in g[1:])


def test_workspace_reporting_and_refusals():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    plan = _plan(spec, rec["dtype"])
    assert plan.total_bytes == plan.workspace_bytes + plan.persistent_bytes
    assert any(t.kind == 6 for t in plan.tensors)   # hoisted H accumulators
    # (the emulator's arenas are exactly the reported bytes: any access beyond them raises)
    with pytest.raises(NotImplementedError):
        _plan(spec, rec["dtype"], strip_exponent=True)
    with pytest.raises(ValueError):
        _plan(spec, rec["dtype"], wrt=[len(spec.inputs)])


def test_tf32_32x32_selected_for_small_single_precision_results_only():
    from cotengra_b200.lowering import VAR_DMMA_32x32, VAR_TF32_32x32, build_pair_desc, classify_pair
    from cotengra_b200.vjp import choose_vjp_variant

    assert choose_vjp_variant("complex64", 1, 1 << 20, 8, 1 << 20) is None       # a big result
    assert choose_vjp_variant("complex64", 1, 8, 8, 1 << 20) == VAR_TF32_32x32
    assert choose_vjp_variant("float32", 1, 32, 32, 1 << 14) == VAR_TF32_32x32
    assert choose_vjp_variant("float32", 1, 32, 32, (1 << 14) - 1) is None
    assert choose_vjp_variant("complex64", 1, 4, 4, 1 << 20) is None              # DOTSTREAM4 keeps it
    assert choose_vjp_variant("complex128", 1, 8, 8, 1 << 20) is None
    dims = classify_pair("km", (1 << 14, 8), "kn", (1 << 14, 8), "mn")
    plan = build_pair_desc(dims, "complex64", variant=VAR_TF32_32x32, c_dense_elems=64, sm_count=132)
    assert plan.variant == VAR_TF32_32x32 and plan.splitk > 1
    assert build_pair_desc(dims, "complex128", variant=VAR_TF32_32x32).variant == VAR_DMMA_32x32


# ---------------------------------------------------------------------------- public interface


def _emulated_executor(monkeypatch, name, **kw):
    emu_device.install(monkeypatch)
    rec = next(r for r in TREES if r["name"] == name)
    spec = tree_spec(rec)
    return rec, spec, cb.TreeExecutor(spec, dtype=rec["dtype"], **kw)


@pytest.mark.parametrize("name", ["lattice4x4_sliced", "rand_r3_o1_hi1_ho1_None_s42_sliced_out", "projected"])
def test_contract_tree_backward(monkeypatch, name):
    rec, spec, ex = _emulated_executor(monkeypatch, name)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    ts = [torch.tensor(a, requires_grad=(i % 2 == 0)) for i, a in enumerate(arrays)]
    out = cb.contract_tree(ex, ts)
    assert out.grad_fn is not None
    cot = make_arrays([tuple(out.shape)], rec["dtype"], seed=4)[0]
    out.backward(torch.tensor(cot))
    wrt = [i for i in range(len(ts)) if i % 2 == 0]
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot, wrt=wrt)
    for i, t in enumerate(ts):
        if i in wrt:
            assert nrel(t.grad.numpy(), want[i]) < 1e-10
        else:
            assert t.grad is None
    # the executor's own entry point, over a slice range
    g = ex.vjp([torch.tensor(a) for a in arrays], torch.tensor(cot), wrt=[0])
    assert g[1] is None and nrel(g[0].numpy(), want[0]) < 1e-10


def test_paths_without_gradients_are_unchanged(monkeypatch):
    rec, spec, ex = _emulated_executor(monkeypatch, "lattice4x4_sliced")
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    calls = []
    monkeypatch.setattr(cb.contract, "_differentiable", lambda *a: calls.append(a))
    assert isinstance(cb.contract_tree(ex, arrays), np.ndarray)
    before = emu_device.FakeLib.launches
    out = cb.contract_tree(ex, [torch.tensor(a) for a in arrays])
    fwd_launches = sum(1 if nd["phase"] == 0 else ex.plan.nslices for nd in ex.plan.nodes)
    assert emu_device.FakeLib.launches - before == fwd_launches  # the forward plan, once
    assert out.grad_fn is None
    with torch.no_grad():
        out = cb.contract_tree(ex, [torch.tensor(a, requires_grad=True) for a in arrays])
    assert out.grad_fn is None and not calls


def test_strip_exponent_with_grad_warns(monkeypatch):
    rec, spec, ex = _emulated_executor(monkeypatch, "lattice4x4_sliced", strip_exponent=True)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
    m0, e0 = cb.contract_tree(ex, [torch.tensor(a) for a in arrays])
    with pytest.warns(UserWarning, match="no gradient") as warned:
        m, e = cb.contract_tree(ex, [torch.tensor(a, requires_grad=True) for a in arrays])
    assert e == e0 and torch.equal(m, m0) and m.grad_fn is None
    # the warning points at the caller's line
    assert [w.filename for w in warned if "no gradient" in str(w.message)] == [__file__]
    with pytest.raises(NotImplementedError):
        ex.vjp([torch.tensor(a) for a in arrays], torch.ones(ex.plan.out_shape, dtype=m.dtype))


# ---------------------------------------------------------------------------- drop-in


@pytest.fixture()
def ctg(monkeypatch):
    have = os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "cotengra", "__init__.py"))
    if not have:
        pytest.skip("cotengra is not installed in oracle/_ref/")
    sys.path[:0] = [os.path.join(ROOT, "oracle", "refshim"), os.path.join(ROOT, "oracle", "_ref")]
    try:
        import autoray
        import cotengra

        # the numpy-only autoray stand-in, made to dispatch torch tensors to torch (the slice
        # sum / stack of gather_slices), so that cotengra's own control flow records the graph
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
        emu_device.install(monkeypatch)
        yield cotengra
    finally:
        del sys.path[:2]


@pytest.mark.reference
@pytest.mark.parametrize("sliced_out", [False, True])
def test_installed_tree_contract_backward(ctg, sliced_out):
    """``cb.install(tree)``; cotengra's real ``tree.contract`` on torch tensors; ``.backward()``."""
    con = ctg.utils.lattice_equation([3, 3], d_min=2, d_max=3, seed=1) if not sliced_out else \
        ctg.utils.rand_equation(8, 3, n_out=2, seed=3, d_min=2, d_max=3)
    tree = ctg.array_contract_tree(con.inputs, con.output, con.size_dict, optimize="greedy")
    tree.slice_(target_slices=4)
    if sliced_out:
        tree.remove_ind_(tree.output[0])
        assert set(tree.sliced_inds) & set(tree.output)
    assert tree.nslices > 1
    arrays = ctg.utils.make_arrays_from_inputs(con.inputs, con.size_dict, seed=0, dtype="complex128")
    cb.install(tree)
    ts = [torch.tensor(np.asarray(a), requires_grad=True) for a in arrays]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        out = tree.contract(ts)
    cot = make_arrays([tuple(out.shape)], "complex128", seed=6)[0]
    out.backward(torch.tensor(cot))
    spec = cb.TreeSpec.from_cotengra(tree)
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(),
                             [np.asarray(a) for a in arrays], cot)
    for t, w in zip(ts, want):
        assert nrel(t.grad.numpy(), w) < 1e-10
