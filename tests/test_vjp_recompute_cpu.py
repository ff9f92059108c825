"""Reverse mode under a workspace budget (``VjpPlan(max_bytes=...)``) on the CPU: per-slice forward
values recomputed in phase 2, walked by the descriptor emulator in exact-size, NaN-filled arenas
(a slot released too early spoils the result), against the unbudgeted plan bit for bit and the
torch-CPU gradient oracle; planner properties; full-size planning of the benchmarked trees; the
public interface with the device launch emulated."""

import gc
import time

import numpy as np
import pytest
import torch

import cotengra_b200 as cb
from cotengra_b200 import VjpPlan
from cotengra_b200.executor import PHASE_VAR_BWD
from cotengra_b200.fusion import fuse_stems
from oracle import grad_oracle as go
from tests import emu_device
from tests.desc_emulator import emulate_plan
from tests.helpers import load_json, make_arrays, tree_spec
from tests.test_vjp_cpu import ctg  # noqa: F401  (the drop-in fixture)

TREES = load_json("trees.json")
GIB = 1 << 30


@pytest.fixture(autouse=True)
def _collect_while_emulated(monkeypatch):
    yield
    gc.collect()


def _bytes_only(dtype, B, M, N, K, elems):
    return 1e-9 * elems + 1e-12 * B * M * N * K


def _plan(ir, spec, dtype, sm_count=8, **kw):
    return VjpPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype,
                   sm_count=sm_count, **kw)


def min_bytes(ir, spec, dtype, **kw):
    """The smallest budget the planner reaches (a budget of one byte is refused with it)."""
    with pytest.raises(MemoryError) as e:
        _plan(ir, spec, dtype, max_bytes=1, **kw)
    assert str(e.value.min_bytes) in str(e.value)
    return e.value.min_bytes


def recomputed(plan):
    return [nd for nd in plan.nodes if nd.get("recompute")]


def _same_plan(a, b):
    assert (a.workspace_bytes, a.persistent_bytes, a.cotangent_offset) == \
        (b.workspace_bytes, b.persistent_bytes, b.cotangent_offset)
    assert len(a.nodes) == len(b.nodes)
    ia = {id(t): i for i, t in enumerate(a.tensors)}
    ib = {id(t): i for i, t in enumerate(b.tensors)}
    for x, y in zip(a.nodes, b.nodes):
        assert (x["kind"], x["phase"], x["zero_fill"]) == (y["kind"], y["phase"], y["zero_fill"])
        assert np.array_equal(x["words"], y["words"])
        for s in ("a", "b", "c"):
            assert (x[s] is None) == (y[s] is None)
            if x[s] is not None:
                assert ia[id(x[s])] == ib[id(y[s])]
    for s, t in zip(a.tensors, b.tensors):
        assert (s.kind, s.offset, s.nbytes, s.input_index) == (t.kind, t.offset, t.nbytes, t.input_index)


def _check_budgets(ir, spec, dt, arrays, cot, want, **kw):
    base = _plan(ir, spec, dt, **kw)
    ref = emulate_plan(base, arrays, cotangent=cot)
    lo = min_bytes(ir, spec, dt, **kw)
    fwd_words = [np.asarray(nd["words"]) for nd in base.fwd.nodes]
    for budget in sorted({lo, (lo + base.total_bytes) // 2, base.total_bytes}):
        plan = _plan(ir, spec, dt, max_bytes=budget, **kw)
        assert plan.total_bytes <= budget and plan.min_bytes == (lo if budget < base.total_bytes
                                                                  else base.total_bytes)
        if budget >= base.total_bytes:
            _same_plan(plan, base)
            assert plan.recompute_macs == 0
        for nd in recomputed(plan):
            assert nd["phase"] == PHASE_VAR_BWD
            assert any(np.array_equal(nd["words"], w) for w in fwd_words)
        got = emulate_plan(plan, arrays, cotangent=cot)
        for g, r, w in zip(got, ref, want):
            assert np.array_equal(g, r)  # the same descriptors on the same operands
            d = np.linalg.norm(w)
            assert np.linalg.norm(g - w) <= 1e-10 * (d if d else 1.0)
    return base, lo


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_budgeted_gradients_bit_identical(rec):
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    ir = spec.contractions()
    base = _plan(ir, spec, dt)
    cot = make_arrays([base.out_shape], dt, seed=rec["seed"] + 1)[0]
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, arrays, cot)
    _check_budgets(ir, spec, dt, arrays, cot, want)
    _check_budgets(ir, spec, dt, arrays, cot, want, hoist=False)
    fused, _info = fuse_stems(spec, dt, min_big=2, ratio=1.0, min_gain=-1.0, model=_bytes_only)
    _check_budgets(fused.contractions(), spec, dt, arrays, cot, want)


def test_budget_refusals():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    ir = spec.contractions()
    lo = min_bytes(ir, spec, rec["dtype"])
    with pytest.raises(MemoryError, match=str(lo)):
        _plan(ir, spec, rec["dtype"], max_bytes=lo - 1)
    for bad in (0, -5, 1.5, "1", True):
        with pytest.raises(ValueError):
            _plan(ir, spec, rec["dtype"], max_bytes=bad)
    base = _plan(ir, spec, rec["dtype"])
    assert base.min_bytes == base.total_bytes and base.recompute_macs == 0
    _same_plan(_plan(ir, spec, rec["dtype"], max_bytes=10 * base.total_bytes), base)


@pytest.mark.parametrize("width", [10])
def test_sycamore_stems_at_small_width(width):
    """The m20 tree sliced to W = 2^width, stem fusion on, one slice: a budget at the planner's
    minimum recomputes along both stems; the gradients are bit-identical to the unbudgeted plan's."""
    from tests.slicing_util import appxB_at_width

    spec = appxB_at_width(width)
    dt = "complex64"
    fused, _info = fuse_stems(spec, dt, min_big=1 << (width - 6))
    ir = fused.contractions()
    base = _plan(ir, spec, dt, sm_count=132)
    lo = min_bytes(ir, spec, dt, sm_count=132)
    plan = _plan(ir, spec, dt, sm_count=132, max_bytes=lo)
    assert plan.total_bytes <= lo < base.total_bytes / 2
    # the subtree (root operand) every forward node belongs to; every subtree whose root operand is
    # a wide stem end recomputes values of at least a quarter of the width
    nodes = base.fwd.nodes
    owner = {id(nodes[-1]["a"]): 0, id(nodes[-1]["b"]): 1}
    for nd in reversed(nodes[:-1]):
        for s in (nd["a"], nd["b"]):
            if s is not None and id(nd["c"]) in owner:
                owner[id(s)] = owner[id(nd["c"])]
    sides = {owner[id(nodes[i]["c"])] for i in (nd["fwd_index"] for nd in recomputed(plan))
             if nodes[i]["c"].nbytes * 4 >= 8 << width}
    wide = {k for k, s in enumerate((nodes[-1]["a"], nodes[-1]["b"])) if s.nbytes * 4 >= 8 << width}
    assert wide == {0, 1} == sides
    arrays = make_arrays(spec.shapes(), dt, seed=3, scale=0.65)
    cot = np.ones(base.out_shape, dt)
    ref = emulate_plan(base, arrays, cotangent=cot, slice_ids=[0])
    got = emulate_plan(plan, arrays, cotangent=cot, slice_ids=[0])
    for g, r in zip(got, ref):
        assert np.array_equal(g, r)


# planner minimum and recompute MACs (one slice) of the benchmarked trees, stem fusion on, 132 SMs;
# DESIGN.md section 7b quotes them
FULL_SIZE = [
    # (config, dtype, budget or None for the minimum, largest min_bytes, largest recompute_macs as a
    # fraction of the forward's per-slice MACs)
    ("m20", "complex64", 56 * GIB, 41.5 * GIB, 0.46),
    ("m20", "complex128", None, 70.5 * GIB, None),
    ("m12", "complex64", None, 80.1 * GIB, None),
]


@pytest.mark.parametrize("config,dtype,budget,max_min,max_macs", FULL_SIZE)
def test_full_size_planning(config, dtype, budget, max_min, max_macs):
    import bench

    spec, _arrays, _desc = bench.load_workload(config, dtype)
    fused, _info = fuse_stems(spec, dtype)
    ir = fused.contractions()
    t0 = time.perf_counter()
    lo = min_bytes(ir, spec, dtype, sm_count=132)
    plan = _plan(ir, spec, dtype, sm_count=132, max_bytes=budget or lo)
    elapsed = time.perf_counter() - t0
    print(f"{config} {dtype}: min_bytes {lo / GIB:.2f} GiB, plan {plan.total_bytes / GIB:.2f} GiB, "
          f"recompute {plan.recompute_macs / plan.fwd.macs_per_slice:.3f} of the forward MACs, "
          f"{elapsed:.1f} s for both plans")
    assert elapsed < 60
    assert lo <= max_min and plan.total_bytes <= (budget or lo)
    assert 0 < plan.recompute_macs <= plan.fwd.macs_per_slice
    if max_macs is not None:
        assert plan.recompute_macs <= max_macs * plan.fwd.macs_per_slice


# ---------------------------------------------------------------------------- public interface


def test_contract_tree_backward_under_budget(monkeypatch):
    emu_device.install(monkeypatch)
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    grads = []
    for budget in (None, "min"):
        if budget == "min":
            budget = min_bytes(cb.TreeExecutor(spec, dtype=dt)._ir, spec, dt, sm_count=132)
        ts = [torch.tensor(a, requires_grad=True) for a in arrays]
        out = cb.contract_tree(spec, ts, dtype=dt, vjp_max_bytes=budget)
        out.real.sum().backward()
        grads.append([t.grad.numpy() for t in ts])
    for a, b in zip(*grads):
        assert np.array_equal(a, b)
    # an executor's own budget, and the plan it builds
    ex = cb.TreeExecutor(spec, dtype=dt, vjp_max_bytes=budget)
    assert ex.vjp_plan().total_bytes <= budget and recomputed(ex.vjp_plan())
    ts = [torch.tensor(a, requires_grad=True) for a in arrays]
    cb.contract_tree(ex, ts).real.sum().backward()
    for t, g in zip(ts, grads[0]):
        assert np.array_equal(t.grad.numpy(), g)


@pytest.mark.reference
def test_installed_tree_backward_under_budget(ctg):
    """``cb.install(tree, vjp_max_bytes=B)``: cotengra's own ``tree.contract`` backpropagates through
    budgeted plans, to the gradients of the unbudgeted ones."""
    import warnings

    con = ctg.utils.lattice_equation([3, 3], d_min=2, d_max=3, seed=1)
    arrays = ctg.utils.make_arrays_from_inputs(con.inputs, con.size_dict, seed=0, dtype="complex128")
    grads, budget = [], None
    for _ in range(2):
        tree = ctg.array_contract_tree(con.inputs, con.output, con.size_dict, optimize="greedy")
        tree.slice_(target_slices=4)
        fn = cb.install(tree, vjp_max_bytes=budget)
        ts = [torch.tensor(np.asarray(a), requires_grad=True) for a in arrays]
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            out = tree.contract(ts)
        out.real.sum().backward()
        grads.append([t.grad.numpy() for t in ts])
        (flat,) = fn._plans.values()
        (plan,) = flat._vjp_plans.values()
        if budget is None:
            with pytest.raises(MemoryError) as e:
                VjpPlan(*flat._program, (), dtype="complex128", max_bytes=1)
            budget = e.value.min_bytes
            assert budget < plan.total_bytes
        else:
            assert plan.total_bytes <= budget and recomputed(plan)
    for a, b in zip(*grads):
        assert np.array_equal(a, b)
