"""Reverse mode under a workspace budget on the device: budgeted ``VjpPlan``s (per-slice forward
values recomputed in phase 2) against the torch-CPU gradient oracle and the unbudgeted device
plan, the stem kernel families with recomputed operands, the m20 tree at W = 2^26 and at the
benchmarked W = 2^30, and the autograd path."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import torch  # noqa: E402

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import VjpPlan  # noqa: E402
from oracle import grad_oracle as go  # noqa: E402
from tests.helpers import load_json, make_arrays, tree_spec  # noqa: E402
from tests.slicing_util import appxB_at_width  # noqa: E402
from tests.test_gpu_vjp import STEM_CASES, _stem_spec  # noqa: E402

TREES = load_json("trees.json")
BIG = load_json("big_slices.json")
GIB = 1 << 30


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _dev(arrays):
    return [torch.tensor(np.asarray(a)).cuda() for a in arrays]


def _min_bytes(ex):
    with pytest.raises(MemoryError) as e:
        VjpPlan(ex._ir, ex.spec.inputs, ex.spec.output, ex.spec.size_dict, ex.spec.sliced, dtype=ex.dtype,
                max_bytes=1, **ex._plan_opts)
    return e.value.min_bytes


def _grads(ex, arrays, cot, max_bytes=None, **kw):
    g = ex.vjp(_dev(arrays), torch.tensor(np.asarray(cot)).cuda(), max_bytes=max_bytes, **kw)
    torch.cuda.synchronize()
    return [None if x is None else x.cpu().numpy() for x in g]


def _recomputed(plan):
    return [nd for nd in plan.nodes if nd.get("recompute")]


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_budgeted_device_gradients_match_oracle(rec):
    spec = tree_spec(rec)
    dt = rec["dtype"]
    lo_dt = "complex64" if dt == "complex128" else "float32"
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    ir = spec.contractions()
    for prec in (dt, lo_dt):
        ex = cb.TreeExecutor(spec, dtype=prec)
        a = [x.astype(prec) for x in arrays]
        cot = make_arrays([ex.plan.out_shape], dt, seed=rec["seed"] + 1)[0].astype(prec)
        want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, arrays, cot.astype(dt))
        own = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, a, cot)
        full = _grads(ex, a, cot)
        lo, hi = _min_bytes(ex), ex.vjp_plan().total_bytes
        for budget in sorted({lo, (lo + hi) // 2}):
            plan = ex.vjp_plan(max_bytes=budget)
            assert plan.total_bytes <= budget
            got = _grads(ex, a, cot, max_bytes=budget)
            for g, w, r, f in zip(got, want, own, full):
                if prec == dt:
                    assert nrel(g, w) <= 1e-10
                    assert nrel(g, f) <= 1e-10
                else:
                    assert nrel(g, w) <= max(1e-5, 3.0 * nrel(r, w))
                    assert nrel(g, f) <= max(1e-5, 3.0 * nrel(r, w))


@pytest.mark.parametrize("dtype,o,force,expect", STEM_CASES)
def test_stem_backward_reads_recomputed_values(dtype, o, force, expect):
    """``_stem_spec`` at the planner's minimum (the stem end ``ABC`` is recomputed for the root's
    backward step): the kernel family of the case still runs and the gradients hold."""
    spec = _stem_spec(1 << 20, 16, 8, o)
    hi = "complex128" if "complex" in dtype else "float64"
    arrays = make_arrays(spec.shapes(), hi, seed=5)
    cot = make_arrays([(1 << 20,)], hi, seed=6)[0]
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot)
    ex = cb.TreeExecutor(spec, dtype=dtype, fuse=False)
    opts = {} if force is None else {"variant": force}
    mk = lambda **kw: VjpPlan(ex._ir, spec.inputs, spec.output, spec.size_dict, (), dtype=dtype,  # noqa: E731
                              **opts, **kw)
    with pytest.raises(MemoryError) as e:
        mk(max_bytes=1)
    with torch.cuda.device(ex.device):
        plan = mk(max_bytes=e.value.min_bytes).create()
    assert expect in plan.variants(), plan.variants()
    fresh = {id(nd["c"]) for nd in _recomputed(plan)}
    assert [nd for nd in plan.nodes if nd["phase"] == 2 and not nd.get("recompute")
            and {id(nd["a"]), id(nd["b"])} & fresh]
    ex._vjp_plans[tuple(range(4))] = plan
    got = _grads(ex, [a.astype(dtype) for a in arrays], cot.astype(dtype))
    tol = 1e-10 if dtype == hi else 1e-5
    for g, w in zip(got, want):
        assert nrel(g, w) <= tol


@pytest.mark.parametrize("dtype,tol", [("complex128", 1e-10), ("complex64", 1e-5)])
def test_m20_w26_budgeted_matches_unbudgeted(dtype, tol):
    spec = appxB_at_width(26)
    arrays = make_arrays(spec.shapes(), dtype, seed=0, scale=0.65)
    ex = cb.TreeExecutor(spec, dtype=dtype)
    cot = np.ones(ex.plan.out_shape, dtype)
    full = _grads(ex, arrays, cot, begin=0, count=1)
    ex._vjp_plans.clear()
    ex._vjp_ws = None
    torch.cuda.empty_cache()
    lo = _min_bytes(ex)
    assert lo < ex.vjp_plan().total_bytes
    got = _grads(ex, arrays, cot, max_bytes=lo, begin=0, count=1)
    assert _recomputed(ex.vjp_plan(max_bytes=lo))
    for i, (g, f) in enumerate(zip(got, full)):
        assert nrel(g, f) <= tol, i


def _identity_check(width, dtype, budget, tol, amp_tol):
    """Slice 0 of the m20 tree with cotangent 1: the amplitude is linear in every input, so
    ``sum(x_i * conj(g_i))`` equals it for every i."""
    spec = appxB_at_width(width)
    arrays = make_arrays(spec.shapes(), dtype, seed=0, scale=0.65)
    ex = cb.TreeExecutor(spec, dtype=dtype)
    plan_bytes = budget if budget is not None else _min_bytes(ex)
    free = torch.cuda.mem_get_info()[0]
    inputs = 2 * sum(a.nbytes for a in arrays)
    if plan_bytes + inputs + ex.plan.total_bytes > free and plan_bytes + inputs + (1 << 30) > free:
        pytest.skip(f"W = 2^{width} {dtype}: {plan_bytes + inputs} bytes needed, {free} free")
    dev = _dev(arrays)
    amp = complex(ex.contract_device(dev, 0, 1, 1).cpu().numpy().reshape(-1)[0])
    ex._ws = None
    torch.cuda.empty_cache()
    g = ex.vjp(dev, torch.ones(ex.plan.out_shape, dtype=dev[0].dtype, device="cuda"), 0, 1, 1,
               max_bytes=plan_bytes)
    assert ex.vjp_plan(max_bytes=plan_bytes).total_bytes <= plan_bytes
    worst = 0.0
    for x, gi in zip(dev, g):
        s = complex(torch.sum(x * gi.conj()).item())
        scale = float(torch.sum(x.abs() * gi.abs()).item())
        worst = max(worst, abs(s - amp) / scale)
    print(f"m20 W=2^{width} {dtype}: plan {plan_bytes / GIB:.2f} GiB, amplitude {amp}, worst identity error {worst:.2e}")
    assert worst <= tol
    key = f"appxB_w{width}_slice0"
    if key in BIG:
        want = complex(BIG[key]["re"], BIG[key]["im"])
        assert abs(amp - want) / abs(want) < amp_tol
    del dev, g, ex
    torch.cuda.empty_cache()


def test_m20_w30_complex64_identity_under_budget():
    _identity_check(30, "complex64", 56 * GIB, 1e-5, 3e-3)


def test_m20_complex128_identity_at_the_planners_minimum():
    free = torch.cuda.mem_get_info()[0]
    spec = appxB_at_width(30)
    ex = cb.TreeExecutor(spec, dtype="complex128")
    lo = _min_bytes(ex)
    del ex
    width = 30 if lo + (2 << 30) < free else 29
    _identity_check(width, "complex128", None, 1e-12, 1e-10)


def test_autograd_under_budget():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    lo = _min_bytes(cb.TreeExecutor(spec, dtype=dt))
    grads = []
    for budget in (None, lo):
        ts = [torch.tensor(a).cuda().requires_grad_() for a in arrays]
        cb.contract_tree(spec, ts, dtype=dt, vjp_max_bytes=budget).real.sum().backward()
        grads.append([t.grad.cpu().numpy() for t in ts])
    for a, b in zip(*grads):
        assert nrel(a, b) <= 1e-12
