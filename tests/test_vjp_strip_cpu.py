"""Gradients of strip_exponent results (``VjpPlan(strip_exponent=True, stripped_grad=True)``) on the
CPU: the stripped VJP plans' descriptors, factor slots and seeds walked by the plan emulator
(``tests/desc_emulator.py``) against the torch-CPU gradient oracle (``oracle/grad_oracle.py``) with
``dm/dx = 10^-e damp/dx``; central differences of ``log|m| + e ln 10``; the autograd paths of the
public interface with the device launch emulated; and the default path, which is unchanged."""

import gc
import math
import warnings

import numpy as np
import pytest
import torch

import cotengra_b200 as cb
from cotengra_b200 import ExecPlan, VjpPlan
from cotengra_b200.executor import PHASE_INV_FWD, PHASE_VAR_FWD
from cotengra_b200.fusion import fuse_stems
from oracle import ctg_oracle as orc
from oracle import grad_oracle as go
from tests import emu_device
from tests.desc_emulator import emulate_plan
from tests.helpers import load_json, make_arrays, tree_spec
from tests.test_vjp_cpu import ctg  # noqa: F401  (the drop-in fixture)
from tests.zero_util import zero_one_digit

TREES = {r["name"]: r for r in load_json("trees.json")}
STRIP_TREES = ["lattice4x4_sliced", "lattice6x6_d3_sliced", "peps8x8_d2", "projected",
               "rand_r3_o1_hi1_ho1_None_s42_sliced_out", "rand_r2_o1_hi0_ho2_root_s12_sliced",
               "pre_diag_sliced", "pre_sum_sliced", "single_perm", "single_sum", "single_trace"]


@pytest.fixture(autouse=True)
def _collect_while_emulated(monkeypatch):
    yield
    gc.collect()


def _bytes_only(dtype, B, M, N, K, elems):
    return 1e-9 * elems + 1e-12 * B * M * N * K


def _plan(ir, spec, dtype, **kw):
    return VjpPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype, sm_count=8,
                   strip_exponent=True, stripped_grad=True, **kw)


def _forward(ir, spec, dtype, arrays, slice_ids=None):
    """(m, e) of the stripped forward plan, emulated"""
    fwd = ExecPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype, sm_count=8,
                   strip_exponent=True)
    return emulate_plan(fwd, arrays, slice_ids=slice_ids)


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _want(spec, arrays, cot, e, slice_ids=None):
    """the oracle's dm/dx = 10^-e damp/dx"""
    g = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot,
                          slice_ids=slice_ids)
    return [w * 10.0 ** (-e) for w in g]


def _check(got, want, tol=1e-10):
    assert len(got) == len(want)
    for i, (g, w) in enumerate(zip(got, want)):
        assert g is not None and nrel(g, w) <= tol, (i, nrel(g, w))


def _case(name, scale=1.0):
    rec = TREES[name]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"], scale=scale)
    return rec, spec, arrays


@pytest.mark.parametrize("name", STRIP_TREES)
def test_stripped_gradients_match_oracle(name):
    """every golden shape of tree: hoisted and unhoisted, and stem fusion forced on"""
    rec, spec, arrays = _case(name, scale=7.0)
    dt, ir = rec["dtype"], spec.contractions()
    m, e = _forward(ir, spec, dt, arrays)
    assert math.isfinite(e)
    cot = make_arrays([np.shape(m)], dt, seed=rec["seed"] + 1)[0]
    want = _want(spec, arrays, cot, e)
    plan = _plan(ir, spec, dt)
    _check(emulate_plan(plan, arrays, cotangent=cot, exponent=e), want)
    _check(emulate_plan(_plan(ir, spec, dt, hoist=False), arrays, cotangent=cot, exponent=e), want)
    fused, _info = fuse_stems(spec, dt, min_big=2, ratio=1.0, min_gain=-1.0, model=_bytes_only)
    fir = fused.contractions()
    _check(emulate_plan(_plan(fir, spec, dt), arrays, cotangent=cot, exponent=e), want)
    # the exponent is a parameter: another e scales the gradient by 10^(e - e2)
    got = emulate_plan(plan, arrays, cotangent=cot, exponent=e + 3.5)
    _check(got, [w * 10.0 ** -3.5 for w in want])


def test_single_operand_root_is_seeded():
    rec, spec, arrays = _case("single_sum")
    plan = _plan(spec.contractions(), spec, rec["dtype"])
    root = [nd for nd in plan.nodes if nd["kind"] == 1]
    assert len(plan.nodes) == len(root) == 1
    seed = len(plan.tensors)
    assert plan.scale_slots == ([seed], [-1])
    # (no pairwise node: the forward strips nothing, e = 0; the seed carries any other exponent)
    m, e = _forward(spec.contractions(), spec, rec["dtype"], arrays)
    assert e == 0.0
    cot = make_arrays([np.shape(m)], rec["dtype"], seed=3)[0]
    for ex in (e, 12.25):
        _check(emulate_plan(plan, arrays, cotangent=cot, exponent=ex), _want(spec, arrays, cot, ex))


def test_scale_slots():
    """forward nodes divide by their operands, backward ones by (f_p or the seed, f_r)"""
    rec, spec, _arrays = _case("lattice6x6_d3_sliced")
    plan = _plan(spec.contractions(), spec, rec["dtype"])
    slot = {id(t): i for i, t in enumerate(plan.tensors)}
    seed = len(plan.tensors)
    sa, sb = plan.scale_slots
    n_seeded = 0
    for i, nd in enumerate(plan.nodes):
        if nd["phase"] in (PHASE_INV_FWD, PHASE_VAR_FWD) and nd["kind"] == 0:
            assert (sa[i], sb[i]) == (slot[id(nd["a"])], slot[id(nd["b"])])
        elif nd["kind"] == 0:
            # the value the node reads divides by its own factor, H by its tensor's (or the seed)
            assert 0 <= sa[i] <= seed and 0 <= sb[i] <= seed
            assert slot[id(nd["a"])] in (sa[i], sb[i]) or slot[id(nd["b"])] in (sa[i], sb[i])
            n_seeded += seed in (sa[i], sb[i])
        else:
            assert (sa[i], sb[i]) == (-1, -1)
    assert n_seeded == 2  # the root's two children
    # every non-root pairwise node runs forward, even where no backward step reads its value
    assert sum(1 for nd in plan.nodes if nd["kind"] == 0 and nd["phase"] <= PHASE_VAR_FWD) == \
        sum(1 for nd in plan.fwd.nodes[:-1] if nd["kind"] == 0)


@pytest.mark.parametrize("name", ["lattice6x6_d3_sliced", "peps8x8_d2"])
def test_budgeted_plan_recomputes_with_phase1_factors(name):
    rec, spec, arrays = _case(name, scale=7.0)
    dt, ir = rec["dtype"], spec.contractions()
    fused, _info = fuse_stems(spec, dt, min_big=2, ratio=1.0, min_gain=-1.0, model=_bytes_only)
    ir = fused.contractions()
    with pytest.raises(MemoryError) as err:
        _plan(ir, spec, dt, max_bytes=1)
    lo = err.value.min_bytes
    base = _plan(ir, spec, dt)
    assert lo < base.total_bytes
    plan = _plan(ir, spec, dt, max_bytes=lo)
    rec_nodes = [i for i, nd in enumerate(plan.nodes) if nd.get("recompute")]
    assert rec_nodes and plan.recompute_macs > 0
    # a recomputation divides by the phase-1 factors (slots of phase-1 values) and measures nothing
    produced1 = {id(nd["c"]) for nd in plan.nodes if nd["phase"] <= PHASE_VAR_FWD}
    slot = {id(t): i for i, t in enumerate(plan.tensors)}
    for i in rec_nodes:
        nd = plan.nodes[i]
        if nd["kind"] == 0:
            for k, s in enumerate(nd["scale"]):
                assert plan.scale_slots[k][i] == slot[id(s)]
                assert s.kind == 0 or id(s) in produced1
    m, e = _forward(ir, spec, dt, arrays)
    cot = make_arrays([np.shape(m)], dt, seed=5)[0]
    want = _want(spec, arrays, cot, e)
    _check(emulate_plan(plan, arrays, cotangent=cot, exponent=e), want)
    _check(emulate_plan(base, arrays, cotangent=cot, exponent=e), want)


@pytest.mark.parametrize("name", ["lattice4x4_sliced", "rand_r3_o1_hi1_ho1_None_s42_sliced_out"])
def test_zero_slices_contribute_nothing(monkeypatch, name):
    """A slice with an all-zero intermediate (factor 0) adds nothing, as the reference's check_zero
    early return (0.0, -inf) records no graph; an all-zero result gives zero gradients, not NaN."""
    rec, spec, arrays = _case(name)
    dt, ir = rec["dtype"], spec.contractions()
    arrays, ind = zero_one_digit(spec, arrays, which=0, digit=1)
    n = orc.num_slices(spec.sliced)
    live = [i for i in range(n) if orc.slice_key(spec.sliced, i)[ind] != 1]
    assert 0 < len(live) < n
    m, e = _forward(ir, spec, dt, arrays)
    cot = make_arrays([np.shape(m)], dt, seed=8)[0]
    plan = _plan(ir, spec, dt)
    _check(emulate_plan(plan, arrays, cotangent=cot, exponent=e), _want(spec, arrays, cot, e, slice_ids=live))
    # all zero: e = -inf, every seed 0
    zero = [np.zeros_like(a) if k == 0 else a for k, a in enumerate(arrays)]
    mz, ez = _forward(ir, spec, dt, zero)
    assert ez == -math.inf
    for g in emulate_plan(plan, zero, cotangent=cot, exponent=ez):
        assert np.all(g == 0)
    # a NaN exponent gives NaN gradients
    assert all(np.isnan(g).all() for g in emulate_plan(plan, arrays, cotangent=cot, exponent=math.nan))
    # the public paths: check_zero returns (0.0, -inf) without a graph; without it, zero gradients
    emu_device.install(monkeypatch)
    ex = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True, stripped_grad=True)
    ts = [torch.tensor(a, requires_grad=True) for a in zero]
    assert cb.contract_tree(ex, ts, check_zero=True) == (0.0, -math.inf)
    m2, e2 = cb.contract_tree(ex, ts)
    assert e2 == -math.inf and m2.grad_fn is not None
    torch.abs(m2).sum().backward()
    assert all(t.grad is not None and not torch.isnan(t.grad).any() for t in ts)
    ts = [torch.tensor(a, requires_grad=True) for a in arrays]
    m3, e3 = cb.contract_tree(ex, ts)
    m3.backward(torch.tensor(cot))
    for t, w in zip(ts, _want(spec, arrays, cot, e3, slice_ids=live)):
        assert nrel(t.grad.numpy(), w) < 1e-10


@pytest.mark.parametrize("name", ["lattice4x4_sliced", "pre_sum_sliced", "projected"])
def test_central_differences_of_log_amplitude(monkeypatch, name):
    """d(log|m| + e ln 10)/dx through contract_tree's autograd node against central differences of
    log|amp| (the exponent is a float; its split from m does not change the loss)."""
    emu_device.install(monkeypatch)
    rec = TREES[name]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "float64", seed=rec["seed"], scale=5.0)
    ex = cb.TreeExecutor(spec, dtype="float64", strip_exponent=True, stripped_grad=True)
    ts = [torch.tensor(a, requires_grad=True) for a in arrays]
    m, e = cb.contract_tree(ex, ts)
    assert isinstance(e, float)
    loss = torch.log(torch.abs(m.reshape(-1)[0])) + e * math.log(10.0)
    loss.backward()
    plain = cb.TreeExecutor(spec, dtype="float64")

    def f(xs):
        return math.log(abs(float(np.asarray(cb.contract_tree(plain, xs)).reshape(-1)[0])))

    assert abs(loss.item() - f(arrays)) < 1e-10
    rng = np.random.default_rng(0)
    eps = 1e-6
    for i in rng.choice(len(arrays), size=min(4, len(arrays)), replace=False):
        for flat in rng.choice(arrays[i].size, size=min(3, arrays[i].size), replace=False):
            xp = [a.copy() for a in arrays]
            xm = [a.copy() for a in arrays]
            xp[i].reshape(-1)[flat] += eps
            xm[i].reshape(-1)[flat] -= eps
            fd = (f(xp) - f(xm)) / (2 * eps)
            got = float(ts[i].grad.reshape(-1)[flat])
            assert abs(fd - got) <= 1e-5 * max(1.0, abs(fd)), (i, flat, fd, got)


def test_public_interface(monkeypatch):
    """TreeExecutor.vjp(exponent=), contract_tree and B200Contractor record the mantissa's gradient;
    e is the same float as without stripped_grad"""
    emu_device.install(monkeypatch)
    rec, spec, arrays = _case("rand_r3_o1_hi1_ho1_None_s42_sliced_out", scale=9.0)
    dt = rec["dtype"]
    ex = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True, stripped_grad=True)
    m0, e0 = cb.contract_tree(cb.TreeExecutor(spec, dtype=dt, strip_exponent=True),
                              [torch.tensor(a) for a in arrays])
    ts = [torch.tensor(a, requires_grad=(i % 3 != 1)) for i, a in enumerate(arrays)]
    with warnings.catch_warnings():
        warnings.simplefilter("error")
        m, e = cb.contract_tree(ex, ts)
    assert isinstance(e, float) and e == e0 and torch.equal(m.detach(), m0) and m.grad_fn is not None
    cot = make_arrays([tuple(m.shape)], dt, seed=4)[0]
    m.backward(torch.tensor(cot))
    want = _want(spec, arrays, cot, e)
    for i, t in enumerate(ts):
        if i % 3 != 1:
            assert nrel(t.grad.numpy(), want[i]) < 1e-10
        else:
            assert t.grad is None
    g = ex.vjp([torch.tensor(a) for a in arrays], torch.tensor(cot), wrt=[0], exponent=e)
    assert g[1] is None and nrel(g[0].numpy(), want[0]) < 1e-10
    with pytest.raises(ValueError, match="exponent"):
        ex.vjp([torch.tensor(a) for a in arrays], torch.tensor(cot))
    # the per-slice drop-in contractor (flat, unsliced records)
    con = cb.B200Contractor.from_tree(spec, strip_exponent=True, stripped_grad=True)
    sl = go.slice_arrays(spec.inputs, spec.sliced, arrays, 0)
    xs = [torch.tensor(np.ascontiguousarray(a), requires_grad=True) for a in sl]
    ms, es = con(*xs)
    assert isinstance(es, float) and ms.grad_fn is not None
    c1 = make_arrays([tuple(ms.shape)], dt, seed=6)[0]
    ms.backward(torch.tensor(c1))
    leaves = [torch.tensor(np.ascontiguousarray(a), requires_grad=True) for a in sl]
    ref = go.run_contractions(spec.contractions(), leaves)
    w1 = torch.autograd.grad(ref, leaves, grad_outputs=torch.tensor(c1).reshape(ref.shape))
    for x, w in zip(xs, w1):
        assert nrel(x.grad.numpy(), w.numpy() * 10.0 ** -es) < 1e-10


def test_default_path_unchanged(monkeypatch):
    """without stripped_grad: the warning, no graph, and NotImplementedError from the plan"""
    emu_device.install(monkeypatch)
    rec, spec, arrays = _case("lattice4x4_sliced")
    ex = cb.TreeExecutor(spec, dtype=rec["dtype"], strip_exponent=True)
    with pytest.warns(UserWarning, match="no gradient") as warned:
        m, _e = cb.contract_tree(ex, [torch.tensor(a, requires_grad=True) for a in arrays])
    assert m.grad_fn is None
    # the same from the per-slice drop-in contractor; both warnings point at the caller's line
    con = cb.B200Contractor.from_tree(spec, strip_exponent=True)
    sl = go.slice_arrays(spec.inputs, spec.sliced, arrays, 0)
    with pytest.warns(UserWarning, match="no gradient") as warned_con:
        ms, _es = con(*[torch.tensor(np.ascontiguousarray(a), requires_grad=True) for a in sl])
    assert ms.grad_fn is None
    for w in (warned, warned_con):
        assert [x.filename for x in w if "no gradient" in str(x.message)] == [__file__]
    with pytest.raises(NotImplementedError):
        VjpPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced,
                dtype=rec["dtype"], strip_exponent=True)
    # stripped_grad alone changes nothing
    a = VjpPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced,
                dtype=rec["dtype"], sm_count=8)
    b = VjpPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced,
                dtype=rec["dtype"], sm_count=8, stripped_grad=True)
    assert a.scale_slots is None and b.scale_slots is None and not b.strip_exponent
    assert len(a.nodes) == len(b.nodes)
    for x, y in zip(a.nodes, b.nodes):
        assert np.array_equal(x["words"], y["words"]) and x["phase"] == y["phase"]


@pytest.mark.reference
def test_installed_tree_contract_stripped_backward(ctg, monkeypatch):  # noqa: F811
    """``cb.install(tree, strip_exponent=True, stripped_grad=True)``; cotengra's own
    ``tree.contract(..., strip_exponent=True)`` on torch tensors combines the slices' (m_s, e_s);
    ``backward()`` through that combiner gives 10^-e damp/dx."""
    emu_device.install(monkeypatch)  # (the fixture's emulated launch, with stripped VJP plans)
    con = ctg.utils.lattice_equation([3, 3], d_min=2, d_max=3, seed=1)
    tree = ctg.array_contract_tree(con.inputs, con.output, con.size_dict, optimize="greedy")
    tree.slice_(target_slices=4)
    assert tree.nslices > 1
    arrays = ctg.utils.make_arrays_from_inputs(con.inputs, con.size_dict, seed=0, dtype="complex128")
    arrays = [np.asarray(a) * 30.0 for a in arrays]
    cb.install(tree, strip_exponent=True, stripped_grad=True)
    ts = [torch.tensor(a, requires_grad=True) for a in arrays]
    with warnings.catch_warnings():
        warnings.simplefilter("ignore")
        m, e = tree.contract(ts, strip_exponent=True)
    e = float(e)
    assert e > 5
    cot = make_arrays([tuple(m.shape)], "complex128", seed=6)[0]
    m.backward(torch.tensor(cot).reshape(m.shape))
    spec = cb.TreeSpec.from_cotengra(tree)
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot)
    for t, w in zip(ts, want):
        assert nrel(t.grad.numpy(), w * 10.0 ** -e) < 1e-10
