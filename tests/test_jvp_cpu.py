"""Forward mode (``cotengra_b200/jvp.py``) on the CPU: the JVP plans' records walked by the emulator
(``tests/desc_emulator.py``) against the exact multilinear oracle ``J v = sum_i f(x_1, ..., v_i, ..., x_n)``,
and the plans' structure."""

import numpy as np
import pytest

from cotengra_b200 import ExecPlan, VjpPlan
from cotengra_b200.executor import K_TANGENT, K_TOUT, PHASE_INV_FWD
from cotengra_b200.fusion import fuse_stems
from cotengra_b200.jvp import JvpPlan, two_term_fits
from tests.desc_emulator import emulate_plan
from tests.helpers import jvp_oracle, load_json, make_arrays, tree_spec

TREES = load_json("trees.json")
DT = "complex128"


def _plan(spec, contractions=None, **kw):
    ir = spec.contractions() if contractions is None else contractions
    return JvpPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=DT, sm_count=8, **kw)


def _nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _subsets(n, seed):
    rng = np.random.default_rng(seed)
    return [[int(rng.integers(n))], sorted(rng.choice(n, size=max(1, n // 2), replace=False).tolist()),
            list(range(n))]


def _bytes_only(dtype, B, M, N, K, elems):
    return 1e-9 * elems + 1e-12 * B * M * N * K


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_jvp_matches_multilinear_oracle(rec):
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), DT, seed=rec["seed"])
    n = len(arrays)
    ir = spec.contractions()
    fused, _ = fuse_stems(spec, DT, min_big=2, ratio=1.0, min_gain=-1.0, model=_bytes_only)
    for wrt in _subsets(n, rec["seed"]):
        tans = make_arrays([arrays[i].shape for i in wrt], DT, seed=rec["seed"] + 7)
        want = jvp_oracle(spec, ir, arrays, tans, wrt)
        want_out = jvp_oracle(spec, ir, arrays, [arrays[wrt[0]]], [wrt[0]])  # f(x) itself
        for contractions in (None, fused.contractions()):
            plan = _plan(spec, contractions, wrt=wrt)
            out, tout = emulate_plan(plan, arrays, tangents=tans)
            assert _nrel(tout, want) <= 1e-12, (wrt, _nrel(tout, want))
            assert _nrel(out, want_out) <= 1e-12
            # without the primal the root is skipped and the tangent is the same
            assert _nrel(emulate_plan(plan, arrays, tangents=tans, primal=False), want) <= 1e-12
    plan = _plan(spec, hoist=False)
    tans = make_arrays(spec.shapes(), DT, seed=rec["seed"] + 7)
    assert _nrel(emulate_plan(plan, arrays, tangents=tans, primal=False), jvp_oracle(spec, ir, arrays, tans, range(n))) <= 1e-12
    if plan.nslices > 1:
        # slice ranges add up to the whole
        h = plan.nslices // 2
        t1 = emulate_plan(plan, arrays, tangents=tans, slice_ids=range(h), primal=False)
        t2 = emulate_plan(plan, arrays, tangents=tans, slice_ids=range(h, plan.nslices), primal=False)
        assert _nrel(t1, jvp_oracle(spec, ir, arrays, tans, range(n), slice_ids=range(h))) <= 1e-12
        assert _nrel(t1 + t2, emulate_plan(plan, arrays, tangents=tans, primal=False)) <= 1e-12


def _below(plan):
    """fwd node index -> the set of inputs below it"""
    fwd = plan.fwd
    below, out = {}, {}
    for i, nd in enumerate(fwd.nodes):
        s = set()
        for t in (nd["a"], nd["b"], nd.get("d")):
            if t is None:
                continue
            s |= {t.input_index} if t.kind == 0 else below[id(t)]
        below[id(nd["c"])] = out[i] = s
    return out


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_plan_structure(rec):
    spec = tree_spec(rec)
    n = len(spec.inputs)
    for wrt in _subsets(n, rec["seed"]):
        plan = _plan(spec, wrt=wrt)
        fwd = plan.fwd
        below = _below(plan)
        # only nodes above wrt carry a tangent, and every such node does
        assert plan.differentiated == [i for i in range(len(fwd.nodes)) if below[i] & set(wrt)]
        tangent_slots = {id(nd["c"]) for nd in plan.tangent_nodes} | {id(t) for t in plan.tensors
                                                                         if t.kind == K_TANGENT}
        assert {t.input_index for t in plan.tensors if t.kind == K_TANGENT} == set(wrt)
        per_node = {}
        for nd in plan.tangent_nodes:
            per_node.setdefault(nd["fwd_index"], []).append(nd)
            # a tangent record runs in its value's phase: invariant tangents are formed once, in phase 0
            assert nd["phase"] == fwd.nodes[nd["fwd_index"]]["phase"]
            if nd["phase"] == PHASE_INV_FWD:
                assert nd["c"].kind != K_TOUT
        for i, recs in per_node.items():
            f = fwd.nodes[i]
            ops = [t for t in (f["a"], f["b"], f.get("d")) if t is not None]
            carrying = [t for t in ops if (t.input_index in wrt if t.kind == 0 else bool(below[_index(fwd, t)] & set(wrt)))]
            if f["kind"] == 0 and f.get("d") is None and len(carrying) == 2 and two_term_fits(f["words"]):
                assert [r["kind"] for r in recs] == [2]
            else:
                # one ordinary launch per term, the later ones accumulating
                assert len(recs) == len(carrying) and all(r["kind"] == f["kind"] for r in recs)
                for r in recs[1:]:
                    assert int(np.asarray(r["words"])[_flags_word(r)]) & 1
            for r in recs:
                assert id(r["c"]) in tangent_slots
        assert plan.two_term_nodes == sum(1 for nd in plan.tangent_nodes if nd["kind"] == 2)
    # the two-launch form has the same records but no two-term node
    p2 = _plan(spec, _two_term=False)
    assert p2.two_term_nodes == 0


def _index(fwd, t):
    return next(i for i, nd in enumerate(fwd.nodes) if nd["c"] is t)


def _flags_word(r):
    from cotengra_b200 import lowering as L

    return L.W_FLAGS if r["kind"] == 0 else L.S_FLAGS


def test_forward_and_vjp_plans_unchanged():
    """Building JVP plans leaves the forward and VJP plans of the same trees word for word as they were."""
    def snapshot():
        out = []
        for rec in TREES:
            spec = tree_spec(rec)
            args = (spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced)
            f = ExecPlan(*args, dtype=DT, sm_count=8)
            v = VjpPlan(*args, dtype=DT, sm_count=8)
            out.append([np.asarray(nd["words"]).tobytes() for p in (f, v) for nd in p.nodes]
                       + [f.workspace_bytes, f.persistent_bytes, v.workspace_bytes, v.persistent_bytes])
        return out

    before = snapshot()
    for rec in TREES:
        _plan(tree_spec(rec))
    assert snapshot() == before


def test_two_term_fits_follows_the_kernel_limits():
    from cotengra_b200 import lowering as L

    w = np.zeros(L.DESC_WORDS, dtype=np.int64)
    for v, n, k, ok in [(L.VAR_ROWSTREAM, 8, 8, True), (L.VAR_ROWSTREAM_K, 8, 64, True),
                        (L.VAR_DMMASTREAM, 16, 64, True), (L.VAR_DMMASTREAM, 32, 32, True),
                        (L.VAR_DMMASTREAM, 32, 64, False), (L.VAR_DMMASTREAM, 64, 16, True),
                        (L.VAR_DMMASTREAM, 64, 32, False), (L.VAR_DMMA_256x16, 8, 8, False),
                        (L.VAR_TC05_128x64, 8, 8, False)]:
        w[L.W_VARIANT], w[L.W_NTA], w[L.W_KTA] = v, n, k
        assert two_term_fits(w) == ok, (v, n, k)


def test_strip_exponent_refused():
    spec = tree_spec(TREES[0])
    with pytest.raises(NotImplementedError):
        _plan(spec, strip_exponent=True)
    with pytest.raises(ValueError):
        _plan(spec, wrt=[len(spec.inputs)])
