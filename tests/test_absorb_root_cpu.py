"""Absorb-root nodes (``ExecPlan(absorb_root=True)``, csrc/absorbdot.cuh) -- no GPU needed.

The fused Sycamore-m20 complex128 plan folds the last absorption of its second stem into the
DMMA_32x32 product that reads it; every other plan kind keeps its nodes.  The emulator walks the new
node, checked against einsum."""

import string

import numpy as np
import pytest

import cotengra_b200 as cb
from cotengra_b200 import lowering as L
from cotengra_b200.fusion import fuse_stems
from tests.desc_emulator import emulate_absorb, emulate_plan
from tests.helpers import decode_sliced, load_json


def _m20(name="sycamore_m20_appxB"):
    rec = next(r for r in load_json("sycamore_m20.json") if r["name"] == name)
    spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]))
    return fuse_stems(spec, "complex128")[0]


def _plan(spec, **kw):
    return cb.ExecPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced, sm_count=132, **kw)


def _signature(plan):
    return [(nd["kind"], nd["phase"], np.asarray(nd["words"]).tobytes()) for nd in plan.nodes], \
        (plan.workspace_bytes, plan.persistent_bytes)


def test_m20_plan_has_one_absorb_root_node():
    spec = _m20()
    two = _plan(spec, dtype="complex128")
    one = _plan(spec, dtype="complex128", absorb_root=True)
    fused = [i for i, nd in enumerate(one.nodes) if nd.get("d") is not None]
    assert len(fused) == 1 and len(one.nodes) == len(two.nodes) - 1
    i = fused[0]
    F = one.nodes[i]
    P, R = two.nodes[i], two.nodes[i + 1]
    assert tuple(P["sizes"]) == (1, 1 << 23, 128, 16) and int(P["plan"].variant) == L.VAR_DMMA_64x128
    assert tuple(R["sizes"]) == (1, 32, 32, 1 << 25) and int(R["plan"].variant) == L.VAR_DMMA_32x32
    assert int(F["plan"].variant) == L.VAR_ABSORB_ROOT and tuple(F["sizes"]) == tuple(R["sizes"])
    assert not F["invariant"] and sorted(nd["pos"] for nd in two.nodes if nd in (P, R)) == [375, 376]
    # it reads A (2^27), V (2^30) and Bs (2^11) and writes R; X (2^30) has no slot
    assert [int(np.prod(F[x].shape)) for x in ("a", "b", "d", "c")] == [1 << 27, 1 << 30, 1 << 11, 1024]
    assert len(one.tensors) == len(two.tensors) - 1
    assert one.macs_per_slice == two.macs_per_slice
    # the nodes before and after are the same, word for word
    sig1, sig2 = _signature(one)[0], _signature(two)[0]
    assert sig1[:i] == sig2[:i] and sig1[i + 1:] == sig2[i + 2:]
    assert one.workspace_bytes == two.workspace_bytes  # X shared its slot with V's twin before
    w = F["words"]
    assert [int(w[k]) for k in (L.AB_M, L.AB_N, L.AB_K, L.AB_C, L.AB_CCP, L.AB_KL, L.AB_UNITS)] == \
        [32, 32, 16, 32, 32, 2, 1 << 19]


@pytest.mark.parametrize("kw", [dict(dtype="complex64"), dict(dtype="complex128", strip_exponent=True),
                                dict(dtype="complex128", variant=L.VAR_DMMA_64x128)])
def test_other_plans_keep_their_nodes(kw):
    spec = _m20()
    assert _signature(_plan(spec, absorb_root=True, **kw)) == _signature(_plan(spec, **kw))


def test_unfused_and_reverse_mode_plans_keep_their_nodes():
    """``fuse=False`` runs the reference's sequence (no absorb-root); reverse-mode plans never take it."""
    import inspect

    from cotengra_b200 import contract
    from cotengra_b200.vjp import VjpPlan

    src = inspect.getsource(contract.TreeExecutor.__init__)
    assert "absorb_root=bool(fuse) and contractions is None" in src
    assert "absorb_root" not in inspect.signature(VjpPlan).parameters
    rec = next(r for r in load_json("sycamore_m20.json") if r["name"] == "sycamore_m20_appxB")
    spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]))
    assert not any(nd.get("d") is not None for nd in _plan(spec, dtype="complex128", absorb_root=True).nodes)


def test_golden_trees_with_an_absorb_root_node():
    got = []
    for f in ("trees.json", "live_trees.json", "sycamore_m20.json"):
        for rec in load_json(f):
            spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"],
                               decode_sliced(rec["sliced"]))
            spec = fuse_stems(spec, "complex128")[0]
            n = sum(1 for nd in _plan(spec, dtype="complex128", absorb_root=True).nodes if nd.get("d") is not None)
            if n:
                got.append((rec["name"], n))
    assert got == [("sycamore_m20_appxB", 1), ("sycamore_m20_medium", 1)]


def _synthetic(seed=0, n_sliced=0):
    """A[rows, k', k] . Bs[k, cc, ck] -> X, X . V[k', cc, n] -> R over 2^15 contracted elements, all
    extents 2 and index orders shuffled: the pattern of the m20 stem end, small."""
    rng = np.random.default_rng(seed)
    letters = iter(string.ascii_letters)
    groups = {"rows": 3, "ck": 2, "cc": 5, "kp": 10 + n_sliced, "k": 4, "n": 5}
    names = {g: [next(letters) for _ in range(c)] for g, c in groups.items()}

    def term(*gs):
        t = [ix for g in gs for ix in names[g]]
        rng.shuffle(t)
        return "".join(t)

    ta, tb, tv, tr = term("rows", "kp", "k"), term("k", "cc", "ck"), term("kp", "cc", "n"), term("n", "rows", "ck")
    size = {ix: 2 for t in (ta, tb, tv) for ix in t}
    spec = cb.TreeSpec([ta, tb, tv], tr, size, [(0, 1), (2, 3)], [(ix, 2, None) for ix in names["kp"][:n_sliced]])
    arrays = [rng.standard_normal((2,) * len(t)) + 1j * rng.standard_normal((2,) * len(t)) for t in (ta, tb, tv)]
    return spec, arrays, np.einsum(f"{ta},{tb},{tv}->{tr}", *arrays)


@pytest.mark.parametrize("n_sliced", [0, 2])
def test_emulated_plan_against_einsum(n_sliced):
    """The plan's one absorb-root node, emulated, against einsum and the emulated two-node plan; with
    sliced k' indices the node reads sliced input views and adds every slice into the output."""
    spec, arrays, want = _synthetic(n_sliced=n_sliced)
    plan = _plan(spec, dtype="complex128", absorb_root=True)
    assert [int(nd["plan"].variant) for nd in plan.nodes] == [L.VAR_ABSORB_ROOT]
    got = emulate_plan(plan, arrays)
    assert np.abs(got.reshape(want.shape) - want).max() <= 1e-12 * np.abs(want).max()
    ref = emulate_plan(_plan(spec, dtype="complex128"), arrays)
    assert np.abs(got - ref).max() <= 1e-12 * np.abs(want).max()


def test_descriptor_refuses_what_the_kernel_cannot_take():
    spec, arrays, _want = _synthetic(1)
    plan = _plan(spec, dtype="complex128")
    P, R = plan.nodes
    assert L.build_absorb_desc(P["dims"], R["dims"], R["terms"][0] is P["c"]) is not None
    # 40 rows of X: more than the 32 of the kernel
    dp = L.classify_pair("mqk", (40, 64, 4), "kc", (4, 8), "mqc")
    dr = L.classify_pair("qcn", (64, 8, 32), "mqc", (40, 64, 8), "nm")
    assert L.build_absorb_desc(dp, dr, False) is None
    dp = L.classify_pair("mqk", (8, 64, 4), "kc", (4, 8), "mqc")
    dr = L.classify_pair("qcn", (64, 8, 32), "mqc", (8, 64, 8), "nm")
    ab = L.build_absorb_desc(dp, dr, False, c_dense_elems=256)
    C = np.zeros(256, complex)
    rng = np.random.default_rng(2)
    A, Bs, V = (rng.standard_normal(s) + 0j for s in ((8, 64, 4), (4, 8), (64, 8, 32)))
    emulate_absorb(ab.words, A.reshape(-1), Bs.reshape(-1), V.reshape(-1), C)
    want = np.einsum("mqk,kc,qcn->nm", A, Bs, V).reshape(-1)
    assert np.abs(C - want).max() <= 1e-12 * np.abs(want).max()
