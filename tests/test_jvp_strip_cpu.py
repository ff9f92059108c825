"""Forward-mode derivatives of strip_exponent results (``JvpPlan(strip_exponent=True,
stripped_grad=True)``) on the CPU: the stripped JVP plans' records, factor slots and running exponent
walked by the lazy-scheme model (``tests/emu_jvp_strip.py``) against the exact multilinear oracle with
``dm = 10^-e d(amp)``; zero slices and results; central differences of ``log|m| + e ln 10``; forward AD
through the public interface with the device launch emulated; two gloo ranks; and the plans that must
not change, against digests of the parent's descriptors (``tests/golden/plan_digests.json``)."""

import gc
import hashlib
import json
import math
import os
import socket
import warnings

import numpy as np
import pytest
import torch
import torch.multiprocessing as mp

import cotengra_b200 as cb
from cotengra_b200 import ExecPlan, VjpPlan
from cotengra_b200.fusion import fuse_stems
from cotengra_b200.jvp import JvpPlan
from oracle import ctg_oracle as orc
from tests import emu_jvp_strip
from tests.desc_emulator import emulate_plan
from tests.emu_jvp import jvp_oracle
from tests.emu_jvp_strip import emulate_stripped_jvp
from tests.helpers import GOLDEN_DIR, load_json, make_arrays, tree_spec
from tests.test_vjp_cpu import ctg  # noqa: F401  (the drop-in fixture)
from tests.zero_util import zero_one_digit

TREES = load_json("trees.json")
BY_NAME = {r["name"]: r for r in TREES}
DT = "complex128"


@pytest.fixture(autouse=True)
def _collect_while_emulated(monkeypatch):
    yield
    gc.collect()


def _bytes_only(dtype, B, M, N, K, elems):
    return 1e-9 * elems + 1e-12 * B * M * N * K


def _args(spec, ir=None):
    return (spec.contractions() if ir is None else ir, spec.inputs, spec.output, spec.size_dict, spec.sliced)


def _plan(spec, ir=None, dtype=DT, **kw):
    return JvpPlan(*_args(spec, ir), dtype=dtype, sm_count=8, strip_exponent=True, stripped_grad=True, **kw)


def _forward(spec, arrays, ir=None, dtype=DT, slice_ids=None, **kw):
    fwd = ExecPlan(*_args(spec, ir), dtype=dtype, sm_count=8, strip_exponent=True, **kw)
    return emulate_plan(fwd, arrays, slice_ids=slice_ids)


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _subsets(n, seed):
    rng = np.random.default_rng(seed)
    return [[int(rng.integers(n))], list(range(n))]


# ------------------------------------------------------------------ plans that must not change
OPTION_SETS = [("complex128", {}), ("complex128", {"hoist": False}), ("complex64", {}),
               ("complex64", {"precision": "tf32"}), ("complex64", {"accumulate": "double"}),
               ("float64", {}), ("float32", {"accumulate": "double"})]


def _digest(plan):
    h = hashlib.sha256()
    for nd in plan.nodes:
        h.update(np.asarray([nd["kind"], nd["phase"], int(nd.get("root", 0))], dtype=np.int64).tobytes())
        h.update(np.asarray(nd["words"], dtype=np.int64).tobytes())
    h.update(np.asarray([plan.workspace_bytes, plan.persistent_bytes], dtype=np.int64).tobytes())
    return h.hexdigest()


def plan_digests():
    """sha256 of the records of the unstripped JVP plan and the (stripped and unstripped) forward and
    VJP plans of every golden tree, one per tree and plan kind over all option sets (the fixture holds
    the parent's)."""
    out = {}
    for rec in TREES:
        spec = tree_spec(rec)
        args = _args(spec)
        per_kind = {}
        for dt, opts in OPTION_SETS:
            vopts = {k: v for k, v in opts.items() if k != "accumulate"}
            plans = {
                "jvp": lambda: JvpPlan(*args, dtype=dt, sm_count=8, **opts),
                "fwd": lambda: ExecPlan(*args, dtype=dt, sm_count=8, **opts),
                "fwd_strip": lambda: ExecPlan(*args, dtype=dt, sm_count=8, strip_exponent=True, **opts),
                "vjp": lambda: VjpPlan(*args, dtype=dt, sm_count=8, **vopts),
                "vjp_strip": lambda: VjpPlan(*args, dtype=dt, sm_count=8, strip_exponent=True, stripped_grad=True,
                                             **vopts),
            }
            for kind, make in plans.items():
                h = per_kind.setdefault(kind, hashlib.sha256())
                try:
                    h.update(_digest(make()).encode())
                except ValueError as exc:  # (an option a dtype refuses)
                    h.update(f"ValueError: {exc}".encode())
        out.update({f"{rec['name']}|{kind}": h.hexdigest() for kind, h in per_kind.items()})
    return out


def test_other_plans_unchanged():
    with open(os.path.join(GOLDEN_DIR, "plan_digests.json")) as f:
        want = json.load(f)
    got = plan_digests()
    assert got.keys() == want.keys()
    assert [k for k in want if got[k] != want[k]] == []


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_primal_records_are_the_stripped_forward(rec):
    spec = tree_spec(rec)
    n = len(spec.inputs)
    fwd = ExecPlan(*_args(spec), dtype=DT, sm_count=8, strip_exponent=True)
    for wrt in _subsets(n, rec["seed"]):
        plan = _plan(spec, wrt=wrt)
        primal = [nd for nd, t in zip(plan.nodes, plan.tangent_marks) if not t]
        order = sorted(fwd.nodes, key=lambda nd: nd["phase"])  # (the order the library runs them in)
        assert len(primal) == len(order)
        for p, f in zip(primal, order):
            assert np.array_equal(p["words"], f["words"]) and p["kind"] == f["kind"] and p["phase"] == f["phase"]
        slot = {id(t): i for i, t in enumerate(plan.tensors)}
        sa, sb = plan.scale_slots
        for i, nd in enumerate(plan.nodes):
            if nd["kind"] == 1:
                assert (sa[i], sb[i]) == (-1, -1)
            elif not plan.tangent_marks[i]:
                assert (sa[i], sb[i]) == (slot[id(nd["a"])], slot[id(nd["b"])])
            else:
                # a tangent record divides by its primal node's operands' factors
                f = plan.fwd.nodes[nd["fwd_index"]]
                assert (sa[i], sb[i]) == (slot[id(f["a"])], slot[id(f["b"])])
        assert sum(plan.tangent_marks) == len(plan.tangent_nodes)


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_stripped_tangent_matches_oracle(rec):
    """m * 10^e and dm * 10^e against the stripped forward and the exact JVP: hoisted and unhoisted, stem
    fusion forced on, one input and all of them, and slice ranges"""
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), DT, seed=rec["seed"], scale=3.0)
    n = len(arrays)
    ir = spec.contractions()
    fused, _ = fuse_stems(spec, DT, min_big=2, ratio=1.0, min_gain=-1.0, model=_bytes_only)
    for wrt in _subsets(n, rec["seed"]):
        tans = make_arrays([arrays[i].shape for i in wrt], DT, seed=rec["seed"] + 7)
        want = jvp_oracle(spec, ir, arrays, tans, wrt)
        for contractions, opts in ((None, {}), (None, {"hoist": False}), (fused.contractions(), {})):
            m0, e0 = _forward(spec, arrays, contractions, **opts)
            m, e, dm = emulate_stripped_jvp(_plan(spec, contractions, wrt=wrt, **opts), arrays, tans)
            assert abs(e - e0) <= 1e-12 and nrel(m, m0) <= 1e-12
            assert nrel(dm * 10.0 ** e, want) <= 1e-11, (wrt, opts, nrel(dm * 10.0 ** e, want))
    plan = _plan(spec)
    tans = make_arrays(spec.shapes(), DT, seed=rec["seed"] + 9)
    if plan.nslices > 1:
        h = plan.nslices // 2
        ids = range(h, plan.nslices)
        m, e, dm = emulate_stripped_jvp(plan, arrays, tans, slice_ids=ids)
        assert abs(e - _forward(spec, arrays, slice_ids=ids)[1]) <= 1e-12
        assert nrel(dm * 10.0 ** e, jvp_oracle(spec, ir, arrays, tans, range(n), slice_ids=ids)) <= 1e-11


def test_constants(monkeypatch):
    """folded constants: the exponent of the folds is added to e and leaves dm as it is"""
    emu_jvp_strip.install(monkeypatch)
    rec = BY_NAME["lattice6x6_d3_sliced"]
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"], scale=4.0)
    n = len(arrays)
    const = {i: arrays[i] for i in range(0, n, 2)}
    var = [i for i in range(n) if i not in const]
    ex = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True, stripped_grad=True, constants=const)
    tans = make_arrays([arrays[i].shape for i in var], dt, seed=5)
    (m, e), dm = ex.jvp([torch.tensor(arrays[i]) for i in var], [torch.tensor(t) for t in tans])
    e = float(e.item())
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, var)
    assert nrel(dm.numpy() * 10.0 ** e, want) <= 1e-11
    m0, e0 = _forward(spec, arrays, dtype=dt)
    assert abs(e - e0) < 1e-9 and nrel(m.numpy() * 10.0 ** (e - e0), m0) < 1e-11
    # primal=False: relative to the exponent given
    dm2 = ex.jvp([torch.tensor(arrays[i]) for i in var], [torch.tensor(t) for t in tans], primal=False,
                 exponent=e + 2.0)
    assert nrel(dm2.numpy(), dm.numpy() * 1e-2) < 1e-12


@pytest.mark.parametrize("name", ["lattice4x4_sliced", "rand_r3_o1_hi1_ho1_None_s42_sliced_out"])
def test_zero_slices_and_results(name):
    """a slice with an all-zero intermediate adds nothing; an all-zero result gives a zero tangent, no NaN"""
    rec = BY_NAME[name]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), DT, seed=rec["seed"])
    arrays, ind = zero_one_digit(spec, arrays, which=0, digit=1)
    live = [i for i in range(orc.num_slices(spec.sliced)) if orc.slice_key(spec.sliced, i)[ind] != 1]
    # the tangent of the zeroed input too: the zero slices stay zero along it
    tans, _ = zero_one_digit(spec, make_arrays(spec.shapes(), DT, seed=3), which=0, digit=1)
    plan = _plan(spec)
    m, e, dm = emulate_stripped_jvp(plan, arrays, tans)
    assert math.isfinite(e) and not np.isnan(dm).any()
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, range(len(arrays)), slice_ids=live)
    assert nrel(dm * 10.0 ** e, want) <= 1e-11
    zero = [np.zeros_like(a) for a in arrays]
    mz, ez, dmz = emulate_stripped_jvp(plan, zero, tans)
    assert ez == -math.inf and np.all(dmz == 0) and np.all(mz == 0)
    # a NaN in the inputs: NaN exponent, NaN tangent
    bad = [a.copy() for a in arrays]
    bad[1].reshape(-1)[0] = np.nan
    _mn, en, dmn = emulate_stripped_jvp(plan, bad, tans)
    assert math.isnan(en) and np.isnan(dmn).all()


@pytest.mark.parametrize("name", ["lattice4x4_sliced", "pre_sum_sliced", "projected"])
def test_central_differences_of_log_amplitude(name):
    """d/dt (log|m| + e ln 10) along v is Re(conj(m) dm) / |m|^2: against central differences"""
    rec = BY_NAME[name]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "float64", seed=rec["seed"], scale=5.0)
    tans = make_arrays(spec.shapes(), "float64", seed=rec["seed"] + 1)
    plan = _plan(spec, dtype="float64")
    m, e, dm = emulate_stripped_jvp(plan, arrays, tans)
    m0, dm0 = np.asarray(m).reshape(-1)[0], np.asarray(dm).reshape(-1)[0]
    got = float(np.real(np.conj(m0) * dm0) / abs(m0) ** 2)

    def f(xs):
        mm, ee = _forward(spec, xs, dtype="float64")
        return math.log(abs(float(np.asarray(mm).reshape(-1)[0]))) + ee * math.log(10.0)

    eps = 1e-6
    fd = (f([a + eps * t for a, t in zip(arrays, tans)]) - f([a - eps * t for a, t in zip(arrays, tans)])) / (2 * eps)
    assert abs(fd - got) <= 1e-6 * max(1.0, abs(fd)), (fd, got)


def _dual(xs, tans):
    from torch.autograd import forward_ad

    return [forward_ad.make_dual(torch.tensor(x), torch.tensor(t)) for x, t in zip(xs, tans)]


def test_forward_ad_through_public_entry_points(monkeypatch):
    """contract_tree, B200Contractor and make_contractor record dm; e stays a float; check_zero
    returns (0.0, -inf) without a tangent; without stripped_grad the warning and no tangent"""
    from torch.autograd import forward_ad

    from oracle import grad_oracle as go

    emu_jvp_strip.install(monkeypatch)
    rec = BY_NAME["rand_r3_o1_hi1_ho1_None_s42_sliced_out"]
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"], scale=9.0)
    tans = make_arrays(spec.shapes(), dt, seed=11)
    ex = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True, stripped_grad=True)
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, range(len(arrays)))
    with forward_ad.dual_level():
        xs = _dual(arrays, tans)
        with warnings.catch_warnings():
            warnings.simplefilter("error", UserWarning)
            m, e = cb.contract_tree(ex, xs)
        assert isinstance(e, float)
        dm = forward_ad.unpack_dual(m).tangent
        assert dm is not None and nrel(dm.numpy() * 10.0 ** e, want) <= 1e-11
        # the per-slice drop-in contractor (flat records), and make_contractor
        sl = go.slice_arrays(spec.inputs, spec.sliced, arrays, 0)
        tsl = go.slice_arrays(spec.inputs, spec.sliced, tans, 0)
        sl = [np.ascontiguousarray(a) for a in sl]
        tsl = [np.ascontiguousarray(a) for a in tsl]
        leaves = [torch.tensor(a) for a in sl]
        want1 = sum(go.run_contractions(spec.contractions(), [torch.tensor(tsl[j]) if j == i else x
                                                                for j, x in enumerate(leaves)]).numpy()
                    for i in range(len(sl)))
        for con in (cb.B200Contractor.from_tree(spec, strip_exponent=True, stripped_grad=True),
                    cb.make_contractor(spec, strip_exponent=True, stripped_grad=True)):
            ms, es = con(*_dual(sl, tsl))
            assert isinstance(es, float)
            dms = forward_ad.unpack_dual(ms).tangent
            assert nrel(dms.numpy() * 10.0 ** es, np.asarray(want1).reshape(dms.shape)) <= 1e-11
        # check_zero on an all-zero result: (0.0, -inf), no tangent
        zero = [np.zeros_like(a) for a in arrays]
        assert cb.contract_tree(ex, _dual(zero, tans), check_zero=True) == (0.0, -math.inf)
        mz, ez = cb.contract_tree(ex, _dual(zero, tans))
        assert ez == -math.inf and torch.all(forward_ad.unpack_dual(mz).tangent == 0)
        # without stripped_grad: unchanged, a warning and no tangent
        plain = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True)
        with pytest.warns(UserWarning, match="no forward-mode tangent"):
            m2, _e2 = cb.contract_tree(plain, _dual(arrays, tans))
        assert forward_ad.unpack_dual(m2).tangent is None
    with pytest.raises(NotImplementedError):
        plain.jvp([torch.tensor(a) for a in arrays], [torch.tensor(t) for t in tans])
    with pytest.raises(ValueError, match="exponent"):
        ex.jvp([torch.tensor(a) for a in arrays], [torch.tensor(t) for t in tans], primal=False)
    # an exponent the call would not use is refused
    with pytest.raises(ValueError, match="exponent"):
        ex.jvp([torch.tensor(a) for a in arrays], [torch.tensor(t) for t in tans], exponent=1.0)


@pytest.mark.reference
def test_installed_tree_contract_forward_ad(ctg, monkeypatch):  # noqa: F811
    """``cb.install(tree, strip_exponent=True, stripped_grad=True)``; cotengra's own stripped slice
    combiner propagates the slices' tangents through torch ops"""
    from torch.autograd import forward_ad

    emu_jvp_strip.install(monkeypatch)
    con = ctg.utils.lattice_equation([3, 3], d_min=2, d_max=3, seed=1)
    tree = ctg.array_contract_tree(con.inputs, con.output, con.size_dict, optimize="greedy")
    tree.slice_(target_slices=4)
    assert tree.nslices > 1
    arrays = ctg.utils.make_arrays_from_inputs(con.inputs, con.size_dict, seed=0, dtype="complex128")
    arrays = [np.asarray(a) * 30.0 for a in arrays]
    tans = make_arrays([a.shape for a in arrays], "complex128", seed=2)
    cb.install(tree, strip_exponent=True, stripped_grad=True)
    with forward_ad.dual_level():
        with warnings.catch_warnings():
            warnings.simplefilter("ignore")
            m, e = tree.contract(_dual(arrays, tans), strip_exponent=True)
        e = float(e)
        assert e > 5
        dm = forward_ad.unpack_dual(m).tangent
    spec = cb.TreeSpec.from_cotengra(tree)
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, range(len(arrays)))
    assert nrel(dm.numpy() * 10.0 ** e, np.asarray(want).reshape(dm.shape)) <= 1e-10


# ------------------------------------------------------------------ two ranks
def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _rank_tangent(rec, ids):
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), DT, seed=rec["seed"], scale=3.0)
    tans = make_arrays(spec.shapes(), DT, seed=rec["seed"] + 1)
    _m, e, dm = emulate_stripped_jvp(_plan(spec), arrays, tans, slice_ids=ids)
    return np.array(dm), e


def _worker(rank, world, port, name, q):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rec = BY_NAME[name]
        begin, step, count = cb.rank_slices(rank, world, tree_spec(rec).nslices)
        dm, e = _rank_tangent(rec, range(begin, begin + step * count, step))
        tot, emax = cb.reduce_partials(torch.as_tensor(dm), torch.tensor([e], dtype=torch.float64))
        q.put((rank, tot.numpy(), float(emax.item())))
    finally:
        dist.destroy_process_group()


def test_two_ranks_reduce_partials():
    name = "lattice6x6_d3_sliced"
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, name, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {r: (dm, e) for r, dm, e in (q.get(timeout=120) for _ in procs)}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    dm1, e1 = _rank_tangent(BY_NAME[name], None)
    for r in (0, 1):
        dm, e = got[r]
        assert e == e1 and nrel(dm, dm1) < 1e-12


# ------------------------------------------------------------------ a slice whose amplitude is exactly zero
def zero_amplitude_case(zero_slice):
    """A sliced tree ``X[j] = sum_i A[i,s] B[i,j]``, ``R[k] = sum_j X[j] C[j,s,k]`` whose slice
    ``zero_slice`` has an exactly zero root product while X is not: integer operands, C orthogonal to X
    on that slice and max|X| a power of two, so neither the lazy scaling by 1/max|X| nor any summation
    order leaves a residue.  Its root factor is 0 (``e_s = -inf``) and
    ``e'_s`` is finite; the tangent is not zero.  Returns ``(spec, arrays, tangents)``, float64."""
    spec = cb.TreeSpec([("i", "s"), ("i", "j"), ("j", "s", "k")], ("k",), {"i": 3, "j": 2, "k": 2, "s": 2},
                       [(0, 1), (3, 2)], [("s", 2, None)])
    rng = np.random.default_rng(5)
    A = rng.integers(-3, 4, size=(3, 2)).astype(np.float64)
    B = rng.integers(-3, 4, size=(3, 2)).astype(np.float64)
    A[:, zero_slice] = [1.0, 0.0, 0.0]
    B[0] = [4.0, -2.0]  # X of the zero slice: [4, -2]
    C = rng.integers(-3, 4, size=(2, 2, 2)).astype(np.float64)
    X = A[:, zero_slice] @ B
    C[:, zero_slice, 0] = [X[1], -X[0]]
    C[:, zero_slice, 1] = [-2 * X[1], 2 * X[0]]
    other = 1 - zero_slice
    assert np.any(np.einsum("i,ij,jk->k", A[:, other], B, C[:, other, :]) != 0)
    tans = make_arrays([A.shape, B.shape, C.shape], "float64", seed=8)
    return spec, [A, B, C], tans


@pytest.mark.parametrize("zero_slice", [0, 1], ids=["zero_slice_first", "zero_slice_second"])
def test_zero_amplitude_slice_keeps_its_tangent(zero_slice):
    """Folded first (the running exponent still -inf) or after a non-zero slice, the zero-amplitude
    slice contributes its tangent: dm 10^e equals the exact JVP in both orders, and in a reversed
    slice order and as two interleaved one-slice calls combined by exponent"""
    spec, arrays, tans = zero_amplitude_case(zero_slice)
    plan = _plan(spec, dtype="float64")
    want = jvp_oracle(spec, spec.contractions(), arrays, tans, range(3))
    zero_only = jvp_oracle(spec, spec.contractions(), arrays, tans, range(3), slice_ids=[zero_slice])
    assert np.linalg.norm(zero_only) > 0.1 * np.linalg.norm(want)  # (the slice's tangent matters)
    for ids in ([0, 1], [1, 0]):
        m, e, dm = emulate_stripped_jvp(plan, arrays, tans, slice_ids=ids)
        assert math.isfinite(e)
        assert nrel(dm * 10.0 ** e, want) <= 1e-13, (ids, nrel(dm * 10.0 ** e, want))
    # one call per slice, combined as reduce_partials does: additive over slices
    parts = [emulate_stripped_jvp(plan, arrays, tans, slice_ids=[s]) for s in (0, 1)]
    emax = max(p[1] for p in parts)
    tot = sum(p[2] * (0.0 if p[1] == -math.inf else 10.0 ** (p[1] - emax)) for p in parts)
    # (the zero slice's own call has e = -inf: alone it is a zero result, with a zero tangent)
    assert np.all(parts[zero_slice][2] == 0) and parts[zero_slice][1] == -math.inf
    assert nrel(tot * 10.0 ** emax, want - zero_only) <= 1e-13
    # the zero slice alone, with the exponent of the other slice given as the running exponent it
    # continues from: its tangent is kept
    other = parts[1 - zero_slice]
    m2, e2, dm2 = emulate_stripped_jvp(plan, arrays, tans, slice_ids=[zero_slice], out=np.array(other[0]).reshape(-1),
                                       tout=np.array(other[2]).reshape(-1), exponent=other[1])
    assert nrel(dm2 * 10.0 ** e2, want) <= 1e-13
