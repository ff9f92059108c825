"""Constant inputs of the tree executor (``TreeExecutor(constants=...)``, ``constants.py``) on the CPU:
the fold planner, the folded and main plans walked by the descriptor emulator
(``tests/desc_emulator.py`` through ``tests/emu_device.py``) against the golden values and the
unfolded executor, gradients on the variables, budgets, errors, ``array_contract_expression``,
checkpoint tags and a two-rank gloo run."""

import gc
import math
import os
import socket

import numpy as np
import pytest
import torch

import cotengra_b200 as cb
from cotengra_b200 import ExecPlan
from cotengra_b200.constants import plan_folds
from tests import emu_device
from tests.helpers import load_json, load_npz, make_arrays, rel_err, tree_spec

TREES = load_json("trees.json")
TVALS = load_npz("trees_values.npz")
BY_NAME = {r["name"]: r for r in TREES}
GRAD_TREES = [r for r in TREES if r["sliced"] or r["name"].startswith(("pre_", "single_", "lattice4x4"))
              or r["name"] in ("config1_rand10_hyper", "projected")]


@pytest.fixture
def emu(monkeypatch):
    emu_device.install(monkeypatch)
    yield
    gc.collect()  # (autograd graphs hold executors: free them while the emulator is installed)


def constant_sets(n, seed):
    """none, all but one, about half and all of ``n`` inputs, seeded"""
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n).tolist()
    return [[], sorted(perm[1:]), sorted(perm[: n // 2]) if n > 1 else [], list(range(n))]


def split(arrays, consts):
    return {i: arrays[i] for i in consts}, [a for i, a in enumerate(arrays) if i not in consts]


def call_macs(plan):
    return plan.macs_per_slice * plan.nslices + plan.macs_invariant


def golden(rec):
    return TVALS[rec["name"]] if rec["name"] in TVALS else None


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_folded_values(emu, rec):
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    base = cb.TreeExecutor(spec, dtype=dt)
    want = base(arrays)
    gold = golden(rec)
    if gold is not None:
        assert rel_err(want, gold) < 1e-11
    base_s = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True)
    for consts in constant_sets(len(arrays), rec["seed"]):
        cmap, var = split(arrays, consts)
        ex = cb.TreeExecutor(spec, dtype=dt, constants=cmap)
        got = ex(var)
        assert isinstance(got, np.ndarray)
        assert rel_err(got, want if gold is None else gold) < 1e-11, (consts, ex.folded)
        # the MACs a fold removes are exactly the folded subtrees' (the planner's unfolded count)
        assert call_macs(ex.plan) == call_macs(base.plan) - sum(f.macs for f in ex.folded) or len(consts) == len(arrays)
        assert ex.folded_bytes == sum(f.bytes for f in ex.folded)
        m, e = cb.TreeExecutor(spec, dtype=dt, constants=cmap, strip_exponent=True)(var)
        assert rel_err(np.asarray(m) * 10.0 ** e, want if gold is None else gold) < 1e-11
        # slice by slice and as two round-robin ranks, the same as the unfolded executor
        if spec.nslices > 1:
            for i in range(spec.nslices):
                assert rel_err(ex.contract_host(var, i, 1, 1), base.contract_host(arrays, i, 1, 1)) < 1e-12
            for r in range(2):
                b, s, c = cb.rank_slices(r, 2, spec.nslices)
                assert rel_err(ex.contract_host(var, b, s, c), base.contract_host(arrays, b, s, c)) < 1e-12
            fm, fe = cb.TreeExecutor(spec, dtype=dt, constants=cmap, strip_exponent=True).contract_host(var, 1, 1, 1)
            bm, be = base_s.contract_host(arrays, 1, 1, 1)
            assert rel_err(fm * 10.0 ** fe, bm * 10.0 ** be) < 1e-12
        if any(ix in rec["output"] for ix, _s, _p in spec.sliced):
            got_c = list(ex.gen_output_chunks(var, with_key=True))
            want_c = list(base.gen_output_chunks(arrays, with_key=True))
            assert [k for _c, k in got_c] == [k for _c, k in want_c]
            for (c1, _k1), (c2, _k2) in zip(got_c, want_c):
                assert rel_err(c1, c2) < 1e-12


@pytest.mark.parametrize("rec", GRAD_TREES, ids=[r["name"] for r in GRAD_TREES])
def test_variable_gradients(emu, rec):
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    n = len(arrays)
    base = cb.TreeExecutor(spec, dtype=dt)
    cot = torch.from_numpy(make_arrays([base.plan.out_shape], dt, seed=rec["seed"] + 1)[0])
    dev = [torch.from_numpy(a) for a in arrays]
    base_s = cb.TreeExecutor(spec, dtype=dt, strip_exponent=True, stripped_grad=True)
    for consts in constant_sets(n, rec["seed"])[:3]:
        variables = [i for i in range(n) if i not in consts]
        cmap, var = split(dev, consts)
        ex = cb.TreeExecutor(spec, dtype=dt, constants=cmap)
        want = base.vjp(dev, cot, wrt=variables)
        got = ex.vjp(var, cot)
        for j, i in enumerate(variables):
            assert rel_err(got[j], want[i]) < 1e-10, (consts, i)
        sub = variables[::2]
        got = ex.vjp(var, cot, wrt=range(0, len(variables), 2))
        for j, i in enumerate(variables):
            assert (got[j] is None) == (i not in sub)
        # stripped: the executor's exponent includes the folds', the plan's does not
        exs = cb.TreeExecutor(spec, dtype=dt, constants=cmap, strip_exponent=True, stripped_grad=True)
        _m, e = exs.contract_device(var)
        bm, be = base_s.contract_device(dev)
        got = exs.vjp(var, cot, exponent=e)
        want = base_s.vjp(dev, cot, wrt=variables, exponent=be)
        for j, i in enumerate(variables):
            assert rel_err(got[j], want[i]) < 1e-10, (consts, i)
        # torch autograd through the call records the variables only
        ts = [t.clone().requires_grad_() for t in var]
        out = ex(ts)
        grads = torch.autograd.grad(out, ts, grad_outputs=cot)
        want = base.vjp(dev, cot, wrt=variables)
        for j, i in enumerate(variables):
            assert rel_err(grads[j], want[i]) < 1e-10


def _words(plan):
    return [(nd["kind"], nd["phase"], list(np.asarray(nd["words"]))) for nd in plan.nodes]


@pytest.mark.parametrize("name", ["rand_r3_o1_hi0_ho1_None_s42_sliced_out", "projected", "pre_diag_sliced",
                                  "lattice6x6_d3_sliced", "single_trace"])
def test_unfolded_plans_unchanged(emu, name):
    rec = BY_NAME[name]
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    base = cb.TreeExecutor(spec, dtype=dt)
    none = cb.TreeExecutor(spec, dtype=dt, constants={})
    assert _words(none.plan) == _words(base.plan) and none.folded == []
    consts = constant_sets(len(arrays), 1)[2]
    cmap, var = split(arrays, consts)
    zero = cb.TreeExecutor(spec, dtype=dt, constants=cmap, fold_max_bytes=0)
    assert zero.folded == [] and zero.folded_bytes == 0
    assert _words(zero.plan) == _words(base.plan)
    assert rel_err(zero(var), base(arrays)) < 1e-12


@pytest.mark.parametrize("name", ["peps8x8_d2", "lattice6x6_d3_sliced"])
def test_budgets(emu, name):
    rec = BY_NAME[name]
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    want = cb.TreeExecutor(spec, dtype=dt)(arrays)
    var_pos = len(arrays) - 1
    cmap, var = split(arrays, [i for i in range(len(arrays)) if i != var_pos])
    full = cb.TreeExecutor(spec, dtype=dt, constants=cmap, fold_max_bytes=1 << 40)
    assert full.folded
    biggest = max(f.bytes for f in full.folded)
    descended = False
    for budget in (1 << 40, full.folded_bytes, biggest - 1, biggest // 4, 16):
        ex = cb.TreeExecutor(spec, dtype=dt, constants=cmap, fold_max_bytes=budget)
        assert ex.folded_bytes <= budget
        descended |= any(f.ssa not in {g.ssa for g in full.folded} for f in ex.folded)
        assert rel_err(ex(var), want) < 1e-11
    assert descended
    # deterministic
    again = cb.TreeExecutor(spec, dtype=dt, constants=cmap, fold_max_bytes=biggest // 4)
    assert [(f.ssa, f.term, f.bytes, f.macs) for f in again.folded] == \
        [(f.ssa, f.term, f.bytes, f.macs) for f in cb.TreeExecutor(spec, dtype=dt, constants=cmap,
                                                                    fold_max_bytes=biggest // 4).folded]


def test_sycamore_m20_planner():
    """The planner host-side on the Sycamore-m20 Appendix-B tree with one variable leaf."""
    rec = next(r for r in load_json("sycamore_m20.json") if r["name"] == "sycamore_m20_appxB")
    spec = tree_spec(rec)
    from cotengra_b200.fusion import fuse_stems

    xspec, _info = fuse_stems(spec, "complex64")
    ir = xspec.contractions()
    cost = ExecPlan(ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype="complex64", sm_count=132)
    var = max(range(len(spec.inputs)), key=lambda i: math.prod(spec.size_dict[ix] for ix in spec.inputs[i]))
    consts = [i for i in range(len(spec.inputs)) if i != var]
    fp = plan_folds(xspec, ir, consts, "complex64", None, cost)
    assert fp.folds
    assert sum(f.bytes for f in fp.folds) <= cost.workspace_bytes
    main = ExecPlan(fp.records, fp.inputs, spec.output, spec.size_dict, spec.sliced, dtype="complex64",
                    sm_count=132, input_ids=fp.input_ids)
    assert call_macs(main) == fp.macs_unfolded - sum(f.macs for f in fp.folds)
    assert fp.variables == (var,)


def test_errors(emu):
    rec = BY_NAME["lattice4x4_sliced"]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=0)
    with pytest.raises(ValueError):
        cb.TreeExecutor(spec, constants={len(arrays): arrays[0]})
    with pytest.raises(ValueError):
        cb.TreeExecutor(spec, constants={-1: arrays[-1]})
    with pytest.raises(ValueError):
        cb.TreeExecutor(spec, constants={0: np.zeros((7,), complex)})
    with pytest.raises(ValueError):
        cb.TreeExecutor(spec, constants=[(0, arrays[0]), (0, arrays[0])])
    with pytest.raises(TypeError):
        cb.TreeExecutor(spec, constants={0: arrays[0].astype(np.complex64)})
    ex = cb.TreeExecutor(spec, constants={0: arrays[0], 3: arrays[3]})
    with pytest.raises(ValueError):
        ex(arrays)  # every input, not the variables
    with pytest.raises(ValueError):
        ex.vjp([torch.from_numpy(a) for a in arrays[1:3] + arrays[4:]], torch.zeros(ex.plan.out_shape,
               dtype=torch.complex128), wrt=[len(arrays) - 2])


def test_all_constant_returns_copies(emu):
    rec = BY_NAME["lattice4x4_sliced"]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    want = cb.TreeExecutor(spec)(arrays)
    ex = cb.TreeExecutor(spec, constants=dict(enumerate(arrays)))
    a, b = ex([]), ex([])
    assert isinstance(a, np.ndarray) and rel_err(a, want) < 1e-12
    a[...] = 0
    assert rel_err(b, want) < 1e-12 and rel_err(ex([]), want) < 1e-12
    ext = cb.TreeExecutor(spec, constants={i: torch.from_numpy(x) for i, x in enumerate(arrays)},
                          strip_exponent=True)
    (m1, e1), (m2, _e2) = ext([]), ext([])
    assert isinstance(m1, torch.Tensor) and m1.data_ptr() != m2.data_ptr()
    assert rel_err(m1.numpy() * 10.0 ** e1, want) < 1e-12


def test_constants_are_copied(emu):
    rec = BY_NAME["lattice4x4_sliced"]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    want = cb.TreeExecutor(spec)(arrays)
    consts = {i: torch.from_numpy(arrays[i].copy()) for i in range(0, len(arrays), 2)}
    ex = cb.TreeExecutor(spec, constants=consts, fold_max_bytes=0)
    for t in consts.values():
        t.zero_()
    assert rel_err(ex([a for i, a in enumerate(arrays) if i % 2]), want) < 1e-12


def test_array_contract_expression(emu):
    rec = BY_NAME["rand_r3_o1_hi0_ho1_None_s42_sliced_out"]
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    want = cb.TreeExecutor(spec, dtype=dt)(arrays)
    cmap, var = split(arrays, [0, 2, 5])
    expr = cb.array_contract_expression(spec.inputs, spec.output, size_dict=spec.size_dict, optimize=spec,
                                        constants=cmap)
    assert expr.executor.dtype == dt
    assert rel_err(expr(*var), want) < 1e-11
    assert rel_err(expr(*var, backend="numpy"), want) < 1e-11
    m, e = cb.array_contract_expression(spec.inputs, shapes=spec.shapes(), optimize=spec, constants=cmap,
                                        strip_exponent=True)(*var)
    assert rel_err(m * 10.0 ** e, want) < 1e-11
    plain = cb.array_contract_expression(spec.inputs, spec.output, optimize=spec)
    assert plain.executor is None and rel_err(plain(*arrays), want) < 1e-11
    other = tree_spec(BY_NAME["rand_r3_o1_hi0_ho1_None_s42"])
    with pytest.raises(ValueError):
        cb.array_contract_expression(other.inputs[::-1], other.output, optimize=spec)
    with pytest.raises(ValueError):
        cb.array_contract_expression(spec.inputs, spec.output[::-1], optimize=spec)
    with pytest.raises(ValueError):
        cb.array_contract_expression(spec.inputs, spec.output, size_dict={ix: 5 for ix in spec.size_dict},
                                     optimize=spec)
    with pytest.raises(ValueError):
        cb.array_contract_expression(spec.inputs, spec.output, optimize="auto")


def test_checkpoint_tag(emu, tmp_path):
    rec = BY_NAME["lattice4x4_sliced"]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    want = cb.TreeExecutor(spec)(arrays)
    cmap, var = split(arrays, [1, 4, 9])
    ck = str(tmp_path / "c.npz")
    got = cb.contract_checkpointed(spec, var, ck, every=1, executor=cb.TreeExecutor(spec, constants=cmap))
    assert rel_err(got, want) < 1e-12
    # the same constants resume; other constant values are refused
    cb.contract_checkpointed(spec, var, ck, executor=cb.TreeExecutor(spec, constants=cmap))
    other = {**cmap, 4: arrays[4] * 2}
    with pytest.raises(ValueError):
        cb.contract_checkpointed(spec, var, ck, executor=cb.TreeExecutor(spec, constants=other))
    # executors without constants hash as before: a file of the plain executor resumes with an empty dict
    ck2 = str(tmp_path / "d.npz")
    cb.contract_checkpointed(spec, arrays, ck2, every=1)
    assert rel_err(cb.contract_checkpointed(spec, arrays, ck2, executor=cb.TreeExecutor(spec, constants={})),
                   want) < 1e-12


def _free_port():
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    return port


def _worker(rank, world, port, q):
    import torch.distributed as dist

    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    mp = pytest.MonkeyPatch()
    emu_device.install(mp)
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        rec = BY_NAME["lattice6x6_d3_sliced"]
        spec = tree_spec(rec)
        arrays = make_arrays(spec.shapes(), rec["dtype"], seed=rec["seed"])
        cmap, var = split(arrays, list(range(0, len(arrays), 3)))
        ex = cb.TreeExecutor(spec, dtype=rec["dtype"], constants=cmap)
        q.put((rank, cb.contract_distributed(spec, var, executor=ex), len(ex.folded)))
        del ex
    finally:
        dist.destroy_process_group()
        gc.collect()  # (the emulated plans are released while the emulator is installed)
        mp.undo()


def test_two_ranks_gloo():
    import torch.multiprocessing as tmp

    want = TVALS["lattice6x6_d3_sliced"]
    ctx = tmp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    got = {r: (out, nf) for r, out, nf in (q.get(timeout=300) for _ in procs)}
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for r in range(2):
        assert got[r][1] > 0
        assert rel_err(got[r][0], want) < 1e-11
