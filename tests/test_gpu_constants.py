"""Constant inputs of the tree executor on the device (``TreeExecutor(constants=...)``): every
golden tree with none, all but one, about half and all of its inputs constant, in complex128 and
complex64, against the golden values and the unfolded executor; gradients, precision and
accumulation modes, strip_exponent, and the benchmark's peps8x8 and m10s workloads."""

import numpy as np
import pytest
import torch

import bench
import cotengra_b200 as cb
from tests.helpers import load_json, load_npz, make_arrays, rel_err, tree_spec

pytestmark = pytest.mark.gpu

TREES = load_json("trees.json")
TVALS = load_npz("trees_values.npz")
BY_NAME = {r["name"]: r for r in TREES}


def constant_sets(n, seed):
    rng = np.random.default_rng(seed)
    perm = rng.permutation(n).tolist()
    return [[], sorted(perm[1:]), sorted(perm[: n // 2]) if n > 1 else [], list(range(n))]


def split(arrays, consts):
    return {i: arrays[i] for i in consts}, [a for i, a in enumerate(arrays) if i not in consts]


def host(x):
    return x.cpu().numpy() if isinstance(x, torch.Tensor) else np.asarray(x)


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_folded_matrix(rec):
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    d128 = [torch.from_numpy(a).cuda() for a in arrays]
    d64 = [t.to(torch.complex64) for t in d128]
    ref = cb.TreeExecutor(spec, dtype="complex128")(d128)
    if rec["dtype"] == "complex128" and rec["name"] in TVALS:
        assert rel_err(host(ref), TVALS[rec["name"]]) < 1e-10
    ref = host(ref)
    base128 = cb.TreeExecutor(spec, dtype="complex128")
    runs = [base128(d128), base128(d128)]
    base64 = host(cb.TreeExecutor(spec, dtype="complex64")(d64))
    tol64 = 3 * max(rel_err(base64, ref), 1e-7)
    for consts in constant_sets(len(arrays), rec["seed"]):
        c128, v128 = split(d128, consts)
        c64, v64 = split(d64, consts)
        got = cb.TreeExecutor(spec, dtype="complex128", constants=c128)(v128)
        assert isinstance(got, torch.Tensor) and got.is_cuda
        assert rel_err(host(got), ref) < 1e-10, consts
        got64 = cb.TreeExecutor(spec, dtype="complex64", constants=c64)(v64)
        assert rel_err(host(got64), ref) <= tol64, consts
        if consts and len(consts) < len(arrays):
            # nothing folded: the very same launches as the unfolded executor
            zero = cb.TreeExecutor(spec, dtype="complex128", constants=c128, fold_max_bytes=0)(v128)
            same_launches(zero, runs)
    same_launches(cb.TreeExecutor(spec, dtype="complex128", constants={})(d128), runs)


def same_launches(got, runs):
    """Bit for bit what the unfolded executor returns; where that executor itself differs between two
    calls (split-K partial sums added atomically, in arrival order), to a few ulps."""
    if torch.equal(runs[0], runs[1]):
        assert torch.equal(got, runs[0])
    else:
        assert rel_err(host(got), host(runs[0])) <= 1e-14


@pytest.mark.parametrize("name", ["lattice6x6_d3_sliced", "rand_r3_o1_hi0_ho1_None_s42_sliced_out", "projected",
                                  "pre_sum_sliced", "peps8x8_d2"])
def test_autograd_through_expression(name):
    rec = BY_NAME[name]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    consts = constant_sets(len(arrays), rec["seed"])[2]
    variables = [i for i in range(len(arrays)) if i not in consts]
    cmap, var = split(dev, consts)
    expr = cb.array_contract_expression(spec.inputs, spec.output, optimize=spec, constants=cmap)
    ts = [t.clone().requires_grad_() for t in var]
    out = expr(*ts)
    cot = torch.from_numpy(make_arrays([tuple(out.shape)], "complex128", seed=1)[0]).cuda()
    grads = torch.autograd.grad(out, ts, grad_outputs=cot)
    base = cb.TreeExecutor(spec, dtype="complex128")
    want = base.vjp(dev, cot, wrt=variables)
    for g, i in zip(grads, variables):
        assert rel_err(host(g), host(want[i])) < 1e-10


@pytest.mark.parametrize("opts", [dict(precision="tf32"), dict(accumulate="double"), dict(strip_exponent=True)],
                         ids=["tf32", "double", "strip"])
def test_modes(opts):
    rec = BY_NAME["lattice6x6_d3_sliced"]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex64", seed=rec["seed"])
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    cmap, var = split(dev, constant_sets(len(arrays), rec["seed"])[1])
    ex = cb.TreeExecutor(spec, dtype="complex64", constants=cmap, **opts)
    assert ex.folded
    want = cb.TreeExecutor(spec, dtype="complex64", **opts)(dev)
    got = ex(var)
    if opts.get("strip_exponent"):
        got, want = host(got[0]) * 10.0 ** got[1], host(want[0]) * 10.0 ** want[1]
    tol = 1e-2 if opts.get("precision") == "tf32" else 1e-5
    assert rel_err(host(got), host(want)) < tol
    if opts.get("accumulate") == "double":
        assert got.dtype == torch.complex128


@pytest.mark.parametrize("config", ["peps8x8", "m10s"])
@pytest.mark.parametrize("k", [1, 4])
def test_benchmark_workloads(config, k):
    spec, arrays, _desc = bench.load_workload(config, "complex128")
    rng = np.random.default_rng(k)
    variables = sorted(rng.choice(len(arrays), size=k, replace=False).tolist())
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    cmap, var = split(dev, [i for i in range(len(arrays)) if i not in variables])
    ex = cb.TreeExecutor(spec, dtype="complex128", constants=cmap)
    assert ex.folded and ex.folded_bytes > 0
    got = ex.contract_device(var)
    want = cb.TreeExecutor(spec, dtype="complex128").contract_device(dev)
    assert rel_err(host(got), host(want)) < 1e-10


def test_all_constant_copies():
    rec = BY_NAME["lattice4x4_sliced"]
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    ex = cb.TreeExecutor(spec, constants=dict(enumerate(dev)))
    a, b = ex([]), ex([])
    assert a.is_cuda and a.data_ptr() != b.data_ptr()
    a.zero_()
    assert rel_err(host(b), TVALS[rec["name"]]) < 1e-10
    assert rel_err(host(ex([])), TVALS[rec["name"]]) < 1e-10
    exn = cb.TreeExecutor(spec, constants=dict(enumerate(arrays)))
    assert isinstance(exn([]), np.ndarray)
