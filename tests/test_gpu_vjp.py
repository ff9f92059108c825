"""Reverse mode on the device: ``ctgb_plan_execute`` of VJP plans against the torch-CPU gradient oracle
(``oracle/grad_oracle.py``), kernel-family coverage of the backward nodes, the autograd paths of
the public interface, and the workspace check."""

import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import torch  # noqa: E402

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import _lib  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from oracle import grad_oracle as go  # noqa: E402
from tests.helpers import GOLDEN_DIR, load_json, make_arrays, tree_spec  # noqa: E402

TREES = load_json("trees.json")
SEEN_VARIANTS = set()  # (dtype class, variant) of every backward node run below


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _dev(arrays):
    return [torch.tensor(np.asarray(a)).cuda() for a in arrays]


def _run(ex, arrays, cot, wrt=None, **kw):
    plan = ex.vjp_plan(wrt)
    fam = "double" if ex.dtype in ("float64", "complex128") else "single"
    SEEN_VARIANTS.update((fam, v) for v in plan.variants())
    g = ex.vjp(_dev(arrays), torch.tensor(np.asarray(cot)).cuda(), wrt=wrt, **kw)
    torch.cuda.synchronize()
    return [None if x is None else x.cpu().numpy() for x in g]


@pytest.mark.parametrize("rec", TREES, ids=[r["name"] for r in TREES])
def test_device_gradients_match_oracle(rec):
    spec = tree_spec(rec)
    dt = rec["dtype"]
    arrays = make_arrays(spec.shapes(), dt, seed=rec["seed"])
    ex = cb.TreeExecutor(spec, dtype=dt)
    cot = make_arrays([ex.plan.out_shape], dt, seed=rec["seed"] + 1)[0]
    ir = spec.contractions()
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, arrays, cot)
    for g, w in zip(_run(ex, arrays, cot), want):
        assert nrel(g, w) <= 1e-10
    # single precision against the double oracle: max(1e-5, 3 x the oracle's own single-precision error)
    lo = "complex64" if dt == "complex128" else "float32"
    a32 = [a.astype(lo) for a in arrays]
    c32 = cot.astype(lo)
    ref32 = go.tree_gradients(spec.inputs, spec.output, spec.sliced, ir, a32, c32)
    ex32 = cb.TreeExecutor(spec, dtype=lo)
    for g, w, r in zip(_run(ex32, a32, c32), want, ref32):
        assert nrel(g, w) <= max(1e-5, 3.0 * nrel(r, w))


def _stem_spec(m, k, n, o):
    """A[m,k] B[k,n] C[n,o] D[o] -> [m], contracted ((A B) C) D: the shapes of a stem absorbing small
    tensors -- its backward has tall x small results (H_A, H_AB, H_ABC) and small results over the
    long m range (H_B, H_C, H_D)."""
    inputs = [("m", "k"), ("k", "n"), ("n", "o"), ("o",)]
    return cb.TreeSpec(inputs, ("m",), {"m": m, "k": k, "n": n, "o": o}, [(0, 1), (4, 2), (5, 3)])


STEM_CASES = [
    # (dtype, o, forced variant, variant that must appear among the backward nodes)
    ("complex128", 4, None, L.VAR_DOTSTREAM4),
    ("complex128", 4, None, L.VAR_ROWSTREAM),
    ("complex128", 4, None, L.VAR_DMMASTREAM),
    ("complex128", 4, None, L.VAR_DMMA_32x32),
    ("complex128", 1, None, L.VAR_DOTSTREAM),
    ("complex128", 4, L.VAR_KRED, L.VAR_KRED),
    ("complex128", 4, L.VAR_SIMT_64x64, L.VAR_SIMT_64x64),
    ("complex128", 4, L.VAR_DMMA_128x64, L.VAR_DMMA_128x64),
    ("float64", 4, L.VAR_DMMA_256x16, L.VAR_DMMA_256x16),
    ("complex64", 4, None, L.VAR_TF32_32x32),
    ("complex64", 4, None, L.VAR_TC05_128x16),
    ("complex64", 4, L.VAR_DMMA_256x16, L.VAR_DMMA_256x16),
    ("float32", 4, None, L.VAR_TF32_32x32),
    ("float32", 4, L.VAR_DMMA_128x64, L.VAR_DMMA_128x64),
    ("float32", 4, L.VAR_SIMT_64x64, L.VAR_SIMT_64x64),
]


@pytest.mark.parametrize("dtype,o,force,expect", STEM_CASES)
def test_backward_kernel_families(dtype, o, force, expect):
    spec = _stem_spec(1 << 20, 16, 8, o)
    hi = "complex128" if "complex" in dtype else "float64"
    arrays = make_arrays(spec.shapes(), hi, seed=5)
    cot = make_arrays([(1 << 20,)], hi, seed=6)[0]
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot)
    opts = {} if force is None else {"variant": force}
    ex = cb.TreeExecutor(spec, dtype=dtype, fuse=False)
    ex._plan_opts = {}
    from cotengra_b200 import VjpPlan

    with torch.cuda.device(ex.device):
        plan = VjpPlan(ex._ir, spec.inputs, spec.output, spec.size_dict, (), dtype=dtype, **opts).create()
    ex._vjp_plans[tuple(range(4))] = plan
    assert expect in plan.variants(), plan.variants()
    got = _run(ex, [a.astype(dtype) for a in arrays], cot.astype(dtype))
    tol = 1e-10 if dtype == hi else 1e-5
    for g, w in zip(got, want):
        assert nrel(g, w) <= tol


def test_every_kernel_family_ran_backward():
    """Row / DMMA streams, dot streams, KRED, DMMA and TF32 tiles, wgmma, SIMT and TF32_32x32."""
    need = {("double", L.VAR_ROWSTREAM), ("double", L.VAR_DMMASTREAM), ("double", L.VAR_DOTSTREAM),
            ("double", L.VAR_DOTSTREAM4), ("double", L.VAR_KRED), ("double", L.VAR_DMMA_128x64),
            ("double", L.VAR_DMMA_32x32), ("single", L.VAR_DMMA_256x16), ("single", L.VAR_TC05_128x16),
            ("double", L.VAR_SIMT_64x64), ("single", L.VAR_TF32_32x32)}
    if not need <= SEEN_VARIANTS:
        pytest.skip("runs after test_backward_kernel_families in the same session")
    assert need <= SEEN_VARIANTS


def test_config2_peps8x8_bond6_gradients():
    """BASELINE config 2 (8x8 PEPS, D = 6) in complex64: the gradient of all 64 tensors against torch
    GPU autograd in complex128 (torch.einsum node by node)."""
    rec = next(r for r in TREES if r["name"] == "peps8x8_d2")
    size_dict = {ix: 6 for ix in rec["size_dict"]}
    spec = cb.TreeSpec(rec["inputs"], rec["output"], size_dict, rec["path"])
    arrays = make_arrays(spec.shapes(), "complex128", seed=11, scale=0.35)
    ts = [torch.from_numpy(a).cuda().requires_grad_() for a in arrays]
    out = go.run_contractions(spec.contractions(), ts)
    want = [g.cpu().numpy() for g in torch.autograd.grad(out, ts, grad_outputs=torch.ones_like(out))]
    a64 = [a.astype(np.complex64) for a in arrays]
    ref64 = go.tree_gradients(spec.inputs, spec.output, (), spec.contractions(), a64, np.ones((), np.complex64))
    ex = cb.TreeExecutor(spec, dtype="complex64")
    got = _run(ex, a64, np.ones(ex.plan.out_shape, np.complex64))
    assert len(got) == 64
    errs = [nrel(g, w) for g, w in zip(got, want)]
    refs = [nrel(r, w) for r, w in zip(ref64, want)]
    print(f"config2 peps8x8 D=6 c64 gradients: worst {max(errs):.2e}, torch-cpu c64 worst {max(refs):.2e}")
    for e, r in zip(errs, refs):
        assert e <= max(1e-5, 3.0 * r)


def test_sliced_sycamore_m10_gate_gradients():
    import json

    path = os.path.join(GOLDEN_DIR, "circuits.json")
    recs = json.load(open(path))
    rec = recs["m10"]
    flat = np.load(os.path.join(GOLDEN_DIR, "circuits_arrays.npz"))["m10_arrays_flat"]
    small = cb.TreeSpec.from_dict(rec["small_spec"])
    arrays, off = [], 0
    for shape in small.shapes():
        n = int(np.prod(shape))
        arrays.append(flat[off:off + n].reshape(shape).astype(np.complex128))
        off += n
    ex = cb.TreeExecutor(small, dtype="complex128")
    cot = make_arrays([ex.plan.out_shape], "complex128", seed=8)[0]
    big = sorted(range(len(arrays)), key=lambda i: -arrays[i].size)
    wrt = sorted({big[0], big[1], len(arrays) // 2, len(arrays) - 1})
    plan = ex.vjp_plan(wrt)
    print(f"m10 small_spec: {ex.nslices} slices, VJP workspace {plan.total_bytes} bytes")
    got = _run(ex, arrays, cot, wrt=wrt, begin=0, step=1, count=2)
    want = go.tree_gradients(small.inputs, small.output, small.sliced, small.contractions(), arrays, cot,
                             wrt=wrt, slice_ids=range(2))
    for i in wrt:
        assert nrel(got[i], want[i]) <= 1e-10


@pytest.mark.parametrize("dtype", ["float64", "complex128"])
def test_gradcheck(dtype):
    rec = next(r for r in TREES if r["name"] == "lattice4x4_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), dtype, seed=1)
    ex = cb.TreeExecutor(spec, dtype=dtype)
    ts = tuple(torch.from_numpy(a).cuda().requires_grad_() for a in arrays)
    assert torch.autograd.gradcheck(lambda *xs: cb.contract_tree(ex, list(xs)), ts, fast_mode=True)


def test_inputs_without_grad_launch_what_they_did():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=1)
    ex = cb.TreeExecutor(spec, dtype=rec["dtype"])
    dev = _dev(arrays)
    ex.contract_device(dev)
    torch.cuda.synchronize()
    n0 = _lib.launch_count()
    ref = ex.contract_device(dev)
    n1 = _lib.launch_count()
    out = cb.contract_tree(ex, dev)
    n2 = _lib.launch_count()
    with torch.no_grad():
        out2 = cb.contract_tree(ex, [t.clone().requires_grad_() for t in dev])
    n3 = _lib.launch_count()
    assert n2 - n1 == n1 - n0 == n3 - n2
    assert out.grad_fn is None and out2.grad_fn is None
    # (split-K partial sums arrive in any order: equal up to rounding)
    assert torch.allclose(out, ref, rtol=1e-12, atol=0) and torch.allclose(out2, ref, rtol=1e-12, atol=0)
    # with requires_grad: the same forward launches, then the VJP plan's on backward()
    xs = [t.clone().requires_grad_() for t in dev]
    out3 = cb.contract_tree(ex, xs)
    n4 = _lib.launch_count()
    assert n4 - n3 == n1 - n0 and torch.allclose(out3.detach(), ref, rtol=1e-12, atol=0)
    out3.backward(torch.ones_like(out3))
    assert all(x.grad is not None for x in xs)


def test_small_workspace_is_refused_before_any_launch():
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), rec["dtype"], seed=1)
    ex = cb.TreeExecutor(spec, dtype=rec["dtype"])
    plan = ex.vjp_plan()
    dev = _dev(arrays)
    cot = torch.ones(plan.out_shape, dtype=dev[0].dtype, device="cuda")
    grads = [torch.zeros_like(t) for t in dev]
    ws = torch.empty(plan.total_bytes - 1, dtype=torch.uint8, device="cuda")
    before = _lib.launch_count()
    with pytest.raises(MemoryError):
        plan.execute([t.data_ptr() for t in dev], cot.data_ptr(), [g.data_ptr() for g in grads], ws.data_ptr(),
                     ws.numel(), 0, 1, plan.nslices, torch.cuda.current_stream().cuda_stream)
    assert _lib.launch_count() == before
