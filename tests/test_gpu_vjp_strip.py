"""Gradients of strip_exponent results on the device (``stripped_grad=True``): the mantissa's
gradient ``dm/dx = 10^-e damp/dx`` against the unstripped device gradient and the torch-CPU oracle,
every backward kernel family with the epilogue / pre-scaled-operand scaling in both single-precision
modes, the m20 tree in complex64 with normalised inputs (whose unstripped amplitude underflows), the
same tree at W = 2^30 under a workspace budget, and an 8x8 PEPS whose unstripped complex64
amplitude overflows."""

import math

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import torch  # noqa: E402

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import VjpPlan  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from oracle import grad_oracle as go  # noqa: E402
from tests.helpers import load_json, make_arrays, tree_spec  # noqa: E402
from tests.slicing_util import appxB_at_width  # noqa: E402
from tests.test_gpu_vjp import STEM_CASES, _stem_spec  # noqa: E402

TREES = load_json("trees.json")
GIB = 1 << 30
SEEN = set()  # (dtype, precision, variant) of every stripped backward node run below


def nrel(got, want):
    d = np.linalg.norm(want)
    return float(np.linalg.norm(np.asarray(got) - want) / (d if d else 1.0))


def _dev(arrays):
    return [torch.tensor(np.asarray(a)).cuda() for a in arrays]


def _stripped(ex, arrays, cot, begin=0, count=None, **kw):
    """(m, e, gradients) of the stripped executor ``ex`` for the mantissa cotangent ``cot``"""
    dev = _dev(arrays)
    m, e = ex.contract_device(dev, begin, 1, count)
    for plan in ex._vjp_plans.values():
        SEEN.update((ex.dtype, ex.precision, v) for v in plan.variants())
    g = ex.vjp(dev, torch.as_tensor(np.asarray(cot)).cuda() if not callable(cot) else cot(m), begin, 1, count,
               exponent=e, **kw)
    torch.cuda.synchronize()
    return m.cpu().numpy(), float(e.item()), [None if x is None else x.cpu().numpy() for x in g]


@pytest.mark.parametrize("rec", [r for r in TREES if r["dtype"] == "complex128"], ids=lambda r: r["name"])
def test_complex128_stripped_equals_unstripped_times_ten_to_minus_e(rec):
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=6.0)
    ex = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True, stripped_grad=True)
    cot = make_arrays([ex.plan.out_shape], "complex128", seed=rec["seed"] + 1)[0]
    m, e, got = _stripped(ex, arrays, cot)
    SEEN.update(("complex128", "3xtf32", v) for v in ex.vjp_plan().variants())
    plain = cb.TreeExecutor(spec, dtype="complex128")
    full = plain.vjp(_dev(arrays), torch.tensor(cot).cuda())
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot)
    for g, f, w in zip(got, full, want):
        assert nrel(g, f.cpu().numpy() * 10.0 ** -e) <= 1e-10
        assert nrel(g, w * 10.0 ** -e) <= 1e-10


CASES = [c + ("3xtf32",) for c in STEM_CASES] + [
    ("complex64", 4, None, L.VAR_TF32_32x32, "tf32"),
    ("complex64", 4, None, L.VAR_TC05_128x16, "tf32"),
    ("float32", 4, L.VAR_DMMA_128x64, L.VAR_DMMA_128x64, "tf32"),
]


@pytest.mark.parametrize("dtype,o,force,expect,precision", CASES)
def test_stripped_backward_kernel_families(dtype, o, force, expect, precision):
    """``_stem_spec``: tall x small backward results and small results over a long range, each
    family forced or chosen as the unstripped plan chooses it; the small operand is pre-scaled
    (``prescale_b``) or the epilogue scales, as ``ctgb_plan_strip_modes`` reports."""
    spec = _stem_spec(1 << 20, 16, 8, o)
    hi = "complex128" if "complex" in dtype else "float64"
    arrays = make_arrays(spec.shapes(), hi, seed=5, scale=3.0)
    cot = make_arrays([(1 << 20,)], hi, seed=6)[0]
    want = go.tree_gradients(spec.inputs, spec.output, spec.sliced, spec.contractions(), arrays, cot)
    ex = cb.TreeExecutor(spec, dtype=dtype, fuse=False, strip_exponent=True, stripped_grad=True,
                         precision=precision)
    opts = {} if force is None else {"variant": force}
    with torch.cuda.device(ex.device):
        plan = VjpPlan(ex._ir, spec.inputs, spec.output, spec.size_dict, (), dtype=dtype, strip_exponent=True,
                       stripped_grad=True, precision=precision, **opts).create()
    ex._vjp_plans[tuple(range(4))] = plan
    assert expect in plan.variants(), plan.variants()
    modes = plan.strip_modes()
    bwd = [i for i, nd in enumerate(plan.nodes) if nd["phase"] >= 2 and nd["kind"] == 0]
    assert all(modes[i][1] == 0 for i in bwd)  # backward nodes measure nothing
    print(f"{dtype} {precision} {expect}: prescaled {[modes[i][0] for i in bwd]}, "
          f"launches/slice {plan.launches_per_slice()}")
    _m, e, got = _stripped(ex, [a.astype(dtype) for a in arrays], cot.astype(dtype))
    tol = 1e-10 if dtype == hi else (1e-5 if precision == "3xtf32" else 5e-3)
    for g, w in zip(got, want):
        assert nrel(g, w * 10.0 ** -e) <= tol


def test_every_family_and_mode_ran_stripped():
    need = {(c[0], c[4], c[3]) for c in CASES}
    assert need <= SEEN, need - SEEN
    assert {p for _d, p, _v in SEEN} == {"3xtf32", "tf32"}


def _m20_identity(width, budget, tol, scale=1.0):
    """Slice 0 of the m20 tree, complex64, inputs without a tuning scale, cotangent 1: the mantissa
    is linear in every input, so ``sum(x_i conj(g_i)) = m`` for every i."""
    spec = appxB_at_width(width)
    arrays = make_arrays(spec.shapes(), "complex64", seed=0, scale=scale)
    ex = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True, stripped_grad=True)
    dev = _dev(arrays)
    m, e = ex.contract_device(dev, 0, 1, 1)
    m = complex(m.cpu().numpy().reshape(-1)[0])
    e = float(e.item())
    ex._ws = None
    torch.cuda.empty_cache()
    g = ex.vjp(dev, torch.ones(ex.plan.out_shape, dtype=dev[0].dtype, device="cuda"), 0, 1, 1,
               max_bytes=budget, exponent=e)
    plan = ex.vjp_plan(max_bytes=budget)
    if budget is not None:
        assert plan.total_bytes <= budget
    worst, gmax = 0.0, 0.0
    for x, gi in zip(dev, g):
        s = complex(torch.sum(x.to(torch.complex128) * gi.to(torch.complex128).conj()).item())
        norm = float(torch.sum(x.abs().double() * gi.abs().double()).item())
        worst = max(worst, abs(s - m) / norm)
        gmax = max(gmax, float(gi.abs().max().item()))
    print(f"m20 W=2^{width} complex64 stripped, scale {scale}: plan {plan.total_bytes / GIB:.2f} GiB, m {m}, e {e:.4f}, "
          f"worst identity error {worst:.2e}, largest input |H~| {gmax:.3e}")
    assert math.isfinite(e) and abs(m) > 0
    assert worst <= tol
    return dev, ex


@pytest.mark.parametrize("scale", [1.0, 0.4])
def test_m20_w26_complex64_untuned_inputs(scale):
    """Inputs without the 0.65 that keeps the unstripped complex64 slice in range: at scale 1 the
    unstripped amplitude is lost to overflow (10^72), at 0.4 it underflows to 0."""
    spec = appxB_at_width(26)
    arrays = make_arrays(spec.shapes(), "complex64", seed=0, scale=scale)
    plain = cb.TreeExecutor(spec, dtype="complex64")
    amp = plain.contract_device(_dev(arrays), 0, 1, 1).cpu().numpy()
    if scale == 1.0:
        assert not np.isfinite(amp).all()
    else:
        assert np.all(amp == 0)
    del plain
    torch.cuda.empty_cache()
    _m20_identity(26, None, 1e-5, scale)


def test_m20_w30_complex64_identity_under_budget():
    free = torch.cuda.mem_get_info()[0]
    if 56 * GIB + (4 << 30) > free:
        pytest.skip(f"{free} bytes free")
    dev, ex = _m20_identity(30, 56 * GIB, 1e-5)
    del dev, ex
    torch.cuda.empty_cache()


def test_peps8x8_d6_log_amplitude_gradient():
    """Inputs scaled so that the unstripped complex64 amplitude overflows: d log|amp| from the
    stripped complex64 plan (cotangent m/|m|^2) against the complex128 amplitude's."""
    import bench

    spec, arrays, _desc = bench.load_workload("peps8x8", "complex128")
    ex128 = cb.TreeExecutor(spec, dtype="complex128")
    amp0 = complex(ex128.contract_device(_dev(arrays)).cpu().numpy().reshape(-1)[0])
    s = (1e45 / abs(amp0)) ** (1.0 / len(arrays))
    arrays = [a * s for a in arrays]
    dev = _dev(arrays)
    amp = ex128.contract_device(dev)
    c = amp / (amp.abs() ** 2)
    want = [g.cpu().numpy() for g in ex128.vjp(dev, c)]
    a64 = [a.astype("complex64") for a in arrays]
    plain = cb.TreeExecutor(spec, dtype="complex64")
    assert not np.isfinite(plain.contract_device(_dev(a64)).cpu().numpy()).all()
    ex = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True, stripped_grad=True)
    m, e, got = _stripped(ex, a64, lambda m: m / (m.abs() ** 2))
    assert abs(e + math.log10(abs(complex(m.reshape(-1)[0]))) - math.log10(abs(complex(amp.item())))) < 1e-4
    worst = max(nrel(g, w) for g, w in zip(got, want))
    print(f"peps8x8 D=6 complex64 stripped: e {e:.4f}, worst d log|amp| error {worst:.2e}")
    assert worst <= 1e-3


def test_autograd_log_amplitude():
    """contract_tree on CUDA tensors: (log|m| + e ln 10).backward() equals the complex128 unstripped
    d log|amp|."""
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex128", seed=rec["seed"], scale=4.0)
    ts = [torch.tensor(a).cuda().requires_grad_() for a in arrays]
    m, e = cb.contract_tree(spec, ts, dtype="complex128", strip_exponent=True, stripped_grad=True)
    assert isinstance(e, float) and m.grad_fn is not None
    (torch.log(torch.abs(m.reshape(-1)[0])) + e * math.log(10.0)).backward()
    ref = [torch.tensor(a).cuda().requires_grad_() for a in arrays]
    amp = cb.contract_tree(spec, ref, dtype="complex128")
    torch.log(torch.abs(amp.reshape(-1)[0])).backward()
    for t, r in zip(ts, ref):
        assert nrel(t.grad.cpu().numpy(), r.grad.cpu().numpy()) <= 1e-10
