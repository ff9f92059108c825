"""``precision="tf32"`` (one round-to-nearest tf32 pass) on the device.

* Every float32 / complex64 tensor-core case of ``tests/kernel_cases.py`` (the wgmma kernel's 106, the
  mma.sync tiles' and ``TF32_32x32``'s), built with ``precision="tf32"``, in the same sentinel-guarded
  buffers as ``test_gpu_kernel_paths.py``.  Each element must lie within ``C_SINGLE * (|A| |B|)_ij`` of
  the numpy model of one tf32 pass (``tests/precision_cases.py``): what is left is fp32 accumulation.
  Every case's model differs from the exact einsum by more than twice that bound
  (``test_precision_cpu.py``), so a three-pass or a truncating kernel fails here.
* Special values: inf and NaN reach the same outputs as in the default mode, and an operand within
  half a tf32 ulp of FLT_MAX does not round to inf.
* Whole trees, forward and VJP, against complex128.
* The default mode launches what it launched without the keyword, and gives the same bits.
"""

import json
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cotengra_b200 as cb  # noqa: E402
from cotengra_b200 import lowering as L  # noqa: E402
from tests import kernel_cases as KC  # noqa: E402
from tests import precision_cases as PC  # noqa: E402
from tests.helpers import GOLDEN_DIR, load_json, load_npz, make_arrays, rel_err  # noqa: E402

CASES = {c.id: c for c in PC.CASES}


def _launch(plan, lay, case):
    import torch

    from cotengra_b200 import _lib

    dev = [torch.from_numpy(b).cuda() for b in lay.bufs]
    es = np.dtype(case.dtype).itemsize
    ptr = [d.data_ptr() + off * es for d, off in zip(dev, lay.offs)]
    pa, pb = (ptr[1], ptr[0]) if plan.swapped else (ptr[0], ptr[1])
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa, pb, ptr[2], 0))
    torch.cuda.synchronize()
    for d, b in zip(dev[:2], lay.bufs[:2]):
        assert d.cpu().numpy().tobytes() == b.tobytes()  # operands untouched
    return dev[2].cpu().numpy()


@pytest.mark.parametrize("cid", list(CASES))
def test_tf32_kernel_path(cid):
    case = CASES[cid]
    plan = PC.build_plan(case, "tf32")
    assert plan.variant in L.TF32_VARIANTS and int(plan.words[L.W_FLAGS]) & L.FLAG_TF32_ONE_PASS
    lay = KC.make_layout(case, seed=zlib.crc32(cid.encode()))
    cbuf = _launch(plan, lay, case)
    got, bad = KC.check_result(case, lay, cbuf)
    assert bad.size == 0, f"{bad.size} sentinel components outside C changed, first at {bad[:8]}"
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} described C elements NaN"
    ref, scale = PC.tf32_reference(case, lay)
    ratio = KC.error_ratio(got, ref, scale)
    assert ratio <= KC.C_SINGLE, ratio


def _special_operands(dtype, rng, M=256, K=64, N=64):
    """A with inf, -inf, the NaNs GPU arithmetic makes (0x7FFFFFFF) and a low-payload one
    (0x7F800001) in rows 3..6, and FLT_MAX (within half a tf32 ulp of it) alone in row 11."""
    rd = np.float32
    cplx = np.dtype(dtype).kind == "c"
    a = rng.uniform(-1, 1, (M, K)) + (1j * rng.uniform(-1, 1, (M, K)) if cplx else 0)
    b = rng.uniform(-1, 1, (K, N)) + (1j * rng.uniform(-1, 1, (K, N)) if cplx else 0)
    a, b = a.astype(dtype), b.astype(dtype)
    comp = a.view(rd).reshape(M, -1)
    comp[3, 0] = np.inf
    comp[4, 2] = -np.inf
    comp[5, 4] = np.array(0x7FFFFFFF, np.uint32).view(rd)
    comp[6, 6] = np.array(0x7F800001, np.uint32).view(rd)
    a[11, :] = 0
    a[11, 0] = np.array(0x7F7FFFFF, np.uint32).view(rd)  # FLT_MAX
    b[0, :] = 0.5 + (0.25j if cplx else 0)
    return a, b


@pytest.mark.parametrize("variant,dtype", [
    (L.VAR_TC05_128x64, "complex64"), (L.VAR_TC05_128x16, "complex64"), (L.VAR_DMMA_128x64, "complex64"),
    (L.VAR_DMMA_256x16, "float32"), (L.VAR_DMMA_64x128, "float32"), (L.VAR_TF32_32x32, "complex64"),
], ids=lambda x: KC.VARIANT_NAMES.get(x, x) if isinstance(x, int) else x)
def test_tf32_special_values(variant, dtype):
    import torch

    from cotengra_b200 import _lib

    a, b = _special_operands(dtype, np.random.default_rng(5))
    dims = L.classify_pair("ab", a.shape, "bc", b.shape, "ac")
    outs = {}
    for precision in ("3xtf32", "tf32"):
        plan = L.build_pair_desc(dims, dtype, variant=variant, c_dense_elems=a.shape[0] * b.shape[1],
                                 precision=precision)
        assert plan.variant == variant
        ta, tb = torch.from_numpy(a).cuda(), torch.from_numpy(b).cuda()
        c = torch.full((a.shape[0], b.shape[1]), float("nan"), dtype=ta.dtype, device="cuda")
        pa, pb = (tb, ta) if plan.swapped else (ta, tb)
        _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa.data_ptr(), pb.data_ptr(),
                                                  c.data_ptr(), 0))
        torch.cuda.synchronize()
        outs[precision] = c.cpu().numpy()
    base, one = outs["3xtf32"], outs["tf32"]
    comp = lambda x: x.view(np.float32).reshape(x.shape[0], -1)  # noqa: E731
    # every non-finite output of the default mode is non-finite here too, and nothing else is
    assert np.array_equal(~np.isfinite(comp(base)), ~np.isfinite(comp(one)))
    assert np.isnan(comp(one)[5:7]).all()  # a NaN operand poisons its whole row
    assert not np.isfinite(comp(one)[3:5]).any()
    # FLT_MAX * 0.5 (+ 0.25i) stays finite: hi is truncated, not rounded up to inf
    want = a[11, 0].astype(np.complex128 if dtype == "complex64" else np.float64) * b[0].astype(np.complex128)
    assert np.isfinite(comp(one)[11]).all()
    assert rel_err(one[11], want) < 2e-3
    # ordinary rows sit near the default mode's result
    assert rel_err(one[20:], base[20:]) < 5e-3


# ---------------------------------------------------------------------------------- whole trees


def _peps():
    rec = next(r for r in load_json("trees.json") if r["name"] == "peps8x8_d2")
    spec = cb.TreeSpec(rec["inputs"], rec["output"], {ix: 6 for ix in rec["size_dict"]}, rec["path"])
    return spec, make_arrays(spec.shapes(), "complex128", seed=11, scale=0.35)


def _m10s():
    with open(os.path.join(GOLDEN_DIR, "circuits.json")) as f:
        rec = json.load(f)["m10s"]
    flat = load_npz("circuits_arrays.npz")["m10s_arrays_flat"]
    spec = cb.TreeSpec.from_dict(rec["spec"])
    arrays, off = [], 0
    for shape in spec.shapes():
        n = int(np.prod(shape))
        arrays.append(np.ascontiguousarray(flat[off:off + n].reshape(shape)).astype(np.complex128))
        off += n
    return spec, arrays


TREE_CASES = {"peps8x8": _peps, "m10s": _m10s}
# Max-norm relative error of one tf32 pass against complex128, measured on an H100 80GB HBM3 at a 700 W
# power limit with these inputs (DESIGN.md §4b), two runs: forward 1.4e-3 and 1.8e-3 (peps8x8; split-K
# summation order moves it), 5.8e-4 (m10s), 1.4e-3 (m10s with strip_exponent); worst gradient 2.4e-3
# (peps8x8) and 2.3e-3 (m10s).  An operand rounded to tf32 is off by up to 2^-11 relative, and these
# trees chain dozens of dependent tensor-core nodes whose errors add up like a random walk, so 1e-3 is
# the expected size; the default mode holds 1e-5 on the same trees.  The bounds leave a margin of 3.5-4x
# over the largest measured value of each quantity.
TREE_TOL = {"peps8x8": 7e-3, "m10s": 5e-3}
GRAD_TOL = {"peps8x8": 1e-2, "m10s": 1e-2}


def _nrel(x, w):
    return float(np.linalg.norm(np.ravel(x - w)) / max(np.linalg.norm(np.ravel(w)), 1e-300))


@pytest.mark.parametrize("name", list(TREE_CASES))
def test_tf32_whole_tree_forward_and_vjp(name):
    import torch

    spec, arrays = TREE_CASES[name]()
    count = min(spec.nslices, 2)
    dev128 = [torch.from_numpy(a).cuda() for a in arrays]
    dev64 = [t.to(torch.complex64) for t in dev128]
    ex128 = cb.TreeExecutor(spec, dtype="complex128")
    ex3 = cb.TreeExecutor(spec, dtype="complex64")
    ex1 = cb.TreeExecutor(spec, dtype="complex64", precision="tf32")
    want = ex128.contract_device(dev128, 0, 1, count).cpu().numpy()
    got3 = ex3.contract_device(dev64, 0, 1, count).cpu().numpy()
    got1 = ex1.contract_device(dev64, 0, 1, count).cpu().numpy()
    e3, e1 = rel_err(got3, want), rel_err(got1, want)
    print(f"{name}: forward rel err 3xtf32 {e3:.2e}, tf32 {e1:.2e}")
    assert e3 < 1e-4
    assert e1 < TREE_TOL[name]
    assert e1 > e3  # the one-pass kernels really ran
    # reverse mode: every input, cotangent of ones
    cot = torch.ones(ex128.plan.out_shape, dtype=torch.complex128, device="cuda")
    g128 = [g.cpu().numpy() for g in ex128.vjp(dev128, cot, 0, 1, count)]
    g1 = [g.cpu().numpy() for g in ex1.vjp(dev64, cot.to(torch.complex64), 0, 1, count)]
    assert ex1.vjp_plan().precision == "tf32"
    worst = max(_nrel(a, w) for a, w in zip(g1, g128))
    print(f"{name}: VJP worst gradient rel err tf32 {worst:.2e}")
    assert worst < GRAD_TOL[name]


def test_tf32_strip_exponent():
    import torch

    # (the strip-exponent epilogues scale what later nodes read, so their tf32 roundings differ from the
    # plain run's: both are held to the complex128 value)
    spec, arrays = _m10s()
    dev128 = [torch.from_numpy(a).cuda() for a in arrays]
    want = cb.TreeExecutor(spec, dtype="complex128").contract_device(dev128).cpu().numpy()
    exs = cb.TreeExecutor(spec, dtype="complex64", precision="tf32", strip_exponent=True)
    m, e = exs.contract_device([t.to(torch.complex64) for t in dev128])
    stripped = m.cpu().numpy() * 10.0 ** float(e.item())
    err = rel_err(stripped, want)
    print(f"m10s strip_exponent: rel err tf32 {err:.2e}")
    assert err < TREE_TOL["m10s"]


def test_default_mode_unchanged():
    import torch

    from cotengra_b200 import _lib

    spec, arrays = _m10s()
    dev = [torch.from_numpy(a).to(torch.complex64).cuda() for a in arrays]
    # planned for one SM the descriptors choose no split-K, and m10s has no dot-stream node: no atomics,
    # so the result is deterministic bit for bit (the launches still use every SM)
    exa = cb.TreeExecutor(spec, dtype="complex64", sm_count=1)
    exb = cb.TreeExecutor(spec, dtype="complex64", precision="3xtf32", sm_count=1)
    pairs = [nd["words"] for nd in exa.plan.nodes if nd["kind"] == 0]
    assert sum(int(w[L.W_VARIANT]) in L.TF32_VARIANTS for w in pairs) > 10
    assert all(int(w[L.W_SPLITK]) == 1 for w in pairs)
    assert not any(int(w[L.W_VARIANT]) in (L.VAR_DOTSTREAM, L.VAR_DOTSTREAM4) for w in pairs)
    assert exa.plan.launches_per_slice() == exb.plan.launches_per_slice()
    outs, launches = [], []
    for ex in (exa, exb, exa):
        n0 = _lib.launch_count()
        outs.append(ex.contract_device(dev).cpu().numpy())
        torch.cuda.synchronize()
        launches.append(_lib.launch_count() - n0)
    assert launches[0] == launches[1] == launches[2]
    assert outs[0].tobytes() == outs[1].tobytes() == outs[2].tobytes()


def test_einsum_keyword_on_device():
    import torch

    rng = np.random.default_rng(7)
    a = torch.from_numpy((rng.uniform(-1, 1, (512, 96)) + 1j * rng.uniform(-1, 1, (512, 96))).astype(np.complex64))
    b = torch.from_numpy((rng.uniform(-1, 1, (96, 64)) + 1j * rng.uniform(-1, 1, (96, 64))).astype(np.complex64))
    want = (a.to(torch.complex128) @ b.to(torch.complex128)).numpy()
    want1 = PC.round_tf32(a.numpy()).astype(np.complex128) @ PC.round_tf32(b.numpy()).astype(np.complex128)
    ein, tdot = cb.implementation(precision="tf32")
    for got in (ein("ab,bc->ac", a.cuda(), b.cuda()), tdot(a.cuda(), b.cuda(), 1)):
        got = got.cpu().numpy()
        assert rel_err(got, want1) < 1e-6 < rel_err(got, want)
    assert rel_err(cb.einsum("ab,bc->ac", a.cuda(), b.cuda()).cpu().numpy(), want) < 1e-6
