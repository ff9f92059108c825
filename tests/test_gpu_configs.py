"""GPU parity on the BASELINE.json configurations other than the bench line:
config 2 (8x8 PEPS, bond 6, complex64, unsliced), config 3 (Sycamore m10
amplitude, real gate tensors, unsliced) and config 4 (Sycamore m12, 256 slices)."""

import json
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

import cotengra_b200 as cb  # noqa: E402
from oracle import ctg_oracle as orc  # noqa: E402
from tests.helpers import GOLDEN_DIR, decode_sliced, load_json, load_npz, make_arrays, rel_err  # noqa: E402


def _circuit(name):
    path = os.path.join(GOLDEN_DIR, "circuits.json")
    if not os.path.exists(path):
        pytest.skip("circuits.json not generated")
    recs = json.load(open(path))
    if name not in recs:
        pytest.skip(f"{name} fixture not generated")
    rec = recs[name]
    flat = load_npz("circuits_arrays.npz")[f"{name}_arrays_flat"]
    spec = cb.TreeSpec.from_dict(rec["spec"])
    arrays, off = [], 0
    for shape in spec.shapes():
        n = int(np.prod(shape))
        arrays.append(flat[off:off + n].reshape(shape))
        off += n
    assert off == flat.size
    return rec, spec, arrays


def test_config2_peps8x8_bond6():
    rec = next(r for r in load_json("trees.json") if r["name"] == "peps8x8_d2")
    size_dict = {ix: 6 for ix in rec["size_dict"]}
    spec = cb.TreeSpec(rec["inputs"], rec["output"], size_dict, rec["path"])
    arrays = make_arrays(spec.shapes(), "complex128", seed=11, scale=0.35)
    want = orc.run_contractions(spec.contractions(), arrays)  # numpy oracle, complex128
    got = cb.contract_tree(spec, arrays)
    assert rel_err(got, want) < 1e-10
    a64 = [a.astype(np.complex64) for a in arrays]
    got64 = cb.contract_tree(spec, a64)
    assert got64.dtype == np.complex64
    # north_star: 1e-5 -- or, where the reference's own numpy complex64 run is itself further than
    # that from the complex128 value (BASELINE.md: 8e-6 on this network), within 3x of its error
    e_ref = rel_err(orc.run_contractions(spec.contractions(), a64), want)
    e_gpu = rel_err(got64, want)
    print(f"config2 peps8x8 D=6 c64: gpu {e_gpu:.2e}, numpy c64 {e_ref:.2e}")
    assert e_gpu < max(1e-5, 3.0 * e_ref)
    # ... and with stripped exponents: the long contracted ranges of this tree are folded into C chunk
    # by chunk by the tcgen05 epilogue, such nodes are measured after the launch (ctg_b200.cu measure_after)
    m, e = cb.contract_tree(spec, a64, strip_exponent=True)
    e_strip = rel_err(complex(m) * 10.0 ** float(e), want)
    print(f"config2 peps8x8 D=6 c64 strip_exponent: gpu {e_strip:.2e}")
    assert e_strip < max(1e-5, 3.0 * e_ref)
    m, e = cb.contract_tree(spec, arrays, strip_exponent=True)
    assert rel_err(complex(m) * 10.0 ** float(e), want) < 1e-10


def test_config3_sycamore_m10_amplitude():
    rec, spec, arrays = _circuit("m10")
    vals = load_npz("circuits_values.npz")
    want = vals["m10_amplitude"]  # reference numpy path, real gate tensors
    got = cb.contract_tree(spec, arrays)
    assert rel_err(got, want) < 1e-10
    a64 = [a.astype(np.complex64) for a in arrays]
    got64 = cb.contract_tree(spec, a64)
    e_ref = rel_err(orc.run_contractions(spec.contractions(), a64), want)
    e_gpu = rel_err(got64, want)
    print(f"config3 m10 c64: gpu {e_gpu:.2e}, numpy c64 {e_ref:.2e}")
    assert e_gpu < max(1e-5, 3.0 * e_ref)
    # slices of the further-sliced copy against the reference
    small = cb.TreeSpec.from_dict(rec["small_spec"])
    ex = cb.TreeExecutor(small, dtype="complex128")
    import torch

    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    for i in (0, 3):
        g = ex.contract_device(dev, begin=i, step=1, count=1).cpu().numpy()
        assert rel_err(g, vals[f"m10_small_slice{i}"]) < 1e-10


def test_config3_sycamore_m10_simplified_network():
    """Config 3 as the reference notebooks run it: the rank-simplified m10 network (164 tensors,
    `Quantum Circuit Example Old.ipynb:143`; cotengra_b200.circuits.rank_simplify), tree searched
    by the unmodified reference; same amplitude as the 1764-tensor network."""
    rec, spec, arrays = _circuit("m10s")
    assert spec.N == 164
    vals = load_npz("circuits_values.npz")
    want = vals["m10s_amplitude"]
    assert rel_err(want, vals["m10_amplitude"]) < 1e-10  # the reference agrees with itself
    got = cb.contract_tree(spec, arrays)
    assert rel_err(got, want) < 1e-10
    small = cb.TreeSpec.from_dict(rec["small_spec"])
    for i in (0, 3):
        g = cb.contract_tree(small, arrays, slice_ids=(i, 1, 1))
        assert rel_err(g, vals[f"m10s_small_slice{i}"]) < 1e-10


def test_config4_sycamore_m12_sliced():
    rec, spec, arrays = _circuit("m12")
    vals = load_npz("circuits_values.npz")
    import torch

    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    small = cb.TreeSpec.from_dict(rec["small_spec"])
    ex = cb.TreeExecutor(small, dtype="complex128")
    for i in (0, 3):
        g = ex.contract_device(dev, begin=i, step=1, count=1).cpu().numpy()
        assert rel_err(g, vals[f"m12_small_slice{i}"]) < 1e-10
    # the 256-slice tree itself (W = 2^32 per slice at complex64 = 32 GiB tensors,
    # > 2^31 elements: 64-bit offsets): one slice must equal the sum of the slices
    # of the further-sliced tree that refine it
    # (~100 GiB of device memory; on an 80 GB H100 the same check runs one slicing step down:
    # W = 2^31 per slice, 16 GiB tensors, byte offsets beyond 2^32)
    from tests.slicing_util import slice_id, slice_one_more

    free, _total = torch.cuda.mem_get_info()
    if free < 120 * 2**30:
        spec, _ix = slice_one_more(spec)
    ex_big = cb.TreeExecutor(spec, dtype="complex64")
    dev64 = [t.to(torch.complex64) for t in dev]
    big = ex_big.contract_device(dev64, begin=0, step=1, count=1).cpu().numpy()
    del ex_big
    torch.cuda.empty_cache()

    child, extra = spec, []
    for _ in range(3):
        child, ix = slice_one_more(child)
        extra.append(ix)
    exc = cb.TreeExecutor(child, dtype="complex128")
    from itertools import product

    tot = 0
    for digs in product(*[range(child.size_dict[ix]) for ix in extra]):
        key = dict(spec.slice_key(0))
        key.update(dict(zip(extra, digs)))
        tot = tot + exc.contract_device(dev, begin=slice_id(child, key), step=1, count=1).cpu().numpy()
    assert rel_err(big, tot) < 1e-4
