"""``accumulate="double"`` on the GPU: the wide dot-stream kernels through ``ctgb_contract_pair``
(double sums of fp32 operands, guard bands intact, run-to-run agreement), the slice sum of trees with
2^14 slices against this package's complex128 result and a numpy model of the sequential fp32 sum,
and every host entry point."""

import numpy as np
import pytest

import cotengra_b200 as cb
from cotengra_b200 import _lib, lowering as L
from tests.helpers import rel_err

pytestmark = pytest.mark.gpu

GUARD = 64  # NaN elements on either side of C
WIDE = {"float32": "float64", "complex64": "complex128"}


def _torch():
    import torch

    return torch


def _operand(torch, shape, dtype, same_sign, seed):
    gen = torch.Generator(device="cuda")
    gen.manual_seed(seed)
    lo, hi = (0.5, 1.0) if same_sign else (-1.0, 1.0)
    rdt = torch.float32
    x = torch.empty(shape, dtype=rdt, device="cuda").uniform_(lo, hi, generator=gen)
    if dtype == "complex64":
        # (same sign: real parts positive, imaginary parts small, so that re(a b) does not cancel)
        y = torch.empty(shape, dtype=rdt, device="cuda").uniform_(lo, hi, generator=gen)
        x = torch.complex(x, 0.25 * y if same_sign else y)
    return x


def _run_pair(torch, eq, a, b, dtype, wide, accumulate, variant):
    """One launch of ``eq`` through ``ctgb_contract_pair``; returns ``(C, prior, guards_intact)``."""
    lhs, out = eq.split("->")
    ta, tb = lhs.split(",")
    dims = L.classify_pair(tuple(ta), tuple(a.shape), tuple(tb), tuple(b.shape), tuple(out))
    n = int(np.prod(dims.out_shape)) if dims.out_shape else 1
    plan = L.build_pair_desc(dims, dtype, accumulate=accumulate, c_dense_elems=n, wide_c=wide,
                             sm_count=_lib.device_info()["sm_count"])
    assert plan.variant == variant
    assert bool(int(plan.words[L.W_FLAGS]) & L.FLAG_WIDE_C) == wide
    cdt = getattr(torch, WIDE[dtype] if wide else dtype)
    buf = torch.full((n + 2 * GUARD,), float("nan"), dtype=cdt, device="cuda")
    prior = (torch.arange(n, device="cuda", dtype=torch.float64) * 0.5 + 1.0).to(cdt)
    buf[GUARD:GUARD + n] = prior  # (accumulate off: must be overwritten)
    before = buf.clone()
    x, y = (b, a) if plan.swapped else (a, b)
    words = np.ascontiguousarray(plan.words)
    _lib.check(_lib.load().ctgb_contract_pair(words.ctypes.data, x.data_ptr(), y.data_ptr(),
                                              buf.data_ptr() + GUARD * buf.element_size(), 0))
    torch.cuda.synchronize()
    raw, raw0 = (t.view(torch.uint8) for t in (buf, before))
    gb = GUARD * buf.element_size()
    intact = bool(torch.equal(raw[:gb], raw0[:gb]) and torch.equal(raw[-gb:], raw0[-gb:]))
    return buf[GUARD:GUARD + n].reshape(dims.out_shape), prior.reshape(dims.out_shape), intact


# (equation, shapes as powers of two filled in per K, variant)
def _shapes(kind, K):
    if kind == "dot":  # operands in differing index orders
        return "abc,cba->", (128, K // (128 * 128), 128), (128, K // (128 * 128), 128), L.VAR_DOTSTREAM
    if kind == "dot4_permuted_c":
        return "km,kn->nm", (K, 4), (K, 3), L.VAR_DOTSTREAM4
    return "akm,kan->mn", (32, K // 32, 3), (K // 32, 32, 2), L.VAR_DOTSTREAM4  # dot4_accumulate


CASES = [("dot", 20), ("dot", 23), ("dot", 26), ("dot4_permuted_c", 20), ("dot4_accumulate", 20),
         ("dot4_accumulate", 22)]


@pytest.mark.parametrize("dtype", ["float32", "complex64"])
@pytest.mark.parametrize("kind,logk", CASES, ids=[f"{k}-2^{e}" for k, e in CASES])
def test_wide_dot_stream_kernels(kind, logk, dtype):
    torch = _torch()
    if logk == 26 and dtype == "complex64":
        logk = 25  # (512 MiB per operand either way)
    eq, sa, sb, variant = _shapes(kind, 1 << logk)
    for same_sign in (True, False):
        a = _operand(torch, sa, dtype, same_sign, 1)
        b = _operand(torch, sb, dtype, same_sign, 2)
        wdt = getattr(torch, WIDE[dtype])
        want = torch.einsum(eq, a.to(wdt), b.to(wdt))
        bound = torch.einsum(eq, a.abs().double(), b.abs().double())  # |A||B|
        for accumulate in (False, True):
            got, prior, intact = _run_pair(torch, eq, a, b, dtype, True, accumulate, variant)
            assert intact, "guard bands of C changed"
            assert got.dtype == wdt
            ref = want + prior if accumulate else want
            err = float(((got - ref).abs() / bound).max())
            assert err < 1e-12, (same_sign, accumulate, err)
        # the native kernel on the same case keeps its own bound, which the wide one is far below
        got32, _p, intact = _run_pair(torch, eq, a, b, dtype, False, False, variant)
        assert intact and got32.dtype == getattr(torch, dtype)
        err32 = float(((got32.to(wdt) - want).abs() / bound).max())
        assert err32 < 4e-6, err32
        if same_sign:
            assert err32 > 1e-10, err32
        del a, b, want, bound


def test_wide_dot_stream_runs_agree():
    torch = _torch()
    eq, sa, sb, variant = _shapes("dot4_permuted_c", 1 << 22)
    a = _operand(torch, sa, "complex64", True, 3)
    b = _operand(torch, sb, "complex64", True, 4)
    r1, _p, _i = _run_pair(torch, eq, a, b, "complex64", True, False, variant)
    r2, _p, _i = _run_pair(torch, eq, a, b, "complex64", True, False, variant)
    assert float(((r1 - r2).abs() / r1.abs()).max()) < 1e-14


def test_launcher_refuses_the_flag_elsewhere():
    torch = _torch()
    dims = L.classify_pair(("k",), (1 << 14,), ("k",), (1 << 14,), ())
    plan = L.build_pair_desc(dims, "complex64", accumulate=True)
    assert plan.variant == L.VAR_KRED
    words = np.ascontiguousarray(plan.words).copy()
    words[L.W_FLAGS] |= L.FLAG_WIDE_C
    a = torch.zeros(1 << 14, dtype=torch.complex64, device="cuda")
    c = torch.zeros(4, dtype=torch.complex128, device="cuda")
    with pytest.raises(ValueError):
        _lib.check(_lib.load().ctgb_contract_pair(words.ctypes.data, a.data_ptr(), a.data_ptr(), c.data_ptr(), 0))
    torch.cuda.synchronize()
    assert not bool(c.abs().any())


# ---------------------------------------------------------------------------- many slices
NB = 14  # sliced bonds: 2^14 slices
BONDS = [f"b{i}" for i in range(NB)]


def _tree(kind):
    """A[bonds, i] M[i, j, o] B[bonds, j] (-> [o]) with every bond sliced: "closed" sums everything,
    "open" keeps o, "sliced_out" also keeps (and slices) the first bond."""
    sizes = {b: 2 for b in BONDS}
    sizes.update(i=8, j=8, o=1 if kind == "closed" else 8)
    out = {"closed": (), "open": ("o",), "sliced_out": (BONDS[0], "o")}[kind]
    m_term = ("i", "j") if kind == "closed" else ("i", "j", "o")
    sizes = {k: v for k, v in sizes.items() if k != "o" or kind != "closed"}
    inputs = [tuple(BONDS) + ("i",), m_term, tuple(BONDS) + ("j",)]
    return cb.TreeSpec(inputs, out, sizes, [(0, 1), (3, 2)], [(b, 2, None) for b in BONDS])


def _same_sign_inputs(spec, scale=1.0):
    rng = np.random.default_rng(11)
    arrays = []
    for shp in spec.shapes():
        re = rng.uniform(0.5, 1.0, size=shp)
        im = 0.25 * rng.uniform(0.5, 1.0, size=shp)
        arrays.append(((re + 1j * im) * scale).astype(np.complex64))
    return arrays


def _per_slice_values(spec, arrays, kind):
    """complex128 value of every slice, in slice order, from numpy."""
    a, m, b = (np.asarray(x, dtype=np.complex128) for x in arrays)
    n = 1 << NB
    a, b = a.reshape(n, -1), b.reshape(n, -1)
    if kind == "closed":
        return np.einsum("si,ij,sj->s", a, m, b)
    return np.einsum("si,ijo,sj->so", a, m, b)


def _sequential_fp32_sum(vals):
    """The running complex64 sum of the slices' (rounded) values, as the native root forms it."""
    return np.cumsum(vals.astype(np.complex64), axis=0, dtype=np.complex64)[-1]


@pytest.mark.parametrize("kind", ["closed", "open", "sliced_out"])
def test_many_slices(kind):
    torch = _torch()
    spec = _tree(kind)
    assert spec.nslices == 1 << NB
    arrays = _same_sign_inputs(spec)
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    truth = cb.TreeExecutor(spec, dtype="complex128").contract_device([t.to(torch.complex128) for t in dev])
    native = cb.TreeExecutor(spec, dtype="complex64").contract_device(dev)
    ex = cb.TreeExecutor(spec, dtype="complex64", accumulate="double")
    wide = ex.contract_device(dev)
    torch.cuda.synchronize()
    assert wide.dtype == torch.complex128 and native.dtype == torch.complex64
    # (a non-dot root: its slices are folded by one extra launch each)
    assert not ex.plan.root_direct
    assert ex.plan.launches_per_slice() == cb.TreeExecutor(spec, dtype="complex64").plan.launches_per_slice() + 1
    truth, native, wide = (t.cpu().numpy() for t in (truth, native, wide))
    e_wide, e_native = rel_err(wide, truth), rel_err(native, truth)
    assert e_wide < 2e-6, e_wide
    assert e_wide * 10 < e_native, (e_wide, e_native)
    if kind != "sliced_out":
        # the numpy model of the sequential fp32 sum reproduces the native error's size
        vals = _per_slice_values(spec, arrays, kind)
        assert rel_err(vals.sum(axis=0).reshape(truth.shape), truth) < 1e-12
        e_model = rel_err(_sequential_fp32_sum(vals).reshape(truth.shape), truth)
        assert 0.1 < e_native / e_model < 10, (e_native, e_model)
    # no slices: the zeroed wide output
    none = ex.contract_device(dev, count=0)
    assert none.dtype == torch.complex128 and not bool(none.abs().any())


def test_many_slices_stripped():
    torch = _torch()
    spec = _tree("closed")
    arrays = _same_sign_inputs(spec, scale=1e-15)  # the complex64 amplitude (~1e-45 * 2^14 * 64) underflows
    dev = [torch.from_numpy(a).cuda() for a in arrays]
    plain = cb.TreeExecutor(spec, dtype="complex64").contract_device(dev)
    assert float(plain.abs().max()) < 1e-38  # denormal or zero: unusable
    mt, et = cb.TreeExecutor(spec, dtype="complex128", strip_exponent=True).contract_device(
        [t.to(torch.complex128) for t in dev])
    mn, en = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True).contract_device(dev)
    mw, ew = cb.TreeExecutor(spec, dtype="complex64", strip_exponent=True, accumulate="double").contract_device(dev)
    torch.cuda.synchronize()
    assert mw.dtype == torch.complex128 and mn.dtype == torch.complex64
    truth = mt.cpu().numpy()

    def err(m, e):
        return rel_err(m.cpu().numpy().astype(np.complex128) * 10.0 ** (float(e.item()) - float(et.item())), truth)

    assert err(mw, ew) < 2e-6, err(mw, ew)
    assert err(mw, ew) * 10 < err(mn, en), (err(mw, ew), err(mn, en))


# ---------------------------------------------------------------------------- entry points
NB_SMALL = 6


def _small(kind="sliced_out"):
    sizes = {f"b{i}": 2 for i in range(NB_SMALL)}
    sizes.update(i=8, j=8, o=8)
    bonds = [f"b{i}" for i in range(NB_SMALL)]
    out = (bonds[0], "o") if kind == "sliced_out" else ("o",)
    spec = cb.TreeSpec([tuple(bonds) + ("i",), ("i", "j", "o"), tuple(bonds) + ("j",)], out, sizes,
                       [(0, 1), (3, 2)], [(b, 2, None) for b in bonds])
    return spec, _same_sign_inputs(spec)


def test_entry_points_return_the_wide_result(tmp_path):
    torch = _torch()
    spec, arrays = _small()
    ex = cb.TreeExecutor(spec, dtype="complex64", accumulate="double")
    want = ex.contract_device([torch.from_numpy(a).cuda() for a in arrays]).cpu().numpy()
    assert want.dtype == np.complex128
    tol = 1e-12 * np.abs(want).max()

    def same(x):
        x = np.asarray(x)
        return x.dtype == np.complex128 and x.shape == want.shape and np.abs(x - want).max() <= tol

    assert same(cb.contract_tree(spec, arrays, accumulate="double"))
    assert same(cb.contract_tree(spec, [torch.from_numpy(a).cuda() for a in arrays], accumulate="double").cpu())
    chunks = list(cb.gen_output_chunks(spec, arrays, accumulate="double"))
    assert len(chunks) == 2 and same(np.stack(chunks))
    # checkpointed: interrupted after two blocks, resumed, and refused by the other mode
    ck = str(tmp_path / "wide.npz")

    class Stop(Exception):
        pass

    def stop(done, _n):
        if done >= 32:
            raise Stop

    with pytest.raises(Stop):
        cb.contract_checkpointed(spec, arrays, ck, every=16, accumulate="double", on_block=stop)
    with pytest.raises(ValueError):
        cb.contract_checkpointed(spec, arrays, ck, every=16)
    seen = []
    got = cb.contract_checkpointed(spec, arrays, ck, every=16, accumulate="double",
                                   on_block=lambda d, n: seen.append(d))
    assert seen == [48, 64] and same(got)
    # the per-slice contractor (make_contractor / install): wide slices, summed by the caller
    fn = cb.make_contractor(spec, accumulate="double")
    from oracle import ctg_oracle as orc

    total = np.zeros(want.shape, dtype=np.complex128)
    for i in range(spec.nslices):
        one = fn(*orc.slice_arrays(spec.inputs, spec.sliced, arrays, i))
        assert one.dtype == np.complex128
        total[i // (spec.nslices // 2)] += one
    assert np.abs(total - want).max() <= 1e-6 * np.abs(want).max()
    # float64 / complex128: "double" is "native", bit for bit
    a128 = [a.astype(np.complex128) for a in arrays]
    assert np.array_equal(cb.contract_tree(spec, a128, accumulate="double"), cb.contract_tree(spec, a128))


@pytest.mark.reference
def test_installed_tree_contracts_wide():
    import os
    import sys

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    sys.path[:0] = [os.path.join(root, "oracle", "refshim"), os.path.join(root, "oracle", "_ref")]
    try:
        import cotengra as ctg

        spec, arrays = _small("open")
        tree = ctg.ContractionTree.from_path(spec.inputs, spec.output, spec.size_dict, path=[(0, 1), (0, 1)])
        for b, _s, _p in spec.sliced:
            tree.remove_ind_(b)
        cb.install(tree, accumulate="double")
        got = tree.contract(arrays)
        want = cb.contract_tree(spec, arrays, accumulate="double")
        assert np.asarray(got).dtype == np.complex128
        assert rel_err(got, want) < 1e-6
    finally:
        del sys.path[:2]


def test_gradients_through_a_wide_result():
    torch = _torch()
    spec, arrays = _small("open")
    grads = {}
    for mode in ("native", "double"):
        ts = [torch.from_numpy(a).cuda().requires_grad_(True) for a in arrays]
        out = cb.contract_tree(spec, ts, accumulate=mode)
        assert out.dtype == (torch.complex128 if mode == "double" else torch.complex64)
        (out.abs() ** 2).sum().backward()
        assert all(t.grad.dtype == torch.complex64 for t in ts)
        grads[mode] = [t.grad.cpu().numpy() for t in ts]
    for g0, g1 in zip(grads["native"], grads["double"]):
        assert rel_err(g1, g0) < 1e-5


@pytest.mark.multigpu
def test_contract_distributed_wide():
    import os
    import socket
    import subprocess
    import sys

    torch = _torch()
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    s = socket.socket()
    s.bind(("127.0.0.1", 0))
    port = s.getsockname()[1]
    s.close()
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2",
           "--master-addr", "127.0.0.1", "--master-port", str(port),
           os.path.join(root, "scripts", "gpu_dist_accumulate_check.py")]
    res = subprocess.run(cmd, cwd=root, capture_output=True, text=True, timeout=600)
    assert res.returncode == 0 and "DIST_ACCUMULATE PASS" in res.stdout, res.stdout[-2000:] + res.stderr[-2000:]
