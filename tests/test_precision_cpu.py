"""The ``precision`` option ("3xtf32", the default, or "tf32": one round-to-nearest tf32 pass) on the
host: descriptors, plans, refusals, the checkpoint tag and the public interface, without a GPU.

With the default every descriptor is word for word what it is without the keyword; with "tf32" the
descriptors differ from the default ones only in flags bit7, set exactly on the float32 / complex64
tensor-core variants (``lowering.TF32_VARIANTS``)."""

import hashlib
import json
import os

import numpy as np
import pytest

import cotengra_b200 as cb
from cotengra_b200 import lowering as L
from tests import emu_device
from tests.helpers import GOLDEN_DIR, load_json, make_arrays, tree_spec

TREES = load_json("trees.json")
M20 = load_json("sycamore_m20.json")
SINGLE = ("float32", "complex64")
BIT = L.FLAG_TF32_ONE_PASS


def _golden_specs():
    out = [(r["name"], tree_spec(r)) for r in TREES + M20]
    with open(os.path.join(GOLDEN_DIR, "circuits.json")) as f:
        for name, rec in json.load(f).items():
            out.append((f"circuit_{name}", cb.TreeSpec.from_dict(rec["spec"])))
    return out


SPECS = _golden_specs()


def _plan(spec, dtype, **kw):
    return cb.ExecPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype,
                       sm_count=132, **kw)


def _pair_words(plan):
    return [(nd["words"], int(nd["words"][L.W_VARIANT])) for nd in plan.nodes if nd["kind"] == 0]


def _check_tf32_words(base, tf32):
    """tf32 words equal the default ones but for bit7, set exactly on the tensor-core variants;
    returns how many nodes carry it."""
    assert len(base) == len(tf32)
    marked = 0
    for (w0, v0), (w1, v1) in zip(base, tf32):
        assert v0 == v1
        on = v0 in L.TF32_VARIANTS
        assert int(w1[L.W_FLAGS]) == int(w0[L.W_FLAGS]) | (BIT if on else 0)
        assert not int(w0[L.W_FLAGS]) & BIT
        rest = np.ones(L.DESC_WORDS, dtype=bool)
        rest[L.W_FLAGS] = False
        assert np.array_equal(w0[rest], w1[rest])
        marked += on
    return marked


@pytest.mark.parametrize("name,spec", SPECS, ids=[n for n, _ in SPECS])
def test_golden_tree_descriptors(name, spec):
    marked = 0
    for dtype in ("complex64", "complex128"):
        base = _pair_words(_plan(spec, dtype))
        same = _pair_words(_plan(spec, dtype, precision="3xtf32"))
        assert all(np.array_equal(a, b) for (a, _), (b, _) in zip(base, same))
        if dtype == "complex64":
            marked += _check_tf32_words(base, _pair_words(_plan(spec, dtype, precision="tf32")))
    if name.startswith("sycamore_m20") or name.startswith("circuit_"):
        assert marked > 0  # these trees have tensor-core nodes: the mode reaches them


def test_float32_descriptors():
    for rec in TREES[:40]:
        spec = tree_spec(rec)
        base = _pair_words(_plan(spec, "float32"))
        _check_tf32_words(base, _pair_words(_plan(spec, "float32", precision="tf32")))


def test_every_tensor_core_variant_takes_the_bit():
    dims = L.classify_pair("ab", (1024, 256), "bc", (256, 128), "ac")
    for dtype in SINGLE:
        for v in L.TF32_VARIANTS:
            if v in L.TC05_VARIANTS and dtype != "complex64":
                continue
            p0 = L.build_pair_desc(dims, dtype, variant=v, force_splitk=1)
            p1 = L.build_pair_desc(dims, dtype, variant=v, force_splitk=1, precision="tf32")
            assert p1.variant == v and int(p1.words[L.W_FLAGS]) == int(p0.words[L.W_FLAGS]) | BIT
        for v in (L.VAR_SIMT_64x64, L.VAR_KRED, L.VAR_ROW_128x8, L.VAR_ROW_256x4):
            p0 = L.build_pair_desc(dims, dtype, variant=v, force_splitk=1)
            p1 = L.build_pair_desc(dims, dtype, variant=v, force_splitk=1, precision="tf32")
            assert np.array_equal(p0.words, p1.words)
    # a wgmma pick that falls back to the mma.sync tiles keeps the bit there
    thin = L.classify_pair("ab", (1296, 216), "bc", (216, 13), "ac")
    p = L.build_pair_desc(thin, "complex64", variant=L.VAR_TC05_128x16, precision="tf32")
    assert p.variant in L.TF32_VARIANTS and int(p.words[L.W_FLAGS]) & BIT


def test_bad_values_and_double_dtypes_raise():
    spec = tree_spec(next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced"))
    dims = L.classify_pair("ab", (256, 64), "bc", (64, 64), "ac")
    for bad in ("fp16", "TF32", "", None, 3):
        with pytest.raises(ValueError):
            L.build_pair_desc(dims, "complex64", precision=bad)
        with pytest.raises(ValueError):
            _plan(spec, "complex64", precision=bad)
    for dtype in ("float64", "complex128"):
        with pytest.raises(ValueError):
            L.build_pair_desc(dims, dtype, precision="tf32")
        with pytest.raises(ValueError):
            _plan(spec, dtype, precision="tf32")
        with pytest.raises(ValueError):
            cb.VjpPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype,
                       sm_count=132, precision="tf32")
    with pytest.raises(ValueError):
        cb.implementation(precision="bf16")
    with pytest.raises(ValueError):
        cb.B200Contractor(spec.contractions(), precision="half")


def _vjp(spec, dtype, **kw):
    return cb.VjpPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype,
                      sm_count=132, **kw)


@pytest.mark.parametrize("name", ["lattice6x6_d3_sliced", "peps8x8_d2", "lattice4x4_sliced"])
def test_vjp_plans_carry_the_bit(name):
    spec = tree_spec(next(r for r in TREES if r["name"] == name))
    base, tf32 = _vjp(spec, "complex64"), _vjp(spec, "complex64", precision="tf32")
    pair = lambda p: [(nd["words"], int(nd["words"][L.W_VARIANT])) for nd in p.nodes if nd["kind"] == 0]  # noqa: E731
    _check_tf32_words(pair(base), pair(tf32))
    assert [nd["phase"] for nd in base.nodes] == [nd["phase"] for nd in tf32.nodes]
    # phase-2 recomputations under the smallest budget are copies of tf32 forward records
    small0 = _vjp(spec, "complex64", max_bytes=base.min_bytes)
    small1 = _vjp(spec, "complex64", max_bytes=base.min_bytes, precision="tf32")
    assert small0.recompute_macs == small1.recompute_macs
    _check_tf32_words(pair(small0), pair(small1))


def test_tree_executor_plans_carry_the_bit(monkeypatch):
    emu_device.install(monkeypatch)
    rec = next(r for r in TREES if r["name"] == "rand_r2_o0_hi0_ho1_None_s666_sliced_out")
    spec = tree_spec(rec)
    ex0 = cb.TreeExecutor(spec, dtype="complex64", fuse=False)
    ex1 = cb.TreeExecutor(spec, dtype="complex64", fuse=False, precision="tf32")
    assert ex0.precision == "3xtf32" and ex1.precision == "tf32"
    for p0, p1 in ((ex0.plan, ex1.plan), (ex0._chunk_plan(), ex1._chunk_plan()), (ex0.vjp_plan(), ex1.vjp_plan())):
        assert p1.precision == "tf32"
        _check_tf32_words(_pair_words(p0), _pair_words(p1))
    with pytest.raises(ValueError):
        cb.TreeExecutor(spec, dtype="complex128", precision="tf32")
    # results through the emulated launch are the same (the emulator computes in wide precision)
    arrays = make_arrays(spec.shapes(), "complex64", seed=rec["seed"])
    a = cb.contract_tree(spec, arrays, dtype="complex64", fuse=False)
    b = cb.contract_tree(spec, arrays, dtype="complex64", fuse=False, precision="tf32")
    assert np.allclose(a, b)
    # gen_output_chunks and contract_distributed (one gloo rank) hand the mode to the plans they launch
    import torch.distributed as dist

    seen = []
    launch = cb.ExecPlan.execute  # (the emulated launch)

    def spy(self, *args, **kw):
        seen.append(self.precision)
        return launch(self, *args, **kw)

    monkeypatch.setattr(cb.ExecPlan, "execute", spy)
    want = list(ex0.gen_output_chunks(arrays))
    for prec in ("3xtf32", "tf32"):
        seen.clear()
        got = list(cb.gen_output_chunks(spec, arrays, dtype="complex64", fuse=False, precision=prec))
        assert len(seen) == len(got) == len(want) and set(seen) == {prec}
        assert all(np.allclose(g, w) for g, w in zip(got, want))
        seen.clear()
        dist.init_process_group("gloo", rank=0, world_size=1, store=dist.HashStore())
        try:
            got = cb.contract_distributed(spec, arrays, dtype="complex64", fuse=False, precision=prec)
        finally:
            dist.destroy_process_group()
        assert seen == [prec] and np.allclose(got, a)


def _tag(spec, dtype, strip, arrays, extra=b""):
    # the checkpoint tag as the default mode has always written it
    h = hashlib.sha256()
    h.update(spec.to_json().encode())
    h.update(f"|{dtype}|{int(bool(strip))}|".encode())
    h.update(extra)
    for a in arrays:
        h.update(str(a.shape).encode())
        h.update(np.asarray(a, dtype=dtype, order="C").tobytes())
    return h.hexdigest()


def test_checkpoint_tag(monkeypatch, tmp_path):
    emu_device.install(monkeypatch)
    rec = next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex64", seed=rec["seed"])
    ck = str(tmp_path / "run.npz")
    want = cb.contract_checkpointed(spec, arrays, ck, every=4, dtype="complex64")
    with np.load(ck) as z:
        assert str(z["tag"]) == _tag(spec, "complex64", False, arrays)  # unchanged by default
    with pytest.raises(ValueError):  # a default-mode file is not resumed in tf32 mode
        cb.contract_checkpointed(spec, arrays, ck, every=4, dtype="complex64", precision="tf32")
    ck1 = str(tmp_path / "run_tf32.npz")
    got = cb.contract_checkpointed(spec, arrays, ck1, every=4, dtype="complex64", precision="tf32")
    with np.load(ck1) as z:
        tag1 = str(z["tag"])
    assert tag1 != _tag(spec, "complex64", False, arrays)
    assert tag1 == _tag(spec, "complex64", False, arrays, b"precision=tf32|")
    with pytest.raises(ValueError):  # ... nor a tf32 file in the default mode
        cb.contract_checkpointed(spec, arrays, ck1, every=4, dtype="complex64")
    assert np.allclose(got, want)


def test_implementation_routes_precision(monkeypatch):
    lib = emu_device.install(monkeypatch)
    seen = []
    orig = type(lib).ctgb_contract_pair

    def spy(self, words_ptr, pa, pb, pc, stream):
        W = emu_device._view(words_ptr, np.int64, L.DESC_WORDS)
        seen.append((int(W[L.W_VARIANT]), int(W[L.W_FLAGS])))
        return orig(self, words_ptr, pa, pb, pc, stream)

    monkeypatch.setattr(type(lib), "ctgb_contract_pair", spy)
    rng = np.random.default_rng(3)
    a = (rng.standard_normal((256, 64)) + 1j * rng.standard_normal((256, 64))).astype(np.complex64)
    b = (rng.standard_normal((64, 64)) + 1j * rng.standard_normal((64, 64))).astype(np.complex64)
    assert cb.implementation() == (cb.einsum, cb.tensordot)
    ein, tdot = cb.implementation(precision="tf32")
    want = a.astype(np.complex128) @ b.astype(np.complex128)
    for fn, args in ((ein, ("ab,bc->ac", a, b)), (tdot, (a, b, 1))):
        got = fn(*args)
        assert np.allclose(got, want, rtol=1e-4, atol=1e-4)
        v, flags = seen[-1]
        assert v in L.TC05_VARIANTS and flags & BIT
    cb.einsum("ab,bc->ac", a, b)
    assert not seen[-1][1] & BIT
    with pytest.raises(ValueError):
        ein("ab,bc->ac", a.astype(np.complex128), b.astype(np.complex128))
    with pytest.raises(ValueError):
        cb.einsum("ab->a", a.astype(np.complex128), precision="tf32")
    # the whole-tree drop-in: make_contractor / install route it to every plan they build
    spec = tree_spec(next(r for r in TREES if r["name"] == "lattice6x6_d3_sliced"))
    con = cb.make_contractor(spec, precision="tf32")
    assert con.precision == "tf32"
    arrays = [np.ones(s, dtype=np.complex64) for s in spec.sliced_shapes()]
    con(*arrays)
    (ex,) = con._plans.values()
    assert ex.plan.precision == "tf32"
    with pytest.raises(ValueError):
        con(*[x.astype(np.complex128) for x in arrays])


def test_kernel_cases_tell_the_modes_apart():
    """Each tf32 kernel case's model of one pass differs from the exact einsum by more than twice
    the per-element bound the GPU test holds the kernel to: a three-pass kernel would fail it."""
    import zlib

    from tests import kernel_cases as KC
    from tests import precision_cases as PC

    assert len(PC.CASES) > 200
    assert {PC.build_plan(c, "tf32").variant for c in PC.CASES} == set(L.TF32_VARIANTS)
    for c in PC.CASES:
        lay = KC.make_layout(c, seed=zlib.crc32(c.id.encode()))
        exact, scale = KC.reference(c, lay)
        model, _ = PC.tf32_reference(c, lay)
        assert KC.error_ratio(model.astype(exact.dtype), exact, scale) > 2 * KC.C_SINGLE, c.id


def _tc05_expected(words, NT, one, sms, smem_optin):
    """B' residency, B' slots and A staging depth as tc05_launch_config derives them, for the one-pass
    kernel (half-size B' k-steps, no A'lo images) or the default one."""
    images = 1 if one else 2
    op_bytes = 8 * (128 * 16 + 64)
    fixed = 2 * images * op_bytes + 8 * (128 + NT + 1024 + 8 + 2 * 8 + 4) + 128
    pair = images * 8 * (2 * NT) * 4 * 4
    pool = smem_optin - 1024 - fixed
    steps, tiles_n = int(words[L.W_STEPS_K]), int(words[L.W_TILES_N])
    b_stat = (int(words[L.W_TILES_B]) == 1 and int(words[L.W_SPLITK]) == 1 and steps <= 8 and tiles_n <= sms
              and pool - steps * pair >= 3 * 128 * 16 * 8)
    nb = steps if b_stat else 3
    return int(b_stat), nb, min(8, (pool - nb * pair) // (128 * 16 * 8))


def test_one_pass_wgmma_launch_config():
    """The one-pass wgmma launch sizes its B' ring (or keeps B' resident) from the halved image and
    frees the A'lo images; chunking and A staging choices do not change."""
    from cotengra_b200 import _lib
    from tests import kernel_cases as KC
    from tests import precision_cases as PC

    wider = 0
    for c in PC.CASES:
        p0, p1 = KC.build_plan(c), PC.build_plan(c, "tf32")
        if p1.variant not in L.TC05_VARIANTS:
            continue
        NT = L.VARIANT_TILES[p1.variant][1]
        for sms in KC.H100_SMS:
            addr = KC.a_operand_addr(c, p1, 1 << 20)
            f0 = _lib.tc05_launch_config(p0.words, addr, sms, KC.H100_SMEM_OPTIN)
            f1 = _lib.tc05_launch_config(p1.words, addr, sms, KC.H100_SMEM_OPTIN)
            for k in ("tm_rank", "bulk", "chunk_steps", "chunks"):
                assert f0[k] == f1[k], (c.id, k)
            assert (f0["b_stat"], f0["nb"], f0["sa"]) == _tc05_expected(p0.words, NT, False, sms, KC.H100_SMEM_OPTIN)
            assert (f1["b_stat"], f1["nb"], f1["sa"]) == _tc05_expected(p1.words, NT, True, sms, KC.H100_SMEM_OPTIN)
            assert f1["smem"] < f0["smem"] or f1["sa"] > f0["sa"] or f1["b_stat"] > f0["b_stat"]
            assert f1["b_stat"] >= f0["b_stat"]
            wider += f1["b_stat"] > f0["b_stat"]
    assert wider > 0  # some B' images only stay resident at half size (ring_past_fit for N tiles 64 and 32)
