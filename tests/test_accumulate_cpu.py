"""``accumulate="double"`` on the host side: default plans are unchanged word for word, the wide-C
flag sits on exactly the dot-stream roots, every other root gets a dense workspace slot and the chunk
descriptor, and the emulated launch of wide plans matches the oracle in double precision."""

import hashlib
import json
import os

import numpy as np
import pytest

import cotengra_b200 as cb
from cotengra_b200 import _lib, executor as X, lowering as L
from oracle import ctg_oracle as orc
from tests import emu_accumulate
from tests.emu_accumulate import emulate_plan
from tests.helpers import GOLDEN_DIR, decode_ir, decode_sliced, load_json, make_arrays, rel_err, tree_spec

TREES = load_json("trees.json")
M20 = load_json("sycamore_m20.json")
SPECS = [(r["name"], tree_spec(r)) for r in TREES + M20]
BIT = L.FLAG_WIDE_C
WIDE = {"float32": "float64", "complex64": "complex128"}


def _plan(spec, dtype, **kw):
    return cb.ExecPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=dtype,
                       sm_count=132, **kw)


def _same_plan(p, q):
    assert len(p.nodes) == len(q.nodes) and len(p.tensors) == len(q.tensors)
    for a, b in zip(p.nodes, q.nodes):
        assert np.array_equal(a["words"], b["words"]) and a["phase"] == b["phase"] and a["kind"] == b["kind"]
    for a, b in zip(p.tensors, q.tensors):
        assert (a.kind, a.offset, a.nbytes, a.strides) == (b.kind, b.offset, b.nbytes, b.strides)
    assert (p.workspace_bytes, p.persistent_bytes, p.acc_dtype) == (q.workspace_bytes, q.persistent_bytes, q.acc_dtype)
    assert (p._chunk_words is None) == (q._chunk_words is None)


def _rec(name):
    return next(r for r in TREES if r["name"] == name)


def _oracle(rec, arrays, **kw):
    """The tree in double precision on the (single-precision) values of ``arrays``."""
    wide = [np.asarray(a, dtype=WIDE[str(a.dtype)]) for a in arrays]
    return orc.contract_tree([tuple(t) for t in rec["inputs"]], tuple(rec["output"]), decode_sliced(rec["sliced"]),
                             decode_ir(rec["contractions"]), wide, **kw)


@pytest.mark.parametrize("name,spec", SPECS, ids=[n for n, _ in SPECS])
def test_golden_tree_plans(name, spec):
    for dtype in ("complex64", "complex128"):
        for strip in (False, True):
            base = _plan(spec, dtype, strip_exponent=strip)
            assert base.acc_dtype == dtype and not base.wide
            _same_plan(base, _plan(spec, dtype, strip_exponent=strip, accumulate="native"))
            assert not any(int(nd["words"][L.W_FLAGS]) & BIT for nd in base.nodes if nd["kind"] == 0)
            wide = _plan(spec, dtype, strip_exponent=strip, accumulate="double")
            if dtype == "complex128":
                _same_plan(base, wide)  # "double" on a double dtype is "native"
                continue
            assert wide.acc_dtype == "complex128" and wide.wide
            # every node but the root is the native one
            for a, b in zip(base.nodes[:-1], wide.nodes[:-1]):
                assert np.array_equal(a["words"], b["words"])
            root, root0 = wide.nodes[-1], base.nodes[-1]
            dot = (root["kind"] == 0 and not strip
                   and int(root0["words"][L.W_VARIANT]) in L.DOTSTREAM_VARIANTS)
            flagged = [nd for nd in wide.nodes if nd["kind"] == 0 and int(nd["words"][L.W_FLAGS]) & BIT]
            assert flagged == ([root] if dot else [])
            if dot:
                # the native root but for the bit: it adds into the (wide) output itself
                rest = np.ones(L.DESC_WORDS, dtype=bool)
                rest[L.W_FLAGS] = False
                assert np.array_equal(root["words"][rest], root0["words"][rest])
                assert int(root["words"][L.W_FLAGS]) == int(root0["words"][L.W_FLAGS]) | BIT
                assert root["c"].kind == X.K_OUTPUT and wide._chunk_words is None and wide.root_direct
            else:
                # a dense slot of the plan dtype in the per-slice workspace, and the chunk descriptor
                assert root["c"].kind == X.K_SCRATCH and not wide.root_direct
                assert root["c"].nbytes == max(int(np.prod(wide.root_shape)), 1) * 8
                assert root["c"].strides == L.row_major_strides(wide.root_shape)
                flags = int(root["words"][L.W_FLAGS if root["kind"] == 0 else L.S_FLAGS])
                assert not flags & 1  # stored, not accumulated
                assert wide._chunk_words is not None and int(wide._chunk_words[L.S_MAGIC]) == L.SDESC_MAGIC
                assert int(wide._chunk_words[L.S_OUT_ELEMS]) == int(np.prod([d for d in wide.root_shape if d != 1]))
            if strip:
                _same_plan_nodes = [np.array_equal(a["words"], b["words"]) for a, b in zip(base.nodes, wide.nodes)]
                assert all(_same_plan_nodes)  # a stripped plan only widens the running mantissa
    if name in ("sycamore_m20_appxB", "sycamore_m20_medium"):
        wide = _plan(spec, "complex64", accumulate="double")
        assert int(wide.nodes[-1]["words"][L.W_FLAGS]) & BIT  # the amplitude's final inner product


def test_circuit_plans_unchanged():
    with open(os.path.join(GOLDEN_DIR, "circuits.json")) as f:
        recs = json.load(f)
    for rec in list(recs.values())[:4]:
        spec = cb.TreeSpec.from_dict(rec["spec"])
        _same_plan(_plan(spec, "complex64"), _plan(spec, "complex64", accumulate="native"))


def _dot_dims(M, N, K, dtype="complex64"):
    ta = ("k",) + (("m",) if M > 1 else ())
    tb = ("k",) + (("n",) if N > 1 else ())
    out = tuple(x for x, e in (("m", M), ("n", N)) if e > 1)
    sa = (K,) + ((M,) if M > 1 else ())
    sb = (K,) + ((N,) if N > 1 else ())
    return L.classify_pair(ta, sa, tb, sb, out)


def test_build_pair_desc_takes_the_flag_on_dot_streams_only():
    for M, N, var in ((1, 1, L.VAR_DOTSTREAM), (4, 3, L.VAR_DOTSTREAM4)):
        dims = _dot_dims(M, N, 1 << 20)
        for dtype in ("float32", "complex64"):
            w0 = L.build_pair_desc(dims, dtype, accumulate=True)
            w1 = L.build_pair_desc(dims, dtype, accumulate=True, wide_c=True)
            assert w0.variant == w1.variant == var
            assert int(w1.words[L.W_FLAGS]) == int(w0.words[L.W_FLAGS]) | BIT
        for dtype in ("float64", "complex128"):
            with pytest.raises(ValueError):
                L.build_pair_desc(dims, dtype, accumulate=True, wide_c=True)
    # any other variant refuses it: chosen (a short contracted range), forced, or reached by a fallback
    with pytest.raises(ValueError):
        L.build_pair_desc(_dot_dims(1, 1, 1 << 14), "complex64", accumulate=True, wide_c=True)
    with pytest.raises(ValueError):
        L.build_pair_desc(_dot_dims(64, 64, 64), "complex64", accumulate=True, wide_c=True)
    for var in (L.VAR_KRED, L.VAR_SIMT_64x64, L.VAR_TF32_32x32):
        with pytest.raises(ValueError):
            L.build_pair_desc(_dot_dims(1, 1, 1 << 20), "complex64", accumulate=True, variant=var, wide_c=True)
    with pytest.raises(ValueError):  # 5 > 4 kept columns: DOTSTREAM4 falls back
        L.build_pair_desc(_dot_dims(5, 2, 1 << 20), "complex64", accumulate=True, variant=L.VAR_DOTSTREAM4,
                          wide_c=True)


def test_bad_values_raise():
    spec = tree_spec(_rec("lattice6x6_d3_sliced"))
    for bad in ("float64", "wide", None, True, ""):
        with pytest.raises(ValueError):
            _plan(spec, "complex64", accumulate=bad)
        with pytest.raises(ValueError):
            cb.TreeExecutor(spec, dtype="complex64", accumulate=bad)
        with pytest.raises(ValueError):
            cb.B200Contractor(spec.contractions(), accumulate=bad)
        with pytest.raises(ValueError):
            L.accumulator_dtype("complex64", bad)
    assert L.accumulator_dtype("float32", "double") == "float64"
    assert L.accumulator_dtype("complex128", "double") == "complex128"
    assert L.accumulator_dtype("complex64", "native") == "complex64"


def test_entry_point_is_exported():
    assert "ctgb_plan_set_accumulator" in _lib.EXPORTS
    assert hasattr(_lib.load(), "ctgb_plan_set_accumulator")


@pytest.mark.parametrize("name", ["lattice6x6_d3_sliced", "rand_r2_o0_hi0_ho1_None_s666_sliced_out"])
@pytest.mark.parametrize("dtype", ["float32", "complex64"])
def test_emulated_wide_plans_match_the_oracle(name, dtype):
    rec = _rec(name)
    if dtype == "float32" and rec["dtype"].startswith("complex"):
        pytest.skip("complex tree")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), dtype, seed=rec["seed"])
    want = _oracle(rec, arrays)
    plan = _plan(spec, dtype, accumulate="double")
    got = emulate_plan(plan, arrays)
    assert got.dtype == np.dtype(WIDE[dtype]) and got.shape == want.shape
    # (the emulation holds every value of a wide plan in the accumulator dtype: tests/emu_accumulate.py)
    assert rel_err(got, want) < 1e-10
    # zero slices: the zeroed wide output
    none = emulate_plan(plan, arrays, slice_ids=[])
    assert none.dtype == got.dtype and not np.any(none)
    # stripped: the running mantissa is wide
    m, e = emulate_plan(_plan(spec, dtype, accumulate="double", strip_exponent=True), arrays)
    assert m.dtype == got.dtype and rel_err(m * 10.0 ** e, want) < 1e-10


def test_emulated_dot_stream_root_sums_in_double():
    """A sliced inner product of 2^20 same-sign terms per slice: the flagged root adds exact double
    products into the wide output, so the emulated plan equals the double dot product to rounding."""
    K, S = 1 << 20, 4
    spec = cb.TreeSpec([("s", "k"), ("s", "k")], (), {"s": S, "k": K}, [(0, 1)], [("s", S, None)])
    rng = np.random.default_rng(5)
    arrays = [rng.uniform(0.5, 1.0, (S, K)).astype(np.float32) for _ in range(2)]
    plan = _plan(spec, "float32", accumulate="double")
    root = plan.nodes[-1]
    assert int(root["words"][L.W_VARIANT]) == L.VAR_DOTSTREAM and int(root["words"][L.W_FLAGS]) & BIT
    assert root["c"].kind == X.K_OUTPUT and plan._chunk_words is None
    got = emulate_plan(plan, arrays)
    want = np.dot(arrays[0].astype(np.float64).ravel(), arrays[1].astype(np.float64).ravel())
    assert got.dtype == np.float64 and abs(got - want) < 1e-12 * want
    native = emulate_plan(_plan(spec, "float32"), arrays)
    assert native.dtype == np.float32 and abs(native - want) > 1e-9 * want  # the bound tells the two apart


def _tag(spec, dtype, strip, arrays, extra=b""):
    # the checkpoint tag as the native mode has always written it
    h = hashlib.sha256()
    h.update(spec.to_json().encode())
    h.update(f"|{dtype}|{int(bool(strip))}|".encode())
    h.update(extra)
    for a in arrays:
        h.update(str(a.shape).encode())
        h.update(np.asarray(a, dtype=dtype, order="C").tobytes())
    return h.hexdigest()


def test_checkpoint_tag_and_entry_points(monkeypatch, tmp_path):
    emu_accumulate.install(monkeypatch)
    rec = _rec("lattice6x6_d3_sliced")
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex64", seed=rec["seed"])
    ck = str(tmp_path / "native.npz")
    native = cb.contract_checkpointed(spec, arrays, ck, every=4, dtype="complex64")
    assert native.dtype == np.complex64
    with np.load(ck) as z:
        assert str(z["tag"]) == _tag(spec, "complex64", False, arrays)  # unchanged
    with pytest.raises(ValueError):  # a native file is not resumed by a wide run
        cb.contract_checkpointed(spec, arrays, ck, every=4, dtype="complex64", accumulate="double")
    ck1 = str(tmp_path / "wide.npz")
    wide = cb.contract_checkpointed(spec, arrays, ck1, every=4, dtype="complex64", accumulate="double")
    with np.load(ck1) as z:
        assert str(z["tag"]) == _tag(spec, "complex64", False, arrays, b"accumulate=complex128|")
        assert z["partial"].dtype == np.complex128
    with pytest.raises(ValueError):  # ... nor a wide file by a native one
        cb.contract_checkpointed(spec, arrays, ck1, every=4, dtype="complex64")
    assert wide.dtype == np.complex128 and rel_err(wide, _oracle(rec, arrays)) < 1e-10
    # complex128: "double" is "native", tag included
    a128 = make_arrays(spec.shapes(), "complex128", seed=rec["seed"])
    ck2 = str(tmp_path / "c128.npz")
    cb.contract_checkpointed(spec, a128, ck2, every=4, dtype="complex128", accumulate="double")
    with np.load(ck2) as z:
        assert str(z["tag"]) == _tag(spec, "complex128", False, a128)
    # the other entry points return the wide dtype and the same values
    ex = cb.TreeExecutor(spec, dtype="complex64", accumulate="double")
    assert ex.out_dtype == "complex128" and ex.accumulate == "double"
    assert ex.vjp_plan().dtype == "complex64"  # reverse mode is the native one
    got = cb.contract_tree(spec, arrays, dtype="complex64", accumulate="double")
    assert got.dtype == np.complex128 and np.allclose(got, wide, rtol=0, atol=1e-12 * np.abs(wide).max())
    one = cb.make_contractor(spec, accumulate="double")(*[np.asarray(a) for a in _slice0(rec, arrays)])
    assert np.asarray(one).dtype == np.complex128


def _slice0(rec, arrays):
    return orc.slice_arrays([tuple(t) for t in rec["inputs"]], decode_sliced(rec["sliced"]), arrays, 0)
