"""Which complex128 nodes the DMMA stream kernel (csrc/dmmastream.cuh) takes, and the instantiation its
launcher picks -- no GPU needed.

tests/golden/sycamore_m20_c128_nodes.json lists the per-slice pair nodes of the fused Sycamore-m20
Appendix-B plan as (B, M, N, K, variant), with the variants chosen before N = 17..32 nodes streamed: the
plan must keep every node and shape, and change only the variant of the nodes the stream kernel now
takes."""

import numpy as np
import pytest

from cotengra_b200 import ExecPlan, TreeSpec
from cotengra_b200 import lowering as L
from cotengra_b200.fusion import fuse_stems
from tests.helpers import decode_sliced, load_json

STAGED_DMMA = (L.VAR_DMMA_256x16, L.VAR_DMMA_256x32, L.VAR_DMMA_128x64, L.VAR_DMMA_64x128)


def _streams(B, M, N, K):
    return B == 1 and 4096 <= M < 1 << 32 and N <= 32 and K <= 64


def test_m20_plan_streams_exactly_the_narrow_nodes():
    rec = next(r for r in load_json("sycamore_m20.json") if r["name"] == "sycamore_m20_appxB")
    spec = TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]))
    new, _ = fuse_stems(spec, "complex128")
    plan = ExecPlan(new.contractions(), new.inputs, new.output, new.size_dict, new.sliced, dtype="complex128",
                    sm_count=132)
    got = [[int(x) for x in nd["sizes"]] + [int(nd["plan"].variant)] for nd in plan.nodes
           if nd["kind"] == 0 and not nd["invariant"]]
    before = load_json("sycamore_m20_c128_nodes.json")
    assert len(got) == len(before) == 184
    assert [g[:4] for g in got] == [b[:4] for b in before]
    moved = {}
    for g, b in zip(got, before):
        B, M, N, K = b[:4]
        if b[4] in STAGED_DMMA and _streams(B, M, N, K):
            assert g[4] == L.VAR_DMMASTREAM, (b, g)
            moved[(N, K)] = moved.get((N, K), 0) + 1
        else:
            assert g[4] == b[4], (b, g)
    # the 14 nodes of N = 32 (K = 16, 32, 64), all from DMMA_256x32; N = 64 stays on DMMA_128x64
    assert sum(moved.values()) == 14
    assert set(n for n, _k in moved) == {32}
    assert all(b[4] == L.VAR_DMMA_128x64 for b in before if b[2] == 64 and b[3] <= 32 and b[1] >= 4096)


@pytest.mark.parametrize("dtype,B,M,N,K", [
    ("complex128", 1, (1 << 25) + (1 << 20) + 24, 64, 64),  # K = 64 at N = 64: s_B would not fit
    ("complex128", 1, 1 << 22, 96, 16),
    ("complex128", 1, 1 << 22, 64, 33),
    ("complex128", 1, 1 << 22, 40, 64),
    ("complex128", 1, 1 << 24, 64, 32),                      # the kernel takes it; DMMA_128x64 is faster
    ("complex128", 1, 1 << 22, 33, 16),
    ("complex128", 4, 1 << 20, 32, 32),                      # batched
    ("float64", 1, 1 << 22, 32, 32),
    ("complex64", 1, 1 << 22, 64, 16),
])
def test_stays_off_the_stream_kernel(dtype, B, M, N, K):
    assert L.choose_variant(dtype, B, M, N, K) != L.VAR_DMMASTREAM


@pytest.mark.parametrize("N,K", [(17, 64), (24, 40), (32, 64), (32, 16), (12, 48), (16, 32)])
def test_routes_to_the_stream_kernel(N, K):
    assert L.choose_variant("complex128", 1, 1 << 20, N, K) == L.VAR_DMMASTREAM


@pytest.mark.parametrize("N,K,want", [(48, 32, L.VAR_DMMA_128x64), (32, 64, L.VAR_DMMA_256x32),
                                      (24, 16, L.VAR_DMMA_256x32), (12, 16, L.VAR_DMMA_256x16)])
def test_ragged_rows_fall_back_to_the_staged_tile(N, K, want):
    """A row extent that the 256-row tile blocks raggedly (4101 = 16 x 256 + 5) leaves the stream
    kernel, asked for by name, for the staged tile choose_variant picks without it (N <= 16: 256x16,
    as before)."""
    M = 4101
    dims = L.classify_pair("ak", (M, K), "kc", (K, N), "ac")
    plan = L.build_pair_desc(dims, "complex128", c_dense_elems=M * N, sm_count=132, variant=L.VAR_DMMASTREAM)
    assert plan.variant == want


def _desc(M, N, K, variant=L.VAR_DMMASTREAM):
    dims = L.classify_pair("ak", (M, K), "kc", (K, N), "ac")
    return L.build_pair_desc(dims, "complex128", c_dense_elems=M * N, sm_count=132, variant=variant)


@pytest.mark.parametrize("N,K,nj,rows", [(8, 64, 1, 32), (16, 32, 2, 32), (17, 64, 4, 32), (32, 64, 4, 32),
                                         (33, 32, 8, 16), (48, 24, 8, 16), (64, 32, 8, 16)])
def test_launcher_instantiation(N, K, nj, rows):
    from cotengra_b200 import _lib

    for M, sms in ((8192, 132), (1 << 24, 132), (12288, 114)):
        plan = _desc(M, N, K)
        assert plan.variant == L.VAR_DMMASTREAM
        f = _lib.dmmastream_launch_config(plan.words, sms)
        assert (f["nj"], f["rows"]) == (nj, rows)
        assert f["grid"] == min(-(-M // (4 * rows)), 12 * sms)


def test_launcher_rejects_what_the_kernel_cannot_take():
    from cotengra_b200 import _lib

    plan = _desc(8192, 64, 32)
    for n, k in ((65, 16), (64, 33), (33, 64)):
        w = plan.words.copy()
        w[L.W_NTA], w[L.W_KTA] = n, k
        with pytest.raises(ValueError):
            _lib.dmmastream_launch_config(w, 132)
    w = _desc(8192, 128, 32, variant=None).words
    assert int(w[L.W_VARIANT]) != L.VAR_DMMASTREAM
    with pytest.raises(ValueError):
        _lib.dmmastream_launch_config(w, 132)
    assert np.array_equal(plan.words, _desc(8192, 64, 32).words)
