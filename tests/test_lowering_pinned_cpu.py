"""Every pair node the lowering produces, pinned to ``tests/golden/pair_lowering_digests.json``.

``lowering.build_pair_desc`` picks the kernel of every pairwise node of every plan, and that choice
decides the project's speed.  This test runs a fixed corpus through it -- the golden pair equations
forced onto every variant, the kernel-path table, a grid of matrix shapes straddling the variant and
admission thresholds, and the forward and VJP plans of every golden tree -- and compares, bucket by
bucket, a sha256 over each case's ``variant``, ``swapped``, ``tiles``, ``splitk`` and descriptor
words (or the class of the exception it raised).

A change that moves nodes on purpose regenerates the fixture, visibly, with

    python -m tests.test_lowering_pinned_cpu --write
"""

from __future__ import annotations

import hashlib
import json
import math
import os
import sys

from cotengra_b200 import ExecPlan, VjpPlan
from cotengra_b200 import lowering as L
from cotengra_b200.fusion import fuse_stems
from tests import kernel_cases as KC
from tests.helpers import GOLDEN_DIR, load_json, tree_spec

FIXTURE = os.path.join(GOLDEN_DIR, "pair_lowering_digests.json")
DTYPES = ("float32", "float64", "complex64", "complex128")
SINGLE = ("float32", "complex64")
VARIANTS = sorted(L.VARIANT_TILES)
NAMES = {None: "unforced", **KC.VARIANT_NAMES}
SM = 132

# the grid: extents on both sides of every threshold of choose_variant and of the admission rules
GRID_M = (1, 4, 5, 32, 33, 64, 128, 4096, 4101, 1 << 20, 1 << 24)
GRID_N = (1, 4, 5, 8, 9, 12, 16, 17, 24, 32, 33, 48, 64, 96, 128)
GRID_K = (1, 4, 8, 9, 16, 33, 64, 65, 256, 8192, 1 << 14, 1 << 20, 1 << 21)
GRID_BATCHED = ((4, 4101, 32, 33), (4, 1 << 20, 8, 8), (4, 4096, 16, 64), (3, 128, 64, 256), (2, 1, 1, 1 << 20),
                (4, 33, 33, 8192), (2, 4, 4, 1 << 20), (8, 128, 12, 16))


class Digests:
    def __init__(self):
        self.h = {}

    def add(self, bucket, build):
        """One case: the plan ``build()`` returns, or the class of what it raises."""
        h = self.h.setdefault(bucket, hashlib.sha256())
        try:
            p = build()
        except Exception as e:  # noqa: BLE001  (the class is part of the pinned behaviour)
            h.update(f"!{type(e).__name__}|".encode())
            return
        h.update(f"{int(p.variant)},{int(bool(p.swapped))},{int(p.tiles)},{int(p.splitk)}|".encode())
        h.update(p.words.tobytes())

    def add_plan(self, bucket, name, build):
        """Every pair node of the plan ``build()`` returns, in order, or the class of what it raises."""
        h = self.h.setdefault(bucket, hashlib.sha256())
        h.update(f"{name}:".encode())
        try:
            plan = build()
        except Exception as e:  # noqa: BLE001
            h.update(f"!{type(e).__name__}|".encode())
            return
        for nd in plan.nodes:
            if nd["kind"] == 0:
                p = nd["plan"]
                h.update(f"{int(p.variant)},{int(bool(p.swapped))},{int(p.tiles)},{int(p.splitk)}|".encode())
                h.update(p.words.tobytes())

    def hexdigests(self):
        return {k: self.h[k].hexdigest() for k in sorted(self.h)}


def _parser_cases(d):
    for n, rec in enumerate(load_json("parsers.json")["pair"]):
        if "error" in rec:
            continue
        terms, out = L.split_equation(rec["eq"])
        dims = L.classify_pair(terms[0], rec["shape_a"], terms[1], rec["shape_b"], out)
        n_out = max(math.prod(dims.out_shape), 1)
        for dtype in DTYPES:
            modes = [("plain", {}), ("acc_splitk3", dict(accumulate=True, force_splitk=3))]
            if dtype in SINGLE:
                modes.append(("tf32", dict(precision="tf32")))
            for mode, kw in modes:
                for v in (None, *VARIANTS):
                    d.add(f"parsers/{dtype}/{mode}/{NAMES[v]}",
                          lambda: L.build_pair_desc(dims, dtype, sm_count=SM, variant=v, c_dense_elems=n_out, **kw))


def _kernel_cases(d):
    for case in KC.CASES:
        d.add(f"kernel_cases/{NAMES[case.variant]}/{case.dtype}", lambda: KC.build_plan(case))


def _grid_cases(d):
    shapes = [(1, M, N, K) for M in GRID_M for N in GRID_N for K in GRID_K] + list(GRID_BATCHED)
    for B, M, N, K in shapes:
        if B == 1:
            dims = L.classify_pair("ak", (M, K), "kc", (K, N), "ac")
        else:
            dims = L.classify_pair("bak", (B, M, K), "bkc", (B, K, N), "bac")
        for dtype in DTYPES:
            for sm in (4, SM):
                d.add(f"grid/{dtype}/sm{sm}/unforced",
                      lambda: L.build_pair_desc(dims, dtype, sm_count=sm, c_dense_elems=B * M * N))
            for v in VARIANTS:
                d.add(f"grid/{dtype}/forced/{NAMES[v]}",
                      lambda: L.build_pair_desc(dims, dtype, sm_count=SM, variant=v, c_dense_elems=B * M * N))
            if dtype in SINGLE:
                # the root of an accumulate="double" plan: added into the output, a wide C
                for v in (None, *VARIANTS):
                    d.add(f"grid/{dtype}/wide_c/{NAMES[v]}",
                          lambda: L.build_pair_desc(dims, dtype, accumulate=True, sm_count=SM, variant=v,
                                                    wide_c=True))


def _bytes_only(dtype, B, M, N, K, elems):
    """A model that always prefers fewer bytes: forces stem fusion on small trees."""
    return 1e-9 * elems + 1e-12 * B * M * N * K


def _tree_cases(d):
    for source in ("trees.json", "live_trees.json", "sycamore_m20.json"):
        for rec in load_json(source):
            spec = tree_spec(rec)
            for dtype in DTYPES:
                # the small trees with stem fusion forced, the Sycamore ones as the default model fuses them
                kw = {} if source == "sycamore_m20.json" else dict(min_big=2, ratio=1.0, min_gain=-1.0,
                                                                   model=_bytes_only)
                fused, _ = fuse_stems(spec, dtype, **kw)
                for form, ir in (("unfused", spec.contractions()), ("fused", fused.contractions())):
                    args = (ir, spec.inputs, spec.output, spec.size_dict, spec.sliced)
                    b = f"trees/{source}/{dtype}/{form}"
                    d.add_plan(f"{b}/exec", rec["name"], lambda: ExecPlan(*args, dtype=dtype, sm_count=SM))
                    d.add_plan(f"{b}/vjp", rec["name"], lambda: VjpPlan(*args, dtype=dtype, sm_count=SM))


def _tree_option_cases(d):
    """Plan options that reach the lowering differently, on the golden trees (not the live ones)."""
    for source in ("trees.json", "sycamore_m20.json"):
        for rec in load_json(source):
            spec, name = tree_spec(rec), rec["name"]
            args = (spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced)
            for dtype in ("complex64", "complex128"):
                b = f"tree_options/{source}/{dtype}"
                d.add_plan(f"{b}/strip_exec", name,
                           lambda: ExecPlan(*args, dtype=dtype, sm_count=SM, strip_exponent=True))
                d.add_plan(f"{b}/no_dmma_exec", name, lambda: ExecPlan(*args, dtype=dtype, sm_count=SM, allow_dmma=False))
                if dtype in SINGLE:
                    d.add_plan(f"{b}/double_exec", name,
                               lambda: ExecPlan(*args, dtype=dtype, sm_count=SM, accumulate="double"))
                    d.add_plan(f"{b}/tf32_exec", name, lambda: ExecPlan(*args, dtype=dtype, sm_count=SM, precision="tf32"))
                if source == "sycamore_m20.json":
                    continue
                d.add_plan(f"{b}/strip_vjp", name, lambda: VjpPlan(*args, dtype=dtype, sm_count=SM,
                                                                    strip_exponent=True, stripped_grad=True))
                d.add_plan(f"{b}/no_dmma_vjp", name, lambda: VjpPlan(*args, dtype=dtype, sm_count=SM, allow_dmma=False))
                if dtype in SINGLE:
                    d.add_plan(f"{b}/tf32_vjp", name, lambda: VjpPlan(*args, dtype=dtype, sm_count=SM, precision="tf32"))
                    # a workspace budget one byte under the plan's own size: per-slice values recomputed
                    d.add_plan(f"{b}/recompute_vjp", name, lambda: VjpPlan(
                        *args, dtype=dtype, sm_count=SM,
                        max_bytes=VjpPlan(*args, dtype=dtype, sm_count=SM).total_bytes - 1))


def digests():
    d = Digests()
    for part in (_parser_cases, _kernel_cases, _grid_cases, _tree_cases, _tree_option_cases):
        part(d)
    return d.hexdigests()


def test_pair_lowering_is_pinned():
    with open(FIXTURE) as f:
        want = json.load(f)
    got = digests()
    assert sorted(got) == sorted(want), sorted(set(got) ^ set(want))[:20]
    moved = [k for k in sorted(want) if got[k] != want[k]]
    assert not moved, f"{len(moved)} buckets moved: {moved[:20]}"


if __name__ == "__main__":
    if sys.argv[1:] != ["--write"]:
        sys.exit("usage: python -m tests.test_lowering_pinned_cpu --write")
    with open(FIXTURE, "w") as f:
        json.dump(digests(), f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"wrote {FIXTURE}")
