"""Accumulation-mode benchmark: complex64 trees under accumulate="native" (the default) and "double",
alternated in one process after warm-up.  Prints one JSON line per workload with the card name and
power limit read in the same run.

    python scripts/bench_accumulate.py [--configs m20,m10s,many] [--rounds 3] [--warmup 1]

Workloads: the m20 tree at W = 2^30 (2 of its slices), the m10s circuit, and a three-tensor tree with
14 sliced bonds (2^14 slices, same-sign inputs, a non-dot root).  Per mode: ms per slice (CUDA events,
median over ``--rounds`` alternations), the root node's time from ``ctgb_plan_profile`` (one separate
untimed slice), launches per slice, and the max-norm error of the result over the timed slices against
this package's complex128 result on the same inputs.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402
from scripts.bench_precision import _card, _timed  # noqa: E402

MODES = ("native", "double")


def _many():
    import cotengra_b200 as cb

    bonds = [f"b{i}" for i in range(14)]
    sizes = {b: 2 for b in bonds}
    sizes.update(i=8, j=8, o=8)
    spec = cb.TreeSpec([tuple(bonds) + ("i",), ("i", "j", "o"), tuple(bonds) + ("j",)], ("o",), sizes,
                       [(0, 1), (3, 2)], [(b, 2, None) for b in bonds])
    rng = np.random.default_rng(11)
    arrays = [(rng.uniform(0.5, 1.0, s) + 0.25j * rng.uniform(0.5, 1.0, s)).astype(np.complex64)
              for s in spec.shapes()]
    return spec, arrays, "three tensors, 14 sliced bonds of 2 (2^14 slices), same-sign inputs, open output"


def main():
    import torch

    import cotengra_b200 as cb

    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="m20,m10s,many")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_accumulate.py needs a CUDA device")
    card = _card()
    for config in args.configs.split(","):
        spec, arrays, desc = _many() if config == "many" else bench.load_workload(config, "complex64")
        count = min(int(spec.nslices), 2 if config == "m20" else 1 << 14)
        dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
        ref_ex = cb.TreeExecutor(spec, dtype="complex128")
        truth = ref_ex.contract_device([t.to(torch.complex128) for t in dev], 0, 1, count).cpu().numpy()
        del ref_ex
        torch.cuda.empty_cache()
        exs = {m: cb.TreeExecutor(spec, dtype="complex64", accumulate=m) for m in MODES}
        res = {m: {"ms_per_slice": []} for m in MODES}
        for m in MODES:
            for _ in range(args.warmup):
                exs[m].contract_device(dev, 0, 1, count)
        torch.cuda.synchronize()
        for _ in range(args.rounds):
            for m in MODES:
                res[m]["ms_per_slice"].append(_timed(torch, lambda: exs[m].contract_device(dev, 0, 1, count), 1) / count)
        for m in MODES:
            ex = exs[m]
            out = ex.contract_device(dev, 0, 1, count).cpu().numpy()
            ex.plan.profile(True)
            ex.contract_device(dev, 0, 1, 1)
            root_ms = ex.plan.profile_read()[-1]
            ex.plan.profile(False)
            r = res[m]
            r["ms_per_slice_all"] = [round(x, 5) for x in r["ms_per_slice"]]
            r["ms_per_slice"] = round(statistics.median(r["ms_per_slice"]), 5)
            r["root_node_ms"] = round(root_ms, 5)
            r["root_variant"] = int(ex.plan.nodes[-1]["words"][cb.lowering.W_VARIANT]) if ex.plan.nodes[-1]["kind"] == 0 else -1
            r["launches_per_slice"] = ex.plan.launches_per_slice()
            r["out_dtype"] = ex.out_dtype
            den = float(np.abs(truth).max())
            r["max_err_vs_complex128"] = float(np.abs(out - truth).max() / den) if den else float(np.abs(out).max())
        print(json.dumps({"bench": "accumulate", "config": config, "workload": desc, "slices": count,
                          "card": card, **res}), flush=True)
        del exs, dev
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
