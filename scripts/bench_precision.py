"""Compute-mode benchmark: complex64 trees under precision="3xtf32" (the default) and "tf32" (one
round-to-nearest tf32 pass), alternated in one process after warm-up.  Prints one JSON line per
workload with the card name and power limit read in the same run.

    python scripts/bench_precision.py [--configs m20,peps8x8,m10s] [--steps 5] [--warmup 2] [--rounds 3]
                                      [--slices 2] [--no-vjp]

For each workload and mode: time per slice (CUDA events, median over ``--rounds`` alternations),
per-node times summed by kernel variant (``ExecPlan.profile``, in a separate untimed slice) and the
relative error of the result against complex128: slice 0 of the m20 tree against the CPU oracle's
golden value (``tests/golden/big_slices.json``), the other trees against this package's complex128
result on the same inputs (which the golden-value tests hold to 1e-10).  peps8x8 also runs its VJP
(every input, cotangent of ones) in both modes, timed the same way, with the worst gradient error
against complex128.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402

MODES = ("3xtf32", "tf32")


def _card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip().splitlines()
        return out[0]
    except Exception:
        import torch

        return torch.cuda.get_device_name(0) + ", power limit unknown"


def _timed(torch, fn, steps):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def _by_variant(ex, tensors):
    """ms per kernel variant of one slice (node events), pairwise nodes only."""
    import torch

    from tests.kernel_cases import VARIANT_NAMES

    plan = ex.plan
    plan.profile(True)
    ex.contract_device(tensors, 0, 1, 1)
    torch.cuda.synchronize()
    ms = plan.profile_read()
    plan.profile(False)
    out = {}
    for nd, t in zip(plan.nodes, ms):
        if nd["kind"] == 0:
            name = VARIANT_NAMES[int(nd["words"][32])]  # W_VARIANT
            out[name] = round(out.get(name, 0.0) + t, 4)
    return out


def run(args):
    import torch

    import cotengra_b200 as cb

    torch.cuda.set_device(0)
    card = _card()
    for config in args.configs.split(","):
        spec, arrays, desc = bench.load_workload(config, "complex128")
        count = min(spec.nslices, args.slices)
        dev128 = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
        dev64 = [t.to(torch.complex64) for t in dev128]
        if config == "m20":
            want = bench.golden_big_slice()
            ref_src = "tests/golden/big_slices.json, slice 0"
            want = None if want is None else np.array(want)
        else:
            ex128 = cb.TreeExecutor(spec, dtype="complex128")
            want = ex128.contract_device(dev128, 0, 1, count).cpu().numpy()
            ref_src = f"complex128 executor, slices 0..{count - 1}"
            del ex128
            torch.cuda.empty_cache()
        exs = {m: cb.TreeExecutor(spec, dtype="complex64", precision=m) for m in MODES}
        line = {"metric": f"{config}_precision", "config": config, "workload": desc, "card": card,
                "slices_per_step": count, "reference": ref_src, "modes": {}}
        for m, ex in exs.items():
            ex.workspace()
            for _ in range(args.warmup):
                ex.contract_device(dev64, 0, 1, count)
        torch.cuda.synchronize()
        times = {m: [] for m in MODES}
        for _ in range(args.rounds):
            for m, ex in exs.items():
                times[m].append(_timed(torch, lambda: ex.contract_device(dev64, 0, 1, count), args.steps) / count)
        for m, ex in exs.items():
            n = 1 if config == "m20" else count
            got = ex.contract_device(dev64, 0, 1, n).cpu().numpy()
            err = None if want is None else float(np.max(np.abs(got - want)) / np.max(np.abs(want)))
            line["modes"][m] = {"ms_per_slice": statistics.median(times[m]), "ms_per_slice_all": times[m],
                                "rel_err_vs_complex128": err, "ms_by_variant": _by_variant(ex, dev64)}
        t3, t1 = line["modes"]["3xtf32"]["ms_per_slice"], line["modes"]["tf32"]["ms_per_slice"]
        line["speedup_tf32_over_3xtf32"] = t3 / t1
        if config == "peps8x8" and not args.no_vjp:
            ex128 = cb.TreeExecutor(spec, dtype="complex128")
            cot = torch.ones(ex128.plan.out_shape, dtype=torch.complex128, device="cuda")
            g128 = [g.cpu().numpy() for g in ex128.vjp(dev128, cot, 0, 1, count)]
            cot64 = cot.to(torch.complex64)
            vt = {m: [] for m in MODES}
            for ex in exs.values():
                for _ in range(args.warmup):
                    ex.vjp(dev64, cot64, 0, 1, count)
            for _ in range(args.rounds):
                for m, ex in exs.items():
                    vt[m].append(_timed(torch, lambda: ex.vjp(dev64, cot64, 0, 1, count), args.steps))
            vjp = {}
            for m, ex in exs.items():
                g = [x.cpu().numpy() for x in ex.vjp(dev64, cot64, 0, 1, count)]
                worst = max(float(np.linalg.norm(a - w) / np.linalg.norm(w)) for a, w in zip(g, g128))
                vjp[m] = {"ms": statistics.median(vt[m]), "ms_all": vt[m], "worst_grad_rel_err_vs_complex128": worst}
            line["vjp"] = vjp
        print(json.dumps(line), flush=True)
        del exs
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="m20,peps8x8,m10s")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--slices", type=int, default=2)
    ap.add_argument("--no-vjp", action="store_true")
    run(ap.parse_args())


if __name__ == "__main__":
    main()
