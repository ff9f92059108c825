"""Constant folding benchmark: a tree with K variable inputs and every other input constant, run by a
folded executor (``TreeExecutor(constants=...)``) and by the unfolded one, per call, forward and
forward + ``vjp`` on the variables.  Prints one JSON line with the card name and power limit.

    python scripts/bench_constants.py --config peps8x8|m10s --dtype complex64|complex128 --variables K
                                      [--seed S] [--steps 10 --warmup 3 --rounds 3]

The K variables are drawn at random (seeded).  The two executors alternate round by round in one
process, after warm-up, each timed window closed by a device synchronise; the line reports the
median per-call times.  ``max_rel_diff`` is the largest difference between the two executors'
results relative to the largest element.  Writes nothing to the tree.
"""
import argparse
import json
import os
import statistics
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402


def run(args):
    import subprocess

    import torch

    import cotengra_b200 as cb

    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        card = torch.cuda.get_device_name(0) + ", power limit unknown"
    spec, arrays, desc = bench.load_workload(args.config, args.dtype)
    n = len(arrays)
    rng = np.random.default_rng(args.seed)
    variables = sorted(rng.choice(n, size=min(args.variables, n), replace=False).tolist())
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    consts = {i: dev[i] for i in range(n) if i not in variables}
    var = [dev[i] for i in variables]
    t0 = time.perf_counter()
    folded = cb.TreeExecutor(spec, dtype=args.dtype, constants=consts)
    build_s = time.perf_counter() - t0
    plain = cb.TreeExecutor(spec, dtype=args.dtype)
    cot = torch.ones(plain.plan.out_shape, dtype=dev[0].dtype, device="cuda")

    def fwd_f():
        return folded.contract_device(var)

    def fwd_p():
        return plain.contract_device(dev)

    def both_f():
        folded.contract_device(var)
        return folded.vjp(var, cot)

    def both_p():
        plain.contract_device(dev)
        return plain.vjp(dev, cot, wrt=variables)

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        for _ in range(args.steps):
            fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t) / args.steps

    for fn in (fwd_f, fwd_p, both_f, both_p):
        for _ in range(args.warmup):
            fn()
    times = {k: [] for k in ("fwd_f", "fwd_p", "both_f", "both_p")}
    for _ in range(args.rounds):
        for k, fn in (("fwd_f", fwd_f), ("fwd_p", fwd_p), ("both_f", both_f), ("both_p", both_p)):
            times[k].append(timed(fn))
    med = {k: statistics.median(v) for k, v in times.items()}
    a, b = fwd_f(), fwd_p()
    diff = float((a - b).abs().max() / max(float(b.abs().max()), 1e-300))
    ga, gb = both_f(), both_p()
    gdiff = max(float((x - gb[i]).abs().max() / max(float(gb[i].abs().max()), 1e-300))
                for x, i in zip(ga, variables))
    macs_plain = plain.plan.macs_per_slice * plain.nslices + plain.plan.macs_invariant
    print(json.dumps({
        "metric": f"{args.config}_constants", "config": args.config, "dtype": args.dtype, "workload": desc,
        "card": card, "variables": variables, "n_inputs": n, "folds": len(folded.folded),
        "folded": [{"ssa": f.ssa, "term": "".join(f.term), "bytes": f.bytes, "macs": f.macs} for f in folded.folded],
        "folded_bytes": folded.folded_bytes, "macs_per_call_unfolded": macs_plain,
        "macs_per_call_removed": sum(f.macs for f in folded.folded), "build_s": build_s,
        "forward_folded_s": med["fwd_f"], "forward_unfolded_s": med["fwd_p"],
        "forward_plus_vjp_folded_s": med["both_f"], "forward_plus_vjp_unfolded_s": med["both_p"],
        "forward_speedup": med["fwd_p"] / med["fwd_f"], "forward_plus_vjp_speedup": med["both_p"] / med["both_f"],
        "max_rel_diff": diff, "max_rel_grad_diff": gdiff, "steps": args.steps, "rounds": args.rounds,
    }))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="peps8x8", choices=["peps8x8", "m10s"])
    ap.add_argument("--dtype", default="complex64", choices=["complex64", "complex128"])
    ap.add_argument("--variables", type=int, default=1)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    run(ap.parse_args())


if __name__ == "__main__":
    main()
