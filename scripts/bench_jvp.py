"""Forward-mode benchmark: per-call times of the forward, the JVP with one input and with every input
carrying a tangent, and the VJP, on one GPU; then the JVP with every input in its two forms -- the
two-term stream nodes in one launch (``ctgb_contract_pair2``) and the same nodes as two launches --
alternated in one process.  Prints one JSON line per (config, dtype) with the card name and power
limit.

    python scripts/bench_jvp.py [--configs peps8x8 m10s] [--dtypes complex64 complex128]
                                [--slices 2 --steps 10 --warmup 3 --rounds 5]
    python scripts/bench_jvp.py --strip [--m20-widths 26 30] ...

``--strip`` times the stripped JVP (``strip_exponent=True, stripped_grad=True``) against the
unstripped one instead, for one input and for every input, alternated round by round, and reports
the launches per slice and the stripped two-term nodes of both plans; ``--m20-widths`` adds slice 0
of the Sycamore-m20 tree at those widths in complex64 (a plan that does not fit the card is reported
with its bytes and not run).

Times are CUDA-event times per call, averaged over ``--steps`` calls after ``--warmup``; the two-form
comparison takes the median of ``--rounds`` alternated rounds.  The trees run as ``TreeExecutor``
builds them (stem fusion on).  Writes nothing to the tree.
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
from tests.helpers import make_arrays  # noqa: E402


def card_name():
    import torch

    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def run(config, dtype, args, card):
    import torch

    import cotengra_b200 as cb

    spec, arrays, desc = bench.load_workload(config, dtype)
    ex = cb.TreeExecutor(spec, dtype=dtype)
    count = min(ex.nslices, args.slices)
    n = len(arrays)
    big = max(range(n), key=lambda i: arrays[i].size)
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    tans = [torch.from_numpy(t).cuda() for t in make_arrays([a.shape for a in arrays], dtype, seed=1, scale=0.35)]
    cot = torch.ones(ex.plan.out_shape, dtype=dev[0].dtype, device="cuda")
    all_plan = ex.jvp_plan()
    two_plan = ex.jvp_plan(_two_term=False)
    line = {"metric": f"{config}_jvp", "config": config, "dtype": dtype, "workload": desc, "card": card,
            "slices": count, "inputs": n, "one_input": big,
            "jvp_workspace_bytes": all_plan.total_bytes, "forward_workspace_bytes": ex.plan.total_bytes,
            "two_term_nodes": all_plan.two_term_nodes,
            "tangent_launches_two_term_form": len(all_plan.tangent_nodes),
            "tangent_launches_two_launch_form": len(two_plan.tangent_nodes)}
    free = torch.cuda.mem_get_info()[0]
    if all_plan.total_bytes + ex.plan.total_bytes > 0.9 * free:
        line["note"] = f"the JVP workspace ({all_plan.total_bytes} bytes) does not fit the card ({free} bytes free)"
        print(json.dumps(line), flush=True)
        return

    def timed(fn, steps=args.steps, warmup=args.warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / steps

    line["forward_s"] = timed(lambda: ex.contract_device(dev, 0, 1, count))
    line["jvp_one_input_s"] = timed(lambda: ex.jvp(dev, [tans[big]], 0, 1, count, wrt=[big], primal=False))
    line["jvp_all_inputs_s"] = timed(lambda: ex.jvp(dev, tans, 0, 1, count, primal=False))
    line["jvp_all_inputs_with_primal_s"] = timed(lambda: ex.jvp(dev, tans, 0, 1, count))
    ex._jvp_ws = None
    torch.cuda.empty_cache()
    if ex.vjp_plan().total_bytes < 0.8 * torch.cuda.mem_get_info()[0]:
        line["vjp_s"] = timed(lambda: ex.vjp(dev, cot, 0, 1, count))
        ex._vjp_ws = None
        torch.cuda.empty_cache()
    else:
        line["vjp_note"] = "VJP workspace does not fit beside the JVP's: not measured"
    # the two forms, alternated (they differ only at the two-term stream nodes)
    one, two = [], []
    for _ in range(args.rounds):
        one.append(timed(lambda: ex.jvp(dev, tans, 0, 1, count, primal=False), warmup=1))
        two.append(timed(lambda: ex.jvp(dev, tans, 0, 1, count, primal=False, _two_term=False), warmup=1))
    t1 = ex.jvp(dev, tans, 0, 1, count, primal=False)
    t2 = ex.jvp(dev, tans, 0, 1, count, primal=False, _two_term=False)
    line.update({"jvp_two_term_form_s": statistics.median(one), "jvp_two_launch_form_s": statistics.median(two),
                 "jvp_two_term_rounds_s": one, "jvp_two_launch_rounds_s": two,
                 "two_forms_max_rel_diff": float(torch.linalg.vector_norm(t1 - t2)
                                                 / max(float(torch.linalg.vector_norm(t2)), 1e-300))})
    print(json.dumps(line), flush=True)


def run_strip(config, dtype, args, card, spec=None, arrays=None, desc=None):
    import torch

    import cotengra_b200 as cb

    if spec is None:
        spec, arrays, desc = bench.load_workload(config, dtype)
    plain = cb.TreeExecutor(spec, dtype=dtype)
    strip = cb.TreeExecutor(spec, dtype=dtype, strip_exponent=True, stripped_grad=True)
    count = min(plain.nslices, args.slices)
    n = len(arrays)
    big = max(range(n), key=lambda i: arrays[i].size)
    line = {"metric": f"{config}_jvp_strip", "config": config, "dtype": dtype, "workload": desc, "card": card,
            "slices": count, "inputs": n, "one_input": big}
    plans = {}
    free = torch.cuda.mem_get_info()[0]
    for name, ex in (("unstripped", plain), ("stripped", strip)):
        for wrt, key in ((None, "all"), ([big], "one")):
            p = ex.jvp_plan(wrt)
            plans[name, key] = p
            line[f"{name}_{key}_launches_per_slice"] = p.launches_per_slice()
            line[f"{name}_{key}_two_term_nodes"] = p.two_term_nodes
            line[f"{name}_{key}_workspace_bytes"] = p.total_bytes
    need = max(p.total_bytes for p in plans.values()) + strip.plan.total_bytes
    if need > 0.9 * free:
        line["note"] = f"the JVP workspace ({need} bytes) does not fit the card ({free} bytes free): not run"
        print(json.dumps(line), flush=True)
        return
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    tans = [torch.from_numpy(t).cuda() for t in make_arrays([a.shape for a in arrays], dtype, seed=1, scale=0.35)]

    def timed(fn, steps=args.steps, warmup=args.warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / steps

    calls = {
        ("unstripped", "one"): lambda: plain.jvp(dev, [tans[big]], 0, 1, count, wrt=[big]),
        ("stripped", "one"): lambda: strip.jvp(dev, [tans[big]], 0, 1, count, wrt=[big]),
        ("unstripped", "all"): lambda: plain.jvp(dev, tans, 0, 1, count),
        ("stripped", "all"): lambda: strip.jvp(dev, tans, 0, 1, count),
    }
    for f in calls.values():
        timed(f, steps=1, warmup=args.warmup)
    rounds = {k: [] for k in calls}
    for _ in range(args.rounds):  # alternated: a drift in clocks hits both forms alike
        for k, f in calls.items():
            rounds[k].append(timed(f, warmup=1))
    for (name, key), r in rounds.items():
        line[f"{name}_{key}_s"] = statistics.median(r)
        line[f"{name}_{key}_rounds_s"] = r
    for key in ("one", "all"):
        line[f"stripped_over_unstripped_{key}"] = line[f"stripped_{key}_s"] / line[f"unstripped_{key}_s"]
    # the stripped tangent times 10^e against the unstripped one (complex128: ~1e-13)
    (_m, e), dm = strip.jvp(dev, tans, 0, 1, count)
    _o, want = plain.jvp(dev, tans, 0, 1, count)
    got = dm.to(torch.complex128) * 10.0 ** float(e.item())
    line["exponent"] = float(e.item())
    line["stripped_vs_unstripped_rel_diff"] = float(torch.linalg.vector_norm(got - want.to(torch.complex128))
                                                    / max(float(torch.linalg.vector_norm(want)), 1e-300))
    print(json.dumps(line), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", nargs="+", default=["peps8x8", "m10s"], choices=sorted(bench.METRICS))
    ap.add_argument("--dtypes", nargs="+", default=["complex64", "complex128"], choices=["complex64", "complex128"])
    ap.add_argument("--slices", type=int, default=2)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--strip", action="store_true", help="stripped against unstripped JVP")
    ap.add_argument("--m20-widths", nargs="*", type=int, default=[], help="with --strip: m20 slice 0 at 2^W")
    args = ap.parse_args()
    card = card_name()
    if args.strip:
        from tests.slicing_util import appxB_at_width

        for config in args.configs:
            for dtype in args.dtypes:
                run_strip(config, dtype, args, card)
        for w in args.m20_widths:
            spec = appxB_at_width(w)
            arrays = make_arrays(spec.shapes(), "complex64", seed=0, scale=0.65)
            run_strip(f"m20_w{w}", "complex64", argparse.Namespace(**{**vars(args), "slices": 1}), card, spec, arrays,
                      f"Sycamore m20 slice 0 at W = 2^{w}")
        return
    for config in args.configs:
        for dtype in args.dtypes:
            run(config, dtype, args, card)


if __name__ == "__main__":
    main()
