"""Gradient benchmark: forward + VJP of one BASELINE configuration on one GPU, against the same
tree under torch GPU autograd.  Prints one JSON line with the card name and power limit.

    python scripts/bench_grad.py --config peps8x8 --dtype complex64 [--steps 10 --warmup 3]
                                 [--slices-per-gpu 2] [--no-fuse] [--vjp-max-gib 56] [--strip]

Gradient TFLOP/s are quoted on the VJP work: the recomputed forward (root excluded) plus, for each
differentiated pairwise node, its MACs times the number of H it forms (8 flops per complex
multiply-add, 2 per real one); with ``--vjp-max-gib`` the plan recomputes per-slice forward values
to stay within that workspace, and ``recompute_macs`` reports the extra forward work per slice.  Trees
whose VJP workspace does not fit the card report the bytes they need.  The torch-autograd baseline
keeps every intermediate, as the unbudgeted plan does: it is skipped when that plan would not fit.
Writes nothing to the tree.
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

import bench  # noqa: E402


def run_grad(args):
    """Forward + VJP (``TreeExecutor.vjp``, every input differentiated, cotangent of ones)
    on one GPU, against the same tree under torch GPU autograd (``torch.einsum`` / ``tensordot`` per
    node, cuBLAS).  Gradient TFLOP/s are quoted on the VJP work: the recomputed forward (root
    excluded) plus, per differentiated pairwise node, its MACs times the number of H it forms."""
    import subprocess

    import torch

    import cotengra_b200 as cb

    try:
        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        card = torch.cuda.get_device_name(0) + ", power limit unknown"
    spec, arrays, desc = bench.load_workload(args.config, args.dtype)
    ex = cb.TreeExecutor(spec, dtype=args.dtype, fuse=not args.no_fuse)
    count = min(ex.nslices, args.slices_per_gpu)
    # the unbudgeted plan's size, planned on the host only
    full = cb.VjpPlan(ex._ir, spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype=ex.dtype,
                      sm_count=ex.plan.sm_count).total_bytes
    budget = None if args.vjp_max_gib is None else int(args.vjp_max_gib * (1 << 30))
    plan = ex.vjp_plan(max_bytes=budget)
    line = {"metric": f"{args.config}_grad", "config": args.config, "dtype": args.dtype, "workload": desc,
            "card": card, "slices": count, "vjp_workspace_bytes": plan.total_bytes,
            "vjp_workspace_bytes_unbudgeted": full, "vjp_max_bytes": budget,
            "vjp_min_bytes": plan.min_bytes, "recompute_macs": plan.recompute_macs,
            "forward_macs": plan.fwd.macs_per_slice}
    free = torch.cuda.mem_get_info()[0]
    if plan.total_bytes > 0.9 * free:
        line["note"] = f"the VJP workspace ({plan.total_bytes} bytes) does not fit the card ({free} bytes free)"
        print(json.dumps(line))
        return
    dev = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in arrays]
    cot = torch.ones(ex.plan.out_shape, dtype=dev[0].dtype, device="cuda")

    def timed(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(args.steps):
            res = fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / 1e3 / args.steps, res

    t_fwd, _ = timed(lambda: ex.contract_device(dev, 0, 1, count))
    both_fit = plan.total_bytes + ex.plan.total_bytes < 0.9 * free
    if not both_fit:
        ex._ws = None  # the forward's workspace and the VJP's do not fit at once
        torch.cuda.empty_cache()
    t_vjp, grads = timed(lambda: ex.vjp(dev, cot, 0, 1, count, max_bytes=budget))
    t_both = t_fwd + t_vjp
    if both_fit:
        t_both, _ = timed(lambda: (ex.contract_device(dev, 0, 1, count),
                                   ex.vjp(dev, cot, 0, 1, count, max_bytes=budget)))
    per_mac = 8 if "complex" in args.dtype else 2

    def torch_step():
        # the caller's tree, slice by slice (every config here has no sliced output index)
        ts = [t.detach().requires_grad_() for t in dev]
        out = None
        for i in range(count):
            r = bench.torch_run_contractions(spec.contractions(), bench.torch_slice_arrays(spec, ts, i))
            out = r if out is None else out + r
        return torch.autograd.grad(out, ts, grad_outputs=torch.ones_like(out))

    line.update({
        "grad_tflops": per_mac * plan.vjp_macs(count) / t_vjp / 1e12,
        "flops_convention": f"{per_mac} flops per scalar multiply-add on the VJP work "
                            "(recomputed forward without the root + MACs x H formed per differentiated node)",
        "forward_s": t_fwd, "vjp_s": t_vjp, "forward_plus_vjp_s": t_both,
        "ratio_forward_plus_vjp_over_forward": t_both / t_fwd,
        "forward_plus_vjp_timed_together": both_fit,
    })
    if not both_fit or full > 0.8 * (free - plan.total_bytes - ex.plan.total_bytes):
        line["torch_note"] = f"torch autograd skipped: it keeps every intermediate (about {full} bytes)"
    else:
        t_torch, tgrads = timed(torch_step)
        diff = max(float(torch.linalg.vector_norm(g - w) / max(float(torch.linalg.vector_norm(w)), 1e-300))
                   for g, w in zip(grads, tgrads))
        line.update({"torch_autograd_s": t_torch, "speedup_vs_torch_autograd": t_torch / t_both,
                     "max_rel_grad_diff_vs_torch": diff})
    if args.strip:
        # the same VJP of the stripped mantissa (stripped_grad): one seed kernel per slice and scaled
        # epilogues / pre-scaled operands on top of the unstripped plan; timed after it, alone
        del grads
        ex._ws = ex._vjp_ws = None
        torch.cuda.empty_cache()
        exs = cb.TreeExecutor(spec, dtype=args.dtype, fuse=not args.no_fuse, strip_exponent=True,
                              stripped_grad=True)
        _m, e = exs.contract_device(dev, 0, 1, count)
        splan = exs.vjp_plan(max_bytes=budget)
        exs._ws = None
        torch.cuda.empty_cache()
        t_svjp, _g = timed(lambda: exs.vjp(dev, cot, 0, 1, count, max_bytes=budget, exponent=e))
        line.update({"strip_vjp_s": t_svjp, "strip_over_unstripped_vjp": t_svjp / t_vjp,
                     "strip_vjp_workspace_bytes": splan.total_bytes,
                     "strip_launches_per_slice": splan.launches_per_slice(),
                     "launches_per_slice": plan.launches_per_slice()})
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="peps8x8", choices=sorted(bench.METRICS))
    ap.add_argument("--dtype", default="complex64", choices=["complex128", "complex64"])
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--slices-per-gpu", type=int, default=2)
    ap.add_argument("--no-fuse", action="store_true", help="differentiate the reference's node sequence one to one")
    ap.add_argument("--vjp-max-gib", type=float, default=None,
                    help="workspace budget of the VJP plan in GiB (per-slice values are recomputed to meet it)")
    ap.add_argument("--strip", action="store_true",
                    help="also time the VJP of the strip_exponent mantissa (stripped_grad=True)")
    run_grad(ap.parse_args())


if __name__ == "__main__":
    main()
