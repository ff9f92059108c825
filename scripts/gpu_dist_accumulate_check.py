"""torchrun --nproc-per-node 2 scripts/gpu_dist_accumulate_check.py
contract_distributed(accumulate="double") over NCCL == the single-GPU wide result to 1e-12: the
ranks all-reduce their float64 / complex128 partials (the exponent MAX first when stripped)."""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch
import torch.distributed as dist

import cotengra_b200 as cb
from tests.helpers import load_json, make_arrays, rel_err, tree_spec

local = int(os.environ.get("LOCAL_RANK", "0"))
torch.cuda.set_device(local)
dist.init_process_group("nccl", device_id=torch.device("cuda", local))
rank = dist.get_rank()
ok = True
for name in ("lattice6x6_d3_sliced", "rand_r3_o1_hi0_ho1_None_s42_sliced_out"):
    rec = next(r for r in load_json("trees.json") if r["name"] == name)
    spec = tree_spec(rec)
    arrays = make_arrays(spec.shapes(), "complex64", seed=rec["seed"])
    want = cb.contract_tree(spec, arrays, accumulate="double")
    got = cb.contract_distributed(spec, arrays, accumulate="double")
    errs = [rel_err(got, want)]
    ok = ok and got.dtype == np.complex128
    if "sliced_out" not in name:
        mw, ew = cb.contract_tree(spec, arrays, accumulate="double", strip_exponent=True)
        m, e = cb.contract_distributed(spec, arrays, accumulate="double", strip_exponent=True)
        ok = ok and m.dtype == np.complex128
        errs.append(rel_err(m * 10.0 ** (e - ew), mw))
    if rank == 0:
        print(f"{name}: " + " ".join(f"{x:.1e}" for x in errs))
    ok = ok and max(errs) < 1e-12
t = torch.tensor([1 if ok else 0], device="cuda")
dist.all_reduce(t, op=dist.ReduceOp.MIN)
if rank == 0:
    print("DIST_ACCUMULATE", "PASS" if int(t.item()) == 1 else "FAIL")
dist.destroy_process_group()
sys.exit(0 if int(t.item()) == 1 else 1)
