"""Time the complex128 root product of the fused Sycamore-m20 slice alone (dev tool).

usage: python scripts/gpu_root_stream.py [reps] [--save=PATH]

The root is the DMMA_32x32 node R[32 x 32] = sum_k A[k, m] B[k, n] over K = 2^25 that stem fusion
leaves (DESIGN.md section 5).  Its descriptor comes from the real plan, with its real strides, and it
runs through ctgb_contract_pair on two 2^30-element complex128 operands (34.4 GB, seeded normal
values) into a zeroed 32 x 32 result.  Prints ms and GB/s of the algorithmic bytes next to the card's
name, power limit and maximum SM clock.  --save writes the result, for comparing two builds."""
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import cotengra_b200 as cb
from cotengra_b200 import _lib, lowering as L
from cotengra_b200.fusion import fuse_stems
from tests.helpers import decode_sliced, load_json

reps = int(sys.argv[1]) if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else 10
save = next((a.split("=", 1)[1] for a in sys.argv if a.startswith("--save=")), None)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
sms = _lib.device_info()["sm_count"]
rec = next(r for r in load_json("sycamore_m20.json") if r["name"] == "sycamore_m20_appxB")
spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]))
spec, _info = fuse_stems(spec, "complex128")
plan = cb.ExecPlan(spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced, dtype="complex128",
                   sm_count=sms)
nd = next(nd for nd in plan.nodes if nd["kind"] == 0 and int(nd["plan"].variant) == L.VAR_DMMA_32x32)
B_, M, N, K = nd["sizes"]
W = np.array(nd["words"], dtype=np.int64)
W[L.W_FLAGS] &= ~1  # alone: no accumulate, C zeroed by the launch
W[L.W_CELEMS] = M * N
na, nb = (int(np.prod(nd[x].shape)) for x in ("a", "b"))
g = torch.Generator(device="cuda").manual_seed(0)
a = torch.empty(na, dtype=torch.complex128, device="cuda")
b = torch.empty(nb, dtype=torch.complex128, device="cuda")
torch.view_as_real(a).normal_(generator=g)
torch.view_as_real(b).normal_(generator=g)
c = torch.empty(M * N, dtype=torch.complex128, device="cuda")
lib = _lib.load()


def launch():
    _lib.check(lib.ctgb_contract_pair(W.ctypes.data, a.data_ptr(), b.data_ptr(), c.data_ptr(), 0))


for _ in range(2):
    launch()
torch.cuda.synchronize()
e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
e0.record()
for _ in range(reps):
    launch()
e1.record()
torch.cuda.synchronize()
ms = e0.elapsed_time(e1) / reps
nbytes = (na + nb + M * N) * 16
print(f"card: {card}")
print(f"root M={M} N={N} K={K}: {ms:.3f} ms  {nbytes / ms / 1e6:.0f} GB/s  {8 * M * N * K / ms / 1e9:.2f} TFLOP/s  "
      f"({reps} launches, variant {int(W[L.W_VARIANT])}, split-K {int(W[L.W_SPLITK])})", flush=True)
if save:
    os.makedirs(os.path.dirname(save) or ".", exist_ok=True)
    np.save(save, c.cpu().numpy())
