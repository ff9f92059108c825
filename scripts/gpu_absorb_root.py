"""Time the last complex128 stem absorption and the 32 x 32 product that reads it, as two nodes and
as one absorb-root node, on the fused Sycamore-m20 slice (dev tool).

usage: python scripts/gpu_absorb_root.py [rounds] [--save=PATH]

The two nodes are X = A . Bs (DMMA_64x128, 2^23 x 128 x 16) and R = X . V (DMMA_32x32, 32 x 32 over
K = 2^25); the absorb-root node (VAR_ABSORB_ROOT, csrc/absorbdot.cuh) computes R from A, Bs and V
without X.  Descriptors come from the real plans (``ExecPlan`` with and without ``absorb_root``),
with their real strides; operands are seeded normal values.  The two ways run alternated, ``rounds``
times each, and the script prints ms per way, the largest difference of R relative to max|R|, and
the card's name, power limit and maximum SM clock."""
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

rounds = int(sys.argv[1]) if len(sys.argv) > 1 and not sys.argv[1].startswith("--") else 5
save = next((a.split("=", 1)[1] for a in sys.argv if a.startswith("--save=")), None)
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                      capture_output=True, text=True).stdout.strip().splitlines()[0]
sms = _lib.device_info()["sm_count"]
rec = next(r for r in load_json("sycamore_m20.json") if r["name"] == "sycamore_m20_appxB")
spec = cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"], decode_sliced(rec["sliced"]))
spec, _info = fuse_stems(spec, "complex128")
args = (spec.contractions(), spec.inputs, spec.output, spec.size_dict, spec.sliced)
two = cb.ExecPlan(*args, dtype="complex128", sm_count=sms)
one = cb.ExecPlan(*args, dtype="complex128", sm_count=sms, absorb_root=True)
F = next(nd for nd in one.nodes if nd.get("d") is not None)
ri = next(i for i, nd in enumerate(two.nodes) if nd["kind"] == 0 and int(nd["plan"].variant) == L.VAR_DMMA_32x32)
R, P = two.nodes[ri], two.nodes[ri - 1]  # (the absorbed node runs right before the product)
assert P["c"] in R["terms"]


def elems(t):
    return int(np.prod(t.shape))


g = torch.Generator(device="cuda").manual_seed(0)


def randn(n):
    x = torch.empty(n, dtype=torch.complex128, device="cuda")
    torch.view_as_real(x).normal_(generator=g)
    return x


# the fused node's operands: A (big), Bs (small), V; P reads A and Bs as its own a / b
A, Bs, V = randn(elems(F["a"])), randn(elems(F["d"])), randn(elems(F["b"]))
X = torch.empty(elems(P["c"]), dtype=torch.complex128, device="cuda")
pa, pb = (A, Bs) if elems(P["a"]) > elems(P["b"]) else (Bs, A)
x_is_ra = R["a"] is P["c"]
ra, rb = (X, V) if x_is_ra else (V, X)
M, N = R["sizes"][1], R["sizes"][2]
c2 = torch.empty(M * N, dtype=torch.complex128, device="cuda")
c1 = torch.empty(M * N, dtype=torch.complex128, device="cuda")
WP = np.array(P["words"], dtype=np.int64)
WR = np.array(R["words"], dtype=np.int64)
WR[L.W_FLAGS] &= ~1
WR[L.W_CELEMS] = M * N
WF = np.array(F["words"], dtype=np.int64)
WF[L.W_FLAGS] &= ~1
WF[L.W_CELEMS] = M * N
lib = _lib.load()


def run_two():
    _lib.check(lib.ctgb_contract_pair(WP.ctypes.data, pa.data_ptr(), pb.data_ptr(), X.data_ptr(), 0))
    _lib.check(lib.ctgb_contract_pair(WR.ctypes.data, ra.data_ptr(), rb.data_ptr(), c2.data_ptr(), 0))


def run_one():
    _lib.check(lib.ctgb_absorb_root(WF.ctypes.data, A.data_ptr(), Bs.data_ptr(), V.data_ptr(), c1.data_ptr(), 0))


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


run_two()
run_one()
torch.cuda.synchronize()
t2, t1 = [], []
for _ in range(rounds):
    t2.append(timed(run_two))
    t1.append(timed(run_one))
err = float((c1 - c2).abs().max() / c2.abs().max())
print(f"card: {card}")
print(f"P {tuple(P['sizes'])} variant {int(P['plan'].variant)} + R {tuple(R['sizes'])} variant {int(R['plan'].variant)}")
print(f"two nodes: {' '.join(f'{t:.3f}' for t in t2)} ms")
print(f"absorb-root: {' '.join(f'{t:.3f}' for t in t1)} ms")
print(f"max|R_one - R_two| / max|R_two| = {err:.2e}", flush=True)
if save:
    os.makedirs(os.path.dirname(save) or ".", exist_ok=True)
    np.save(save, c1.cpu().numpy())
