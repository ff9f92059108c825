"""Every case of tests/kernel_cases.py once through ``ctgb_contract_pair`` on the device.

The operands sit at element offsets inside buffers whose gaps and guard bands are NaN (a stray
read poisons the result); C sits 256-byte aligned inside a buffer whose guard bands and stride
gaps hold a sentinel NaN payload, and a non-accumulating launch starts from an all-NaN C.  After
the launch every sentinel must be bit-identical, no described C element may be NaN, and every
element must lie within c * (|A| |B|)_ij (+ c |C0|_ij) of np.einsum in float64/complex128 -- a
missing or doubled k-step, a row stored one row down or swapped real and imaginary halves fail
that even where the normwise error is small.  The normwise bound (1e-12 double, 1e-5 single) is
checked as well.  Set CTGB_ERROR_REPORT to collect the measured ratios.

A wgmma (complex64) case also asserts the launch-time choices ctgb_tc05_launch_config reports for
this device and the real A pointer (resident B' or ring, A staging, chunking), and that a tensor map
was encoded exactly when one is predicted.
"""

import json
import os
import zlib

import numpy as np
import pytest

pytestmark = pytest.mark.gpu

from cotengra_b200 import lowering as L  # noqa: E402
from tests import kernel_cases as KC  # noqa: E402
from tests.helpers import rel_err  # noqa: E402

CASES = {c.id: c for c in KC.CASES}
REPORT = os.environ.get("CTGB_ERROR_REPORT")


def _note(key, value):
    if not REPORT:
        return
    try:
        path = os.path.abspath(REPORT)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        data = json.load(open(path)) if os.path.exists(path) else {}
        data[key] = value
        json.dump(data, open(path, "w"), indent=1, sort_keys=True)
    except Exception:
        pass


@pytest.mark.parametrize("cid", list(CASES))
def test_kernel_path(cid):
    import torch

    from cotengra_b200 import _lib

    case = CASES[cid]
    plan = KC.build_plan(case)
    assert not KC.plan_mismatches(case, plan), KC.plan_mismatches(case, plan)
    lay = KC.make_layout(case, seed=zlib.crc32(cid.encode()))
    dev = [torch.from_numpy(b).cuda() for b in lay.bufs]
    es = np.dtype(case.dtype).itemsize
    ptr = [d.data_ptr() + off * es for d, off in zip(dev, lay.offs)]
    assert ptr[2] % KC.C_ALIGN == 0
    pa, pb = (ptr[1], ptr[0]) if plan.swapped else (ptr[0], ptr[1])
    wgmma = plan.variant in L.TC05_VARIANTS
    if wgmma:
        # the launch-time choices for this device and this A pointer, and the tensor-map launch counter
        # moving exactly when a tensor map is predicted (an encode that fails shows here too)
        info = _lib.device_info()
        facts = KC.launch_facts(case, plan, pa, info["sm_count"], info["smem_optin"])
        assert not KC.launch_mismatches(case, facts), KC.launch_mismatches(case, facts)
        tmaps = _lib.tensor_map_launches()
    _lib.check(_lib.load().ctgb_contract_pair(plan.words.ctypes.data, pa, pb, ptr[2], 0))
    torch.cuda.synchronize()
    if wgmma:
        # (CTGB_NO_TENSOR_MAP, a measurement setting of the launcher, turns tensor maps off)
        tmap = facts["tm_rank"] and "CTGB_NO_TENSOR_MAP" not in os.environ
        assert _lib.tensor_map_launches() - tmaps == (1 if tmap else 0), facts
    for d, b in zip(dev[:2], lay.bufs[:2]):
        assert d.cpu().numpy().tobytes() == b.tobytes()  # operands untouched
    got, bad = KC.check_result(case, lay, dev[2].cpu().numpy())
    assert bad.size == 0, f"{bad.size} sentinel components outside C changed, first at {bad[:8]}"
    assert not np.isnan(got).any(), f"{int(np.isnan(got).sum())} described C elements NaN"
    ref, scale = KC.reference(case, lay)
    ratio = KC.error_ratio(got, ref, scale)
    _note(f"kernel_paths/{cid}", ratio)
    single = KC.is_single(case.dtype)
    assert ratio <= (KC.C_SINGLE if single else KC.C_DOUBLE), ratio
    assert rel_err(got, ref) < (1e-5 if single else 1e-12)
