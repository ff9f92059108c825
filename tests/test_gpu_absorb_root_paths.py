"""The absorb-root kernel's other paths (csrc/absorbdot.cuh), in the guarded buffers and within the
tolerance of ``test_gpu_absorb_root``: Bs read from shared memory when the contracted c spans more
than one quarter (CCP = 64, 128), two kept Bs columns (the ring that stages 8 A rows), and KL = 1
with k' units that split unevenly over the CTAs, both fewer and many more per CTA than the ring
has stages."""

import pytest

from cotengra_b200 import lowering as L
from tests.test_gpu_absorb_root import _case, _run

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("cc,kp", [((40,), (3, 250)), ((100,), (2, 2, 37)), ((5, 25), (2, 2, 2, 2, 2, 2, 2))])
def test_shared_bs_quarters(cc, kp):
    """CK = 1 and more than 32 contracted columns: 20 distinct A rows and Bs from shared memory."""
    groups = {"rows": (20,), "ck": (), "cc": cc, "kp": kp, "k": (12,), "n": (30,)}
    terms, A, Bs, V = _case(21, groups)
    ab = _run(terms, A, Bs, V, False)
    assert int(ab.words[L.AB_CCP]) > 32


@pytest.mark.parametrize("cc,x_is_a", [((32,), False), ((2,) * 5, True), ((48,), False), ((3, 11), True)])
def test_two_kept_columns(cc, x_is_a):
    """CK = 2: rows 0-7 and 8-15 are the same A rows with the two kept Bs columns, rows 16-31 absent;
    one quarter (Bs in registers) and two (Bs in shared memory)."""
    groups = {"rows": (2, 4), "ck": (2,), "cc": cc, "kp": (2,) * 11, "k": (16,), "n": (32,)}
    terms, A, Bs, V = _case(23, groups)
    ab = _run(terms, A, Bs, V, x_is_a)
    assert int(ab.words[L.AB_M]) == 16


@pytest.mark.parametrize("kp", [(7, 45), (1000, 3)])
@pytest.mark.parametrize("rows,ck", [((3, 2), (3,)), ((5,), ())])
def test_ragged_units_single_k(rows, ck, kp):
    """KL = 1 with 8 staged A rows: 315 units (fewer per CTA than the ring's stages) and 3000 (the
    ring wraps many times), for three kept Bs columns and for 5 rows without any."""
    groups = {"rows": rows, "ck": ck, "cc": (20,), "kp": kp, "k": (7,), "n": (17,)}
    terms, A, Bs, V = _case(29, groups)
    ab = _run(terms, A, Bs, V, False, accumulate=True)
    assert int(ab.words[L.AB_KL]) == 1
