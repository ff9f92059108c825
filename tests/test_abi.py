"""The C-ABI shared library loads (no GPU needed) and exports every symbol that
``include/ctg_b200.h`` declares."""

import ctypes
import os
import re

import pytest

from cotengra_b200 import _lib, lowering

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    src = open(os.path.join(ROOT, "include", "ctg_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(ctgb_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_header_symbols():
    lib = _lib.load()
    names = _declared()
    assert len(names) >= 14
    for name in names:
        assert hasattr(lib, name), name
    assert set(names) == set(_lib.EXPORTS)


def test_layout_constants_agree():
    lib = _lib.load()
    assert lib.ctgb_abi_version() == 2
    assert lib.ctgb_desc_words() == lowering.DESC_WORDS
    assert lib.ctgb_single_desc_words() == lowering.SDESC_WORDS


def test_fails_loudly_without_device():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    with pytest.raises(RuntimeError):
        _lib.device_info()
    import numpy as np

    import cotengra_b200 as cb

    with pytest.raises(RuntimeError):
        cb.einsum("ab,bc->ac", np.ones((2, 2)), np.ones((2, 2)))
