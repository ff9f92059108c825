import importlib.util
import os
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def pytest_configure(config):
    config.addinivalue_line(
        "markers", "gpu: needs a CUDA device (an H100: run with -m gpu)"
    )
    config.addinivalue_line(
        "markers", "multigpu: needs >= 2 GPUs; skipped otherwise"
    )
    config.addinivalue_line(
        "markers",
        "reference: needs the cotengra package, installed into oracle/_ref/ by build() "
        "(oracle/build_ref.py) or importable; skipped otherwise",
    )


def pytest_collection_modifyitems(config, items):
    have_ref = (os.path.isfile(os.path.join(ROOT, "oracle", "_ref", "cotengra", "__init__.py"))
                or importlib.util.find_spec("cotengra") is not None)
    skip_ref = pytest.mark.skip(reason="cotengra is neither in oracle/_ref/ nor installed")
    have_gpu = None
    for item in items:
        if "reference" in item.keywords and not have_ref:
            item.add_marker(skip_ref)
        if "gpu" in item.keywords:
            if have_gpu is None:
                have_gpu = _gpu_ready()
            if have_gpu is not True:
                item.add_marker(pytest.mark.skip(reason=have_gpu))


def _gpu_ready():
    """True, or the reason the ``gpu`` tests cannot run here: a plain ``pytest`` on a machine
    without CUDA skips them instead of failing 200+ times.  With a GPU present they always
    run -- a missing ``libctgb200.so`` must fail loudly there, never skip."""
    try:
        import torch

        if not torch.cuda.is_available():
            return "no CUDA device"
    except Exception as exc:  # pragma: no cover
        return f"torch unavailable: {exc}"
    return True
