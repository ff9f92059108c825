"""Install the unmodified reference (jcmgray/cotengra, pure Python) into ``oracle/_ref/``.

The drop-in tests (``tests/test_dropin_reference.py``) drive cotengra's own control flow
(``ctg.einsum``, ``ContractionTree.contract``) with this package behind it, so they need the
reference itself, not golden data.  ``__graft_entry__.build()`` runs this recipe; ``oracle/_ref/``
is a build product and stays out of git.  The source checkout is ``$COTENGRA_SRC`` (default
``/root/reference``); without one nothing is installed and those tests skip.  The reference's one
dependency, ``autoray``, is stood in for by ``oracle/refshim``.
"""

import os
import shutil

HERE = os.path.dirname(os.path.abspath(__file__))
DEST = os.path.join(HERE, "_ref")


def build(src=None):
    """Copy the ``cotengra`` package of the reference checkout to ``oracle/_ref/cotengra``.
    Returns the installed package directory, or None when no checkout is available."""
    src = src or os.environ.get("COTENGRA_SRC", "/root/reference")
    pkg = os.path.join(src, "cotengra")
    if not os.path.isfile(os.path.join(pkg, "__init__.py")):
        return None
    out = os.path.join(DEST, "cotengra")
    if os.path.isdir(out):
        shutil.rmtree(out)
    shutil.copytree(pkg, out, ignore=shutil.ignore_patterns("__pycache__", "*.pyc"))
    return out


if __name__ == "__main__":
    print(build() or "no reference checkout found: nothing installed")
