"""Helpers shared by the golden generator (``oracle/gen_golden.py``) and the
tests: deterministic synthetic arrays and golden-file decoding."""

import json
import os

import numpy as np

GOLDEN_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def make_arrays(shapes, dtype="complex128", seed=0, scale=1.0):
    """Seeded synthetic operands: uniform(-1, 1) real parts (plus imaginary
    parts for complex dtypes), generated in float64 then cast, so that every
    dtype sees the same underlying values."""
    rng = np.random.default_rng(seed)
    dtype = np.dtype(dtype)
    arrays = []
    for shape in shapes:
        shape = tuple(int(d) for d in shape)
        x = rng.uniform(-1.0, 1.0, size=shape)
        if dtype.kind == "c":
            x = x + 1j * rng.uniform(-1.0, 1.0, size=shape)
        arrays.append(np.asarray(x * scale).astype(dtype))
    return arrays


def load_json(name):
    with open(os.path.join(GOLDEN_DIR, name)) as f:
        return json.load(f)


def load_npz(name):
    return np.load(os.path.join(GOLDEN_DIR, name))


def decode_ir(contractions):
    """JSON -> the reference's contraction records ``(p, l, r, tdot, arg,
    perm)`` with tuples restored."""
    out = []
    for p, l, r, tdot, arg, perm in contractions:
        if tdot:
            arg = (tuple(arg[0]), tuple(arg[1]))
        if perm is not None:
            perm = tuple(perm)
        out.append((p, l, r, bool(tdot), arg, perm))
    return tuple(out)


def decode_sliced(sliced):
    return [(ind, int(size), None if project is None else int(project))
            for ind, size, project in sliced]


def tree_spec(rec):
    """The ``cotengra_b200.TreeSpec`` of a golden tree record (``trees.json``)."""
    import cotengra_b200 as cb

    n_in = len(rec["inputs"])
    node_inds = {int(k): v for k, v in rec["inds"].items() if int(k) >= n_in}
    return cb.TreeSpec(rec["inputs"], rec["output"], rec["size_dict"], rec["path"],
                       decode_sliced(rec["sliced"]), node_inds)


def rel_err(x, ref):
    x = np.asarray(x)
    ref = np.asarray(ref)
    den = np.max(np.abs(ref))
    if den == 0:
        return float(np.max(np.abs(x))) if x.size else 0.0
    return float(np.max(np.abs(x - ref)) / den)


def jvp_oracle(spec, contractions, arrays, tangents, wrt, slice_ids=None):
    """The exact JVP of a multilinear tree: ``sum_{i in wrt} f(x_1, ..., v_i, ..., x_n)`` through the
    torch-CPU oracle (``oracle/grad_oracle.py``), in the arrays' dtype."""
    import torch

    from oracle import grad_oracle as go

    total = 0
    for i, t in zip(wrt, tangents):
        xs = [torch.tensor(t if j == i else a) for j, a in enumerate(arrays)]
        total = total + go.contract_tree(spec.inputs, spec.output, spec.sliced, contractions, xs,
                                         slice_ids=slice_ids).detach().numpy()
    return np.asarray(total)
