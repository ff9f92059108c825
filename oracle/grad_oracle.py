"""Gradient oracle: the reference IR walked node by node with ``torch.einsum`` /
``torch.tensordot`` on CPU tensors (complex128 / float64) under torch autograd.

It mirrors ``ctg_oracle.run_contractions`` and ``ctg_oracle.contract_tree`` -- the slice
loop by view indexing of the inputs (projected indices included), the sum over inner sliced
indices and the stack over sliced output indices -- and shares nothing with the product's
planner or with the descriptor emulator.  Gradients come from ``torch.autograd.grad`` and so
follow torch's complex convention.
"""

import string

import torch

from oracle import ctg_oracle as orc

_LETTERS = string.ascii_letters


def _einsum(eq, *xs):
    # the reference's symbols may lie outside a-zA-Z: relabel them for torch.einsum
    lhs, out = eq.split("->") if "->" in eq else (eq, None)
    if out is None:
        flat = lhs.replace(",", "")
        out = "".join(c for c in sorted(set(flat)) if flat.count(c) == 1)
    chars = []
    for c in lhs + out:
        if c != "," and c not in chars:
            chars.append(c)
    table = {c: _LETTERS[i] for i, c in enumerate(chars)}
    tr = lambda s: "".join(table.get(c, c) for c in s)  # noqa: E731
    return torch.einsum(f"{tr(lhs)}->{tr(out)}", *xs)


def run_contractions(contractions, arrays):
    """``ctg_oracle.run_contractions`` on torch tensors (differentiable)."""
    live = dict(enumerate(arrays))
    out = None
    for p, l, r, tdot, arg, perm in contractions:
        if r is None:
            if l is None:
                live[p] = _einsum(arg, live[p])
                continue
            return _einsum(arg, live[l])
        x, y = live.pop(l), live.pop(r)
        if tdot:
            out = torch.tensordot(x, y, dims=(list(arg[0]), list(arg[1])))
            if perm:
                out = out.permute(*perm)
        else:
            out = _einsum(arg, x, y)
        live[p] = out
    return out


def slice_arrays(inputs, sliced, arrays, i):
    key = orc.slice_key(sliced, i)
    out = list(arrays)
    for c, term in enumerate(inputs):
        if any(ix in key for ix in term):
            out[c] = arrays[c][tuple(key.get(ix, slice(None)) for ix in term)]
    return out


def contract_tree(inputs, output, sliced, contractions, arrays, slice_ids=None):
    """``ctg_oracle.contract_tree`` on torch tensors: per-slice results summed, and stacked over
    sliced output indices.  With ``slice_ids`` the slices left out contribute zeros, so that the
    result keeps the full output's shape."""
    if not sliced:
        return run_contractions(contractions, arrays)
    n = orc.num_slices(sliced)
    ids = range(n) if slice_ids is None else slice_ids
    where = [ix for ix in output if any(ix == s[0] for s in sliced)]
    if not where:
        total = None
        for i in ids:
            r = run_contractions(contractions, slice_arrays(inputs, sliced, arrays, i))
            total = r if total is None else total + r
        return total
    chunks = {}
    for i in ids:
        key = orc.slice_key(sliced, i)
        k = tuple(key[ix] for ix in where)
        r = run_contractions(contractions, slice_arrays(inputs, sliced, arrays, i))
        chunks[k] = chunks[k] + r if k in chunks else r
    info = {s[0]: s for s in sliced}
    pos = {ix: output.index(ix) for ix in where}

    like = next(iter(chunks.values()))

    def stack(prefix, rest):
        if not rest:
            return chunks[prefix] if prefix in chunks else torch.zeros_like(like)
        _ind, size, project = info[rest[0]]
        values = range(size) if project is None else [project]
        return torch.stack([stack(prefix + (d,), rest[1:]) for d in values], pos[rest[0]] - len(prefix))

    return stack((), tuple(where))


def tree_gradients(inputs, output, sliced, contractions, arrays, cotangent, wrt=None, slice_ids=None):
    """Gradients of ``<cotangent, contract_tree(...)>`` with respect to the inputs ``wrt``
    (default all): a list with ``None`` outside ``wrt``; numpy in, numpy out."""
    wrt = set(range(len(arrays))) if wrt is None else set(wrt)
    ts = [torch.tensor(a).requires_grad_(i in wrt) for i, a in enumerate(arrays)]
    out = contract_tree([tuple(t) for t in inputs], tuple(output), sliced, contractions, ts, slice_ids)
    cot = torch.as_tensor(cotangent).reshape(out.shape).to(out.dtype)
    req = [t for t in ts if t.requires_grad]
    grads = torch.autograd.grad(out, req, grad_outputs=cot, allow_unused=True)
    it = iter(grads)
    res = []
    for i, t in enumerate(ts):
        if i in wrt:
            g = next(it)
            res.append(torch.zeros_like(t).numpy() if g is None else g.detach().numpy())
        else:
            res.append(None)
    return res
