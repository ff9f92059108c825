"""Constant inputs of a tree executor (cotengra's ``array_contract_expression(..., constants=...)``,
interface.py:511-574): every subtree whose leaves are all constant is contracted once, when the
executor is built, and each call contracts only what depends on the variables.

The planner works on the records that run (``exec_spec.contractions()``, stem fusion included) and
is host-side integer work:

* a node is *constant* when every leaf below it is; a constant leaf's preprocessing record
  (diagonal or sum) belongs to its subtree;
* the folded array ``F`` of a node holds its per-slice value in the node's own index order
  (``spec.inds[p]``) followed by one axis per non-projected sliced index of the subtree's leaves,
  in ``spec.sliced`` order.  The main plan reads ``F`` as an ordinary sliced input, so every slice
  selects its slab and slice ids keep their meaning; projected indices are applied while ``F`` is
  formed;
* the maximal constant subtrees are taken in decreasing order of the MACs they cost per call (per
  slice x ``nslices`` for variant nodes, once for invariant ones) and folded while ``F`` fits the
  remaining byte budget; a subtree that does not fit queues its constant children.  Leaves are never
  folded: they stay resident inputs of the main plan.

``F`` is formed by one ``ExecPlan`` over the subtree's own records, whose inputs are its constant
leaves and whose output is ``F``'s term: the carried sliced indices are sliced *output* indices of
that plan and are stacked through ``slice_out_stride``.
"""

from __future__ import annotations

import hashlib
import heapq
import math
import numbers
from dataclasses import dataclass, field

import numpy as np

from .lowering import DTYPE_SIZES, dtype_name


@dataclass
class Fold:
    """One folded constant subtree: its root's SSA id, the term and bytes of ``F``, and the MACs
    per call that the main plan no longer runs."""

    ssa: int
    term: tuple
    bytes: int
    macs: int
    leaves: tuple = field(repr=False, default=())
    records: tuple = field(repr=False, default=())
    sliced: list = field(repr=False, default_factory=list)


@dataclass
class FoldPlan:
    """The folds and the program that remains: its records, plan-input terms and the SSA id of every
    plan input (the variables, then the ``F`` arrays, then the constant leaves left unfolded)."""

    folds: list
    records: tuple
    inputs: list
    input_ids: list
    variables: tuple
    resident_leaves: tuple
    macs_unfolded: int


def check_constants(constants, shapes, dtype=None):
    """``{position: array}`` checked against the input ``shapes``: positions are ints in
    ``[0, len(shapes))``, given once, arrays of the input's full shape (``ValueError``) and, when
    ``dtype`` is given, of that dtype (``TypeError``).  A mapping or ``(position, array)`` pairs."""
    items = list(constants.items()) if hasattr(constants, "items") else list(constants)
    out = {}
    for item in items:
        try:
            pos, arr = item
        except (TypeError, ValueError):
            raise ValueError(f"constants must map input positions to arrays, got {item!r}") from None
        if isinstance(pos, bool) or not isinstance(pos, numbers.Integral) or not 0 <= pos < len(shapes):
            raise ValueError(f"constant position {pos!r} is not an input position in 0..{len(shapes) - 1}")
        pos = int(pos)
        if pos in out:
            raise ValueError(f"constant position {pos} is given twice")
        if tuple(arr.shape) != tuple(shapes[pos]):
            raise ValueError(f"constant {pos} has shape {tuple(arr.shape)}, the input {tuple(shapes[pos])}")
        if dtype is not None and dtype_name(arr.dtype) != dtype:
            raise TypeError(f"plan was built for {dtype}, constant {pos} is {arr.dtype}")
        out[pos] = arr
    return out


def _structure(ir, n_inputs):
    """Children and leaves of every SSA node of the records, and the records of each node
    (a pair record, or a leaf's preprocessing record)."""
    children, rec_of = {}, {}
    for k, (p, l, r, *_rest) in enumerate(ir):
        if r is None and l is None:
            rec_of[p] = (k,)  # preprocessing of leaf p
        else:
            children[p] = (l,) if r is None else (l, r)
            rec_of[p] = rec_of.get(p, ()) + (k,)
    leaves = {i: frozenset((i,)) for i in range(n_inputs)}

    def below(p):
        if p not in leaves:
            leaves[p] = frozenset().union(*(below(c) for c in children[p]))
        return leaves[p]

    for p in children:
        below(p)
    return children, rec_of, leaves


def plan_folds(spec, ir, constant_positions, dtype, max_bytes, cost_plan):
    """Choose the subtrees of the records ``ir`` (``spec.contractions()`` of the executed tree, whose
    ``spec.inds`` name every node's indices) to fold for the constant inputs ``constant_positions``,
    within ``max_bytes`` of ``F`` arrays (``None``: the unfolded plan's ``workspace_bytes``).
    ``cost_plan`` is the unfolded ``ExecPlan`` of ``ir`` (host-side, one node per record), which
    gives every node's MACs and whether it runs once or per slice."""
    consts = frozenset(int(i) for i in constant_positions)
    n = len(spec.inputs)
    esize = DTYPE_SIZES[dtype_name(dtype)]
    children, rec_of, leaves = _structure(ir, n)
    budget = cost_plan.workspace_bytes if max_bytes is None else int(max_bytes)
    nslices = cost_plan.nslices
    rec_macs = []
    for nd in cost_plan.nodes:
        macs = math.prod(nd["sizes"]) if nd["kind"] == 0 else 0
        rec_macs.append(macs if nd["invariant"] else macs * nslices)
    macs_unfolded = sum(rec_macs)

    def records(p):
        """every record of the subtree under p, in program order"""
        ks = set()
        stack = [p]
        while stack:
            q = stack.pop()
            ks.update(rec_of.get(q, ()))
            stack.extend(children.get(q, ()))
        return tuple(sorted(ks))

    def is_const(p):
        return leaves[p] <= consts

    node_inds = spec.inds

    def make(p):
        recs = records(p)
        lv = tuple(sorted(leaves[p]))
        ixs = set().union(*(spec.inputs[i] for i in lv))
        carried = tuple(ind for ind, _s, proj in spec.sliced if proj is None and ind in ixs)
        term = tuple(node_inds[p]) + carried
        nbytes = math.prod(spec.size_dict[ix] for ix in term) * esize
        return Fold(p, term, nbytes, sum(rec_macs[k] for k in recs), lv, tuple(ir[k] for k in recs),
                    [s for s in spec.sliced if s[0] in ixs])

    root = ir[-1][0]
    heap = []

    def push(p):
        if p in children:  # (leaves are never folded)
            f = make(p)
            heapq.heappush(heap, (-f.macs, p, f))

    stack = [root]
    while stack:  # the maximal constant subtrees
        p = stack.pop()
        if is_const(p):
            push(p)
        else:
            stack.extend(children.get(p, ()))
    folds, left = [], budget
    while heap:
        _m, p, f = heapq.heappop(heap)
        if f.bytes <= left:
            folds.append(f)
            left -= f.bytes
        else:
            for c in children[p]:
                push(c)
    folds.sort(key=lambda f: f.ssa)

    gone = set()
    for f in folds:
        gone.update(records(f.ssa))
    rest = tuple(rec for k, rec in enumerate(ir) if k not in gone)
    folded_leaves = set().union(*(f.leaves for f in folds)) if folds else set()
    variables = tuple(i for i in range(n) if i not in consts)
    resident = tuple(i for i in sorted(consts) if i not in folded_leaves)
    inputs = [spec.inputs[i] for i in variables] + [f.term for f in folds] + [spec.inputs[i] for i in resident]
    ids = list(variables) + [f.ssa for f in folds] + list(resident)
    return FoldPlan(folds, rest, inputs, ids, variables, resident, macs_unfolded)


def digest(constants, dtype):
    """sha256 of the constants' positions, shapes and values (as ``dtype``), for checkpoint tags."""
    h = hashlib.sha256()
    for pos in sorted(constants):
        x = constants[pos]
        if not isinstance(x, np.ndarray):
            x = x.detach().cpu().numpy()
        a = np.asarray(x, dtype=dtype, order="C")
        h.update(f"{pos}|{a.shape}|".encode())
        h.update(a.tobytes())
    return h.hexdigest()
