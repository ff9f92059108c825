"""Forward mode through the tree executor: the Jacobian-vector product of a whole sliced tree
compiled into one ``ctgb_plan`` (the forward plan's type, with tangent slots) whose slice loop runs
in C++/CUDA.

The tree is multilinear in its inputs, so the tangent of a pairwise node ``p = contract(l, r)`` is

    p' = contract(l', r) + contract(l, r')

two ordinary pairwise contractions with the node's own descriptor: a tangent has the shape and
row-major strides of its value, and the tangent of an input those of the input.  A single-operand
node (diagonal, sum, transpose) is linear: its tangent is the same descriptor applied to the
tangent.  An absorb-root node ``(A . Bs) . V`` is linear in each of its three operands: one launch
per operand that carries a tangent.

A node carries a tangent when an input in ``wrt`` lies below it; only those nodes get tangent
records.  A node with one tangent child gets one launch.  When both children carry one and the
node runs on a stream kernel (``VAR_ROWSTREAM``, ``VAR_ROWSTREAM_K``, ``VAR_DMMASTREAM``), both
terms go into one two-term node (kind 2, ``ctgb_contract_pair2``): the kernel streams the rows of
``l'`` and ``l`` together and stores ``p'`` once.  Every other variant runs the second term as a
second launch with the descriptor's accumulate bit set.

Schedule: the forward plan's nodes, each followed by its tangent records in the same phase, so a
slice-invariant tangent is formed once per call in phase 0 like a hoisted value.  The root's
tangent uses the root's descriptor and accumulates over the slices into the tangent output (kind
8, the output's slice view), so ``accumulate="double"``, sliced output indices and the chunk
descriptor of a dense root apply to it unchanged.  Both arenas are laid out by liveness
(``executor.layout``).

With ``strip_exponent`` and ``stripped_grad`` the plan forms the tangent of the mantissa ``m`` of a
stripped result ``(m, e)`` with the exponent held constant, ``dm = 10^-e d(amp)``.  The primal
records are the stripped forward plan's, descriptor for descriptor: a pairwise value is stored raw,
``S_p = (S_l/f_l)(S_r/f_r)``, and records ``f_p = max|S_p|``.  Each tangent is defined with the same
factors,

    T_p = (T_l S_r + S_l T_r) / (f_l f_r)

one scale shared by both terms, the one its primal node uses; a tangent record divides by its
primal node's two factor slots and records no factor of its own (``tangent_marks``,
``ctgb_plan_set_tangent_scale_slots``).  A one-term record takes the forward's stripped launch path
(a pre-scaled small operand, reusing the copy its primal node has just made, or epilogue scaling); a
two-term record scales B and B' as the kernel stages them.  The primal root always runs, since its
factor sets the slice exponent ``e_s``.  The raw tangent root ``T_s`` is folded against a running
exponent of its own, ``Et' = max(Et, e'_s)``: ``tout <- tout 10^(Et - Et') + T_s 10^(e'_s - Et')``,
``e'_s`` being the slice exponent without the root's factor, and after the slices ``tout`` is brought
to the mantissa's exponent ``E`` once.  ``e'_s`` is finite whenever the factors below the root are,
so a slice whose amplitude is exactly zero keeps its tangent in any slice order.  A slice with a zero
factor below its root adds nothing, a zero result (``E = -inf``) gives a zero tangent, and a NaN
exponent gives NaN.
"""

from __future__ import annotations

import ctypes as C

import numpy as np

from . import _lib
from .executor import (
    K_INPUT,
    K_OUTPUT,
    K_PERSISTENT,
    K_SCRATCH,
    K_TANGENT,
    K_TOUT,
    ExecPlan,
    _DevicePlan,
    _Slot,
    _slots,
    layout,
)
from .lowering import (
    S_FLAGS,
    VAR_DMMASTREAM,
    VAR_ROWSTREAM,
    VAR_ROWSTREAM_K,
    W_FLAGS,
    W_KTA,
    W_NTA,
    W_VARIANT,
)


def two_term_fits(words):
    """Whether the pair descriptor ``words`` runs in the two-term form (``ctgb_contract_pair2``):
    a row-stream node, or a DMMA stream node whose k range fits two copies of B in shared memory
    (csrc/dmmastream.cuh ``ds_two_kb``)."""
    v = int(words[W_VARIANT])
    if v in (VAR_ROWSTREAM, VAR_ROWSTREAM_K):
        return True
    if v != VAR_DMMASTREAM:
        return False
    n = int(words[W_NTA])
    nj = 1 if n <= 8 else 2 if n <= 16 else 4 if n <= 32 else 8
    return int(words[W_KTA]) <= (64 if nj <= 2 else 32 if nj == 4 else 16)


def _accumulating(words, kind):
    """A copy of ``words`` with the accumulate bit set (flags bit 0 of either descriptor kind)."""
    w = np.array(words, dtype=np.int64)
    w[W_FLAGS if kind == 0 else S_FLAGS] |= 1
    return w


class JvpPlan(_DevicePlan):
    """Compile the JVP of ``contractions`` (the executed IR, stem fusion included) for fixed input
    shapes and dtype.  Same arguments as ``ExecPlan`` plus ``wrt``, the inputs that carry a tangent
    (default: all; positions among the plan's inputs).  ``precision``, ``accumulate`` and
    ``absorb_root`` apply to the tangent nodes as to the values.  ``strip_exponent=True`` needs
    ``stripped_grad=True``: the plan then forms the tangent of the mantissa with the exponent held
    constant (see the module notes; ``absorb_root`` stays off) and ``execute`` takes an exponent
    buffer.  Without ``stripped_grad`` it raises ``NotImplementedError``.

    ``_two_term=False`` runs every two-term node as two launches (for measuring the two forms)."""

    def __init__(self, contractions, inputs, output, size_dict, sliced=(), dtype="complex128", wrt=None,
                 strip_exponent=False, hoist=True, allow_dmma=True, sm_count=None, variant=None,
                 precision="3xtf32", accumulate="native", absorb_root=False, input_ids=None, stripped_grad=False,
                 _two_term=True):
        if strip_exponent and not stripped_grad:
            raise NotImplementedError("forward-mode derivatives of strip_exponent results are only defined with "
                                      "stripped_grad=True (the exponent held constant)")
        self.strip_exponent = bool(strip_exponent)
        fwd = ExecPlan(contractions, inputs, output, size_dict, sliced, dtype=dtype, strip_exponent=strip_exponent,
                       hoist=hoist, allow_dmma=allow_dmma, sm_count=sm_count, variant=variant, precision=precision,
                       accumulate=accumulate, absorb_root=absorb_root, input_ids=input_ids)
        self.fwd = fwd
        for k in ("dtype", "esize", "sm_count", "precision", "acc_dtype", "wide", "inputs", "output", "sliced",
                  "nslices", "out_shape", "out_elements", "slice_out_stride", "_chunk_words"):
            setattr(self, k, getattr(fwd, k))
        n_in = len(self.inputs)
        wrt = set(range(n_in)) if wrt is None else {int(i) for i in wrt}
        if any(i < 0 or i >= n_in for i in wrt):
            raise ValueError(f"wrt {sorted(wrt)} names inputs outside 0..{n_in - 1}")
        self.wrt = tuple(sorted(wrt))
        self._build(bool(_two_term))

    def _build(self, two_term):
        fwd = self.fwd
        strip = self.strip_exponent
        tan = {}
        for nd in fwd.nodes:
            for t in (nd["a"], nd["b"], nd.get("d")):
                if t is not None and t.kind == K_INPUT and t.input_index in self.wrt and id(t) not in tan:
                    tan[id(t)] = _Slot(t.shape, t.strides, K_TANGENT, fwd.input_nbytes[t.input_index],
                                       t.input_index, t.slice_pos, t.slice_stride)
        phases = {0: [], 1: []}
        self.tangent_nodes, self.two_term_nodes = [], 0
        for i, nd in enumerate(fwd.nodes):
            rec = {k: nd[k] for k in ("kind", "a", "b", "c", "words", "phase", "root")}
            if nd.get("d") is not None:
                rec["d"] = nd["d"]
            if strip and nd["kind"] == 0:
                rec["scale"] = (nd["a"], nd["b"])  # (the forward's own: its operands' factors)
            phases[nd["phase"]].append(rec)
            a, b, d, c = nd["a"], nd["b"], nd.get("d"), nd["c"]
            ta, tb, td = (tan.get(id(t)) if t is not None else None for t in (a, b, d))
            if ta is None and tb is None and td is None:
                continue
            if c.kind == K_OUTPUT:
                tc = _Slot(c.shape, c.strides, K_TOUT, c.nbytes)
            elif nd["root"]:
                # a dense root (folded into the output after the slice): persistent, so that it cannot
                # share bytes with the dense primal root, which the fold reads as well
                tc = _Slot(c.shape, c.strides, K_PERSISTENT, c.nbytes)
            else:
                tc = _Slot(c.shape, c.strides, K_PERSISTENT if nd["invariant"] else K_SCRATCH, c.nbytes)
            tan[id(c)] = tc
            if nd["kind"] == 1:
                terms = [dict(a=ta, b=None)]
            elif d is not None:  # absorb-root (A . Bs) . V: A in a, V in b, Bs in d
                terms = [dict(a=x, b=y, d=z) for t, (x, y, z) in zip((ta, tb, td), ((ta, b, d), (a, tb, d), (a, b, td)))
                         if t is not None]
            elif ta is not None and tb is not None and two_term and two_term_fits(nd["words"]):
                terms = [dict(kind=2, a=ta, b=b, a2=a, b2=tb)]
                self.two_term_nodes += 1
            else:
                terms = [dict(a=x, b=y) for t, (x, y) in zip((ta, tb), ((ta, b), (a, tb))) if t is not None]
            for k, t in enumerate(terms):
                words = nd["words"] if k == 0 else _accumulating(nd["words"], nd["kind"])
                trec = dict(kind=nd["kind"], c=tc, words=words, phase=nd["phase"], root=2 if nd["root"] else 0,
                            fwd_index=i)
                trec.update(t)  # (a two-term record sets kind 2)
                if strip and nd["kind"] == 0:
                    trec["scale"] = (a, b)  # the primal node's factors; a tangent records none
                phases[nd["phase"]].append(trec)
                self.tangent_nodes.append(trec)
        sched = phases[0] + [None] + phases[1]
        self.nodes = [nd for nd in sched if nd is not None]
        self.tensors = _slots(sched)
        self.workspace_bytes, self.persistent_bytes, _ = layout(sched)
        self.differentiated = sorted({nd["fwd_index"] for nd in self.tangent_nodes})
        if strip:
            self._scale_slots()
            self.tangent_marks = [int("fwd_index" in nd) for nd in self.nodes]
        self._marshal()

    def variants(self):
        """Kernel variants of the pairwise tangent records (two-term ones included)."""
        return [int(nd["words"][W_VARIANT]) for nd in self.tangent_nodes if nd["kind"] != 1]

    # ------------------------------------------------------------------ device side
    def execute(self, input_ptrs, tangent_ptrs, out_ptr, tangent_out_ptr, ws_ptr, ws_bytes, begin, step, count,
                stream=0, exp_ptr=None):
        """``tangent_ptrs``: one device pointer per plan input, ``None`` outside ``wrt``; ``out_ptr``
        may be ``None`` (the primal root is then not run).  A stripped plan needs ``out_ptr`` and
        ``exp_ptr``, the device double of the running exponent (``ctgb_plan_execute_jvp_stripped``)."""
        lib = _lib.load()
        arr = (C.c_void_p * len(input_ptrs))(*input_ptrs)
        tans = (C.c_void_p * len(tangent_ptrs))(*tangent_ptrs)
        if self.strip_exponent:
            _lib.check(lib.ctgb_plan_execute_jvp_stripped(self.handle, arr, tans, out_ptr, tangent_out_ptr, exp_ptr,
                                                          ws_ptr, ws_bytes, int(begin), int(step), int(count),
                                                          stream))
            return
        _lib.check(lib.ctgb_plan_execute_jvp(self.handle, arr, tans, out_ptr, tangent_out_ptr, ws_ptr, ws_bytes,
                                             int(begin), int(step), int(count), stream))

