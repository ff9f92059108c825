"""Reverse mode through the tree executor: the vector-Jacobian product of a whole sliced tree
compiled into one ``ctgb_plan`` (the forward plan's type, with backward phases) whose slice
loop runs in C++/CUDA.

The plan propagates the *conjugated* cotangent ``H = conj(g)``.  For a pairwise node
``p = contract(l, r)`` torch's convention ``g_l = g_p . conj(r)^T`` becomes

    H_l = contract(H_p, r -> term_l)        H_r = contract(l, H_p -> term_r)

plain contractions without any conjugation, so every backward step is an ordinary pairwise
descriptor (``lowering.build_pair_desc``) and runs on the existing kernels.  A single-operand
node (diagonal, sum, transpose) is a real linear map: its adjoint is one single-operand
descriptor -- a sum becomes a stride-0 read, a transpose strides, a diagonal a write along
summed strides.  Conjugation happens only on a copy of the incoming cotangent and on the
finished input gradients (complex dtypes).

Schedule (``ctgb_plan_execute`` runs the phases in this order; a forward plan has 0 and 1 only):

    0  invariant forward   once per call, into the persistent arena (as ``ExecPlan`` hoists)
       -- the H accumulators of slice-invariant tensors are zeroed --
    1  variant forward     per slice; the root is not run (it only receives H_root)
    2  variant backward    per slice, nodes in reverse; H_root is the cotangent's slice view,
                           input gradients accumulate through the inputs' sliced views and the
                           H of invariant tensors accumulates in persistent buffers
    3  invariant backward  once, from the accumulated H

Only nodes on a path from the root to an input in ``wrt`` are differentiated, and a forward
node runs only if some backward step reads its value.  Intermediates live until their last
backward use; both arenas are laid out by liveness over the whole schedule (``executor.layout``,
as for forward plans).  Without a budget the per-slice arena keeps every intermediate the backward
needs.

Under a workspace budget (``max_bytes``) some per-slice forward values are dropped after phase 1
and recomputed in phase 2: a recomputation is a copy of the forward node's record (same
descriptor) with phase 2 and a fresh scratch slot, emitted right before the first phase-2 node
that reads the value and kept until its last read.  A dropped value whose operands were dropped
recomputes them first, from the nearest kept values.  Which values to drop is a greedy search on
the arena size ``executor.layout`` reports (see ``VjpPlan._fit``).

With ``strip_exponent`` and ``stripped_grad`` the plan differentiates the mantissa ``m`` of a
stripped result ``(m, e)``, ``amp = m 10^e``, with the exponent held constant:
``dm/dx = 10^-e damp/dx``.  The forward nodes keep the forward plan's lazy scheme: a pairwise
value is stored raw, ``S_p = (S_l/f_l)(S_r/f_r)``, and records ``f_p = max|S_p|``; every non-root
pairwise node runs in phase 0 or 1 so that the slice exponent without the root's factor, ``e'_s``,
is complete before phase 2.  The plan propagates ``H~ = conj(dm/dp~)`` of the normalised values
``p~ = S_p/f_p``:

    seed        H~_root = conj(g_m)[slice view] * 10^(e'_s - e)      (the divisor 10^(e - e'_s))
    pairwise    H~_l = contract(H~_p, S_r) / (f_p f_r)               (f_p: the seed at the root)
    single      H~_x = adjoint(H~_c)                                 (factor 1; seeded at the root)

Inputs have factor 1, so ``H~_x`` is ``conj(dm/dx)``.  A recomputed value divides by the phase-1
factors of its operands and records none, so it is the quotient phase 1 formed.  A slice with a
zero factor, or a zero result (``e = -inf``), contributes zero; a NaN exponent gives NaN.
"""

from __future__ import annotations

import ctypes as C
import math
import numbers

from . import _lib
from .executor import (
    K_COT,
    K_GRAD,
    K_HACC,
    K_INPUT,
    K_PERSISTENT,
    K_SCRATCH,
    PHASE_INV_BWD,
    PHASE_INV_FWD,
    PHASE_VAR_BWD,
    PHASE_VAR_FWD,
    ExecPlan,
    _DevicePlan,
    _Slot,
    _slots,
    layout,
)
from .fusion import node_time
from .lowering import (
    VAR_TF32_32x32,
    PairDims,
    build_pair_desc,
    build_single_desc,
    row_major_strides,
    split_equation,
    tensordot_terms,
)

def choose_vjp_variant(dtype, B, M, N, K):
    """``VAR_TF32_32x32`` for the single-precision backward nodes with a small result over a long
    contracted range (``H_B[K, N] = sum_m A[m, K] H_p[m, N]`` of a stem absorption), else None
    (``choose_variant``'s pick).  The dot-stream kernels keep the shapes they already serve."""
    M, N = max(M, N), min(M, N)
    if dtype not in ("float32", "complex64") or B != 1 or M > 32 or M * N < 4 or K < 1 << 14:
        return None
    if M <= 4 and N <= 4 and K >= 1 << 20:
        return None  # DOTSTREAM4
    return VAR_TF32_32x32


def _axes(term, shape, strides):
    """extent and (summed, for repeated labels) stride of every label of extent > 1"""
    ext, st = {}, {}
    for ix, d, s in zip(term, shape, strides):
        if int(d) == 1:
            continue
        ext[ix] = int(d)
        st[ix] = st.get(ix, 0) + int(s)
    return ext, st


def _is_diagonal(term, shape):
    seen = set()
    for ix, d in zip(term, shape):
        if int(d) != 1:
            if ix in seen:
                return True
            seen.add(ix)
    return False


def vjp_pair_dims(x, y, t):
    """Index classes of the backward contraction ``T[t] (+)= sum X[x] Y[y]``; each argument is
    ``(term, shape, strides)``.  Beyond ``classify_pair``:

    * a label of the target that neither operand carries (an index summed on one operand only in
      the forward) is a kept dim with stride 0 on both operands -- a broadcast, no copy;
    * a label of extent 1 on the target but longer on an operand (a size-1 broadcast in the
      forward) is contracted;
    * a label repeated on the target (a diagonal) writes along the summed strides.
    """
    (ex, sx), (ey, sy), (et, stt) = _axes(*x), _axes(*y), _axes(*t)
    order = []
    for term in (t[0], x[0], y[0]):
        for ix in term:
            if ix not in order:
                order.append(ix)
    dims = PairDims(out_shape=tuple(int(d) for d in t[1]))
    for ix in order:
        a, b = sx.get(ix, 0), sy.get(ix, 0)
        if ix in et:
            rec = [et[ix], a, b, stt[ix]]
            if ix in sx and ix in sy:
                dims.batch.append(rec)
            elif ix in sy:
                dims.n.append(rec)
            else:
                dims.m.append(rec)
        else:
            e = ex.get(ix, ey.get(ix))
            if e is not None:
                dims.k.append([e, a, b, 0])
    return dims


def vjp_single_dims(h, t):
    """Output dims ``[ext, sH, sT]`` of the adjoint of a single-operand node: ``T[t] (+)= H[h]``
    broadcast over the labels ``h`` lacks (the summed ones)."""
    (_eh, sh), (et, stt) = _axes(*h), _axes(*t)
    order = []
    for ix in t[0]:
        if ix in et and ix not in order:
            order.append(ix)
    return [[et[ix], sh.get(ix, 0), stt[ix]] for ix in order]


class VjpPlan(_DevicePlan):
    """Compile the VJP of ``contractions`` (the executed IR, stem fusion included) for fixed
    input shapes and dtype.  Same arguments as ``ExecPlan`` plus ``wrt``, the inputs that need a
    gradient (default: all; positions among the plan's inputs, as ``input_index``).  ``variant`` forces the kernel of every backward pairwise node.

    ``max_bytes`` bounds ``workspace_bytes + persistent_bytes`` by recomputing per-slice forward
    values in phase 2.  ``None``, or a budget at or above the plan's own size, gives the plan
    without recomputation.  A budget below the smallest the planner reaches raises
    ``MemoryError``.  ``recompute_macs`` are the MACs of the phase-2 forward nodes of one slice;
    ``min_bytes`` is the smallest budget the planner reached (``total_bytes`` without a budget).
    ``precision`` applies to the forward, recomputed and backward nodes alike.

    ``strip_exponent=True`` needs ``stripped_grad=True``: the plan then differentiates the mantissa
    of a stripped result with its exponent held constant (see the module notes), and ``execute``
    takes the forward's exponent.  Without ``stripped_grad`` it raises ``NotImplementedError``."""

    def __init__(self, contractions, inputs, output, size_dict, sliced=(), dtype="complex128",
                 wrt=None, strip_exponent=False, hoist=True, allow_dmma=True, sm_count=None,
                 variant=None, max_bytes=None, precision="3xtf32", stripped_grad=False, input_ids=None):
        if max_bytes is not None and (isinstance(max_bytes, bool) or not isinstance(max_bytes, numbers.Integral)
                                      or max_bytes <= 0):
            raise ValueError(f"max_bytes must be a positive integer, got {max_bytes!r}")
        if strip_exponent and not stripped_grad:
            raise NotImplementedError("gradients of strip_exponent results are only defined with "
                                      "stripped_grad=True (the exponent held constant)")
        self.strip_exponent = bool(strip_exponent)
        fwd = ExecPlan(contractions, inputs, output, size_dict, sliced, dtype=dtype, hoist=hoist,
                       allow_dmma=allow_dmma, sm_count=sm_count, precision=precision, input_ids=input_ids)
        self.fwd = fwd
        self.dtype, self.esize, self.sm_count, self.precision = fwd.dtype, fwd.esize, fwd.sm_count, fwd.precision
        self.inputs, self.output, self.sliced = fwd.inputs, fwd.output, fwd.sliced
        self.nslices, self.out_shape, self.out_elements = fwd.nslices, fwd.out_shape, fwd.out_elements
        self.slice_out_stride = fwd.slice_out_stride
        n_in = len(self.inputs)
        wrt = set(range(n_in)) if wrt is None else {int(i) for i in wrt}
        if any(i < 0 or i >= n_in for i in wrt):
            raise ValueError(f"wrt {sorted(wrt)} names inputs outside 0..{n_in - 1}")
        self.wrt = tuple(sorted(wrt))
        self._build(tuple(contractions), allow_dmma, variant, None if max_bytes is None else int(max_bytes))

    # ------------------------------------------------------------------ build
    def _build(self, contractions, allow_dmma, variant, max_bytes):
        fwd, es, dtype = self.fwd, self.esize, self.dtype
        nodes = fwd.nodes
        # local index terms of every node: [(operand, term)], output term
        ops = []
        for (p, l, r, tdot, arg, perm), nd in zip(contractions, nodes):
            if r is None:
                terms, to = split_equation(arg)
                ops.append(([(nd["a"], tuple(terms[0]))], tuple(to)))
                continue
            A, Bt = (nd["b"], nd["a"]) if nd["plan"].swapped else (nd["a"], nd["b"])
            if tdot:
                ta, tb, to = tensordot_terms((tuple(arg[0]), tuple(arg[1])), len(A.shape), len(Bt.shape), perm)
            else:
                (ta, tb), to = split_equation(arg)
            ops.append(([(A, tuple(ta)), (Bt, tuple(tb))], tuple(to)))

        # which tensors lead to an input in wrt (only they get an H)
        needs = {}
        for nd, (opl, _to) in zip(nodes, ops):
            for t, _term in opl:
                if t.kind == 0:
                    needs[id(t)] = t.input_index in self.wrt
            needs[id(nd["c"])] = any(needs[id(t)] for t, _ in opl)
        need = lambda t: needs.get(id(t), False)  # noqa: E731

        # which forward values are read (by a backward step or a forward node that runs); stripped,
        # every non-root node runs, because e'_s needs every factor
        n_nodes = len(nodes)
        value, runs = set(), [False] * n_nodes
        for i in range(n_nodes - 1, -1, -1):
            nd, (opl, _to) = nodes[i], ops[i]
            if i < n_nodes - 1 and (id(nd["c"]) in value or self.strip_exponent):
                runs[i] = True
                value.update(id(t) for t, _ in opl)
            if need(nd["c"]) and len(opl) == 2:
                (A, _), (Bt, _) = opl
                if need(A):
                    value.add(id(Bt))
                if need(Bt):
                    value.add(id(A))

        # forward values
        vals = {}
        for t in (t for opl, _ in ops for t, _ in opl):
            if t.kind == 0 and id(t) not in vals:
                vals[id(t)] = _Slot(t.shape, t.strides, K_INPUT, fwd.input_nbytes[t.input_index], t.input_index,
                                    t.slice_pos, t.slice_stride)
        for i, nd in enumerate(nodes):
            if runs[i]:
                c = nd["c"]
                kind = K_PERSISTENT if nd["invariant"] else K_SCRATCH
                vals[id(c)] = _Slot(c.shape, row_major_strides(c.shape), kind, max(math.prod(c.shape), 1) * es)

        # H of the root: the (conjugated) cotangent at the slice's output view
        sliced_inds = {s[0] for s in self.sliced}
        full_strides = row_major_strides(self.out_shape)
        root_strides = [s for ix, s in zip(self.output, full_strides) if ix not in sliced_inds]
        root = nodes[-1]
        hs = {id(root["c"]): _Slot(root["c"].shape, root_strides, K_COT, self.out_elements * es)}
        producer_invariant = {id(nd["c"]): bool(nd["invariant"]) for nd in nodes}

        def h_of(t, consumer_invariant):
            v = hs.get(id(t))
            if v is None:
                if t.kind == 0:
                    v = _Slot(t.shape, t.strides, K_GRAD, fwd.input_nbytes[t.input_index], t.input_index,
                              t.slice_pos, t.slice_stride)
                else:
                    # H of an invariant tensor read by the slice loop collects every slice
                    hoisted = producer_invariant[id(t)] and not consumer_invariant
                    kind = K_HACC if hoisted else K_SCRATCH
                    v = _Slot(t.shape, row_major_strides(t.shape), kind, max(math.prod(t.shape), 1) * es)
                hs[id(t)] = v
            return v

        fwd_nodes = {PHASE_INV_FWD: [], PHASE_VAR_FWD: []}
        for i, nd in enumerate(nodes):
            if runs[i]:
                a = vals[id(nd["a"])]
                b = vals[id(nd["b"])] if nd["b"] is not None else None
                ph = PHASE_INV_FWD if nd["invariant"] else PHASE_VAR_FWD
                rec = dict(kind=nd["kind"], a=a, b=b, c=vals[id(nd["c"])], words=nd["words"], phase=ph,
                           zero_fill=False, fwd_index=i)
                if nd["kind"] == 0:
                    rec["plan"] = nd["plan"]
                    if self.strip_exponent:
                        rec["scale"] = (a, b)  # (kept by a recomputation: the phase-1 factors)
                fwd_nodes[ph].append(rec)

        bwd_nodes = {PHASE_VAR_BWD: [], PHASE_INV_BWD: []}
        self.macs_fwd = [0, 0]  # (per slice, once per call)
        self.macs_bwd = [0, 0]
        for rec in fwd_nodes[PHASE_INV_FWD] + fwd_nodes[PHASE_VAR_FWD]:
            if rec["kind"] == 0:
                Bn, M, N, K = rec["plan"].sizes
                self.macs_fwd[rec["phase"] == PHASE_INV_FWD] += Bn * M * N * K
        for i in range(n_nodes - 1, -1, -1):
            nd, (opl, to) = nodes[i], ops[i]
            if not need(nd["c"]):
                continue
            inv = bool(nd["invariant"])
            ph = PHASE_INV_BWD if inv else PHASE_VAR_BWD
            Hc = hs[id(nd["c"])]
            hc_arg = (to, nd["c"].shape, Hc.strides)
            if len(opl) == 1:
                (X, tx), = opl
                if not need(X):
                    continue
                HX = h_of(X, inv)
                odims = vjp_single_dims(hc_arg, (tx, X.shape, HX.strides))
                diag = _is_diagonal(tx, X.shape)
                acc = HX.kind in (K_GRAD, K_HACC) or diag
                words = build_single_desc(odims, [], dtype, accumulate=acc)
                rec = dict(kind=1, a=Hc, b=None, c=HX, words=words, phase=ph,
                           zero_fill=diag and HX.kind == K_SCRATCH, fwd_index=i)
                if self.strip_exponent and i == n_nodes - 1:
                    rec["scale"] = (None,)  # None: the root's seed
                bwd_nodes[ph].append(rec)
                continue
            # stripped: H~_p divides by f_p (the seed at the root), the value read by its factor
            hp_factor = None if i == n_nodes - 1 else vals.get(id(nd["c"]))
            n_h = 0
            for (X, tx), (Y, ty) in ((opl[0], opl[1]), (opl[1], opl[0])):
                if not need(X):
                    continue
                HX = h_of(X, inv)
                Yv = vals[id(Y)]
                dims = vjp_pair_dims(hc_arg, (ty, Y.shape, Yv.strides), (tx, X.shape, HX.strides))
                diag = _is_diagonal(tx, X.shape)
                acc = HX.kind in (K_GRAD, K_HACC) or diag
                dense = 0 if acc else math.prod(X.shape)
                v = variant
                if v is None:
                    v = choose_vjp_variant(dtype, *dims.sizes())
                plan = build_pair_desc(dims, dtype, accumulate=acc, sm_count=self.sm_count,
                                       allow_dmma=allow_dmma, c_dense_elems=dense, variant=v,
                                       precision=self.precision)
                a, b = (Yv, Hc) if plan.swapped else (Hc, Yv)
                rec = dict(kind=0, a=a, b=b, c=HX, words=plan.words, phase=ph,
                           zero_fill=diag and HX.kind == K_SCRATCH, plan=plan, fwd_index=i)
                if self.strip_exponent:
                    rec["scale"] = (Yv, hp_factor) if plan.swapped else (hp_factor, Yv)
                bwd_nodes[ph].append(rec)
                n_h += 1
            if n_h:
                Bn, M, N, K = nd["plan"].sizes
                self.macs_bwd[inv] += n_h * Bn * M * N * K

        sched = (fwd_nodes[PHASE_INV_FWD] + [None] + fwd_nodes[PHASE_VAR_FWD] + bwd_nodes[PHASE_VAR_BWD]
                 + bwd_nodes[PHASE_INV_BWD])
        self.n_backward_nodes = len(bwd_nodes[PHASE_VAR_BWD]) + len(bwd_nodes[PHASE_INV_BWD])
        self.differentiated = sorted({nd["fwd_index"] for nd in sched if nd is not None and nd["phase"] >= PHASE_VAR_BWD})
        # the conjugated cotangent copy comes first in the persistent arena
        cot_bytes = self.out_elements * self.esize if self.dtype.startswith("complex") else 0
        sizes = layout(sched, cot_bytes)
        self.recompute_macs = 0
        self.min_bytes = sizes[0] + sizes[1]
        if max_bytes is not None and sizes[0] + sizes[1] > max_bytes:
            sched, sizes = self._fit(fwd_nodes, bwd_nodes, cot_bytes, sizes, max_bytes)
        self.nodes = [nd for nd in sched if nd is not None]
        self.tensors = _slots(sched)
        self.workspace_bytes, self.persistent_bytes, self.cotangent_offset = sizes
        if self.strip_exponent:
            # factor slot of every operand a node divides by: a tensor slot, or the seed (n_tensors)
            self._scale_slots()
        self._marshal()

    # ------------------------------------------------------------------ recomputation
    def _fit(self, fwd_nodes, bwd_nodes, cot_bytes, sizes, max_bytes):
        """The schedule with recomputation that fits ``max_bytes`` at the least estimated recompute
        time the greedy search finds, and its ``layout``.

        The candidates are the per-slice values a phase-2 node reads that take at least 1/1024 of
        the unbudgeted arena (the stem tensors; smaller values stay kept).  Starting from every
        candidate kept, each step drops the candidate with the largest arena reduction per second of
        added recompute time (``fusion.node_time``), or, where no single drop lowers the arena, the
        largest reduction of the bytes x schedule positions held.  The search runs until no
        candidate is left or no drop helps, so ``min_bytes`` is the smallest arena along its path;
        the plan is the first state of the path within the budget."""
        var_fwd, var_bwd = fwd_nodes[PHASE_VAR_FWD], bwd_nodes[PHASE_VAR_BWD]
        producer = {id(rec["c"]): rec for rec in var_fwd}
        saved = {}
        for nd in var_bwd:
            for s in (nd["a"], nd["b"]):
                if s is not None and id(s) in producer:
                    saved[id(s)] = s
        cost = {}
        for rec in var_fwd:
            elems = sum(math.prod(s.shape) for s in (rec["a"], rec["b"], rec["c"]) if s is not None)
            Bn, M, N, K = rec["plan"].sizes if rec["kind"] == 0 else (1, math.prod(rec["c"].shape), 1, 1)
            cost[id(rec["c"])] = (node_time(self.dtype, Bn, M, N, K, elems), Bn * M * N * K if rec["kind"] == 0 else 0)
        head, tail = fwd_nodes[PHASE_INV_FWD] + [None], bwd_nodes[PHASE_INV_BWD]

        def schedule(dropped):
            # phase 1 forms the kept values and what they are formed from (stripped: every factor)
            kept = saved.keys() - dropped
            want, run1 = set(kept), []
            for rec in reversed(var_fwd):
                if id(rec["c"]) in want or self.strip_exponent:
                    run1.append(rec)
                    want.update(id(s) for s in (rec["a"], rec["b"]) if s is not None)
            run1.reverse()
            # phase 2 recomputes every other per-slice value where it is first read again
            mat, run2, t_rec = {}, [], [0.0, 0]

            def get(s):
                if s is None or id(s) not in producer or id(s) in kept:
                    return s
                r = mat.get(id(s))
                if r is None:
                    rec = producer[id(s)]
                    a, b = get(rec["a"]), get(rec["b"])
                    r = mat[id(s)] = _Slot(s.shape, s.strides, K_SCRATCH, s.nbytes)
                    run2.append(dict(rec, a=a, b=b, c=r, phase=PHASE_VAR_BWD, recompute=True))
                    t_rec[0] += cost[id(s)][0]
                    t_rec[1] += cost[id(s)][1]
                return r

            for nd in var_bwd:
                a, b = get(nd["a"]), get(nd["b"])
                run2.append(nd if a is nd["a"] and b is nd["b"] else dict(nd, a=a, b=b))
            sched = head + run1 + run2 + tail
            ws, ps, off = layout(sched, cot_bytes)
            held = sum(t.nbytes * (t.last_use - t.first_use + 1) for t in _slots(sched) if t.kind == K_SCRATCH)
            return sched, (ws, ps, off), ws + ps, t_rec[0], held, t_rec[1]

        total0 = sizes[0] + sizes[1]
        cands = [k for k, s in saved.items() if s.nbytes * 1024 >= total0]
        dropped = frozenset()
        state = (total0, 0.0, sum(t.nbytes * (t.last_use - t.first_use + 1)
                                  for t in _slots(head + var_fwd + var_bwd + tail) if t.kind == K_SCRATCH))
        path = [(total0, dropped)]
        while cands:
            best = None
            for k in cands:
                _s, _z, total, t, held, _m = schedule(dropped | {k})
                dt = max(t - state[1], 0.0) + 1e-6
                key = (total < state[0], (state[0] - total) / dt if total < state[0] else (state[2] - held) / dt)
                if best is None or key > best[0]:
                    best = (key, k, (total, t, held))
            if not best[0][0] and best[2][2] >= state[2]:
                break  # no drop lowers the arena or the bytes held
            dropped = dropped | {best[1]}
            cands.remove(best[1])
            state = best[2]
            path.append((state[0], dropped))
        self.min_bytes = min(total for total, _d in path)
        fits = [d for total, d in path if total <= max_bytes]
        if not fits:
            err = MemoryError(f"the VJP plan needs at least {self.min_bytes} bytes with recomputation "
                              f"(min_bytes), {total0} without; the budget is {max_bytes}")
            err.min_bytes, err.total_bytes = self.min_bytes, total0
            raise err
        sched, sizes, _total, _t, _held, self.recompute_macs = schedule(fits[0])
        return sched, sizes

    # ------------------------------------------------------------------ work
    def vjp_macs(self, count):
        """Scalar MACs of one call over ``count`` slices: the recomputed forward (root excluded)
        plus, for every differentiated pairwise node, its MACs times the number of H it forms."""
        return (self.macs_fwd[0] + self.macs_bwd[0]) * count + self.macs_fwd[1] + self.macs_bwd[1]

    def variants(self, phases=(PHASE_VAR_BWD, PHASE_INV_BWD)):
        """Kernel variants of the pairwise nodes of the given phases (the backward ones by default)."""
        return [int(nd["words"][32]) for nd in self.nodes if nd["kind"] == 0 and nd["phase"] in phases]

    # ------------------------------------------------------------------ device side
    def execute(self, input_ptrs, cot_ptr, grad_ptrs, ws_ptr, ws_bytes, begin, step, count, stream=0,
                exp_ptr=None):
        """``exp_ptr``: stripped plans, the device double holding the forward's exponent."""
        lib = _lib.load()
        arr = (C.c_void_p * len(input_ptrs))(*input_ptrs)
        grads = (C.c_void_p * len(grad_ptrs))(*grad_ptrs)
        _lib.check(lib.ctgb_plan_execute(self.handle, arr, None, exp_ptr, cot_ptr, grads, ws_ptr, ws_bytes,
                                         int(begin), int(step), int(count), stream))
