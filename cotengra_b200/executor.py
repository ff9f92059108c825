"""Whole-tree execution plans: the reference's linear contraction IR
(cotengra/contract.py:573-651) compiled into one ``ctgb_plan`` whose node loop
(contract.py:791-832) and slice loop (core.py:4015-4030) run in C++/CUDA.

Planning is host-side integer work:

* shapes are propagated through the IR and every node is lowered to a strided
  descriptor (``lowering.py``) -- sliced inputs are *views* of the unsliced
  arrays (base offset per slice + strides of the kept axes, core.py:3811-3817),
  so slicing moves no data;
* nodes whose subtree touches no sliced input are marked slice-invariant and run
  once per execute call into a persistent arena (the reference recontracts them
  for every slice, core.py:4015-4028);
* intermediates are placed in a workspace arena by liveness (children die when
  their parent is formed, contract.py:806-807);
* the root writes straight into the output view selected by the digits of
  sliced *output* indices (gather_slices' stack, core.py:3865-3876) and
  accumulates over inner sliced indices (core.py:3842-3844).

Every node carries the phase it runs in: 0 (invariant forward, once per call)
and 1 (variant forward, per slice) here; a reverse-mode plan (``vjp.py``) adds
2 (variant backward) and 3 (invariant backward); a forward-mode plan (``jvp.py``)
adds tangent records to phases 0 and 1.  All plan kinds are one
``ctgb_plan`` type, laid out by ``layout`` and marshalled and uploaded by
``_DevicePlan``.
"""

from __future__ import annotations

import ctypes as C
import math

import numpy as np

from . import _lib, lowering
from .lowering import (
    DTYPE_CODES,
    DTYPE_SIZES,
    accumulator_dtype,
    build_pair_desc,
    build_single_desc,
    check_precision,
    check_tensordot_shapes,
    classify_pair,
    classify_single,
    dtype_name,
    row_major_strides,
    split_equation,
    tensordot_terms,
)

ALIGN = 256
# node phases and tensor kinds of a plan (include/ctg_b200.h)
PHASE_INV_FWD, PHASE_VAR_FWD, PHASE_VAR_BWD, PHASE_INV_BWD = 0, 1, 2, 3
LOOP_PHASES = (PHASE_VAR_FWD, PHASE_VAR_BWD)  # run once per slice
K_INPUT, K_SCRATCH, K_PERSISTENT, K_OUTPUT, K_COT, K_GRAD, K_HACC = 0, 1, 2, 3, 4, 5, 6
K_TANGENT, K_TOUT = 7, 8  # forward mode (jvp.py): an input's tangent, the output's tangent


def _align(x):
    return (x + ALIGN - 1) // ALIGN * ALIGN


class _Arena:
    """Offset allocator over a linear schedule (best fit + coalescing frees)."""

    def __init__(self):
        self.free = []  # sorted (offset, size)
        self.top = 0
        self.peak = 0

    def alloc(self, size):
        size = _align(max(size, 1))
        best = None
        for i, (off, sz) in enumerate(self.free):
            if sz >= size and (best is None or sz < self.free[best][1]):
                best = i
        if best is not None:
            off, sz = self.free.pop(best)
            if sz > size:
                self.free.append((off + size, sz - size))
                self.free.sort()
            return off
        # extend, reusing a trailing free block if there is one
        if self.free and self.free[-1][0] + self.free[-1][1] == self.top:
            off, sz = self.free.pop()
            self.top = off + size
        else:
            off = self.top
            self.top += size
        self.peak = max(self.peak, self.top)
        return off

    def release(self, off, size):
        size = _align(max(size, 1))
        self.free.append((off, size))
        self.free.sort()
        merged = []
        for o, s in self.free:
            if merged and merged[-1][0] + merged[-1][1] == o:
                merged[-1] = (merged[-1][0], merged[-1][1] + s)
            else:
                merged.append((o, s))
        self.free = merged


def output_chunking(spec):
    """Host-side geometry of ``gen_output_chunks`` (cotengra/core.py:3884-3941) for a
    ``TreeSpec``: ``(chunk_output, stepsize, nchunks)`` -- the output term of one chunk (the
    sliced output indices removed), the number of consecutive slice ids summed into a chunk
    (product of the inner sliced extents) and the number of chunks.  Raises ``ValueError``
    when the sliced indices are not ordered output-first (core.py:3912-3913)."""
    inner_seen = False
    for ind, _size, _proj in spec.sliced:
        if ind in spec.output:
            if inner_seen:
                raise ValueError("gen_output_chunks needs the sliced indices sorted output-first "
                                 "(core.py:3912-3913)")
        else:
            inner_seen = True
    sliced = {s[0] for s in spec.sliced}
    chunk_out = tuple(ix for ix in spec.output if ix not in sliced)
    stepsize = math.prod(size for ind, size, proj in spec.sliced
                         if ind not in spec.output and proj is None)
    return chunk_out, stepsize, spec.nslices // stepsize


class _Slot:
    """A tensor slot while planning; ``kind`` is its ``ctgb_tensor`` kind."""

    __slots__ = ("shape", "strides", "kind", "input_index", "slice_pos", "slice_stride", "nbytes",
                 "offset", "variant", "first_use", "last_use")

    def __init__(self, shape, strides, kind, nbytes, input_index=-1, slice_pos=(), slice_stride=(),
                 variant=False):
        self.shape = tuple(int(d) for d in shape)
        self.strides = [int(s) for s in strides]
        self.kind = kind
        self.nbytes = int(nbytes)
        self.input_index = input_index
        self.slice_pos = list(slice_pos)
        self.slice_stride = list(slice_stride)
        self.offset = 0
        self.variant = variant  # (forward planning) a sliced input lies below it
        self.first_use = None
        self.last_use = -1


def layout(sched, reserve=0):
    """Offsets of the scratch and persistent slots of the node schedule ``sched`` (the order the
    library runs the nodes in, phase by phase) by liveness: a slot is allocated where it is first
    written and released after its last read.  Persistent values read inside the slice loop
    (phases 1 and 2) live to its end; H accumulators live from the ``None`` entry of ``sched``,
    where the slice loop starts and they are zeroed.  ``reserve`` bytes (the conjugated cotangent
    copy) are taken from the persistent arena first.  The liveness fields of the slots are reset on
    entry, so a planner may lay out candidate schedules that share slots one after another.
    Returns ``(workspace_bytes, persistent_bytes, reserve_offset)``, the offset -1 without reserve."""
    for t in _slots(sched):
        t.first_use, t.last_use, t.offset = None, -1, 0
    zero_pos = sched.index(None) if None in sched else 0
    end_loop = max((pos for pos, nd in enumerate(sched) if nd is not None and nd["phase"] in LOOP_PHASES),
                   default=zero_pos)
    for pos, nd in enumerate(sched):
        if nd is None:
            continue
        c = nd["c"]
        if c.first_use is None:
            c.first_use = zero_pos if c.kind == K_HACC else pos
        for s in (nd["a"], nd["b"], nd.get("d"), nd.get("a2"), nd.get("b2")):
            if s is None:
                continue
            s.last_use = max(s.last_use, pos)
            if s.kind == K_PERSISTENT and nd["phase"] in LOOP_PHASES:
                s.last_use = max(s.last_use, end_loop)
    persistent, scratch = _Arena(), _Arena()
    reserved = persistent.alloc(reserve) if reserve else -1
    arena = {K_SCRATCH: scratch, K_PERSISTENT: persistent, K_HACC: persistent}
    allocs, releases = {}, {}
    for t in _slots(sched):
        if t.kind in arena:
            t.last_use = max(t.last_use, t.first_use)
            allocs.setdefault(t.first_use, []).append(t)
            releases.setdefault(t.last_use, []).append(t)
    for pos in range(len(sched)):
        for t in allocs.get(pos, ()):
            t.offset = arena[t.kind].alloc(t.nbytes)
        for t in releases.get(pos, ()):
            arena[t.kind].release(t.offset, t.nbytes)
    return _align(scratch.peak), _align(persistent.peak), reserved


def _slots(sched):
    """The slots of a schedule in order of first appearance."""
    return list(dict.fromkeys(t for nd in sched if nd is not None
                              for t in (nd["a"], nd["b"], nd.get("d"), nd.get("a2"), nd.get("b2"), nd["c"])
                              if t is not None))


class _DevicePlan:
    """A schedule as the library runs it: its ``ctgb_plan_desc``, upload and release.  Subclasses
    set ``dtype``, ``inputs``, ``sliced``, ``slice_out_stride``, ``out_elements``, the arena sizes
    and ``tensors``/``nodes`` before calling ``_marshal``."""

    handle = None
    strip_exponent = False
    cotangent_offset = -1
    acc_dtype = None     # forward plans that sum their slices in double: ctgb_plan_set_accumulator
    _chunk_words = None  # forward plans whose root stores its slice densely: ctgb_plan_set_chunk_desc
    scale_slots = None   # stripped derivative plans: ([slot_a], [slot_b]), from each node's "scale" (_scale_slots)
    tangent_marks = None  # stripped forward-mode plans: 1 per tangent record (ctgb_plan_set_tangent_scale_slots)

    def _scale_slots(self):
        """``scale_slots`` of a stripped derivative plan: the factor slots every node of ``self.nodes``
        divides by, from its ``"scale"`` entry (the operand tensors; ``None`` for the root's seed, slot
        ``n_tensors``); -1 where a node has none."""
        slot = {id(t): i for i, t in enumerate(self.tensors)}
        seed = len(self.tensors)
        scale = [nd.get("scale", ()) for nd in self.nodes]
        self.scale_slots = tuple([-1 if len(s) <= k else seed if s[k] is None else slot[id(s[k])] for s in scale]
                                 for k in (0, 1))

    def _marshal(self):
        keep = self._keep = []
        slot = {id(t): i for i, t in enumerate(self.tensors)}
        ct = (_lib.CtgbTensor * max(len(self.tensors), 1))()
        for i, t in enumerate(self.tensors):
            ct[i].kind = t.kind
            ct[i].input_index = t.input_index
            ct[i].offset = t.offset
            ct[i].nbytes = t.nbytes
            ct[i].n_sliced = len(t.slice_pos)
            if t.slice_pos:
                pos = (C.c_int32 * len(t.slice_pos))(*t.slice_pos)
                st = (C.c_int64 * len(t.slice_stride))(*t.slice_stride)
                keep += [pos, st]
                ct[i].slice_pos = C.cast(pos, C.POINTER(C.c_int32))
                ct[i].slice_stride = C.cast(st, C.POINTER(C.c_int64))
        cn = (_lib.CtgbNode * max(len(self.nodes), 1))()
        for i, nd in enumerate(self.nodes):
            words = np.array(nd["words"], dtype=np.int64)
            if nd.get("d") is not None:
                words[lowering.AB_BS_SLOT] = slot[id(nd["d"])]
            if nd["kind"] == 2:  # a two-term node: the pair words, then the slots of A' and B'
                words = np.append(words, [slot[id(nd["a2"])], slot[id(nd["b2"])]]).astype(np.int64)
            keep.append(words)
            cn[i].kind = nd["kind"]
            cn[i].a = slot[id(nd["a"])]
            cn[i].b = slot[id(nd["b"])] if nd["b"] is not None else -1
            cn[i].c = slot[id(nd["c"])]
            cn[i].phase = nd["phase"]
            cn[i].zero_fill = int(nd.get("zero_fill", False))
            cn[i].is_root = int(nd.get("root", False))
            cn[i].desc = words.ctypes.data_as(C.POINTER(C.c_int64))
        ns = len(self.sliced)
        radix = (C.c_int64 * max(ns, 1))(*[s for _i, s, _p in self.sliced])
        proj = (C.c_int64 * max(ns, 1))(*[(-1 if p is None else p) for _i, _s, p in self.sliced])
        ostr = (C.c_int64 * max(ns, 1))(*self.slice_out_stride)
        keep += [ct, cn, radix, proj, ostr]
        pd = self._pd = _lib.CtgbPlanDesc()
        pd.dtype = DTYPE_CODES[self.dtype]
        pd.n_inputs = len(self.inputs)
        pd.n_tensors = len(self.tensors)
        pd.tensors = C.cast(ct, C.POINTER(_lib.CtgbTensor))
        pd.n_nodes = len(self.nodes)
        pd.nodes = C.cast(cn, C.POINTER(_lib.CtgbNode))
        pd.n_sliced = ns
        pd.slice_radix = C.cast(radix, C.POINTER(C.c_int64))
        pd.slice_project = C.cast(proj, C.POINTER(C.c_int64))
        pd.slice_out_stride = C.cast(ostr, C.POINTER(C.c_int64))
        pd.out_elements = self.out_elements
        pd.workspace_bytes = self.workspace_bytes
        pd.persistent_bytes = self.persistent_bytes
        pd.strip_exponent = int(self.strip_exponent)
        pd.cotangent_offset = self.cotangent_offset
        self.total_bytes = self.workspace_bytes + self.persistent_bytes

    def create(self):
        """Upload the plan to the current CUDA device."""
        if self.handle is not None:
            return self
        lib = _lib.load()
        h = C.c_void_p()
        _lib.check(lib.ctgb_plan_create(C.byref(self._pd), C.byref(h)))
        self.handle = h
        if self._chunk_words is not None:
            w = self._chunk_words
            _lib.check(lib.ctgb_plan_set_chunk_desc(h, w.ctypes.data_as(C.c_void_p)))
        if self.acc_dtype not in (None, self.dtype):
            _lib.check(lib.ctgb_plan_set_accumulator(h, DTYPE_CODES[self.acc_dtype]))
        if self.scale_slots is not None:
            n = len(self.nodes)
            sa, sb = ((C.c_int32 * max(n, 1))(*s) for s in self.scale_slots)
            if self.tangent_marks is None:
                _lib.check(lib.ctgb_plan_set_scale_slots(h, sa, sb, n))
            else:
                marks = (C.c_int32 * max(n, 1))(*self.tangent_marks)
                _lib.check(lib.ctgb_plan_set_tangent_scale_slots(h, sa, sb, marks, n))
        return self

    def destroy(self):
        if self.handle is not None:
            _lib.load().ctgb_plan_destroy(self.handle)
            self.handle = None

    def launches_per_slice(self):
        return int(_lib.load().ctgb_plan_launches_per_slice(self.handle))

    def strip_modes(self):
        """strip_exponent plans: ``(prescale_b, measure_after)`` of every node of ``self.nodes``
        (ctgb_plan_strip_modes; prescale_b is -1 for single-operand nodes)."""
        n = len(self.nodes)
        pre, after = (C.c_int32 * n)(), (C.c_int32 * n)()
        _lib.check(_lib.load().ctgb_plan_strip_modes(self.handle, pre, after, n))
        return [(int(a), int(b)) for a, b in zip(pre, after)]

    def __del__(self):
        try:
            self.destroy()
        except Exception:
            pass


class ExecPlan(_DevicePlan):
    """Compile ``contractions`` (reference IR) for fixed input shapes / dtype.

    Parameters
    ----------
    contractions : the reference IR records ``(p, l, r, tdot, arg, perm)``.
    inputs : the index term of every network input (full, unsliced).
    output : the full output term.
    size_dict : extent of every index.
    sliced : ordered ``[(ind, size, project)]`` as ``tree.sliced_inds``.
    precision : ``"3xtf32"`` (default) or ``"tf32"``, the compute mode of the float32 / complex64
        tensor-core nodes (``lowering.PRECISIONS``); ``"tf32"`` with a double dtype raises ``ValueError``.
    accumulate : ``"native"`` (default) sums the slices in the plan dtype.  ``"double"`` gives a
        float32 / complex64 plan a float64 / complex128 output (``acc_dtype``) that every slice is added
        to in double: a dot-stream root sums in double inside the kernel (``lowering.FLAG_WIDE_C``) and
        adds into the output itself, any other root stores its slice densely in the workspace and one
        extra launch folds it in through the chunk descriptor.  For float64 / complex128 it is
        ``"native"``.
    absorb_root : fold a complex128 stem absorption ``X = A . Bs`` into the ``DMMA_32x32`` product
        ``R = X . V`` that reads it next (``lowering.build_absorb_desc``), so that X is never stored:
        one ``VAR_ABSORB_ROOT`` node reads A, Bs and V and writes R.  Off by default: the plan is then
        node for node the reference's sequence.  Not with ``strip_exponent`` or a forced ``variant``.
    input_ids : the SSA id each plan input stands for (default ``range(len(inputs))``), so that a plan
        input may be an intermediate node formed elsewhere (a folded constant subtree,
        ``constants.py``); the records keep their own SSA ids.
    """

    def __init__(self, contractions, inputs, output, size_dict, sliced=(), dtype="complex128",
                 strip_exponent=False, hoist=True, allow_dmma=True, sm_count=None,
                 variant=None, precision="3xtf32", accumulate="native", absorb_root=False, input_ids=None):
        self.dtype = dtype_name(dtype)
        self.precision = check_precision(precision, self.dtype)
        self.esize = DTYPE_SIZES[self.dtype]
        self.acc_dtype = accumulator_dtype(self.dtype, accumulate)
        self.wide = self.acc_dtype != self.dtype
        self.contractions = tuple(contractions)
        self.inputs = [tuple(t) for t in inputs]
        self.input_ids = tuple(range(len(self.inputs))) if input_ids is None else tuple(int(i) for i in input_ids)
        if len(self.input_ids) != len(self.inputs):
            raise ValueError(f"{len(self.input_ids)} input_ids for {len(self.inputs)} inputs")
        self.output = tuple(output)
        self.size_dict = dict(size_dict)
        self.sliced = [(i, int(s), None if p is None else int(p)) for i, s, p in sliced]
        self.strip_exponent = bool(strip_exponent)
        if sm_count is None:
            try:
                sm_count = _lib.device_info()["sm_count"]
            except Exception:
                sm_count = 132  # H100 SXM
        self.sm_count = sm_count
        self.absorb_root = bool(absorb_root) and self.dtype == "complex128" and not self.strip_exponent \
            and variant is None
        self._build(hoist, allow_dmma, variant)

    # ------------------------------------------------------------------ build
    def _build(self, hoist, allow_dmma, variant):
        sliced_pos = {ind: j for j, (ind, _s, _p) in enumerate(self.sliced)}
        nslices = math.prod(s for _i, s, p in self.sliced if p is None)
        self.nslices = nslices
        real_slicing = bool(self.sliced)
        hoist = hoist and real_slicing

        # full output geometry (projected output indices keep extent 1)
        def out_ext(ix):
            if ix in sliced_pos and self.sliced[sliced_pos[ix]][2] is not None:
                return 1
            return self.size_dict[ix]

        self.out_shape = tuple(out_ext(ix) for ix in self.output)
        out_full_strides = row_major_strides(self.out_shape)
        self.out_elements = math.prod(self.out_shape)
        root_term = tuple(ix for ix in self.output if ix not in sliced_pos)
        root_strides = [s for ix, s in zip(self.output, out_full_strides) if ix not in sliced_pos]
        self.root_shape = tuple(self.size_dict[ix] for ix in root_term)
        self.slice_out_stride = [0] * len(self.sliced)
        for ix, s in zip(self.output, out_full_strides):
            if ix in sliced_pos and self.sliced[sliced_pos[ix]][2] is None:
                self.slice_out_stride[sliced_pos[ix]] += s

        # network inputs as strided views of the unsliced arrays
        cur = {}
        self.input_nbytes = []
        for i, term in enumerate(self.inputs):
            full_shape = [self.size_dict[ix] for ix in term]
            fs = row_major_strides(full_shape)
            self.input_nbytes.append(math.prod(full_shape) * self.esize)
            keep = [k for k, ix in enumerate(term) if ix not in sliced_pos]
            cut = [k for k, ix in enumerate(term) if ix in sliced_pos]
            # (nbytes: the whole unsliced array, which strip_exponent copies scaled)
            cur[self.input_ids[i]] = _Slot([full_shape[k] for k in keep], [fs[k] for k in keep], K_INPUT,
                                           self.input_nbytes[-1], i, [sliced_pos[term[k]] for k in cut],
                                           [fs[k] for k in cut], variant=bool(cut))
        tensors = list(cur.values())
        self.sliced_shapes = [t.shape for t in tensors]

        nodes = []  # dicts
        # does the root write (accumulate into) the output itself?  Not with strip_exponent, and in a
        # wide plan only a dot-stream root (decided where the root is lowered)
        direct = not self.strip_exponent and not self.wide
        n_rec = len(self.contractions)
        for step, (p, l, r, tdot, arg, perm) in enumerate(self.contractions):
            is_last = step == n_rec - 1
            if r is None:
                src = cur[p] if l is None else cur[l]
                terms, out = split_equation(arg)
                if len(terms) != 1:
                    raise ValueError(f"expected a single-term equation, got {arg!r}")
                is_root = l is not None
                if is_root and not is_last:
                    raise ValueError("single-input record must be the only contraction")
                ostr = root_strides if (is_root and direct) else None
                odims, sdims, oshape = classify_single(terms[0], src.shape, out, out_strides=ostr,
                                                      strides_x=src.strides)
                if is_root:
                    self._check_root_shape(oshape)
                # the root always accumulates into the (zeroed) output, so that
                # slice sums, split-K atomics and plain stores share one path
                acc = is_root and direct
                words = build_single_desc(odims, sdims, self.dtype, accumulate=acc)
                dst = _Slot(oshape, row_major_strides(oshape), K_SCRATCH, max(math.prod(oshape), 1) * self.esize,
                            variant=src.variant)
                nodes.append(dict(kind=1, a=src, b=None, c=dst, words=words, root=is_root))
                tensors.append(dst)
                cur[p] = dst
                continue

            A, Bt = cur.pop(l), cur.pop(r)
            if tdot:
                axes = (tuple(arg[0]), tuple(arg[1]))
                check_tensordot_shapes(axes, A.shape, Bt.shape)
                ta, tb, to = tensordot_terms(axes, len(A.shape), len(Bt.shape), perm)
            else:
                terms, to = split_equation(arg)
                if len(terms) != 2:
                    raise ValueError(f"expected a two-term equation, got {arg!r}")
                ta, tb = terms
            is_root = is_last

            def lower(into_output, wide_c=False):
                ostr = root_strides if into_output else None
                dims = classify_pair(ta, A.shape, tb, Bt.shape, to, out_strides=ostr,
                                     strides_a=A.strides, strides_b=Bt.strides)
                dense = 0 if into_output else math.prod(dims.out_shape)
                return dims, dense, build_pair_desc(dims, self.dtype, accumulate=into_output,
                                                    sm_count=self.sm_count, allow_dmma=allow_dmma,
                                                    c_dense_elems=dense, variant=variant,
                                                    precision=self.precision, wide_c=wide_c)

            if is_root and self.wide and not self.strip_exponent:
                # only the dot-stream kernels sum in double: such a root adds into the wide output
                # itself, any other one stores its slice densely for add_chunk_wide
                direct = lower(True)[2].variant in lowering.DOTSTREAM_VARIANTS
                dims, dense, plan = lower(direct, wide_c=direct)
            else:
                dims, dense, plan = lower(is_root and direct)
            if is_root:
                self._check_root_shape(dims.out_shape)
            acc = is_root and direct
            dst = _Slot(dims.out_shape, row_major_strides(dims.out_shape), K_SCRATCH,
                        max(math.prod(dims.out_shape), 1) * self.esize, variant=A.variant or Bt.variant)
            a, b = (Bt, A) if plan.swapped else (A, Bt)
            nodes.append(dict(kind=0, a=a, b=b, c=dst, words=plan.words, root=is_root, plan=plan,
                              sizes=plan.sizes, dims=dims, acc=acc, dense=dense, terms=(A, Bt)))
            tensors.append(dst)
            cur[p] = dst
            if self.absorb_root:
                self._absorb(nodes, tensors)

        if not nodes:
            raise ValueError("empty contraction program")
        self.root_direct = direct
        if direct:
            nodes[-1]["c"].kind = K_OUTPUT  # the root writes the output accumulator directly
        # invariance: hoisted results live in the persistent arena
        for nd in nodes:
            srcs = [t for t in (nd["a"], nd["b"], nd.get("d")) if t is not None]
            nd["invariant"] = bool(hoist and not nd["root"] and not any(s.variant for s in srcs))
            nd["phase"] = PHASE_INV_FWD if nd["invariant"] else PHASE_VAR_FWD
            if nd["invariant"]:
                nd["c"].kind = K_PERSISTENT
            else:
                nd["c"].variant = True
        # schedule: invariant pass then variant pass (the C side runs them so)
        order = [nd for nd in nodes if nd["invariant"]] + [nd for nd in nodes if not nd["invariant"]]
        for pos, nd in enumerate(order):
            nd["pos"] = pos
        self.workspace_bytes, self.persistent_bytes, _ = layout(order)
        self.nodes = nodes
        self.n_variant_nodes = sum(1 for nd in nodes if not nd["invariant"])

        # cost bookkeeping (scalar MACs and ideal element traffic per slice)
        self.macs_per_slice = 0
        self.macs_invariant = 0
        self.elements_per_slice = 0
        for nd in nodes:
            if nd["kind"] != 0:
                continue
            macs = nd["plan"].macs if nd.get("d") is not None else math.prod(nd["sizes"])
            el = sum(math.prod(nd[x].shape) for x in ("a", "b", "d", "c") if nd.get(x) is not None)
            if nd["invariant"]:
                self.macs_invariant += macs
            else:
                self.macs_per_slice += macs
                self.elements_per_slice += el

        self.tensors = tensors
        self._marshal()
        if not direct:
            # dense root result -> its chunk of the (strided) output
            rs = self.root_shape
            dense = row_major_strides(rs)
            odims = [[e, sx, so] for e, sx, so in zip(rs, dense, root_strides) if e != 1]
            self._chunk_words = build_single_desc(odims, [], self.dtype)

    def _absorb(self, nodes, tensors):
        """Replace the last two pair nodes by one absorb-root node when the last one is a
        ``DMMA_32x32`` product reading the other's result (``lowering.build_absorb_desc``)."""
        if len(nodes) < 2:
            return
        P, R = nodes[-2], nodes[-1]
        if P["kind"] != 0 or R["kind"] != 0 or P.get("d") is not None or R["plan"].variant != lowering.VAR_DMMA_32x32:
            return
        X = P["c"]
        if X not in R["terms"]:
            return
        ab = lowering.build_absorb_desc(P["dims"], R["dims"], R["terms"][0] is X, accumulate=R["acc"],
                                        sm_count=self.sm_count, c_dense_elems=R["dense"])
        if ab is None:
            return
        pa, pb = P["terms"]
        small, big = (pa, pb) if ab.small_is_a else (pb, pa)
        V = R["terms"][1] if R["terms"][0] is X else R["terms"][0]
        tensors.remove(X)
        nodes[-2:] = [dict(kind=0, a=big, b=V, d=small, c=R["c"], words=ab.words, root=R["root"], plan=ab,
                           sizes=ab.sizes, dims=None, acc=R["acc"], dense=R["dense"], terms=None)]

    def _check_root_shape(self, shape):
        if tuple(shape) != tuple(self.root_shape):
            raise ValueError(
                f"contraction program produces shape {tuple(shape)}, "
                f"tree output expects {tuple(self.root_shape)}"
            )

    # ------------------------------------------------------------------ device side
    def host_staging_bytes(self):
        extra = _align(self.total_bytes) - self.total_bytes
        for n in self.input_nbytes:
            extra += _align(n)
        return extra + _align(self.out_elements * DTYPE_SIZES[self.acc_dtype]) + 512

    def execute(self, input_ptrs, out_ptr, exp_ptr, ws_ptr, ws_bytes, begin, step, count, stream=0):
        lib = _lib.load()
        arr = (C.c_void_p * len(input_ptrs))(*input_ptrs)
        _lib.check(lib.ctgb_plan_execute(self.handle, arr, out_ptr, exp_ptr, None, None, ws_ptr, ws_bytes,
                                         int(begin), int(step), int(count), stream))

    def execute_host(self, host_arrays, host_out, ws_ptr, ws_bytes, begin, step, count, stream=0):
        lib = _lib.load()
        ptrs = (C.c_void_p * len(host_arrays))(*[a.ctypes.data for a in host_arrays])
        nb = (C.c_int64 * len(host_arrays))(*[a.nbytes for a in host_arrays])
        exp = C.c_double(0.0)
        _lib.check(lib.ctgb_plan_execute_host(self.handle, ptrs, nb, host_out.ctypes.data,
                                              C.byref(exp), ws_ptr, ws_bytes, int(begin), int(step),
                                              int(count), stream))
        return exp.value

    def profile(self, enable=True):
        _lib.check(_lib.load().ctgb_plan_profile(self.handle, int(enable)))

    def profile_read(self):
        """Milliseconds of every node (plan order) for the last executed slice."""
        n = len(self.nodes)
        ms = (C.c_float * n)()
        _lib.check(_lib.load().ctgb_plan_profile_read(self.handle, ms, n))
        return [float(x) for x in ms]
