"""Stem fusion: keep the big operand of a contraction *stem* from making a round
trip through HBM for every small tensor it absorbs (SURVEY.md section 8 f-2, H4).

A sliced Sycamore tree is a stem: one huge intermediate (2^28-2^30 elements)
absorbs ~50 small tensors one at a time, and for the skinny steps (few kept /
contracted indices on the small side) each absorption is a pure HBM pass --
read 16 GiB, write 16 GiB, a handful of flops per element.  Two consecutive
absorptions

    x = (a . b1)        y = (x . b2)

are fused by never materialising ``x``: the executor contracts the two small
tensors first and streams the big operand once,

    t = (b1 . b2)       y = (a . t)

which is the same multilinear map (contraction is associative; the result
differs from the reference's by floating-point summation order only, inside the
1e-10 / 1e-5 parity bounds) with half the traffic.  Likewise the last small
tensors of a stem are peeled over the final inner product,

    ((a . b1) . v)  ->  ((a . v) . b1),

so that the largest tensor of the tree is read once instead of written and read
again.  Whether a group is fused is decided by a per-node roofline estimate
(flops against the tensor rate of the kernel the node would get, bytes against
HBM), with a dynamic program over every maximal stem; the search, the
hyper-optimiser and the SliceFinder stay in cotengra and are not touched -- this
is an execution-plan transformation of the tree they return
(cf. ``sort_contraction_indices``, cotengra/core.py:3421-3506, and the stem
cost model of cotengra/core_multi.py:39-72).

Everything here is host-side integer work on a ``TreeSpec``.
"""

from __future__ import annotations

import math

from .tree import TreeSpec

# ---- per-node time model (seconds).  Relative kernel rates (not re-measured on H100); they only
# have to rank alternatives, not predict times.
_LAUNCH = 4e-6
_RATES = {
    # dtype-class: (stream_bw, staged_bw, tensor rates by K, tiny-MN-huge-K bandwidth)
    "complex128": dict(stream=5.8e12, dstream=5.2e12, dstream_tf=25e12, staged=4.4e12,
                       tf={64: 34e12, 32: 32.5e12, 16: 24.5e12, 0: 13e12}, dot=6.4e12, flop=8),
    "float64": dict(stream=5.8e12, dstream=5.0e12, dstream_tf=9e12, staged=4.4e12,
                    tf={64: 30e12, 32: 28e12, 16: 20e12, 0: 10e12}, dot=6.4e12, flop=2),
    "complex64": dict(stream=5.8e12, dstream=4.8e12, dstream_tf=60e12, staged=4.8e12,
                      tf={64: 140e12, 32: 120e12, 16: 90e12, 0: 30e12}, dot=6.2e12, flop=8),
    "float32": dict(stream=5.8e12, dstream=4.8e12, dstream_tf=30e12, staged=4.8e12,
                    tf={64: 45e12, 32: 40e12, 16: 30e12, 0: 12e12}, dot=6.2e12, flop=2),
}
_ESIZE = {"float32": 4, "float64": 8, "complex64": 8, "complex128": 16}


def node_time(dtype, B, M, N, K, elems):
    """Estimated seconds of one pairwise node ``C[b,m,n] = sum_k A[b,m,k] B[b,k,n]``
    that moves ``elems`` tensor elements, on the kernel ``choose_variant`` would pick."""
    r = _RATES[dtype]
    if N > M:
        M, N = N, M
    flops = r["flop"] * B * M * N * K
    nbytes = elems * _ESIZE[dtype]
    if M <= 4 and N <= 4 and B == 1:
        if K >= 1 << 20:
            return _LAUNCH + nbytes / r["dot"]      # dot-stream kernels
        return _LAUNCH + nbytes / 2.5e12 + flops / 2e12
    if dtype in ("complex128", "float64") and M <= 32 and N <= 32 and B == 1 and K >= 1 << 14:
        # one 32 x 32 DMMA tile, split-K over two CTAs per SM (measured on M = N = 32, K = 2^25:
        # 4.0 TB/s and 32 TFLOP/s at once)
        return _LAUNCH + max(nbytes / 4.2e12, r["flop"] * 32.0 * 32.0 * K / 33e12)
    if K >= 1 << 12 and (M < 64 or M * N <= 1 << 14):
        # a small result over a long contracted range and no dot-stream kernel for it: a handful
        # of (mostly empty) tensor tiles with split-K atomics -- far from either roofline
        # (measured: M=128 N=16 K=2^23 complex64 at 1.05 TB/s, 15 TFLOP/s)
        return _LAUNCH + max(nbytes / 1.0e12, flops / 12e12)
    if N <= 8 and K <= 8 and B == 1:
        bw = r["stream"] if N * K <= 16 else 0.8 * r["stream"]
        return _LAUNCH + nbytes / bw
    if dtype == "complex128" and B == 1 and ((N <= 16 and K <= 32) or (N <= 8 and K <= 64)):
        return _LAUNCH + max(nbytes / r["dstream"], flops * (8.0 / N if N < 8 else 1.0) / r["dstream_tf"])
    if N <= 8:
        return _LAUNCH + max(nbytes / 3.7e12, flops / 13e12)  # staged row policy
    if dtype == "complex128" and N <= 16 and K <= 32 and B == 1:
        return _LAUNCH + max(nbytes / r["dstream"], flops / r["dstream_tf"])
    tf = r["tf"][64 if K >= 64 else 32 if K >= 32 else 16 if K >= 16 else 0]
    staged_bw = r["staged"]
    if N < 24:
        tf *= 0.8
        if dtype == "complex64":
            staged_bw = 3.2e12  # wgmma 128 x 16 tiles
    # tile occupancy of the staged tensor-core variants (lowering.choose_variant)
    MT, NT = (64, 128) if N >= 96 else (128, 64) if N >= 48 else (256, 32) if N >= 24 else (256, 16)
    util = (M / (-(-M // MT) * MT)) * (N / (-(-N // NT) * NT))
    return _LAUNCH + max(nbytes / staged_bw, flops / (tf * util))


class _Node:
    __slots__ = ("leaves", "left", "right", "leaf", "counts", "inds", "size", "old_id")

    def __init__(self, leaves, counts, left=None, right=None, leaf=None):
        self.leaves, self.counts = leaves, counts
        self.left, self.right, self.leaf = left, right, leaf
        self.inds = None
        self.size = 1
        self.old_id = None


class _Ctx:
    """Index bookkeeping of one (sliced) network."""

    def __init__(self, spec: TreeSpec, dtype):
        self.spec, self.dtype = spec, dtype
        self.sliced = {s[0] for s in spec.sliced}
        self.size = {ix: int(d) for ix, d in spec.size_dict.items()}
        self.app = dict(spec.appearances)
        self.pair_evals = 0
        self.ratio, self.min_big, self.min_gain = _RATIO, _MIN_BIG, 0.03
        self.model = node_time

    def finish(self, node):
        node.inds = tuple(ix for ix, c in node.counts.items() if c < self.app[ix])
        node.size = math.prod(self.size[ix] for ix in node.inds)
        return node

    def leaf(self, i):
        counts = {}
        for ix in self.spec.inputs[i]:
            if ix not in self.sliced:
                counts[ix] = counts.get(ix, 0) + 1
        return self.finish(_Node(frozenset((i,)), counts, leaf=i))

    def join(self, x, y):
        counts = dict(x.counts)
        for ix, c in y.counts.items():
            counts[ix] = counts.get(ix, 0) + c
        return self.finish(_Node(x.leaves | y.leaves, counts, left=x, right=y))

    def pair_sizes(self, x, y, z):
        """(B, M, N, K) of ``z = (x . y)``."""
        kept = set(z.inds)
        xi, yi = set(x.inds), set(y.inds)
        Bn = M = N = K = 1
        for ix in xi | yi:
            d = self.size[ix]
            if ix in kept:
                if ix in xi and ix in yi:
                    Bn *= d
                elif ix in xi:
                    M *= d
                else:
                    N *= d
            else:
                K *= d
        return Bn, M, N, K

    def cost(self, x, y, z=None):
        z = self.join(x, y) if z is None else z
        self.pair_evals += 1
        Bn, M, N, K = self.pair_sizes(x, y, z)
        return self.model(self.dtype, Bn, M, N, K, x.size + y.size + z.size), z


def _build(ctx, spec):
    nodes = {i: ctx.leaf(i) for i in range(spec.N)}
    nxt = spec.N
    for l, r in spec.path:
        n = ctx.join(nodes[l], nodes[r])
        n.old_id = nxt
        nodes[nxt] = n
        nxt += 1
    return nodes[nxt - 1] if spec.N > 1 else nodes[0]


# a "stem step": the big child dwarfs the small one and is itself worth a kernel's attention
_RATIO = 32
_MIN_BIG = 1 << 18
_MAX_GROUP = 4
_MAX_T = 1 << 14


def _big_small(ctx, node):
    l, r = node.left, node.right
    big, small = (l, r) if l.size >= r.size else (r, l)
    if big.size >= ctx.min_big and big.size >= ctx.ratio * small.size:
        return big, small
    return None, None


def _fold(ctx, parts):
    """Left-to-right product of small tensors; returns (node, cost)."""
    t, c = parts[0], 0.0
    for s in parts[1:]:
        dc, t = ctx.cost(t, s)
        c += dc
    return t, c


def _chain_of(ctx, node):
    """Walk down the big children: returns (base, [small_1 .. small_L]) with
    node = (..((base . s_1) . s_2).. . s_L)."""
    smalls = []
    cur = node
    while cur.leaf is None:
        big, small = _big_small(ctx, cur)
        if big is None:
            break
        smalls.append(small)
        cur = big
    smalls.reverse()
    return cur, smalls


def _plan_chain(ctx, base, smalls):
    """Dynamic program over the partitions of a stem into fused groups.
    Returns (f, choice, ys): f[i] = best time to materialise the i-th stem tensor,
    choice[i] = start j of the last group, ys[i] = the stem tensors (as nodes)."""
    L = len(smalls)
    ys = [base]
    for s in smalls:
        ys.append(ctx.join(ys[-1], s))
    f = [0.0] + [math.inf] * L
    choice = [0] * (L + 1)
    for i in range(1, L + 1):
        for j in range(max(0, i - _MAX_GROUP), i):
            t, ct = _fold(ctx, smalls[j:i])
            if i - j > 1 and t.size > _MAX_T:
                continue
            c, _z = ctx.cost(ys[j], t, ys[i])
            # a fused group must beat its unfused chain clearly (the model is coarse)
            total = f[j] + ct + c * (1.0 if i - j == 1 else 1.03)
            if total < f[i]:
                f[i], choice[i] = total, j
    return f, choice, ys


def _emit_chain(ctx, rebuilt_base, smalls, choice, upto):
    """Materialise the partition chosen by the DP for stem tensors 1..upto."""
    cuts, i = [], upto
    while i > 0:
        cuts.append((choice[i], i))
        i = choice[i]
    cuts.reverse()
    cur = rebuilt_base
    for j, i in cuts:
        t, _c = _fold(ctx, smalls[j:i])
        cur = ctx.join(cur, t)
    return cur


def _rebuild(ctx, node, stats):
    if node.leaf is not None:
        return node
    base, smalls = _chain_of(ctx, node)
    if not smalls:
        # no stem here: maybe the meeting point of two stems (the root of an amplitude tree)
        peeled = _peel_root(ctx, node, stats)
        if peeled is not None:
            return peeled
        new = ctx.join(_rebuild(ctx, node.left, stats), _rebuild(ctx, node.right, stats))
        return new
    new_smalls = [_rebuild(ctx, s, stats) for s in smalls]
    new_base = _rebuild(ctx, base, stats)
    f, choice, _ys = _plan_chain(ctx, new_base, new_smalls)
    L = len(smalls)
    unfused = sum(ctx.cost(a, s)[0] for a, s in zip(_ys[:-1], new_smalls))
    stats["chains"].append(dict(length=L, unfused_s=unfused, fused_s=f[L]))
    if f[L] > (1.0 - ctx.min_gain) * unfused:
        choice = list(range(-1, L))  # not worth it: keep every step on its own
        choice[0] = 0
    return _emit_chain(ctx, new_base, new_smalls, choice, L)


def _peel_root(ctx, node, stats):
    """``node = (u . v)`` with two big children that are (ends of) stems: try
    ``((a . v) . T)`` for the last group(s) ``T`` of u's and/or v's stem."""
    u, v = node.left, node.right
    if min(u.size, v.size) < ctx.min_big or max(u.size, v.size) > ctx.ratio * min(u.size, v.size):
        return None
    if node.size > 4096:
        return None
    sides = []
    for w in (u, v):
        base, smalls = _chain_of(ctx, w)
        new_smalls = [_rebuild(ctx, s, stats) for s in smalls]
        new_base = _rebuild(ctx, base, stats)
        f, choice, ys = _plan_chain(ctx, new_base, new_smalls)
        sides.append((new_base, new_smalls, f, choice, ys))
    (bu, su, fu, cu, yu), (bv, sv, fv, cv, yv) = sides
    Lu, Lv = len(su), len(sv)
    best = None
    for pu in range(0, min(3, Lu) + 1):
        for pv in range(0, min(3, Lv) + 1):
            ju, jv = Lu - pu, Lv - pv
            if math.isinf(fu[ju]) or math.isinf(fv[jv]):
                continue
            c, R = ctx.cost(yu[ju], yv[jv])
            total = fu[ju] + fv[jv] + c
            if pu or pv:
                if R.size > 4096:
                    continue
                rest = su[ju:] + sv[jv:]
                cur = R
                for s in rest:
                    dc, cur = ctx.cost(cur, s)
                    total += dc
            if best is None or total < best[0] - 1e-9:
                best = (total, pu, pv)
    total, pu, pv = best
    stats["root_peel"] = dict(peel_left=pu, peel_right=pv, est_s=total)
    ju, jv = Lu - pu, Lv - pv
    for smalls, f, ys, j in ((su, fu, yu, ju), (sv, fv, yv, jv)):
        if j > 0:
            unfused = sum(ctx.cost(a, s_)[0] for a, s_ in zip(ys[:j], smalls[:j]))
            stats["chains"].append(dict(length=j, unfused_s=unfused, fused_s=f[j]))
    a = _emit_chain(ctx, bu, su, cu, ju)
    b = _emit_chain(ctx, bv, sv, cv, jv)
    cur = ctx.join(a, b)
    for s in su[ju:] + sv[jv:]:
        cur = ctx.join(cur, s)
    return cur


def _peak(node):
    """Largest tensor in the subtree."""
    if node.leaf is not None:
        return node.size
    return max(node.size, _peak(node.left), _peak(node.right))


def _emit_path(root, n_leaves):
    """SSA path by post-order; the heavier subtree first, so that at most one big
    intermediate waits while its sibling subtree is contracted."""
    path, ids = [], {}
    order = []
    nxt = [n_leaves]

    def visit(n):
        if n.leaf is not None:
            ids[id(n)] = n.leaf
            return
        first, second = (n.left, n.right) if _peak(n.left) >= _peak(n.right) else (n.right, n.left)
        visit(first)
        visit(second)
        path.append((ids[id(n.left)], ids[id(n.right)]))
        ids[id(n)] = nxt[0]
        order.append(n)
        nxt[0] += 1

    import sys

    old = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old, 10000))
    try:
        visit(root)
    finally:
        sys.setrecursionlimit(old)
    return path, order


def fuse_stems(spec: TreeSpec, dtype="complex128", min_big=None, ratio=None, min_gain=None, model=None):
    """Return ``(new_spec, info)``: the tree of ``spec`` with its stems re-associated where
    the roofline model says the fused form is faster; ``info`` reports what was done
    (estimated seconds before/after per stem, root peel, nodes added/removed).
    ``new_spec is spec`` when nothing is worth changing."""
    if spec.N < 3:
        return spec, {"changed": False}
    import sys

    ctx = _Ctx(spec, dtype)
    if min_big is not None:
        ctx.min_big = int(min_big)
    if ratio is not None:
        ctx.ratio = ratio
    if min_gain is not None:
        ctx.min_gain = float(min_gain)
    if model is not None:
        ctx.model = model  # (dtype, B, M, N, K, elements) -> seconds
    old_limit = sys.getrecursionlimit()
    sys.setrecursionlimit(max(old_limit, 10000))
    try:
        root = _build(ctx, spec)
        stats = {"chains": []}
        new_root = _rebuild(ctx, root, stats)
    finally:
        sys.setrecursionlimit(old_limit)
    path, order = _emit_path(new_root, spec.N)

    def leafsets(r):
        out = set()

        def rec(n):
            if n.leaf is None:
                out.add(n.leaves)
                rec(n.left)
                rec(n.right)
        sys.setrecursionlimit(max(old_limit, 10000))
        try:
            rec(r)
        finally:
            sys.setrecursionlimit(old_limit)
        return out

    before, after = leafsets(root), leafsets(new_root)
    info = {
        "changed": before != after,
        "nodes_removed": len(before - after),
        "chains": [c for c in stats["chains"] if c["fused_s"] < (1.0 - ctx.min_gain) * c["unfused_s"]],
        "root_peel": stats.get("root_peel"),
    }
    if not info["changed"]:
        return spec, info
    # custom index orders (sort_contraction_indices) survive on nodes that still exist
    old_by_set = {}
    if spec.node_inds:
        def rec_old(n):
            if n.leaf is None:
                if n.old_id in spec.node_inds:
                    old_by_set[n.leaves] = spec.node_inds[n.old_id]
                rec_old(n.left)
                rec_old(n.right)
        sys.setrecursionlimit(max(old_limit, 10000))
        try:
            rec_old(root)
        finally:
            sys.setrecursionlimit(old_limit)
    node_inds = {}
    for k, n in enumerate(order):
        if n.leaves in old_by_set and n is not order[-1]:
            node_inds[spec.N + k] = old_by_set[n.leaves]
    new = TreeSpec(spec.inputs, spec.output, spec.size_dict, path, spec.sliced, node_inds)
    return new, info


def tree_work(spec: TreeSpec):
    """Scalar multiply-adds and ideal element traffic of one slice of ``spec`` as the
    reference counts them (``contraction_cost() / nslices``, core.py:1362; every operand read
    once, every result written once), split into the slice-dependent part and the part that
    does not depend on the slice id: ``(macs_variant, macs_invariant, elements_variant)``."""
    ctx = _Ctx(spec, "complex128")
    sliced_inputs = spec.sliced_inputs
    nodes = {i: (ctx.leaf(i), i in sliced_inputs) for i in range(spec.N)}
    nxt = spec.N
    macs_v = macs_i = elems_v = 0
    for l, r in spec.path:
        (x, vx), (y, vy) = nodes[l], nodes[r]
        z = ctx.join(x, y)
        Bn, M, N, K = ctx.pair_sizes(x, y, z)
        var = vx or vy or not spec.sliced
        if var:
            macs_v += Bn * M * N * K
            elems_v += x.size + y.size + z.size
        else:
            macs_i += Bn * M * N * K
        nodes[nxt] = (z, var)
        nxt += 1
    return macs_v, macs_i, elems_v
