"""Test-only numpy emulator of the device-side addressing.

Walks a descriptor (``cotengra_b200/csrc/gett_desc.h`` word layout) exactly the
way ``gett_kernel`` does -- work items, grid-base offsets, k-step bases, the
per-element load tables, partial-tile validity, strided stores, split-K -- but
with numpy on the CPU, and walks every plan kind the way ``plan_run`` runs it.
It lets the ``-m "not gpu"`` suite verify all host-side integer work
(classification, coalescing, tiling, arenas, slice offsets) against
``numpy.einsum`` / the golden vectors without a GPU.  It is NOT a fallback and
is never imported by the product.
"""

import math

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L
from cotengra_b200.jvp import JvpPlan
from cotengra_b200.vjp import VjpPlan


def _rows(W, off, n, width):
    return [tuple(int(x) for x in W[off + i * width: off + (i + 1) * width]) for i in range(n)]


def _local_offsets(tile, count, col):
    """offset of every local index under the tile dims (dim 0 fastest)."""
    out = np.zeros(count, dtype=np.int64)
    for idx in range(count):
        e, o = idx, 0
        for d in tile:
            o += (e % d[0]) * d[col]
            e //= d[0]
        out[idx] = o
    return out


def emulate_pair(W, A, B, C):
    """C (flat, modified in place) (+)= contraction described by ``W`` of flat
    arrays ``A`` and ``B``."""
    W = np.asarray(W)
    assert W[L.W_MAGIC] == L.DESC_MAGIC
    n_tm, n_tn, n_tk = (int(W[i]) for i in (L.W_NTM, L.W_NTN, L.W_NTK))
    n_gm, n_gn, n_gk, n_gb = (int(W[i]) for i in (L.W_NGM, L.W_NGN, L.W_NGK, L.W_NGB))
    MTa, NTa, KTa = (int(W[i]) for i in (L.W_MTA, L.W_NTA, L.W_KTA))
    tiles_m, tiles_n, tiles_b, steps_k = (int(W[i]) for i in (L.W_TILES_M, L.W_TILES_N, L.W_TILES_B, L.W_STEPS_K))
    splitk = int(W[L.W_SPLITK])
    MT, NT, KT = L.VARIANT_TILES[int(W[L.W_VARIANT])]
    if int(W[L.W_VARIANT]) == L.VAR_DOTSTREAM4 and int(W[L.W_DTYPE]) != L.DTYPE_CODES["complex128"]:
        KT = 2048
    assert MTa <= MT and NTa <= NT and KTa <= KT, (MTa, NTa, KTa, MT, NT, KT)
    accumulate = bool(W[L.W_FLAGS] & 1)
    tm = _rows(W, L.OFF_TM, n_tm, 3)
    tn = _rows(W, L.OFF_TN, n_tn, 3)
    gm = _rows(W, L.OFF_GM, n_gm, 4)
    gn = _rows(W, L.OFF_GN, n_gn, 4)
    gk = _rows(W, L.OFF_GK, n_gk, 4)
    gb = _rows(W, L.OFF_GB, n_gb, 5)
    lda = _rows(W, L.OFF_LDA, int(W[L.W_NLDA]), 4)
    ldb = _rows(W, L.OFF_LDB, int(W[L.W_NLDB]), 4)
    assert math.prod(d[0] for d in lda) == MTa * KTa
    assert math.prod(d[0] for d in ldb) == NTa * KTa

    def part(base):
        return tuple(int(W[base + i]) for i in range(4))

    pgm, mfull, mtext, mw = part(L.W_PGM)
    pgn, nfull, ntext, nw = part(L.W_PGN)
    pgk, kfull, ktext, kw = part(L.W_PGK)

    offMC = _local_offsets(tm, MTa, 2)
    offNC = _local_offsets(tn, NTa, 2)

    def table(ld, count):
        g = np.zeros(count, dtype=np.int64)
        x = np.zeros(count, dtype=np.int64)
        y = np.zeros(count, dtype=np.int64)
        for e0 in range(count):
            e = e0
            for ext, s, w1, w2 in ld:
                dig = e % ext
                e //= ext
                g[e0] += dig * s
                x[e0] += dig * w1
                y[e0] += dig * w2
        return g, x, y

    gA, rA, kA = table(lda, MTa * KTa)
    gB, kB, cB = table(ldb, NTa * KTa)

    def decode(idx, grid, ncols, pg):
        offs = [0] * ncols
        blk = 0
        for j, g in enumerate(grid):
            dig = (idx // g[1]) % g[0]
            for c in range(ncols):
                offs[c] += dig * g[2 + c]
            if j == pg:
                blk = dig
        return offs, blk

    if splitk > 1 and not accumulate:
        n = int(W[L.W_CELEMS])
        assert n > 0, "split-K into a strided C needs accumulate"
        C[:n] = 0
    per = -(-steps_k // splitk)
    for w in range(tiles_m * tiles_n * tiles_b * splitk):
        t = w
        in_ = t % tiles_n
        t //= tiles_n
        im_ = t % tiles_m
        t //= tiles_m
        ib_ = t % tiles_b
        ks = t // tiles_b
        (mA, mC), mblk = decode(im_, gm, 2, pgm)
        (nB, nC), nblk = decode(in_, gn, 2, pgn)
        (bA, bB, bC), _ = decode(ib_, gb, 3, -1)
        m_valid = MTa if pgm < 0 else min(mtext, mfull - mblk * mtext) * mw
        n_valid = NTa if pgn < 0 else min(ntext, nfull - nblk * ntext) * nw
        baseA, baseB, baseC = mA + bA, nB + bB, mC + nC + bC
        acc = np.zeros((MTa, NTa), dtype=C.dtype)
        for step in range(ks * per, min(steps_k, ks * per + per)):
            (kAo, kBo), kblk = decode(step, gk, 2, pgk)
            k_valid = KTa if pgk < 0 else min(ktext, kfull - kblk * ktext) * kw
            ta = np.zeros((MTa, KTa), dtype=C.dtype)
            okA = (rA < m_valid) & (kA < k_valid)
            ta[rA[okA], kA[okA]] = A[baseA + kAo + gA[okA]]
            tb = np.zeros((KTa, NTa), dtype=C.dtype)
            okB = (cB < n_valid) & (kB < k_valid)
            tb[kB[okB], cB[okB]] = B[baseB + kBo + gB[okB]]
            acc += ta @ tb
        rr, cc = np.meshgrid(np.arange(MTa), np.arange(NTa), indexing="ij")
        ok = (rr < m_valid) & (cc < n_valid)
        addr = baseC + offMC[rr[ok]] + offNC[cc[ok]]
        if accumulate or splitk > 1:
            np.add.at(C, addr, acc[ok])
        else:
            C[addr] = acc[ok]


def emulate_single(W, X, out):
    W = np.asarray(W)
    assert W[L.S_MAGIC] == L.SDESC_MAGIC
    n_o, n_s = int(W[L.S_NO]), int(W[L.S_NS])
    od = _rows(W, L.OFF_SO, n_o, 3)
    sd = _rows(W, L.OFF_SS, n_s, 2)
    accumulate = bool(W[L.S_FLAGS] & 1)
    for o in range(int(W[L.S_OUT_ELEMS])):
        e, xo, oo = o, 0, 0
        for ext, sx, so in od:
            dig = e % ext
            e //= ext
            xo += dig * sx
            oo += dig * so
        acc = 0
        for s in range(int(W[L.S_SUM_ELEMS])):
            e2, xs = s, 0
            for ext, sx in sd:
                xs += (e2 % ext) * sx
                e2 //= ext
            acc = acc + X[xo + xs]
        out[oo] = out[oo] + acc if accumulate else acc


def emulate_single_scaled(W, X, out, scale):
    n_o = int(W[L.S_NO])
    od = _rows(W, L.OFF_SO, n_o, 3)
    for o in range(int(W[L.S_OUT_ELEMS])):
        e, xo, oo = o, 0, 0
        for ext, sx, so in od:
            dig = e % ext
            e //= ext
            xo += dig * sx
            oo += dig * so
        out[oo] = out[oo] + X[xo] * scale


def emulate_absorb(W, A, Bs, V, C):
    """C (flat, modified in place) (+)= the absorb-root node ``W`` (``lowering.build_absorb_desc``,
    csrc/absorbdot.cuh): R[r, n] = sum_{k', c} (sum_k A[r, k', k] Bs[k, ck(r), c]) V[k', c, n] through
    the word tables."""
    W = np.asarray(W)
    assert W[L.W_MAGIC] == L.DESC_MAGIC and int(W[L.W_VARIANT]) == L.VAR_ABSORB_ROOT
    N, K, CC, CCP, KL, NG = (int(W[i]) for i in (L.AB_N, L.AB_K, L.AB_C, L.AB_CCP, L.AB_KL, L.AB_NG))
    grid = [tuple(int(x) for x in W[L.AB_G + 4 * j:L.AB_G + 4 * j + 4]) for j in range(NG)]
    units = int(W[L.AB_UNITS])
    assert units == math.prod(g[0] for g in grid)
    u = np.arange(units, dtype=np.int64)
    kA = sum((u // g[1]) % g[0] * g[2] for g in grid) + np.zeros(units, dtype=np.int64)
    kV = sum((u // g[1]) % g[0] * g[3] for g in grid) + np.zeros(units, dtype=np.int64)
    kA = (kA[:, None] + np.arange(KL) * int(W[L.AB_KLA])).reshape(-1)  # every k' of the node
    kV = (kV[:, None] + np.arange(KL) * int(W[L.AB_KLV])).reshape(-1)
    ma, mc = W[L.AB_TMA:L.AB_TMA + 32], W[L.AB_TMC:L.AB_TMC + 32]
    nv, nc = W[L.AB_TNV:L.AB_TNV + N], W[L.AB_TNC:L.AB_TNC + N]
    ka, kb = W[L.AB_TKA:L.AB_TKA + K], W[L.AB_TKB:L.AB_TKB + K]
    tcb, cv = W[L.AB_TCB:L.AB_TCB + 128], W[L.AB_TCV:L.AB_TCV + CC]
    Vt = V[kV[:, None, None] + cv[None, :, None] + nv[None, None, :]]  # [k', c, n]
    accumulate = bool(W[L.W_FLAGS] & 1)
    for r in range(32):
        if mc[r] < 0:
            continue
        ck = int(W[L.AB_TBCK + r // 8])
        cols = tcb[ck * CCP:ck * CCP + CC]
        assert (cols >= 0).all()
        a = A[ma[r] + kA[:, None] + ka[None, :]]                     # [k', k]
        x = a @ Bs[kb[:, None] + cols[None, :]]                      # [k', c]
        row = np.einsum("qc,qcn->n", x, Vt)
        dst = mc[r] + nc
        C[dst] = C[dst] + row if accumulate else row


def check_wide_plan(plan):
    """The invariants of a wide forward or forward-mode plan the library relies on
    (``ctgb_plan_set_accumulator``)."""
    assert plan.wide and plan.acc_dtype == L.WIDE_DTYPES[plan.dtype]
    flagged = [nd for nd in plan.nodes if nd["kind"] == 0 and int(nd["words"][L.W_FLAGS]) & L.FLAG_WIDE_C]
    root = _roots(plan)[0]
    if plan.strip_exponent:
        # the mantissa slot keeps the plan dtype; only the running mantissa is wide
        assert not flagged and root["c"].kind == X.K_SCRATCH and plan._chunk_words is not None
    elif getattr(plan, "fwd", plan).root_direct:
        # (the root's tangent records run the root's descriptor into the tangent output)
        assert flagged == [nd for nd in plan.nodes if nd["root"]]
        assert int(root["words"][L.W_VARIANT]) in L.DOTSTREAM_VARIANTS
        assert int(root["words"][L.W_FLAGS]) & 1 and root["c"].kind == X.K_OUTPUT and plan._chunk_words is None
    else:
        assert not flagged and root["c"].kind == X.K_SCRATCH and plan._chunk_words is not None
        flags = int(root["words"][L.W_FLAGS if root["kind"] == 0 else L.S_FLAGS])
        assert not flags & 1, "a dense root slot is stored, not accumulated"


def _roots(plan):
    """The primal root node and the last node that writes the root's tangent (``None`` for a plan
    without them), as ``ctgb_plan_create`` finds them."""
    last = {r: nd for nd in plan.nodes for r in (nd.get("root"),) if r}
    return last.get(1), last.get(2)


def _exponent_max(a, b):
    """gett_kernels.cuh exponent_max: NaN if either is"""
    return math.nan if (math.isnan(a) or math.isnan(b)) else max(a, b)


def _pow10(x):
    return float(np.power(10.0, x))


node_runs = 0  # nodes emulate_plan has run, over all calls (tests/emu_device.py counts them as launches)


def emulate_plan(plan, arrays, *, slice_ids=None, cotangent=None, grads=None, exponent=None, tangents=None,
                 primal=True, out=None, tout=None):
    """Run an ``ExecPlan``, ``VjpPlan`` or ``JvpPlan``, stripped or not, wide or not, on the CPU step for
    step as ``plan_run`` (csrc/ctg_b200.cu) runs it over the slices ``slice_ids`` (default all, taken in
    the order given).

    The arenas are exactly the reported bytes and filled with NaN, as uninitialised device memory may
    be: an access outside them raises and a read of memory nothing wrote spoils the result.  A wide plan
    holds every value in its accumulator dtype (the arenas keep their element counts and offsets): the
    emulator checks the host's integer work, not device rounding.

    ``strip_exponent`` is the lazy scheme of ``strip_setup``: one factor slot per tensor slot (1.0
    unless a node records max|C| there), the seed slot ``len(plan.tensors)``, and every node's product
    divided by its two slots of ``plan.scale_slots``, or for a forward plan a pairwise node's by its own
    operands' (1/0 counts as 0; the emulator scales the operand B, or A of a single-operand node, as
    the kernels' pre-scaled copy does).  Pairwise nodes of phases 0 and 1 that are not tangent records
    (``plan.tangent_marks``) measure max|C|.

    The buffers are those ``ctgb_plan_execute*`` takes: ``cotangent`` and ``grads`` (flat or shaped,
    default fresh zeros) of a VJP plan, whose stripped form needs the forward's ``exponent``; the
    ``tangents`` of a JVP plan, one per input in ``plan.wrt``, whose primal root is skipped with
    ``primal=False``.  ``out``, ``tout`` (flat, accumulator dtype) and ``exponent`` continue an earlier
    call's sums.  Returns, by plan kind: forward ``out``, stripped ``(out, E)``; VJP the gradients
    (``None`` outside ``plan.wrt``); JVP ``(out, tout)``, ``tout`` alone with ``primal=False``, stripped
    ``(out, E, tout)``."""
    is_jvp, is_vjp = isinstance(plan, JvpPlan), isinstance(plan, VjpPlan)
    strip = plan.strip_exponent
    wide = plan.acc_dtype not in (None, plan.dtype)
    if wide:
        check_wide_plan(plan)
    dt = np.dtype(plan.acc_dtype if wide else plan.dtype)
    es = plan.esize
    assert plan.workspace_bytes % es == 0 and plan.persistent_bytes % es == 0
    persistent = np.full(plan.persistent_bytes // es, np.nan, dtype=dt)
    scratch = np.full(plan.workspace_bytes // es, np.nan, dtype=dt)
    n_out = max(plan.out_elements, 1)
    out = np.zeros(n_out, dtype=dt) if out is None else out
    tout = np.zeros(n_out, dtype=dt) if tout is None else tout
    flats = [np.ascontiguousarray(a, dtype=dt).reshape(-1) for a in arrays]
    tflats = [None] * len(flats)
    if is_jvp:
        assert len(tangents) == len(plan.wrt)
        for i, t in zip(plan.wrt, tangents):
            tflats[i] = np.ascontiguousarray(t, dtype=dt).reshape(-1)
    if is_vjp:
        assert cotangent is not None and (exponent is not None or not strip)
        if grads is None:
            grads = [np.zeros(a.size, dtype=dt) if i in plan.wrt else None for i, a in enumerate(flats)]
        grads = [None if g is None else g.reshape(-1) for g in grads]
    root, troot = _roots(plan)

    seed = len(plan.tensors)
    factors = np.ones(seed + 2)
    slot = {id(t): i for i, t in enumerate(plan.tensors)}
    if plan.scale_slots is not None:
        scale_a, scale_b = plan.scale_slots
    else:  # strip_setup(p, nullptr, nullptr): a pairwise node divides by its own operands' slots
        scale_a, scale_b = ([slot[id(nd[k])] if nd["kind"] == 0 else -1 for nd in plan.nodes] for k in "ab")
    marks = plan.tangent_marks or [0] * len(plan.nodes)

    def inv(k):
        return 1.0 if k < 0 else 0.0 if factors[k] == 0 else 1.0 / float(factors[k])

    def view(t, digits, out_off):
        if t.kind in (X.K_INPUT, X.K_GRAD, X.K_TANGENT):
            src = {X.K_INPUT: flats, X.K_GRAD: grads, X.K_TANGENT: tflats}[t.kind][t.input_index]
            assert src is not None, "a gradient or tangent slot of an input outside wrt"
            return src[sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride)):]
        if t.kind in (X.K_SCRATCH, X.K_PERSISTENT, X.K_HACC):
            assert t.offset % es == 0
            return (scratch if t.kind == X.K_SCRATCH else persistent)[t.offset // es:]
        assert t.kind in (X.K_COT, X.K_OUTPUT, X.K_TOUT), t.kind
        return {X.K_COT: cot, X.K_OUTPUT: out, X.K_TOUT: tout}[t.kind][out_off:]

    def run(phase, digits, out_off):
        """Runs the phase's nodes; returns the sums of log10 of the factors they measure, without the
        primal root's and the primal root's alone."""
        global node_runs
        exp = exp_root = 0.0
        for i, nd in enumerate(plan.nodes):
            if nd["phase"] != phase or (is_jvp and not primal and nd is root):
                continue
            node_runs += 1
            c = view(nd["c"], digits, out_off)
            if nd.get("zero_fill"):
                c[: nd["c"].nbytes // es] = 0
            s = inv(scale_a[i]) * inv(scale_b[i]) if strip else 1.0

            def v(k, scaled=False):
                x = view(nd[k], digits, out_off)
                return x * s if scaled and s != 1.0 else x

            if nd["kind"] == 2:  # both products into one C, under one scale
                w = np.array(nd["words"][:L.DESC_WORDS], dtype=np.int64)
                emulate_pair(w, v("a"), v("b", True), c)
                w[L.W_FLAGS] |= 1
                emulate_pair(w, v("a2"), v("b2", True), c)
            elif nd.get("d") is not None:
                emulate_absorb(nd["words"], v("a"), v("d"), v("b", True), c)
            elif nd["kind"] == 0:
                emulate_pair(nd["words"], v("a"), v("b", True), c)
            else:
                emulate_single(nd["words"], v("a", True), c)
            if strip and nd["kind"] == 0 and phase <= X.PHASE_VAR_FWD and not marks[i]:
                f = float(np.max(np.abs(c[: math.prod(nd["c"].shape)])))
                factors[slot[id(nd["c"])]] = f
                lg = math.log10(f) if f != 0 else -math.inf
                if nd is root:
                    exp_root = lg
                else:
                    exp += lg
        return exp, exp_root

    with np.errstate(invalid="ignore", over="ignore"):  # (NaN and inf propagate as on the device)
        # 1. the conjugated cotangent copy
        cot = None if cotangent is None else np.ascontiguousarray(cotangent, dtype=dt).reshape(-1)
        if plan.cotangent_offset >= 0:
            o = plan.cotangent_offset // es
            persistent[o:o + cot.size] = np.conj(cot)
            cot = persistent[o:o + cot.size]
        # 2. phase 0, with the invariant factor slots; 3. the H accumulators zeroed
        ns = len(plan.sliced)
        inv_exp = sum(run(X.PHASE_INV_FWD, [0] * ns, 0))
        for t in plan.tensors:
            if t.kind == X.K_HACC:
                persistent[t.offset // es: (t.offset + t.nbytes) // es] = 0
        E = Et = -math.inf if exponent is None else float(exponent)
        wide_fold = wide and not strip and root["c"].kind != X.K_OUTPUT  # (add_chunk_wide)
        # 4. the slices
        for sid in range(plan.nslices) if slice_ids is None else slice_ids:
            digits, rem = [0] * ns, sid  # (decode_slice: least-significant digit first)
            for j in reversed(range(ns)):
                _i, radix, project = plan.sliced[j]
                if project is None:
                    digits[j], rem = rem % radix, rem // radix
                else:
                    digits[j] = project
            out_off = sum(d * s for d, s in zip(digits, plan.slice_out_stride))
            e_wo, e_root = run(X.PHASE_VAR_FWD, digits, out_off)
            e_t = inv_exp + e_wo  # e'_s, without the root's factor
            e_s = e_t + e_root
            if strip and is_vjp:  # the seed divisor 10^(e - e'_s) (strip_seed_kernel)
                factors[seed] = (math.nan if math.isnan(E) or math.isnan(e_s) else
                                 0.0 if -math.inf in (E, e_s) else _pow10(E - e_s))
            run(X.PHASE_VAR_BWD, digits, out_off)
            if strip and not is_vjp:
                # the raw root (and the raw tangent root) into the output against the running exponent
                # (rescale_out_kernel, add_chunk_kernel, commit_exponent_kernel)
                e, et = _exponent_max(E, e_s), _exponent_max(Et, e_t)
                out *= 1.0 if E == e else _pow10(E - e)
                sn = 1.0 if e_s == e else _pow10(e_s - e)
                if root["kind"] == 0:
                    froot = factors[slot[id(root["c"])]]
                    sn = sn / froot if froot != 0 else 0.0
                emulate_single_scaled(plan._chunk_words, view(root["c"], digits, 0), out[out_off:], sn)
                if is_jvp:
                    tout *= 1.0 if Et == et else _pow10(Et - et)
                    st = 0.0 if et == -math.inf else 1.0 if e_t == et else _pow10(e_t - et)
                    emulate_single_scaled(plan._chunk_words, view(troot["c"], digits, 0), tout[out_off:], st)
                E, Et = e, et
            if wide_fold and not (is_jvp and not primal):
                emulate_single_scaled(plan._chunk_words, view(root["c"], digits, 0), out[out_off:], 1.0)
            if wide_fold and troot is not None:
                emulate_single_scaled(plan._chunk_words, view(troot["c"], digits, 0), tout[out_off:], 1.0)
        # 5. the tangent from Et to E (tangent_to_exponent_kernel: 0 for a zero result, NaN with a NaN)
        if strip and is_jvp:
            if math.isnan(E) or math.isnan(Et):
                tout[:] = math.nan
            elif E == -math.inf:
                tout[:] = 0
            else:
                tout *= 1.0 if Et == E else _pow10(Et - E)
        # 6. phase 3; 7. the conjugated gradients
        run(X.PHASE_INV_BWD, [0] * ns, 0)
    if is_vjp:
        res = []
        for i, g in enumerate(grads):
            if g is None or i not in plan.wrt:
                res.append(None)
                continue
            if dt.kind == "c":
                g[:] = np.conj(g)
            res.append(g.reshape(np.shape(arrays[i])))
        return res
    m, t = (x[: plan.out_elements].reshape(plan.out_shape) for x in (out, tout))
    if is_jvp:
        return (m, E, t) if strip else (m, t) if primal else t
    return (m, E) if strip else m
