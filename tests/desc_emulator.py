"""Test-only numpy emulator of the device-side addressing.

Walks a descriptor (``cotengra_b200/csrc/gett_desc.h`` word layout) exactly the
way ``gett_kernel`` does -- work items, grid-base offsets, k-step bases, the
per-element load tables, partial-tile validity, strided stores, split-K -- but
with numpy on the CPU.  It lets the ``-m "not gpu"`` suite verify all host-side
integer work (classification, coalescing, tiling, arenas, slice offsets) against
``numpy.einsum`` / the golden vectors without a GPU.  It is NOT a fallback and is
never imported by the product.
"""

import math

import numpy as np

from cotengra_b200 import executor as X
from cotengra_b200 import lowering as L


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


def emulate_plan(plan, arrays, cotangent=None, slice_ids=None, grads=None):
    """Run an ``ExecPlan`` or, given the output ``cotangent``, a ``VjpPlan`` on the CPU the way
    ``ctgb_plan_execute`` does: the conjugated cotangent copy, phase 0, the zeroed H accumulators,
    per slice phases 1 and 2, phase 3 and the conjugated gradients; slice digits, input, output,
    cotangent and gradient views, zero fills, and strip_exponent per node.  The arenas are exactly
    the reported bytes and filled with NaN, as uninitialised device memory may be: an access
    outside them raises and a read of memory nothing wrote spoils the result.  Returns the output
    of the slices ``slice_ids`` (default all), with its exponent under strip_exponent, or their
    gradients (``None`` outside ``plan.wrt``)."""
    dt = np.dtype(plan.dtype)
    es = plan.esize
    assert plan.workspace_bytes % es == 0 and plan.persistent_bytes % es == 0
    persistent = np.full(plan.persistent_bytes // es, np.nan, dtype=dt)
    scratch = np.full(plan.workspace_bytes // es, np.nan, dtype=dt)
    out = np.zeros(max(plan.out_elements, 1), dtype=dt)
    flats = [np.ascontiguousarray(a, dtype=dt).reshape(-1) for a in arrays]
    if cotangent is not None:
        if grads is None:
            grads = [np.zeros(a.size, dtype=dt) if i in plan.wrt else None for i, a in enumerate(flats)]
        cot = np.ascontiguousarray(cotangent, dtype=dt).reshape(-1)
        if plan.cotangent_offset >= 0:
            o = plan.cotangent_offset // es
            persistent[o:o + cot.size] = np.conj(cot)
            cot = persistent[o:o + cot.size]
    ns = len(plan.sliced)
    radix = [s for _i, s, _p in plan.sliced]
    proj = [p for _i, _s, p in plan.sliced]
    E = -math.inf

    def view(t, digits, out_off):
        if t.kind in (X.K_INPUT, X.K_GRAD):
            off = sum(digits[p] * s for p, s in zip(t.slice_pos, t.slice_stride))
            return (flats if t.kind == X.K_INPUT else grads)[t.input_index][off:]
        if t.kind in (X.K_SCRATCH, X.K_PERSISTENT, X.K_HACC):
            assert t.offset % es == 0
            return (scratch if t.kind == X.K_SCRATCH else persistent)[t.offset // es:]
        if t.kind == X.K_COT:
            return cot[out_off:]
        assert t.kind == X.K_OUTPUT
        return out[out_off:]

    def run(phase, digits, out_off, exp=0.0):
        for nd in plan.nodes:
            if nd["phase"] != phase:
                continue
            c = view(nd["c"], digits, out_off)
            if nd.get("zero_fill"):
                c[: nd["c"].nbytes // es] = 0
            a = view(nd["a"], digits, out_off)
            if nd["kind"] == 0:
                emulate_pair(nd["words"], a, view(nd["b"], digits, out_off), c)
                if plan.strip_exponent:
                    n = math.prod(nd["c"].shape)
                    f = np.max(np.abs(c[:n]))
                    # strip_kernel: an all-zero intermediate keeps its zeros, exponent -> -inf
                    exp += math.log10(f) if f > 0 else -math.inf
                    if f > 0:
                        c[:n] = c[:n] / f
            else:
                emulate_single(nd["words"], a, c)
        return exp

    zero = [0] * ns
    inv_exp = run(X.PHASE_INV_FWD, zero, 0)
    for t in plan.tensors:
        if t.kind == X.K_HACC:
            persistent[t.offset // es: (t.offset + t.nbytes) // es] = 0
    strides = [1] * ns
    for j in range(ns - 2, -1, -1):
        strides[j] = strides[j + 1] * radix[j + 1]
    for i in range(plan.nslices) if slice_ids is None else slice_ids:
        digits, rem = [0] * ns, i
        for j in range(ns):
            if proj[j] is not None:
                digits[j] = proj[j]
            else:
                digits[j] = rem // strides[j]
                rem %= strides[j]
        out_off = sum(d * s for d, s in zip(digits, plan.slice_out_stride))
        exp = run(X.PHASE_VAR_FWD, digits, out_off, inv_exp)
        run(X.PHASE_VAR_BWD, digits, out_off)
        if plan.strip_exponent:
            root = plan.nodes[-1]
            m = view(root["c"], digits, 0)
            e = max(E, exp)
            so = 1.0 if E == e else 10.0 ** (E - e)
            sn = 1.0 if exp == e else 10.0 ** (exp - e)
            out *= so
            chunk = out[out_off:]
            emulate_single_scaled(plan._chunk_words, m, chunk, sn)
            E = e
    run(X.PHASE_INV_BWD, zero, 0)
    if cotangent is not None:
        res = []
        for i, g in enumerate(grads):
            if g is None or i not in plan.wrt:
                res.append(None)
                continue
            if dt.kind == "c":
                g[:] = np.conj(g)
            res.append(g.reshape(np.shape(arrays[i])))
        return res
    res = out[: plan.out_elements].reshape(plan.out_shape)
    return (res, E) if plan.strip_exponent else res


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
