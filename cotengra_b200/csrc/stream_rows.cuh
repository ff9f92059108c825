// stream_rows.cuh -- what the row-stream kernels (rowstream.cuh) and the DMMA stream kernel
// (dmmastream.cuh) share: the descriptor words they read, the per-CTA offset tables and
// zero-padded copy of B, the row decoder, and the FMA kernels' fused strip_exponent scan and
// row store.  Each kernel keeps its own main loop: their register budgets differ (80 to 255
// registers for two or three blocks per SM) and a shared loop would move the allocation.
// The two-term instantiations (TWO) form C (+)= A.B + A'.B' for A' laid out as A and B' as B: both
// products go into the same accumulators before the one row store, so C is written once.  With scale
// words (and no factor slot of C) they scale both copies of B as they stage them (copy_b<true>).
// (included inside namespace ctgb)
#pragma once

constexpr int RS_MAXDIMS = MAX_T + MAX_G;

// descriptor flags a stream kernel reads (once, before its row loop)
struct StreamFlags {
  bool accumulate;  // bit0: C += the product
  bool pair_ok;     // bit1: pairs of 16-byte columns adjacent -> store_pair_of
  bool pow2;        // bit3: every m dim (tile and grid) is a power of two
  bool quad8;       // 8-byte elements: bit4 = groups of four columns are adjacent and 32-byte aligned,
  bool pair8;       // bit5 = pairs of columns adjacent and 16-byte aligned -> 2 x 128-bit / 128-bit row stores
};
template <typename T>
__device__ __forceinline__ StreamFlags stream_flags(const int64_t* __restrict__ D) {
  StreamFlags f;
  f.accumulate = (D[W_FLAGS] & 1) != 0;
  f.pair_ok = (D[W_FLAGS] & 2) != 0 && !f.accumulate && sizeof(T) == 16;
  f.pow2 = (D[W_FLAGS] & 8) != 0;
  f.quad8 = (D[W_FLAGS] & 16) != 0 && !f.accumulate && sizeof(T) == 8;
  f.pair8 = (D[W_FLAGS] & 32) != 0 && !f.accumulate && sizeof(T) == 8;
  return f;
}

// The shared-memory tables of a stream kernel: offsets of the KMAX k and NMAX n positions, the m
// dims, and B as a zero-padded [KB][NMAX] copy (KB < KMAX where a full copy would not fit).  The
// kernel declares the arrays (STREAM_TABLES) and this names them: ptxas allocates registers
// differently for one shared struct, which moved the row loops' registers and spills.
#define STREAM_TABLES(T, KMAX, NMAX, KB)                                                  \
  __shared__ long long s_akoff[KMAX], s_bkoff[KMAX], s_bnoff[NMAX], s_cnoff[NMAX];     \
  __shared__ long long s_msA[RS_MAXDIMS], s_msC[RS_MAXDIMS];                           \
  __shared__ unsigned s_mext[RS_MAXDIMS];                                              \
  __shared__ T s_B[(KB) * (NMAX)];                                                     \
  const StreamTables<T, KMAX, NMAX, KB> s{s_akoff, s_bkoff, s_bnoff, s_cnoff, s_msA, s_msC, s_mext, s_B}
template <typename T, int KMAX, int NMAX, int KB = KMAX>
struct StreamTables {
  static_assert(KMAX <= 64 && NMAX <= 64, "threads 0-63 fill the k table, 64-127 the n table");
  long long *akoff, *bkoff, *bnoff, *cnoff;
  long long *msA, *msC;
  unsigned* mext;
  T* B;

  // Every thread of the CTA (at least 128) calls this once; K <= KB and N <= NMAX.  Returns the
  // number of m dims.  (SCALED: copy_b's)
  template <bool SCALED = false>
  __device__ __forceinline__ int load(const int64_t* __restrict__ D, const T* __restrict__ Bg, int K, int N) const {
    const int tid = threadIdx.x;
    const int n_tm = (int)D[W_NTM], n_gm = (int)D[W_NGM], n_tk = (int)D[W_NTK], n_tn = (int)D[W_NTN];
    const int n_m = n_tm + n_gm;
    // m dims in enumeration order: tile dims (dim 0 fastest) then grid dims
    for (int d = tid; d < n_m; d += blockDim.x) {
      if (d < n_tm) {
        const int64_t* L = D + OFF_TM + d * 3;
        mext[d] = (unsigned)L[0];
        msA[d] = L[1];
        msC[d] = L[2];
      } else {
        const int64_t* G = D + OFF_GM + (d - n_tm) * 4;
        mext[d] = (unsigned)G[0];
        msA[d] = G[2];
        msC[d] = G[3];
      }
    }
    if (tid < KMAX) {
      long long a = 0, b = 0;
      if (tid < K) {
        unsigned e = tid;
        for (int d = 0; d < n_tk; ++d) {
          const int64_t* L = D + OFF_TK + d * 3;
          const unsigned ext = (unsigned)L[0];
          a += (long long)(e % ext) * L[1];
          b += (long long)(e % ext) * L[2];
          e /= ext;
        }
      }
      akoff[tid] = a;
      bkoff[tid] = b;
    }
    if (tid >= 64 && tid < 64 + NMAX) {
      const int c = tid - 64;
      long long b = 0, o = 0;
      if (c < N) {
        unsigned e = c;
        for (int d = 0; d < n_tn; ++d) {
          const int64_t* L = D + OFF_TN + d * 3;
          const unsigned ext = (unsigned)L[0];
          b += (long long)(e % ext) * L[1];
          o += (long long)(e % ext) * L[2];
          e /= ext;
        }
      }
      bnoff[c] = b;
      cnoff[c] = o;
    }
    __syncthreads();
    copy_b<SCALED>(Bg, B, K, N, D);
    return n_m;
  }

  // A zero-padded [KB][NMAX] copy of an operand laid out as B (offsets bkoff, bnoff) into dst; the
  // two-term kernels make a second one of B'.  SCALED (the two-term kernels): a descriptor with scale
  // words (W_SCALE_A / W_SCALE_B, a stripped two-term node: C (+)= (A.B + A'.B') / (fA fB)) scales the
  // copy by 1/(fA fB) as it is staged, a zero factor by 0 as strip_begin; a runtime branch
  template <bool SCALED = false>
  __device__ __forceinline__ void copy_b(const T* __restrict__ Bg, T* dst, int K, int N,
                                         [[maybe_unused]] const int64_t* __restrict__ D = nullptr) const {
    [[maybe_unused]] double sa = 1.0, sb = 1.0;
    [[maybe_unused]] bool scaled = false;
    if constexpr (SCALED) {
      const double* pa = reinterpret_cast<const double*>(D[W_SCALE_A]);
      scaled = pa != nullptr;  // (uniform over the CTA)
      if (scaled) {
        const double fa = *pa, fb = *reinterpret_cast<const double*>(D[W_SCALE_B]);
        sa = fa != 0.0 ? 1.0 / fa : 0.0;
        sb = fb != 0.0 ? 1.0 / fb : 0.0;
      }
    }
    for (int i = threadIdx.x; i < KB * NMAX; i += blockDim.x) {
      const int kk = i / NMAX, c = i % NMAX;
      T v = (kk < K && c < N) ? Bg[bkoff[kk] + bnoff[c]] : zero_of<T>();
      if constexpr (SCALED) {
        if (scaled) v = scale2_of(v, sa, sb);
      }
      dst[i] = v;
    }
    __syncthreads();
  }

  // offsets in A and C of row e: its mixed-radix digits over the m dims, by shift and mask when
  // every extent is a power of two (one loop per case, so neither pays for the other's test).
  // SPLIT = false: one loop that selects per digit, which the long-k kernel keeps (with the split
  // loops ptxas moves its spills, 256 / 176 -> 272 / 192 bytes for complex64).
  template <bool SPLIT = true>
  __device__ __forceinline__ void row(int n_m, bool pow2, unsigned e, long long& oa, long long& oc) const {
    long long xa = 0, xc = 0;
    if (!SPLIT) {
      for (int d = 0; d < n_m; ++d) {
        const unsigned ext = mext[d];
        const unsigned dig = pow2 ? (e & (ext - 1)) : (e % ext);
        e = pow2 ? (e >> (31 - __clz(ext))) : (e / ext);
        xa += (long long)dig * msA[d];
        xc += (long long)dig * msC[d];
      }
    } else if (pow2) {
      for (int d = 0; d < n_m; ++d) {
        const unsigned ext = mext[d];
        const unsigned dig = e & (ext - 1);
        e >>= 31 - __clz(ext);
        xa += (long long)dig * msA[d];
        xc += (long long)dig * msC[d];
      }
    } else {
      for (int d = 0; d < n_m; ++d) {
        const unsigned ext = mext[d];
        const unsigned dig = e % ext;
        e /= ext;
        xa += (long long)dig * msA[d];
        xc += (long long)dig * msC[d];
      }
    }
    oa = xa;
    oc = xc;
  }
};

// Fused strip_exponent over the accumulators of columns c0 .. c0 + CH - 1 of a row (those below N):
// scaled when the operands carry factors, else an integer scan and, rarely, a look at the values
// (see gett_ws.cuh)
template <typename T, int CH>
__device__ __forceinline__ void strip_row(StripCtx& sctx, T (&acc)[CH], int c0, int N) {
  if (sctx.scale) {
#pragma unroll
    for (int c = 0; c < CH; ++c)
      if (c0 + c < N) acc[c] = strip_apply(sctx, acc[c]);
  } else {
    int hmax = 0;
#pragma unroll
    for (int c = 0; c < CH; ++c)
      if (c0 + c < N) hmax = max(hmax, strip_hi(acc[c]));
    if (strip_hot<T>(sctx, hmax)) {
#pragma unroll
      for (int c = 0; c < CH; ++c)
        if (c0 + c < N) strip_note(sctx, acc[c]);
    }
  }
}

// Columns c0 .. c0 + CH - 1 of a row (those below N) into C at pc + cnoff[column]: four 8-byte
// columns as two 128-bit stores (quad8), pairs as one 128-bit store (pair8, 8-byte) or two
// (pair_ok, 16-byte), else one store per element, added to C's value when accumulating.
// PAIRS = false compiles the pair paths out (the long-k kernel's stores).
template <bool PAIRS, typename T, int CH>
__device__ __forceinline__ void store_row(T* pc, const long long* cnoff, const T (&acc)[CH], int c0, int N,
                                          const StreamFlags& f) {
  if constexpr (sizeof(T) == 8) {
    if (f.quad8) {
#pragma unroll
      for (int c = 0; c + 3 < CH; c += 4)
        if (c0 + c < N) {
          const unsigned long long* q = reinterpret_cast<const unsigned long long*>(&acc[c]);
          st_quad8(pc + cnoff[c0 + c], q);
        }
      return;
    }
    if (PAIRS && f.pair8) {
#pragma unroll
      for (int c = 0; c + 1 < CH; c += 2)
        if (c0 + c < N) {
          const unsigned long long* q = reinterpret_cast<const unsigned long long*>(&acc[c]);
          asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(pc + cnoff[c0 + c]), "l"(q[0]), "l"(q[1]) : "memory");
        }
      return;
    }
  }
  if (PAIRS && f.pair_ok) {
#pragma unroll
    for (int c = 0; c < CH; c += 2)
      if (c0 + c < N) store_pair_of(pc + cnoff[c0 + c], acc[c], acc[c + 1]);
  } else {
#pragma unroll
    for (int c = 0; c < CH; ++c)
      if (c0 + c < N) {
        T* p = pc + cnoff[c0 + c];
        *p = f.accumulate ? add_of(*p, acc[c]) : acc[c];
      }
  }
}
