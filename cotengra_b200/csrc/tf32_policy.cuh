// tf32_policy.cuh -- single-precision tensor-core policy (included inside
// namespace ctgb from gett_kernels.cuh).
//
// float32 / complex64 contractions on the tensor pipe with the 3xTF32 split:
//     a = a_hi + a_lo,  a_hi = tf32(a),  a_lo = tf32(a - a_hi)
//     a*b ~= a_lo*b_hi + a_hi*b_lo + a_hi*b_hi        (fp32 accumulate)
// which keeps ~fp32 accuracy (the dropped a_lo*b_lo term is 2^-22 relative), as
// BASELINE.json's 1e-5 bound for complex64 requires (a single TF32 pass is 1e-3).
// Instruction: mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32.
// Complex products are four real products per fragment pair:
//     Cr += Ar*Br - Ai*Bi ;  Ci += Ar*Bi + Ai*Br      -> 12 MMAs.
// ONE_PASS (descriptor flags bit7, opt-in): a*b ~= a_hi*b_hi, one MMA per product (4 per complex
// fragment pair), with the same round-to-nearest a_hi and the same per-k8 folding.
#pragma once

__device__ __forceinline__ unsigned to_tf32(float x) {
  unsigned r;
  asm("cvt.rna.tf32.f32 %0, %1;\n" : "=r"(r) : "f"(x));
  return r;
}
// a finite x within half a tf32 ulp of FLT_MAX rounds to inf (and hi + lo = inf - inf): truncate it
// instead; inf and NaN inputs pass through
__device__ __forceinline__ unsigned hi_tf32(float x) {
  unsigned hi = to_tf32(x);
  if ((hi & 0x7FFFFFFFu) == 0x7F800000u && (__float_as_uint(x) & 0x7FFFFFFFu) != 0x7F800000u)
    hi = __float_as_uint(x) & 0xFFFFE000u;
  return hi;
}
// the one-pass operand: no lo term carries a NaN into the product, and cvt.rna turns a NaN whose payload
// lies in the low 13 bits (0x7F800001) into inf, so a NaN gets its quiet bit set instead
__device__ __forceinline__ unsigned one_pass_tf32(float x) {
  const unsigned u = __float_as_uint(x);
  return (u & 0x7FFFFFFFu) > 0x7F800000u ? (u | 0x00400000u) : hi_tf32(x);
}
__device__ __forceinline__ void split_tf32(float x, unsigned& hi, unsigned& lo) {
  hi = hi_tf32(x);
  lo = to_tf32(x - __uint_as_float(hi));
}
__device__ __forceinline__ void mma_tf32(float (&c)[4], const unsigned (&a)[4], const unsigned (&b)[2]) {
  asm volatile(
      "mma.sync.aligned.m16n8k8.row.col.f32.tf32.tf32.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
      : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
      : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b[0]), "r"(b[1]));
}
// c += a*b with the 3-term split (small terms first)
__device__ __forceinline__ void mma_3xtf32(float (&c)[4], const unsigned (&ah)[4], const unsigned (&al)[4],
                                           const unsigned (&bh)[2], const unsigned (&bl)[2]) {
  mma_tf32(c, al, bh);
  mma_tf32(c, ah, bl);
  mma_tf32(c, ah, bh);
}

template <typename T, int WARPS_M, int WARPS_N, int FM, int FN, int KT_, int STAGES_, bool ONE_PASS = false>
struct Tf32Policy {
  // T is float (real) or float2 (complex)
  static constexpr bool CPLX = sizeof(T) == 8;
  static constexpr int MT = WARPS_M * FM * 16, NT = WARPS_N * FN * 8, KT = KT_, STAGES = STAGES_;
  static constexpr int THREADS = WARPS_M * WARPS_N * 32;
  static constexpr int A_ELEMS = MT * KT, B_ELEMS = NT * KT;
  static constexpr int SCRATCH_ELEMS = 0;
  static constexpr int CONSUMER_REGS = (THREADS == 256) ? 232 : 0, PRODUCER_REGS = 40;
  static constexpr bool HAS_BCACHE = false;
  static constexpr int MIN_BLOCKS = 1;
  static_assert(KT % 8 == 0, "KT must be a multiple of the MMA k");
  static constexpr bool SCAN_OK = true;
  struct Acc {
    float re[FM][FN][4];
    float im[CPLX ? FM : 1][CPLX ? FN : 1][4];
  };
  // [k/4][row][k%4]: fragment rows are contiguous -> conflict-free LDS
  __device__ static __forceinline__ int idxA(int r, int kk) { return ((kk >> 2) * MT + r) * 4 + (kk & 3); }
  __device__ static __forceinline__ int idxB(int c, int kk) { return ((kk >> 2) * NT + c) * 4 + (kk & 3); }
  __device__ static __forceinline__ void clear(Acc& acc) {
#pragma unroll
    for (int i = 0; i < FM; ++i)
#pragma unroll
      for (int j = 0; j < FN; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          acc.re[i][j][e] = 0.f;
          if constexpr (CPLX) acc.im[i][j][e] = 0.f;
        }
  }
  __device__ static __forceinline__ float re_of(float v) { return v; }
  __device__ static __forceinline__ float re_of(float2 v) { return v.x; }
  __device__ static __forceinline__ float im_of(float v) { return 0.f; }
  __device__ static __forceinline__ float im_of(float2 v) { return v.y; }
  // operand conversion and product of the mode (lo is left unset, and never read, in one pass)
  __device__ static __forceinline__ void split(float x, unsigned& hi, unsigned& lo) {
    if constexpr (ONE_PASS) hi = one_pass_tf32(x);
    else split_tf32(x, hi, lo);
  }
  __device__ static __forceinline__ void mma(float (&c)[4], const unsigned (&ah)[4], const unsigned (&al)[4],
                                             const unsigned (&bh)[2], const unsigned (&bl)[2]) {
    if constexpr (ONE_PASS) mma_tf32(c, ah, bh);
    else mma_3xtf32(c, ah, al, bh, bl);
  }

  __device__ static __forceinline__ void compute(const T* __restrict__ sA, const T* __restrict__ sB, Acc& acc,
                                                 int kvalid, int ncols) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = warp % WARPS_M, wn = warp / WARPS_M;
    const int g = lane >> 2, t = lane & 3;
    const T* pa = sA + ((wm * FM * 16 + g) * 4 + t);
    const T* pb = sB + ((wn * FN * 8 + g) * 4 + t);
#pragma unroll
    for (int k8 = 0; k8 < KT / 8; ++k8) {
      if (k8 * 8 >= kvalid) break;  // uniform: trailing k of a ragged step are zero
      // B fragments (k = t / t+4, n = g), split once per k8 and reused over FM
      unsigned brh[FN][2], brl[FN][2], bih[CPLX ? FN : 1][2], bil[CPLX ? FN : 1][2];
#pragma unroll
      for (int j = 0; j < FN; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          const T v = pb[((2 * k8 + h) * NT + j * 8) * 4];
          split(re_of(v), brh[j][h], brl[j][h]);
          if constexpr (CPLX) split(im_of(v), bih[j][h], bil[j][h]);
        }
#pragma unroll
      for (int i = 0; i < FM; ++i) {
        // A fragment: a0 (g, t), a1 (g+8, t), a2 (g, t+4), a3 (g+8, t+4)
        unsigned arh[4], arl[4], aih[4], ail[4], nih[4], nil[4];
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const T v = pa[((2 * k8 + (e >> 1)) * MT + i * 16 + (e & 1) * 8) * 4];
          split(re_of(v), arh[e], arl[e]);
          if constexpr (CPLX) {
            split(im_of(v), aih[e], ail[e]);
            nih[e] = aih[e] ^ 0x80000000u;  // -Ai
            if constexpr (!ONE_PASS) nil[e] = ail[e] ^ 0x80000000u;
          }
        }
#pragma unroll
        for (int j = 0; j < FN; ++j) {
          // The tensor core adds into its accumulator with truncation; chained
          // over many k-steps that bias grows linearly (2e-4 on a K=1296 PEPS
          // node).  So every k8 step is accumulated from ZERO inside the MMA and
          // folded into the running sum with a round-to-nearest FADD
          // (Ootomo & Yokota's error-corrected scheme).
          float tr[4] = {0.f, 0.f, 0.f, 0.f};
          mma(tr, arh, arl, brh[j], brl[j]);
          if constexpr (CPLX) {
            float ti[4] = {0.f, 0.f, 0.f, 0.f};
            mma(ti, arh, arl, bih[j], bil[j]);
            mma(tr, nih, nil, bih[j], bil[j]);
            mma(ti, aih, ail, brh[j], brl[j]);
#pragma unroll
            for (int e = 0; e < 4; ++e) acc.im[i][j][e] += ti[e];
          }
#pragma unroll
          for (int e = 0; e < 4; ++e) acc.re[i][j][e] += tr[e];
        }
      }
    }
  }
  __device__ static __forceinline__ void finalize(Acc&) {}
  template <typename F, typename F2>
  __device__ static __forceinline__ void epilogue(Acc& acc, T* scratch, F&& store, F2&& store_pair, bool pair_ok,
                                                  int ncols) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int wm = warp % WARPS_M, wn = warp / WARPS_M;
    const int g = lane >> 2, t = lane & 3;
#pragma unroll
    for (int i = 0; i < FM; ++i)
#pragma unroll
      for (int j = 0; j < FN; ++j)
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          // c0 (g, 2t), c1 (g, 2t+1), c2 (g+8, 2t), c3 (g+8, 2t+1)
          const int r = (wm * FM + i) * 16 + g + (e >> 1) * 8;
          const int c = (wn * FN + j) * 8 + t * 2 + (e & 1);
          if constexpr (CPLX) {
            store(r, c, make_float2(acc.re[i][j][e], acc.im[i][j][e]));
          } else {
            store(r, c, acc.re[i][j][e]);
          }
        }
  }
};
