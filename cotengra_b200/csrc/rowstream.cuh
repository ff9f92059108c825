// rowstream.cuh -- streaming kernel for skinny nodes (N <= 8, K <= 8, no batch):
// one output row per thread, operands read straight from global memory
// (coalesced 128-bit loads when consecutive rows are adjacent in A, which the
// host's dim ordering arranges), the small operand held in registers or
// broadcast from shared memory, 128-bit stores.  No shared-memory staging and
// no producer warps: HBM-bound nodes want LSU wavefronts and instructions per
// row at the minimum and many resident warps to cover latency (ncu showed the
// staged row policy bound by the LSU data pipe).
// The offset tables, row decoder, strip scan and row store are in stream_rows.cuh.
// (included inside namespace ctgb)
#pragma once

// STRIP: fused strip_exponent (a separate instantiation: its few live registers would spill
// inside the row loop of the register-bound variants otherwise)
// TWO: C (+)= A.B + A2.B2 (stream_rows.cuh), B2 from shared memory, two blocks per SM (the A2 row
// doubles the operand registers); not with BREG or STRIP.  A stripped two-term node scales the staged
// B and B2 instead (copy_b<true>: a runtime branch in the prologue)
template <typename T, int NMAX, int KMAX, bool BREG, bool STRIP = false, bool TWO = false>
__global__ void __launch_bounds__(256, (BREG || TWO) ? 2 : 3)
rowstream_kernel(const int64_t* __restrict__ D, const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C,
                 const T* __restrict__ A2, const T* __restrict__ B2) {
  static_assert(!TWO || (!BREG && !STRIP), "the two-term form reads B' from shared memory, unstripped");
  STREAM_TABLES(T, KMAX, NMAX, KMAX);
  __shared__ T s_B2[TWO ? KMAX * NMAX : 1];
  const int tid = threadIdx.x;
  const int K = (int)D[W_KTA], N = (int)D[W_NTA];
  const StreamFlags f = stream_flags<T>(D);
  const int n_m = s.template load<TWO>(D, B, K, N);
  if constexpr (TWO) s.template copy_b<true>(B2, s_B2, K, N, D);
  [[maybe_unused]] T breg[BREG ? KMAX : 1][BREG ? NMAX : 1];
  if constexpr (BREG) {
#pragma unroll
    for (int kk = 0; kk < KMAX; ++kk)
#pragma unroll
      for (int c = 0; c < NMAX; ++c) breg[kk][c] = s.B[kk * NMAX + c];
  }
  long long akoff[KMAX];
#pragma unroll
  for (int kk = 0; kk < KMAX; ++kk) akoff[kk] = s.akoff[kk];

  [[maybe_unused]] StripCtx sctx;
  if constexpr (STRIP) sctx = strip_begin(D);
  const unsigned long long M = (unsigned long long)D[W_MTA] * (unsigned long long)D[W_TILES_M];
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  // rows per thread and iteration: narrow element types need more loads in flight
  // per thread to cover HBM latency (Little's law at <= 24 resident warps / SM)
  constexpr int R = sizeof(T) >= 16 ? 1 : ((sizeof(T) == 8 && KMAX <= 4) ? 4 : 2);
  for (unsigned long long m0 = (unsigned long long)blockIdx.x * blockDim.x + tid; m0 < M; m0 += stride * R) {
    long long oa[R], oc[R];
    bool live[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const unsigned long long m = m0 + (unsigned long long)i * stride;
      live[i] = m < M;
      s.row(n_m, f.pow2, live[i] ? (unsigned)m : 0u, oa[i], oc[i]);
    }
    T a[R][KMAX];
    [[maybe_unused]] T a2[TWO ? R : 1][TWO ? KMAX : 1];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int kk = 0; kk < KMAX; ++kk)
        if (kk < K) {
          a[i][kk] = A[oa[i] + akoff[kk]];
          if constexpr (TWO) a2[i][kk] = A2[oa[i] + akoff[kk]];
        }
    // 16-byte types read s.B afresh for every row: through an index the compiler cannot see
    // through, which keeps it from hoisting all KMAX x NMAX reads out of the row loop (for N = K = 8,
    // 64 complex128 values = 256 registers: ptxas spilled them to a 984-byte stack frame and the
    // m20 slice's 2^23 x 8 x 8 nodes streamed at 0.56 TB/s)
    [[maybe_unused]] int sb0 = 0;
    if constexpr (!BREG && sizeof(T) >= 16) asm volatile("" : "+r"(sb0));
    // columns in chunks of CH: 16-byte types with 8 columns would otherwise hold 8 accumulators
    // + 8 operand elements per row (114 registers, 2 blocks / SM; ncu: 25 % of the warps resident,
    // short-scoreboard bound) -- 4 + 8 fit three blocks
    constexpr int CH = (NMAX > 4 && sizeof(T) >= 16) ? 4 : NMAX;
#pragma unroll
    for (int i = 0; i < R; ++i) {
      if (!live[i]) continue;
      T* pc = C + oc[i];
#pragma unroll
      for (int c0 = 0; c0 < NMAX; c0 += CH) {
        if (c0 >= N) break;
        T acc[CH];
#pragma unroll
        for (int c = 0; c < CH; ++c) acc[c] = zero_of<T>();
#pragma unroll
        for (int kk = 0; kk < KMAX; ++kk) {
          if (kk < K) {
#pragma unroll
            for (int c = 0; c < CH; ++c) {
              if constexpr (BREG) {
                mac(acc[c], a[i][kk], breg[kk][c0 + c]);
              } else {
                if (c0 + c < N) mac(acc[c], a[i][kk], s.B[sb0 + kk * NMAX + c0 + c]);
              }
            }
          }
        }
        if constexpr (TWO) {
#pragma unroll
          for (int kk = 0; kk < KMAX; ++kk)
            if (kk < K) {
#pragma unroll
              for (int c = 0; c < CH; ++c)
                if (c0 + c < N) mac(acc[c], a2[i][kk], s_B2[sb0 + kk * NMAX + c0 + c]);
            }
        }
        if constexpr (STRIP) strip_row(sctx, acc, c0, N);
        store_row<true>(pc, s.cnoff, acc, c0, N, f);
      }
    }
  }
  if constexpr (STRIP) strip_end(sctx);
}

// ---- skinny nodes whose contracted space is too long for the kernel above (N <= 8, 8 < K <= 64;
// 8-byte and narrower element types -- complex128 takes the DMMA stream kernel): the same
// thread-per-row stream with the k range walked in chunks of 8.  The m12 slice has an
// M = 2^26, N = 8, K = 64 complex64 node that the staged row policy ran at 0.32 of its roofline.
// Two rows per thread; the offset of element k is chunk_base[k / 8] + in_chunk[k % 8] (the host
// only picks this kernel when the k offsets decompose that way), B is broadcast from shared
// memory, the 8 accumulators of a row stay in registers across the chunks.
constexpr int RSK_KMAX = 64, RSK_NMAX = 8;

// TWO: C (+)= A.B + A2.B2, the chunks of A2 after those of A into the same accumulators (stripped:
// the staged B and B2 scaled, as above)
template <typename T, bool STRIP = false, bool TWO = false>
__global__ void __launch_bounds__(256, 3)
rowstream_longk_kernel(const int64_t* __restrict__ D, const T* __restrict__ A, const T* __restrict__ B,
                       T* __restrict__ C, const T* __restrict__ A2, const T* __restrict__ B2) {
  static_assert(!TWO || !STRIP, "the two-term form is unstripped");
  STREAM_TABLES(T, RSK_KMAX, RSK_NMAX, RSK_KMAX);
  __shared__ T s_B2[TWO ? RSK_KMAX * RSK_NMAX : 1];
  const int tid = threadIdx.x;
  const int K = (int)D[W_KTA], N = (int)D[W_NTA];
  const StreamFlags f = stream_flags<T>(D);
  const int n_m = s.template load<TWO>(D, B, K, N);
  if constexpr (TWO) s.template copy_b<true>(B2, s_B2, K, N, D);
  long long inoff[8];  // offsets inside a chunk of 8 k
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) inoff[kk] = s.akoff[kk];
  const int nchunks = (K + 7) >> 3;
  [[maybe_unused]] StripCtx sctx;
  if constexpr (STRIP) sctx = strip_begin(D);
  const unsigned long long M = (unsigned long long)D[W_MTA] * (unsigned long long)D[W_TILES_M];
  const unsigned long long stride = (unsigned long long)gridDim.x * blockDim.x;
  constexpr int R = 2;
  for (unsigned long long m0 = (unsigned long long)blockIdx.x * blockDim.x + tid; m0 < M; m0 += stride * R) {
    long long oa[R], oc[R];
    bool live[R];
#pragma unroll
    for (int i = 0; i < R; ++i) {
      const unsigned long long m = m0 + (unsigned long long)i * stride;
      live[i] = m < M;
      s.template row<false>(n_m, f.pow2, live[i] ? (unsigned)m : 0u, oa[i], oc[i]);
    }
    T acc[R][RSK_NMAX];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int c = 0; c < RSK_NMAX; ++c) acc[i][c] = zero_of<T>();
    for (int kt = 0; kt < (TWO ? 2 : 1) * nchunks; ++kt) {
      const bool second = TWO && kt >= nchunks;
      const int kc = second ? kt - nchunks : kt;
      const T* __restrict__ At = second ? A2 : A;
      const T* Bt = second ? s_B2 : s.B;
      const long long cb = s.akoff[kc * 8];  // chunk base (in_chunk[0] is 0)
      T a[R][8];
#pragma unroll
      for (int i = 0; i < R; ++i)
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) a[i][kk] = (kc * 8 + kk < K) ? At[oa[i] + cb + inoff[kk]] : zero_of<T>();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int c = 0; c < RSK_NMAX; ++c) {
          const T b = Bt[(kc * 8 + kk) * RSK_NMAX + c];
#pragma unroll
          for (int i = 0; i < R; ++i) mac(acc[i][c], a[i][kk], b);
        }
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      if (!live[i]) continue;
      if constexpr (STRIP) strip_row(sctx, acc[i], 0, N);
      store_row<false>(C + oc[i], s.cnoff, acc[i], 0, N, f);
    }
  }
  if constexpr (STRIP) strip_end(sctx);
}
