// rowstream.cuh -- streaming kernel for skinny nodes (N <= 8, K <= 8, no batch):
// one output row per thread, operands read straight from global memory
// (coalesced 128-bit loads when consecutive rows are adjacent in A, which the
// host's dim ordering arranges), the small operand held in registers or
// broadcast from shared memory, 128-bit stores.  No shared-memory staging and
// no producer warps: HBM-bound nodes want LSU wavefronts and instructions per
// row at the minimum and many resident warps to cover latency (ncu showed the
// staged row policy bound by the LSU data pipe).
// (included inside namespace ctgb)
#pragma once

constexpr int RS_MAXDIMS = MAX_T + MAX_G;

// STRIP: fused strip_exponent (a separate instantiation: its few live registers would spill
// inside the row loop of the register-bound variants otherwise)
template <typename T, int NMAX, int KMAX, bool BREG, bool STRIP = false>
__global__ void __launch_bounds__(256, BREG ? 2 : 3)
rowstream_kernel(const int64_t* __restrict__ D, const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C) {
  __shared__ long long s_akoff[KMAX], s_bkoff[KMAX], s_bnoff[NMAX], s_cnoff[NMAX];
  __shared__ long long s_msA[RS_MAXDIMS], s_msC[RS_MAXDIMS];
  __shared__ unsigned s_mext[RS_MAXDIMS];
  __shared__ T s_B[KMAX * NMAX];
  const int tid = threadIdx.x;
  const int n_tm = (int)D[W_NTM], n_gm = (int)D[W_NGM], n_tk = (int)D[W_NTK], n_tn = (int)D[W_NTN];
  const int K = (int)D[W_KTA], N = (int)D[W_NTA];
  const int n_m = n_tm + n_gm;
  const bool accumulate = (D[W_FLAGS] & 1) != 0;
  const bool pair_ok = (D[W_FLAGS] & 2) != 0 && !accumulate && sizeof(T) == 16;
  // 8-byte elements: bit4 = groups of four columns are adjacent and 32-byte aligned,
  // bit5 = pairs of columns adjacent and 16-byte aligned -> 2 x 128-bit / 128-bit row stores
  [[maybe_unused]] const bool quad8 = (D[W_FLAGS] & 16) != 0 && !accumulate && sizeof(T) == 8;
  [[maybe_unused]] const bool pair8 = (D[W_FLAGS] & 32) != 0 && !accumulate && sizeof(T) == 8;
  const bool pow2 = (D[W_FLAGS] & 8) != 0;  // every m dim (tile and grid) is a power of two
  // m dims in enumeration order: tile dims (dim 0 fastest) then grid dims
  for (int d = tid; d < n_m; d += blockDim.x) {
    if (d < n_tm) {
      const int64_t* L = D + OFF_TM + d * 3;
      s_mext[d] = (unsigned)L[0];
      s_msA[d] = L[1];
      s_msC[d] = L[2];
    } else {
      const int64_t* G = D + OFF_GM + (d - n_tm) * 4;
      s_mext[d] = (unsigned)G[0];
      s_msA[d] = G[2];
      s_msC[d] = G[3];
    }
  }
  if (tid < KMAX) {
    long long a = 0, b = 0;
    if (tid < K) {
      unsigned e = tid;
      for (int d = 0; d < n_tk; ++d) {
        const int64_t* L = D + OFF_TK + d * 3;
        unsigned ext = (unsigned)L[0];
        a += (long long)(e % ext) * L[1];
        b += (long long)(e % ext) * L[2];
        e /= ext;
      }
    }
    s_akoff[tid] = a;
    s_bkoff[tid] = b;
  }
  if (tid >= 32 && tid < 32 + NMAX) {
    const int c = tid - 32;
    long long b = 0, o = 0;
    if (c < N) {
      unsigned e = c;
      for (int d = 0; d < n_tn; ++d) {
        const int64_t* L = D + OFF_TN + d * 3;
        unsigned ext = (unsigned)L[0];
        b += (long long)(e % ext) * L[1];
        o += (long long)(e % ext) * L[2];
        e /= ext;
      }
    }
    s_bnoff[c] = b;
    s_cnoff[c] = o;
  }
  __syncthreads();
  if (tid < KMAX * NMAX) {
    const int kk = tid / NMAX, c = tid % NMAX;
    s_B[tid] = (kk < K && c < N) ? B[s_bkoff[kk] + s_bnoff[c]] : zero_of<T>();
  }
  __syncthreads();
  [[maybe_unused]] T breg[BREG ? KMAX : 1][BREG ? NMAX : 1];
  if constexpr (BREG) {
#pragma unroll
    for (int kk = 0; kk < KMAX; ++kk)
#pragma unroll
      for (int c = 0; c < NMAX; ++c) breg[kk][c] = s_B[kk * NMAX + c];
  }
  long long akoff[KMAX];
#pragma unroll
  for (int kk = 0; kk < KMAX; ++kk) akoff[kk] = s_akoff[kk];

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
      unsigned e = live[i] ? (unsigned)m : 0u;
      long long xa = 0, xc = 0;
      if (pow2) {
        for (int d = 0; d < n_m; ++d) {
          const unsigned ext = s_mext[d];
          const unsigned dig = e & (ext - 1);
          e >>= 31 - __clz(ext);
          xa += (long long)dig * s_msA[d];
          xc += (long long)dig * s_msC[d];
        }
      } else {
        for (int d = 0; d < n_m; ++d) {
          const unsigned ext = s_mext[d];
          const unsigned dig = e % ext;
          e /= ext;
          xa += (long long)dig * s_msA[d];
          xc += (long long)dig * s_msC[d];
        }
      }
      oa[i] = xa;
      oc[i] = xc;
    }
    T a[R][KMAX];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int kk = 0; kk < KMAX; ++kk)
        if (kk < K) a[i][kk] = A[oa[i] + akoff[kk]];
    // 16-byte types read s_B afresh for every row: through an index the compiler cannot see
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
                if (c0 + c < N) mac(acc[c], a[i][kk], s_B[sb0 + kk * NMAX + c0 + c]);
              }
            }
          }
        }
        if constexpr (STRIP) {
          if (sctx.scale) {
#pragma unroll
            for (int c = 0; c < CH; ++c)
              if (c0 + c < N) acc[c] = strip_apply(sctx, acc[c]);
          } else {
            // integer scan, then (rarely) a look at the values: see gett_ws.cuh
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
        bool done = false;
        if constexpr (sizeof(T) == 8) {
          if (quad8) {
#pragma unroll
            for (int c = 0; c + 3 < CH; c += 4)
              if (c0 + c < N) {
                const unsigned long long* q = reinterpret_cast<const unsigned long long*>(&acc[c]);
                st_quad8(pc + s_cnoff[c0 + c], q);
              }
            done = true;
          } else if (pair8) {
#pragma unroll
            for (int c = 0; c + 1 < CH; c += 2)
              if (c0 + c < N) {
                const unsigned long long* q = reinterpret_cast<const unsigned long long*>(&acc[c]);
                asm volatile("st.global.v2.b64 [%0], {%1,%2};" ::"l"(pc + s_cnoff[c0 + c]), "l"(q[0]), "l"(q[1])
                             : "memory");
              }
            done = true;
          }
        }
        if (done) continue;
        if (pair_ok) {
#pragma unroll
          for (int c = 0; c < CH; c += 2)
            if (c0 + c < N) store_pair_of(pc + s_cnoff[c0 + c], acc[c], acc[c + 1]);
        } else {
#pragma unroll
          for (int c = 0; c < CH; ++c)
            if (c0 + c < N) {
              T* p = pc + s_cnoff[c0 + c];
              *p = accumulate ? add_of(*p, acc[c]) : acc[c];
            }
        }
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

template <typename T, bool STRIP = false>
__global__ void __launch_bounds__(256, 3)
rowstream_longk_kernel(const int64_t* __restrict__ D, const T* __restrict__ A, const T* __restrict__ B,
                       T* __restrict__ C) {
  __shared__ long long s_akoff[RSK_KMAX], s_bkoff[RSK_KMAX], s_bnoff[RSK_NMAX], s_cnoff[RSK_NMAX];
  __shared__ long long s_msA[RS_MAXDIMS], s_msC[RS_MAXDIMS];
  __shared__ unsigned s_mext[RS_MAXDIMS];
  __shared__ T s_B[RSK_KMAX * RSK_NMAX];
  const int tid = threadIdx.x;
  const int n_tm = (int)D[W_NTM], n_gm = (int)D[W_NGM], n_tk = (int)D[W_NTK], n_tn = (int)D[W_NTN];
  const int K = (int)D[W_KTA], N = (int)D[W_NTA];
  const int n_m = n_tm + n_gm;
  const bool accumulate = (D[W_FLAGS] & 1) != 0;
  [[maybe_unused]] const bool quad8 = (D[W_FLAGS] & 16) != 0 && !accumulate && sizeof(T) == 8;
  const bool pow2 = (D[W_FLAGS] & 8) != 0;
  for (int d = tid; d < n_m; d += blockDim.x) {
    if (d < n_tm) {
      const int64_t* L = D + OFF_TM + d * 3;
      s_mext[d] = (unsigned)L[0];
      s_msA[d] = L[1];
      s_msC[d] = L[2];
    } else {
      const int64_t* G = D + OFF_GM + (d - n_tm) * 4;
      s_mext[d] = (unsigned)G[0];
      s_msA[d] = G[2];
      s_msC[d] = G[3];
    }
  }
  if (tid < RSK_KMAX) {
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
    s_akoff[tid] = a;
    s_bkoff[tid] = b;
  }
  if (tid >= 64 && tid < 64 + RSK_NMAX) {
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
    s_bnoff[c] = b;
    s_cnoff[c] = o;
  }
  __syncthreads();
  for (int i = tid; i < RSK_KMAX * RSK_NMAX; i += blockDim.x) {
    const int kk = i / RSK_NMAX, c = i % RSK_NMAX;
    s_B[i] = (kk < K && c < N) ? B[s_bkoff[kk] + s_bnoff[c]] : zero_of<T>();
  }
  __syncthreads();
  long long inoff[8];  // offsets inside a chunk of 8 k
#pragma unroll
  for (int kk = 0; kk < 8; ++kk) inoff[kk] = s_akoff[kk];
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
      unsigned e = live[i] ? (unsigned)m : 0u;
      long long xa = 0, xc = 0;
      for (int d = 0; d < n_m; ++d) {
        const unsigned ext = s_mext[d];
        const unsigned dig = pow2 ? (e & (ext - 1)) : (e % ext);
        e = pow2 ? (e >> (31 - __clz(ext))) : (e / ext);
        xa += (long long)dig * s_msA[d];
        xc += (long long)dig * s_msC[d];
      }
      oa[i] = xa;
      oc[i] = xc;
    }
    T acc[R][RSK_NMAX];
#pragma unroll
    for (int i = 0; i < R; ++i)
#pragma unroll
      for (int c = 0; c < RSK_NMAX; ++c) acc[i][c] = zero_of<T>();
    for (int kc = 0; kc < nchunks; ++kc) {
      const long long cb = s_akoff[kc * 8];  // chunk base (in_chunk[0] is 0)
      T a[R][8];
#pragma unroll
      for (int i = 0; i < R; ++i)
#pragma unroll
        for (int kk = 0; kk < 8; ++kk) a[i][kk] = (kc * 8 + kk < K) ? A[oa[i] + cb + inoff[kk]] : zero_of<T>();
#pragma unroll
      for (int kk = 0; kk < 8; ++kk)
#pragma unroll
        for (int c = 0; c < RSK_NMAX; ++c) {
          const T b = s_B[(kc * 8 + kk) * RSK_NMAX + c];
#pragma unroll
          for (int i = 0; i < R; ++i) mac(acc[i][c], a[i][kk], b);
        }
    }
#pragma unroll
    for (int i = 0; i < R; ++i) {
      if (!live[i]) continue;
      if constexpr (STRIP) {
        if (sctx.scale) {
#pragma unroll
          for (int c = 0; c < RSK_NMAX; ++c)
            if (c < N) acc[i][c] = strip_apply(sctx, acc[i][c]);
        } else {
          int hmax = 0;
#pragma unroll
          for (int c = 0; c < RSK_NMAX; ++c)
            if (c < N) hmax = max(hmax, strip_hi(acc[i][c]));
          if (strip_hot<T>(sctx, hmax)) {
#pragma unroll
            for (int c = 0; c < RSK_NMAX; ++c)
              if (c < N) strip_note(sctx, acc[i][c]);
          }
        }
      }
      T* pc = C + oc[i];
      bool done = false;
      if constexpr (sizeof(T) == 8) {
        if (quad8) {
#pragma unroll
          for (int c = 0; c + 3 < RSK_NMAX; c += 4)
            if (c < N) {
              const unsigned long long* q = reinterpret_cast<const unsigned long long*>(&acc[i][c]);
              st_quad8(pc + s_cnoff[c], q);
            }
          done = true;
        }
      }
      if (!done) {
#pragma unroll
        for (int c = 0; c < RSK_NMAX; ++c)
          if (c < N) {
            T* p = pc + s_cnoff[c];
            *p = accumulate ? add_of(*p, acc[i][c]) : acc[i][c];
          }
      }
    }
  }
  if constexpr (STRIP) strip_end(sctx);
}
