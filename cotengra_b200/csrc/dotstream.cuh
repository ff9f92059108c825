// dotstream.cuh -- the final inner product of a contraction tree (M = N = 1, one batch):
// out = sum_k A[k] * B[k] over two operands of up to 2^30 elements whose index orders differ.
//
// The staged KRED policy moves every element with its own cp.async; for 8-byte types that
// is one LSU wavefront per lane (LSU bound for complex64).  Here a thread
// owns the same DS_U tile-local elements of every 2048-element tile: their offsets in A and
// in B (the tile dims' digits times the strides) are launch-invariant and live in registers,
// the tile base (grid dims) is computed once per tile by each warp (one lane per grid dim +
// warp reduction), and the operands come straight from global memory with 2 * DS_U loads in
// flight per thread -- neighbouring lanes read neighbouring elements of A, and a permutation
// of them in B that stays inside the same few sectors (L1 serves the rest).
// Block partial sums are added atomically into the (zeroed) output.
// (included inside namespace ctgb)
#pragma once

constexpr int DOT_KT = 2048, DOT_THREADS = 256, DOT_U = DOT_KT / DOT_THREADS;
// the same stream with a small kept space on both operands (M, N <= 4): the last small tensor
// of a stem peeled over the final inner product (cotengra_b200/fusion.py),
//   R[m, n] = sum_k A[k, m] * B[k, n],
// 16 accumulators per thread, 4 k per thread and tile (16 + 16 loads in flight: 128 KB per SM,
// what the 1x1 kernel needs to stream at HBM rate; 2 k per thread were measurably slower)
constexpr int DOT4_MN = 4;
// k per thread and tile: 4 for 16-byte elements, 8 for narrower ones (the same 128 KB in flight)
template <typename T> constexpr int dot4_u() { return sizeof(T) >= 16 ? 4 : 8; }
template <typename T> constexpr int dot4_kt() { return dot4_u<T>() * DOT_THREADS; }

// CT is the type of C and of every sum on the way to it.  CT = T is the plan dtype's own arithmetic.
// CT = WideOf<T> (descriptor flags bit8, float32 / complex64 roots of accumulate="double" plans) loads
// the operands exactly as above and converts them in registers: products and per-thread sums are
// DFMAs, the warp and block reductions and the one atomicAdd per block and real component are double,
// so the result is the dot product of the fp32 operands to about 1e-15 * sum |a||b|.
template <typename T, int MT, int NT, int U, typename CT = T>
__global__ void __launch_bounds__(DOT_THREADS, (MT * NT > 1) ? 1 : 2)
dotstream_kernel(const int64_t* __restrict__ D, const T* __restrict__ A, const T* __restrict__ B, CT* __restrict__ C) {
  __shared__ CT s_part[DOT_THREADS / 32][MT * NT];
  // the 16 double accumulators of the wide M, N <= 4 kernel (64 registers for complex64) leave no room
  // for the launch-invariant offsets next to the 16 + 16 loads in flight (128 registers): there they
  // wait in shared memory, 2 * U conflict-free and MT + NT broadcast reads per tile of 2 * U * 4 loads
  constexpr bool OFFS_SMEM = MT * NT > 1 && sizeof(CT) > sizeof(T);
  __shared__ long long s_am[OFFS_SMEM ? MT : 1], s_bn[OFFS_SMEM ? NT : 1];
  __shared__ long long s_la[OFFS_SMEM ? U : 1][OFFS_SMEM ? DOT_THREADS : 1], s_lb[OFFS_SMEM ? U : 1][OFFS_SMEM ? DOT_THREADS : 1];
  const int tid = threadIdx.x, lane = tid & 31;
  const int n_tk = (int)D[W_NTK], n_gk = (int)D[W_NGK];
  const int KTa = (int)D[W_KTA], MTa = (int)D[W_MTA], NTa = (int)D[W_NTA];
  const unsigned steps = (unsigned)D[W_STEPS_K];  // the host guarantees < 2^31
  // offsets of the kept indices (all of M and N sit inside the tile)
  long long am[MT], bn[NT];
#pragma unroll
  for (int i = 0; i < MT; ++i) {
    long long a = 0;
    unsigned e = (unsigned)i;
    if (MT > 1 && i < MTa)
      for (int d = 0; d < (int)D[W_NTM]; ++d) {
        const int64_t* L = D + OFF_TM + d * 3;
        a += (long long)(e % (unsigned)L[0]) * L[1];
        e /= (unsigned)L[0];
      }
    am[i] = a;
    if (OFFS_SMEM && tid == 0) s_am[i] = a;
  }
#pragma unroll
  for (int i = 0; i < NT; ++i) {
    long long b = 0;
    unsigned e = (unsigned)i;
    if (NT > 1 && i < NTa)
      for (int d = 0; d < (int)D[W_NTN]; ++d) {
        const int64_t* L = D + OFF_TN + d * 3;
        b += (long long)(e % (unsigned)L[0]) * L[1];
        e /= (unsigned)L[0];
      }
    bn[i] = b;
    if (OFFS_SMEM && tid == 0) s_bn[i] = b;
  }
  if (OFFS_SMEM) __syncthreads();
  // tile-local offsets of this thread's elements (tile dims: dim 0 fastest)
  long long la[U], lb[U];
  bool in_tile[U];
#pragma unroll
  for (int j = 0; j < U; ++j) {
    unsigned e = (unsigned)(tid + j * DOT_THREADS);
    in_tile[j] = e < (unsigned)KTa;
    if (!in_tile[j]) e = 0;
    long long a = 0, b = 0;
    for (int d = 0; d < n_tk; ++d) {
      const int64_t* L = D + OFF_TK + d * 3;
      const unsigned ext = (unsigned)L[0];
      a += (long long)(e % ext) * L[1];
      b += (long long)(e % ext) * L[2];
      e /= ext;
    }
    la[j] = a;
    lb[j] = b;
    if (OFFS_SMEM) {
      s_la[j][tid] = a;
      s_lb[j][tid] = b;
    }
  }
  // this lane's grid dims (at most 2 per lane: MAX_G = 40 <= 64)
  unsigned g_ext[2] = {1u, 1u};
  unsigned g_div[2] = {1u, 1u};
  long long g_sa[2] = {0, 0}, g_sb[2] = {0, 0};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = lane + 32 * h;
    if (q < n_gk) {
      const int64_t* G = D + OFF_GK + q * 4;
      g_ext[h] = (unsigned)G[0];
      g_div[h] = (unsigned)G[1];
      g_sa[h] = G[2];
      g_sb[h] = G[3];
    }
  }
  CT acc[MT][NT];
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int c = 0; c < NT; ++c) acc[i][c] = zero_of<CT>();
  for (unsigned t = blockIdx.x; t < steps; t += gridDim.x) {
    long long ta = 0, tb = 0;
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      const unsigned dig = (t / g_div[h]) % g_ext[h];
      ta += (long long)dig * g_sa[h];
      tb += (long long)dig * g_sb[h];
    }
    ta = warp_sum_ll(ta);
    tb = warp_sum_ll(tb);
    T a[U][MT], b[U][NT];
#pragma unroll
    for (int j = 0; j < U; ++j) {
#pragma unroll
      for (int i = 0; i < MT; ++i)
        a[j][i] = (in_tile[j] && i < MTa) ? A[ta + (OFFS_SMEM ? s_la[j][tid] + s_am[i] : la[j] + am[i])] : zero_of<T>();
#pragma unroll
      for (int c = 0; c < NT; ++c)
        b[j][c] = (in_tile[j] && c < NTa) ? B[tb + (OFFS_SMEM ? s_lb[j][tid] + s_bn[c] : lb[j] + bn[c])] : zero_of<T>();
    }
#pragma unroll
    for (int j = 0; j < U; ++j)
#pragma unroll
      for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int c = 0; c < NT; ++c) mac(acc[i][c], a[j][i], b[j][c]);
  }
  // block reduction, one atomic per block and output element
#pragma unroll
  for (int i = 0; i < MT; ++i)
#pragma unroll
    for (int c = 0; c < NT; ++c) {
      CT v = acc[i][c];
#pragma unroll
      for (int d = 16; d > 0; d >>= 1) v = add_of(v, shfl_down_of(v, d));
      if (lane == 0) s_part[tid >> 5][i * NT + c] = v;
    }
  __syncthreads();
  if (tid < MT * NT) {
    const int i = tid / NT, c = tid % NT;
    if (i < MTa && c < NTa) {
      CT v = s_part[0][tid];
      for (int w = 1; w < DOT_THREADS / 32; ++w) v = add_of(v, s_part[w][tid]);
      StripCtx sctx = strip_begin(D);  // strip_exponent: partial sums are only scaled here
      if (sctx.scale) v = strip_apply(sctx, v);
      long long oc = 0;
      unsigned e = (unsigned)i;
      for (int d = 0; d < (int)D[W_NTM]; ++d) {
        const int64_t* L = D + OFF_TM + d * 3;
        oc += (long long)(e % (unsigned)L[0]) * L[2];
        e /= (unsigned)L[0];
      }
      e = (unsigned)c;
      for (int d = 0; d < (int)D[W_NTN]; ++d) {
        const int64_t* L = D + OFF_TN + d * 3;
        oc += (long long)(e % (unsigned)L[0]) * L[2];
        e /= (unsigned)L[0];
      }
      atomic_add_of(C + oc, v);
    }
  }
}
