// tc05_policy.cuh -- operand preparation for the wgmma (tf32) complex64 kernel.
// Included inside namespace ctgb.  The kernel itself is tc05_kernel.cuh.
//
// A complex tile product C[128 x NT] += A[128 x 16] * B[16 x NT] is run as the real
// product  C'[128 x 2NT] += A'[128 x 32] * B'[2NT x 32]^T  where A' is A's own
// (re, im)-interleaved image and B' is the 2x2-block embedding
//   B'[2n][2k] = Br   B'[2n][2k+1] = -Bi   B'[2n+1][2k] = Bi   B'[2n+1][2k+1] = Br
// so that C' is C's own interleaved image.  fp32 accuracy comes from the 3xTF32
// split  D = A'hi*B'hi + (A'lo*B'hi + A'hi*B'lo)  (hi = rn_tf32(x), lo = rn_tf32(x - hi); the tensor
// core itself would only truncate, which biases a deep tree).  The opt-in one-pass mode (descriptor
// flags bit7) keeps D = A'hi*B'hi: the same round-to-nearest hi, no lo images.
//
// B' (hi and lo, already in shared-memory tile order: wgmma's K-major no-swizzle
// core-matrix layout [chunk = k'/4][row][k'%4]) is prepared once per launch by
// bprime_kernel -- B is the small operand, <= a few MB -- so that each k-step's pair
// of tiles is ONE contiguous TMA bulk copy.
#pragma once

__device__ __forceinline__ uint64_t gmma_desc_kmajor(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
  // wgmma matrix descriptor (PTX ISA, "Matrix Descriptor Format"): start>>4 [0,14), LBO>>4 [16,30),
  // SBO>>4 [32,46), base offset [49,52) = 0, layout [62,64) = 0 (no swizzle).  K-major, no swizzle:
  // LBO = stride between the two core matrices along K, SBO = stride between 8-row groups
  return (uint64_t)((saddr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
         ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
// Round to nearest (ties away) onto the tf32 grid with integer ALU ops.  The tensor core only truncates,
// and a truncating split (hi = trunc(x), lo = x - hi, lo truncated again by the MMA) biases every product
// towards zero by ~2^-22: over the dependent nodes of a deep tree that bias adds up linearly.
// cvt.rna.tf32.f32 does the same with a slower instruction; add + mask are full-rate.
__device__ __forceinline__ float trunc_tf32(float x) { return __uint_as_float(__float_as_uint(x) & 0xFFFFE000u); }
// the low half: the MMA drops the 13 low bits itself, adding half a tf32 ulp first makes that a rounding
__device__ __forceinline__ float half_up_tf32(float x) { return __uint_as_float(__float_as_uint(x) + 0x1000u); }
// The fast 3xTF32 split: hi = round_tf32(x), lo = half_up_tf32(x - hi) (x - hi is exact).  Its integer add
// must not reach the exponent field, and for three kinds of input it does: a NaN whose top mantissa bits
// are set (0x7FFFFFFF, the NaN GPU arithmetic makes) carries into the sign bit and becomes +-0, a finite x
// within half a tf32 ulp of FLT_MAX becomes inf, and a NaN with its payload in the low 13 bits (0x7F800001)
// becomes inf.  Exactly for those (and for +-inf) x - hi is not finite, which is how the producer's scatter
// (tc05_kernel.cuh) finds them and sends them to tc05_split; bprime_kernel calls tc05_split directly.
__device__ __forceinline__ float round_tf32(float x) {
  return __uint_as_float((__float_as_uint(x) + 0x1000u) & 0xFFFFE000u);
}
// hi for every input: a finite x whose rounding would carry into the exponent is truncated (lo stays
// finite and exact), inf stays inf, a NaN gets its quiet bit set (the MMA reads only the top 10 mantissa
// bits, so 0x7F800001 would otherwise be read as inf).  The one-pass mode's operand is this hi alone.
__device__ __forceinline__ float tc05_hi(float x) {
  const unsigned u = __float_as_uint(x), a = u & 0x7FFFFFFFu;
  unsigned h = (u + 0x1000u) & 0xFFFFE000u;
  if (a >= 0x7F7FF000u) h = a > 0x7F800000u ? (u | 0x00400000u) : a == 0x7F800000u ? u : (u & 0xFFFFE000u);
  return __uint_as_float(h);
}
// The split for every input.  lo of an inf or NaN is whatever the add makes of x - hi: the product is
// non-finite either way.
__device__ __forceinline__ void tc05_split(float x, float& hi, float& lo) {
  hi = tc05_hi(x);
  lo = half_up_tf32(x - hi);
}

// B -> B'hi / B'lo in shared-memory tile order:
//   Bp[((ib*tiles_n + in)*steps_k + step)][chunk 0..7][row 0..4NT-1: hi rows, then lo rows][4 floats]
// ONE (a single tf32 pass): B'hi alone, rows 0..2NT-1 of every chunk.
template <int NT, bool ONE = false>
__global__ void __launch_bounds__(256) bprime_kernel(const int64_t* __restrict__ D, const float2* __restrict__ B,
                                                     float* __restrict__ Bp) {
  constexpr int TILE = 8 * (2 * NT) * 4;
  const int n_tn = (int)D[W_NTN], n_tk = (int)D[W_NTK], n_gn = (int)D[W_NGN], n_gk = (int)D[W_NGK], n_gb = (int)D[W_NGB];
  const unsigned tiles_n = (unsigned)D[W_TILES_N], tiles_b = (unsigned)D[W_TILES_B], steps_k = (unsigned)D[W_STEPS_K];
  const unsigned long long total = (unsigned long long)tiles_b * tiles_n * steps_k * TILE;
  for (unsigned long long idx = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; idx < total;
       idx += (unsigned long long)gridDim.x * blockDim.x) {
    const unsigned e = (unsigned)(idx % TILE);
    unsigned t = (unsigned)(idx / TILE);
    const unsigned step = t % steps_k;
    t /= steps_k;
    const unsigned in_ = t % tiles_n, ib_ = t / tiles_n;
    const unsigned j = e & 3, row = (e >> 2) % (2 * NT), chunk = (e >> 2) / (2 * NT);
    const unsigned kp = chunk * 4 + j, kk = kp >> 1, p = kp & 1, c = row >> 1, q = row & 1;
    long long off = 0;
    {
      unsigned x = c;
      for (int d = 0; d < n_tn; ++d) {
        const int64_t* L = D + OFF_TN + d * 3;
        off += (long long)(x % (unsigned)L[0]) * L[1];
        x /= (unsigned)L[0];
      }
      x = kk;
      for (int d = 0; d < n_tk; ++d) {
        const int64_t* L = D + OFF_TK + d * 3;
        off += (long long)(x % (unsigned)L[0]) * L[2];
        x /= (unsigned)L[0];
      }
      for (int d = 0; d < n_gn; ++d) {
        const int64_t* G = D + OFF_GN + d * 4;
        off += (long long)((in_ / (unsigned)G[1]) % (unsigned)G[0]) * G[2];
      }
      for (int d = 0; d < n_gk; ++d) {
        const int64_t* G = D + OFF_GK + d * 4;
        off += (long long)((step / (unsigned)G[1]) % (unsigned)G[0]) * G[3];
      }
      for (int d = 0; d < n_gb; ++d) {
        const int64_t* G = D + OFF_GB + d * 5;
        off += (long long)((ib_ / (unsigned)G[1]) % (unsigned)G[0]) * G[3];
      }
    }
    const float2 b = B[off];
    const float v = (q == p) ? b.x : (q == 0 ? -b.y : b.y);
    if constexpr (ONE) {
      Bp[(idx / TILE) * TILE + ((unsigned long long)chunk * (2 * NT) + row) * 4 + j] = tc05_hi(v);
      continue;
    }
    // stacked along N: chunk c holds 4NT rows -- rows [0, 2NT) are B'hi, rows [2NT, 4NT) are B'lo --
    // so that one wgmma of N = 4NT multiplies A'hi with both and one of N = 2NT takes B'hi alone
    const unsigned long long base = (idx / TILE) * (2ull * TILE) + ((unsigned long long)chunk * (4 * NT)) * 4 + j;
#ifdef CTGB_TC05_TRUNC_SPLIT  // A/B knob: the truncating split (inf gives lo = inf - inf = NaN: a product
                              // with an inf operand comes out NaN, not inf; not run by the test suite)
    Bp[base + row * 4] = v;
    Bp[base + (row + 2 * NT) * 4] = v - trunc_tf32(v);
#else
    float vh, vl;
    tc05_split(v, vh, vl);
    Bp[base + row * 4] = vh;                   // hi
    Bp[base + (row + 2 * NT) * 4] = vl;        // lo
#endif
  }
}
