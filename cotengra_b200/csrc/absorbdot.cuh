// absorbdot.cuh -- complex128 stem absorption folded into the 32 x 32 product that reads it
// (VAR_ABSORB_ROOT, descriptor layout in gett_desc.h):
//
//     R[m, n] (+)= sum_{k', c} X[m, k', c] V[k', c, n],   X[m, k', c] = sum_k A[m, k', k] Bs[k, c]
//
// with N <= 32, K <= 16.  R's 32 rows are A rows, in blocks of 8 that each take one kept column
// ck of Bs (the absorption's columns that R does not contract; one block per ck when there are
// any).  X (the absorption's result, as large as V) is never stored: each CTA walks its own range of k' units and forms X one 8-column block at a time in
// DMMA accumulators, which are exactly the B fragments of the product with V.
//
// A k' unit is one value of the grid k' dims times the tile k' dim (extent KL = 1 or 2, the k' dim
// of smallest V stride).  A stage is one unit and
// one quarter of the contracted c (32 columns): V[KL x 32 n x 32 c] (32 KB) and A[KL x 32 m x 16 k]
// (16 KB), filled by 16-byte cp.async (zero beyond the extents) into a ring of AB_STAGES stages; Bs is copied once.
// Eight warps: warp w takes rows 16 (w / 4) .. + 16 (two 8-row blocks mb) and columns (w % 4) * 8 .. + 8
// of the quarter, for each k' of the unit.  Per k' and warp, with g = lane / 4, t = lane % 4:
//   X[mb]  [Xr; Xi](8 m x 8 c)  += [Ar; Ai] . Br  +  [-Ai; Ar] . Bi        (8 DMMAs per row block)
//   R^T[nb][mb]  [Rr; Ri]^T(8 n x 8 m) += [Vr; Vi] . Xr + [-Vi; Vr] . Xi   (the transposed complex
//   issue of DESIGN.md section 4, contracting c in two steps of four: lane t's X accumulator holds
//   columns 2t and 2t + 1, so step p takes c = 2t + p)
// A warp keeps a 16 x 32 partial R (32 accumulator doubles per lane); at the end the four column
// blocks' partials are summed in shared memory and added atomically into C (zeroed by the launcher
// unless the descriptor accumulates).
// (included inside namespace ctgb)
#pragma once

constexpr int AB_STAGES = 4;
constexpr int AB_THREADS = 256;
constexpr int AB_VSTAGE = 2 * 32 * 32;  // complex elements of a stage's V tile [kl][n][c]
constexpr int AB_ASTAGE = 2 * 32 * 16;  // ... of its A tile [kl][m][k]
constexpr size_t AB_SMEM = (size_t)(128 * 16 + AB_STAGES * (AB_VSTAGE + AB_ASTAGE)) * sizeof(double2);

__device__ __forceinline__ double ab_neg(double x) { return __longlong_as_double(__double_as_longlong(x) ^ (1ll << 63)); }

__global__ void __launch_bounds__(AB_THREADS, 1)
absorbdot_kernel(const int64_t* __restrict__ D, const double2* __restrict__ A, const double2* __restrict__ Bs,
                 const double2* __restrict__ V, double2* __restrict__ C) {
  extern __shared__ __align__(16) double2 ab_smem[];
  double2* sB = ab_smem;              // [c][k ^ ((c & 1) << 2)], zero beyond (K, C)
  double2* sV = sB + 128 * 16;        // stage s: [kl][n][c ^ (n & 1)]
  double2* sA = sV + AB_STAGES * AB_VSTAGE;  // stage s: [kl][m][k ^ ((m & 1) << 2)]
  __shared__ long long t_ma[32], t_mc[32], t_nv[32], t_cv[128], t_ka[16];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = (int)D[AB_N], K = (int)D[AB_K], CC = (int)D[AB_C], CCP = (int)D[AB_CCP], KL = (int)D[AB_KL];
  const int NG = (int)D[AB_NG];
  const long long kla = D[AB_KLA], klv = D[AB_KLV];
  for (int i = tid; i < 32; i += AB_THREADS) {
    t_ma[i] = D[AB_TMA + i];
    t_mc[i] = D[AB_TMC + i];
    t_nv[i] = D[AB_TNV + i];
  }
  for (int i = tid; i < 128; i += AB_THREADS) t_cv[i] = D[AB_TCV + i];
  for (int i = tid; i < 16; i += AB_THREADS) t_ka[i] = D[AB_TKA + i];
  for (int i = tid; i < 128 * 16; i += AB_THREADS) {
    const int c = i >> 4, k = i & 15;
    const long long cb = D[AB_TCB + c];
    const bool ok = cb >= 0 && k < K;
    cp_async_zfill<16>(sB + c * 16 + (k ^ ((c & 1) << 2)), ok ? Bs + D[AB_TKB + k] + cb : Bs, ok);
  }
  __syncthreads();

  // this CTA's k' units
  const unsigned long long U = (unsigned long long)D[AB_UNITS];
  const unsigned u0 = (unsigned)(U * blockIdx.x / gridDim.x), u1 = (unsigned)(U * (blockIdx.x + 1) / gridDim.x);
  const int nq = CCP >> 5;
  const long long nstage = (long long)(u1 - u0) * nq;

  // unit -> (A, V) base offsets: one lane per grid dim, summed over the warp
  // (the launcher keeps the units below 2^32); the lane's dim is loaded once
  unsigned g_ext = 1, g_div = 1;
  long long g_sa = 0, g_sv = 0;
  if (lane < NG) {
    g_ext = (unsigned)D[AB_G + lane * 4];
    g_div = (unsigned)D[AB_G + lane * 4 + 1];
    g_sa = D[AB_G + lane * 4 + 2];
    g_sv = D[AB_G + lane * 4 + 3];
  }
  auto unit_base = [&](unsigned u, long long& oa, long long& ov) {
    const long long dgt = (long long)((u / g_div) % g_ext);
    long long a = dgt * g_sa, v = dgt * g_sv;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      a += __shfl_xor_sync(0xffffffffu, a, o);
      v += __shfl_xor_sync(0xffffffffu, v, o);
    }
    oa = a;
    ov = v;
  };

  // load cursor
  unsigned lu = u0;
  int lq = 0;
  long long la = 0, lv = 0;
  if (nstage > 0) unit_base(lu, la, lv);
  long long issued = 0;
  auto issue = [&]() {
    if (issued < nstage) {
      const int slot = (int)(issued % AB_STAGES);
      double2* dv = sV + slot * AB_VSTAGE;
      double2* da = sA + slot * AB_ASTAGE;
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        const int e = j * AB_THREADS + tid, cq = e & 31, kl = (e >> 5) & 1, n = e >> 6, c = lq * 32 + cq;
        const bool ok = kl < KL && n < N && c < CC;
        cp_async_zfill<16>(dv + (kl * 32 + n) * 32 + (cq ^ (n & 1)), ok ? V + lv + kl * klv + t_nv[n] + t_cv[c] : V, ok);
      }
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const int e = j * AB_THREADS + tid, k = e & 15, kl = (e >> 4) & 1, m = e >> 5;
        const bool ok = k < K && kl < KL && t_mc[m] >= 0;
        cp_async_zfill<16>(da + (kl * 32 + m) * 16 + (k ^ ((m & 1) << 2)), ok ? A + la + kl * kla + t_ka[k] + t_ma[m] : A,
                           ok);
      }
      ++issued;
      if (++lq == nq) {
        lq = 0;
        ++lu;
        if (issued < nstage) unit_base(lu, la, lv);
      }
    }
    cp_async_commit();
  };
#pragma unroll 1
  for (int s = 0; s < AB_STAGES - 1; ++s) issue();

  const int g = lane >> 2, t = lane & 3;
  const int wmh = warp >> 2, wcb = warp & 3;  // row blocks 2 wmh, 2 wmh + 1; column block of the quarter
  int bofs[2];  // where row block mb's columns start in s.B: its kept column ck of Bs
#pragma unroll
  for (int i = 0; i < 2; ++i) bofs[i] = (int)D[AB_TBCK + 2 * wmh + i] * CCP * 16;
  double Rr[4][2][2], Ri[4][2][2];  // [nb][row block][column pair]
#pragma unroll
  for (int nb = 0; nb < 4; ++nb)
#pragma unroll
    for (int i = 0; i < 2; ++i) Rr[nb][i][0] = Rr[nb][i][1] = Ri[nb][i][0] = Ri[nb][i][1] = 0.0;

#pragma unroll 1
  for (long long s = 0; s < nstage; ++s) {
    cp_async_wait<AB_STAGES - 2>();
    __syncthreads();
    issue();
    const int slot = (int)(s % AB_STAGES), q = (int)(s % nq);
    if (q * 32 + wcb * 8 >= CC) continue;  // warp-uniform: nothing of this block exists
    const double2* vb = sB + (q * 32 + wcb * 8 + g) * 16;
#pragma unroll
    for (int kl = 0; kl < 2; ++kl) {
      if (kl >= KL) break;
      const double2* va = sA + slot * AB_ASTAGE + (kl * 32 + wmh * 16) * 16;
      const double2* vv = sV + slot * AB_VSTAGE + kl * 32 * 32;
      // X block: rows (2 wmh + i) * 8 + g, columns q * 32 + wcb * 8 + 2t, 2t + 1
      double Xr[2][2], Xi[2][2];
#pragma unroll
      for (int i = 0; i < 2; ++i) Xr[i][0] = Xr[i][1] = Xi[i][0] = Xi[i][1] = 0.0;
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) {
        const int kk = (ks * 4 + t) ^ ((g & 1) << 2);
#pragma unroll
        for (int i = 0; i < 2; ++i) {
          const double2 b = vb[bofs[i] + kk];
          const double2 a = va[(i * 8 + g) * 16 + kk];
          dmma16x8x4(Xr[i], Xi[i], a.x, a.y, b.x);
          dmma16x8x4(Xr[i], Xi[i], ab_neg(a.y), a.x, b.y);
        }
      }
#pragma unroll
      for (int p = 0; p < 2; ++p) {
#pragma unroll
        for (int nb = 0; nb < 4; ++nb) {
          const double2 v = vv[(nb * 8 + g) * 32 + ((wcb * 8 + 2 * t + p) ^ (g & 1))];
          const double nvi = ab_neg(v.y);
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            dmma16x8x4(Rr[nb][i], Ri[nb][i], v.x, v.y, Xr[i][p]);
            dmma16x8x4(Rr[nb][i], Ri[nb][i], nvi, v.x, Xi[i][p]);
          }
        }
      }
    }
  }
  cp_async_wait<0>();
  __syncthreads();

  // sum the four column blocks' partials (lane holds R[m = (2 wmh + i) * 8 + 2t + e][n = nb * 8 + g])
  // and add into C
  double2* red = sV;  // 4 x 1024 complex, the ring is idle now
#pragma unroll
  for (int nb = 0; nb < 4; ++nb)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        red[wcb * 1024 + ((2 * wmh + i) * 8 + 2 * t + e) * 32 + nb * 8 + g] = make_double2(Rr[nb][i][e], Ri[nb][i][e]);
  __syncthreads();
  for (int i = tid; i < 1024; i += AB_THREADS) {
    const int m = i >> 5, n = i & 31;
    if (t_mc[m] < 0 || n >= N) continue;
    double2 sum = red[i];
#pragma unroll
    for (int w = 1; w < 4; ++w) sum = add_of(sum, red[w * 1024 + i]);
    atomic_add_of(C + t_mc[m] + D[AB_TNC + n], sum);
  }
}
