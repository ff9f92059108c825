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
// of smallest V stride).  A stage is one unit and one quarter of the contracted c (32 columns):
// V[KL x 32 n x 32 c] (32 KB) and A[KL x AROWS m x 16 k], filled by 16-byte cp.async (zero beyond
// the extents); Bs is copied once.  When the 32 rows are 8 A rows repeated once per ck (A8: CK > 1,
// or at most 8 rows) a stage holds those 8 rows (4 KB), else all 32 (16 KB).
//
// Warp specialised: a producer warpgroup issues every gather into a ring of AbRing::STAGES stages
// behind full / empty mbarriers (gett_ws.cuh), so the eight consumer warps only load fragments and
// issue DMMAs, and no CTA-wide barrier runs in the loop.  The producers hand registers to the
// consumers (setmaxnreg: 56 and 224 per thread; a 12-warp CTA starts at 168, as the register file
// is split over the four SM sub-partitions).  Consumer warp w takes rows 16 (w / 4) .. + 16 (two
// 8-row blocks mb) and columns (w % 4) * 8 .. + 8 of the quarter, for each k' of the unit.
// Per k' and warp, with g = lane / 4, t = lane % 4:
//   X[mb]  [Xr; Xi](8 m x 8 c)  += [Ar; Ai] . Br  +  [-Ai; Ar] . Bi        (8 DMMAs per row block)
//   R^T[nb][mb]  [Rr; Ri]^T(8 n x 8 m) += [Vr; Vi] . Xr + [-Vi; Vr] . Xi   (the transposed complex
//   issue of DESIGN.md section 4, contracting c in two steps of four: lane t's X accumulator holds
//   columns 2t and 2t + 1, so step p takes c = 2t + p)
// With A8 both row blocks read the same A fragment, loaded once.  With one quarter (CCP = 32) a
// warp's column block never changes, so its Bs fragments are held in registers for the whole loop.
// A warp keeps a 16 x 32 partial R (32 accumulator doubles per lane); at the end the four column
// blocks' partials are summed in shared memory and added atomically into C (zeroed by the launcher
// unless the descriptor accumulates).
// (included inside namespace ctgb, after gett_ws.cuh)
#pragma once

constexpr int AB_CONSUMERS = 256;               // eight DMMA warps
constexpr int AB_THREADS = AB_CONSUMERS + 128;  // and a producer warpgroup
constexpr int AB_VSTAGE = 2 * 32 * 32;         // complex elements of a stage's V tile [kl][n][c]

template <bool A8>
struct AbRing {
  static constexpr int AROWS = A8 ? 8 : 32;     // A rows a stage holds
  static constexpr int ASTAGE = 2 * AROWS * 16;  // complex elements of its A tile [kl][m][k]
  static constexpr int STAGES = A8 ? 5 : 4;      // as deep as 227 KB of shared memory allows
  static constexpr size_t SMEM = (size_t)(128 * 16 + STAGES * (AB_VSTAGE + ASTAGE)) * sizeof(double2);
};

__device__ __forceinline__ double ab_neg(double x) { return __longlong_as_double(__double_as_longlong(x) ^ (1ll << 63)); }

template <bool A8, bool BREG>
__global__ void __launch_bounds__(AB_THREADS, 1)
absorbdot_kernel(const int64_t* __restrict__ D, const double2* __restrict__ A, const double2* __restrict__ Bs,
                 const double2* __restrict__ V, double2* __restrict__ C) {
  using RG = AbRing<A8>;
  extern __shared__ __align__(16) double2 ab_smem[];
  double2* sB = ab_smem;              // [c][k ^ ((c & 1) << 2)], zero beyond (K, C)
  double2* sV = sB + 128 * 16;        // stage s: [kl][n][c ^ (n & 1)]
  double2* sA = sV + RG::STAGES * AB_VSTAGE;  // stage s: [kl][m][k ^ ((m & 1) << 2)]
  __shared__ long long t_ma[32], t_mc[32], t_nv[32], t_cv[128], t_ka[16];
  __shared__ unsigned long long bar_full[RG::STAGES], bar_empty[RG::STAGES];

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int N = (int)D[AB_N], K = (int)D[AB_K], CC = (int)D[AB_C], CCP = (int)D[AB_CCP], KL = (int)D[AB_KL];
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
  if (tid == 0) {
    for (int s = 0; s < RG::STAGES; ++s) {
      mbar_init(&bar_full[s], AB_THREADS - AB_CONSUMERS);
      mbar_init(&bar_empty[s], AB_CONSUMERS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  cp_async_commit();
  cp_async_wait<0>();
  __syncthreads();

  // this CTA's k' units
  const unsigned long long U = (unsigned long long)D[AB_UNITS];
  const unsigned u0 = (unsigned)(U * blockIdx.x / gridDim.x), u1 = (unsigned)(U * (blockIdx.x + 1) / gridDim.x);
  const int nq = CCP >> 5;
  const long long nstage = (long long)(u1 - u0) * nq;

  if (warp >= AB_CONSUMERS / 32) {
    reg_dealloc<56>();
    // producer warp pw: unit -> (A, V) base offsets, one lane per grid dim summed over the warp (the
    // launcher keeps the units below 2^32); the lane's dim is loaded once
    const int pw = warp - AB_CONSUMERS / 32;
    const int NG = (int)D[AB_NG];
    const long long kla = D[AB_KLA], klv = D[AB_KLV];
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
    // V: a lane copies the k' vkl and the columns vc, vc + 16 of the quarter, for n = 8 pw .. + 8; the
    // lane bits are (c0, kl, c1, c2, c3), so the two k' of the 64-byte runs V has where c0 and kl are
    // its two smallest strides are copied by one instruction.  A: the k' akl and the k ak, for the
    // rows pw + 4j.
    const int vkl = (lane >> 1) & 1, vc = (lane & 1) | ((lane >> 2) << 1);
    const int akl = lane >> 4, ak = lane & 15;
    unsigned lu = u0;
    int lq = 0;
    long long la = 0, lv = 0;
    unit_base(lu, la, lv);
    int slot = 0;
    unsigned ph = 0;
#pragma unroll 1
    for (long long s = 0; s < nstage; ++s) {
      mbar_wait(&bar_empty[slot], ph ^ 1);
      double2* dv = sV + slot * AB_VSTAGE + vkl * 32 * 32;
      double2* da = sA + slot * RG::ASTAGE + akl * RG::AROWS * 16;
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const int cq = vc + 16 * h, c = lq * 32 + cq;
        const bool okc = vkl < KL && c < CC;
        const double2* src = V + lv + vkl * klv + t_cv[c];
#pragma unroll
        for (int n = 8 * pw; n < 8 * pw + 8; ++n) {
          const bool ok = okc && n < N;
          cp_async_zfill<16>(dv + n * 32 + (cq ^ (n & 1)), ok ? src + t_nv[n] : V, ok);
        }
      }
      {
        const bool okk = ak < K && akl < KL;
        const double2* src = A + la + akl * kla + t_ka[ak];
#pragma unroll
        for (int m = pw; m < RG::AROWS; m += 4) {
          const bool ok = okk && t_mc[m] >= 0;
          cp_async_zfill<16>(da + m * 16 + (ak ^ ((m & 1) << 2)), ok ? src + t_ma[m] : A, ok);
        }
      }
      mbar_arrive_cp_async(&bar_full[slot]);
      if (++slot == RG::STAGES) {
        slot = 0;
        ph ^= 1;
      }
      if (++lq == nq) {
        lq = 0;
        ++lu;
        if (s + 1 < nstage) unit_base(lu, la, lv);
      }
    }
    cp_async_commit();
    cp_async_wait<0>();
    return;
  }

  reg_alloc<224>();
  const int g = lane >> 2, t = lane & 3;
  const int wmh = warp >> 2, wcb = warp & 3;  // row blocks 2 wmh, 2 wmh + 1; column block of the quarter
  int bofs[2];  // where row block mb's columns start in s.B: its kept column ck of Bs
#pragma unroll
  for (int i = 0; i < 2; ++i) bofs[i] = (int)D[AB_TBCK + 2 * wmh + i] * CCP * 16;
  double2 breg[2][4];  // BREG: the warp's Bs fragments [row block][k step]
  if constexpr (BREG) {
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int ks = 0; ks < 4; ++ks) breg[i][ks] = sB[(wcb * 8 + g) * 16 + bofs[i] + ((ks * 4 + t) ^ ((g & 1) << 2))];
  }
  double Rr[4][2][2], Ri[4][2][2];  // [nb][row block][column pair]
#pragma unroll
  for (int nb = 0; nb < 4; ++nb)
#pragma unroll
    for (int i = 0; i < 2; ++i) Rr[nb][i][0] = Rr[nb][i][1] = Ri[nb][i][0] = Ri[nb][i][1] = 0.0;

  int slot = 0, q = 0;
  unsigned ph = 0;
#pragma unroll 1
  for (long long s = 0; s < nstage; ++s) {
    mbar_wait(&bar_full[slot], ph);
    if (q * 32 + wcb * 8 < CC) {  // warp-uniform: else nothing of this block exists
      const double2* vb = sB + (q * 32 + wcb * 8 + g) * 16;
#pragma unroll
      for (int kl = 0; kl < 2; ++kl) {
        if (kl >= KL) break;
        const double2* va = sA + slot * RG::ASTAGE + kl * RG::AROWS * 16 + (A8 ? 0 : wmh * 16 * 16);
        const double2* vv = sV + slot * AB_VSTAGE + kl * 32 * 32;
        // X block: rows (2 wmh + i) * 8 + g, columns q * 32 + wcb * 8 + 2t, 2t + 1
        double Xr[2][2], Xi[2][2];
#pragma unroll
        for (int i = 0; i < 2; ++i) Xr[i][0] = Xr[i][1] = Xi[i][0] = Xi[i][1] = 0.0;
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
          const int kk = (ks * 4 + t) ^ ((g & 1) << 2);
          double2 a[2];
          a[0] = va[g * 16 + kk];
          a[1] = A8 ? a[0] : va[(8 + g) * 16 + kk];
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            const double2 b = BREG ? breg[i][ks] : vb[bofs[i] + kk];
            dmma16x8x4(Xr[i], Xi[i], a[i].x, a[i].y, b.x);
            dmma16x8x4(Xr[i], Xi[i], ab_neg(a[i].y), a[i].x, b.y);
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
    __syncwarp();
    if (lane == 0) mbar_arrive(&bar_empty[slot]);
    if (++slot == RG::STAGES) {
      slot = 0;
      ph ^= 1;
    }
    if (++q == nq) q = 0;
  }
  named_sync<1, AB_CONSUMERS>();  // every consumer is done with the ring, and every stage has landed

  // sum the four column blocks' partials (lane holds R[m = (2 wmh + i) * 8 + 2t + e][n = nb * 8 + g])
  // and add into C
  double2* red = sV;  // 4 x 1024 complex
#pragma unroll
  for (int nb = 0; nb < 4; ++nb)
#pragma unroll
    for (int i = 0; i < 2; ++i)
#pragma unroll
      for (int e = 0; e < 2; ++e)
        red[wcb * 1024 + ((2 * wmh + i) * 8 + 2 * t + e) * 32 + nb * 8 + g] = make_double2(Rr[nb][i][e], Ri[nb][i][e]);
  named_sync<1, AB_CONSUMERS>();
  for (int i = tid; i < 1024; i += AB_CONSUMERS) {
    const int m = i >> 5, n = i & 31;
    if (t_mc[m] < 0 || n >= N) continue;
    double2 sum = red[i];
#pragma unroll
    for (int w = 1; w < 4; ++w) sum = add_of(sum, red[w * 1024 + i]);
    atomic_add_of(C + t_mc[m] + D[AB_TNC + n], sum);
  }
}
