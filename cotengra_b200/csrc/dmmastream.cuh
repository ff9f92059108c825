// dmmastream.cuh -- fp64 tensor-core streaming kernel for narrow complex128 nodes
// (N <= 8*NJ, K <= 64 -- K <= 32 for NJ = 8 --, no batch): the rowstream idea with DMMA fragments.
//
// Every warp owns blocks of 8*RG output rows and runs them start to finish on its own:
// A fragments straight from global memory into registers (a lane holds one complex element
// per 8-row group: two LDG.64, 8*RG of them in flight per lane), B fragments from a
// zero-padded shared-memory copy made once per CTA, 4 real m16n8k4 DMMAs per pair of 8-row
// groups and B fragment, 128-bit stores.  No operand staging, no producer warps, no CTA
// barriers in the loop: the warps of an SM drift apart, so loads, DMMAs and stores of different row blocks overlap by themselves
// -- which the staged 256x16 policy could not do (all consumer warps share one phase: ncu
// showed its N=16 K=16 node with compute and HBM time adding up instead of overlapping).
// The offset tables and the row decoder are in stream_rows.cuh.
// (included inside namespace ctgb)
#pragma once

constexpr int DS_KMAX = 64;       // k rows of the s.B copy for NJ <= 4
constexpr int DS_KMAX_WIDE = 32;  // ... for NJ = 8 (64 x 64 complex doubles would be 64 KB of static shared memory)

// NJ = column fragments (N <= 8*NJ), RG = 8-row groups per warp block (4: 32 rows, 2: 16 rows -- one
// m16 pair).  128 threads x 3 blocks (NJ <= 2: <= 170 registers) or x 2 blocks (NJ = 4 at 32 rows and
// NJ = 8 at 16 rows: both 64 accumulator doubles per lane).  NJ = 1 serves skinny nodes
// whose contracted space is too long for the row-stream kernel (N <= 8, 8 < K <= 64: the staged
// row policy ran the M = 2^22, N = 8, K = 64 node of the Sycamore slice at 0.57 of its roofline)
// The two-term form (TWO: C (+)= A.B + A2.B2) holds copies of B and B2: with both within the 48 KB of
// static shared memory its k range is shorter for the wide instantiations (ds_two_kb)
__host__ __device__ constexpr int ds_two_kb(int nj) { return nj <= 2 ? DS_KMAX : nj == 4 ? 32 : 16; }

template <int NJ, int RG, bool STRIP = false, bool TWO = false>
__global__ void __launch_bounds__(128, NJ <= 2 ? 3 : 2)
dmmastream_kernel(const int64_t* __restrict__ D, const double2* __restrict__ A, const double2* __restrict__ B,
                  double2* __restrict__ C, const double2* __restrict__ A2, const double2* __restrict__ B2) {
  static_assert(RG == 2 || RG == 4, "a warp block is one or two m16 fragment pairs");
  static_assert(!TWO || !STRIP, "the two-term form is unstripped");
  constexpr int DS_NMAX = NJ * 8, ROWS = RG * 8;
  constexpr int DS_KB = TWO ? ds_two_kb(NJ) : NJ <= 4 ? DS_KMAX : DS_KMAX_WIDE;
  // s.B: [k][n], zero beyond (K, N); the launcher keeps K <= DS_KB
  STREAM_TABLES(double2, DS_KMAX, DS_NMAX, DS_KB);
  __shared__ double2 s_B2[TWO ? DS_KB * DS_NMAX : 1];
  const int tid = threadIdx.x, lane = tid & 31;
  const int K = (int)D[W_KTA], N = (int)D[W_NTA];
  // (a stripped two-term node: both copies / (fA fB))
  const int n_m = s.template load<TWO>(D, B, K, N);
  if constexpr (TWO) s.template copy_b<true>(B2, s_B2, K, N, D);
  // (the flags after the tables: read before them, ptxas gives <8, 2, true> 248 registers, not 244)
  const StreamFlags f = stream_flags<double2>(D);

  [[maybe_unused]] StripCtx sctx;  // fused strip_exponent: its own instantiation (register-bound loop)
  if constexpr (STRIP) sctx = strip_begin(D);
  const int frow = lane >> 2, fk = lane & 3, fc = (lane & 3) * 2;
  const int n8s = (N + 7) >> 3;       // column fragments in use
  const int kchunks = (K + 15) >> 4;  // chunks of 16 k (4 k4-steps each)
  const unsigned long long M = (unsigned long long)D[W_MTA] * (unsigned long long)D[W_TILES_M];
  const unsigned long long nblk = (M + ROWS - 1) / ROWS;
  const unsigned long long wstride = (unsigned long long)gridDim.x * (blockDim.x >> 5);
  for (unsigned long long blk = (unsigned long long)blockIdx.x * (blockDim.x >> 5) + (tid >> 5); blk < nblk;
       blk += wstride) {
    // the lane's RG rows, one per 8-row group (groups 0,1 and 2,3 each form an m16 fragment)
    long long oa[RG], oc[RG];
    bool live[RG];
#pragma unroll
    for (int i = 0; i < RG; ++i) {
      const unsigned long long m = blk * ROWS + (unsigned)(i * 8 + frow);
      live[i] = m < M;
      s.row(n_m, f.pow2, live[i] ? (unsigned)m : 0u, oa[i], oc[i]);
    }
    double re[RG][NJ][2], im[RG][NJ][2];
#pragma unroll
    for (int i = 0; i < RG; ++i)
#pragma unroll
      for (int j = 0; j < NJ; ++j) re[i][j][0] = re[i][j][1] = im[i][j][0] = im[i][j][1] = 0.0;
    // (TWO: the k chunks of A2.B2 follow those of A.B into the same accumulators)
    for (int kt = 0; kt < (TWO ? 2 : 1) * kchunks; ++kt) {
      const bool second = TWO && kt >= kchunks;
      const int kc = second ? kt - kchunks : kt;
      const double2* __restrict__ At = second ? A2 : A;
      const double2* Bt = second ? s_B2 : s.B;
      // 8*RG independent 64-bit loads per lane: element (row i*8 + frow, k = kc*16 + k4*4 + fk).
      // Not one 128-bit load per element: an m16n8k4 A operand is the real (or imaginary)
      // parts of two rows in adjacent registers, and 128-bit loads make ptxas copy them
      // there, which spilled the NJ = 2 kernels.
      double2 a[RG][4];
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        const int kk = kc * 16 + k4 * 4 + fk;
        const long long ko = s.akoff[kk & (DS_KMAX - 1)];
        const bool kin = kk < K;
#pragma unroll
        for (int i = 0; i < RG; ++i) {
          const double* pa = reinterpret_cast<const double*>(At + oa[i] + ko);
          a[i][k4].x = kin ? __ldg(pa) : 0.0;
          a[i][k4].y = kin ? __ldg(pa + 1) : 0.0;
        }
      }
#pragma unroll
      for (int k4 = 0; k4 < 4; ++k4) {
        if (kc * 16 + k4 * 4 >= K) break;  // uniform
        // B fragment: lane holds B[k = .. + fk][n = j*8 + frow]
        double2 b[NJ];
#pragma unroll
        for (int j = 0; j < NJ; ++j) b[j] = Bt[(kc * 16 + k4 * 4 + fk) * DS_NMAX + j * 8 + frow];
#pragma unroll
        for (int i = 0; i < RG; i += 2)
#pragma unroll
          for (int j = 0; j < NJ; ++j)
            if (j < n8s) dmma16x8x4(re[i][j], re[i + 1][j], a[i][k4].x, a[i + 1][k4].x, b[j].x);
#pragma unroll
        for (int i = 0; i < RG; i += 2)
#pragma unroll
          for (int j = 0; j < NJ; ++j)
            if (j < n8s) dmma16x8x4(im[i][j], im[i + 1][j], a[i][k4].x, a[i + 1][k4].x, b[j].y);
#pragma unroll
        for (int i = 0; i < RG; i += 2)
#pragma unroll
          for (int j = 0; j < NJ; ++j)
            if (j < n8s) dmma16x8x4(re[i][j], re[i + 1][j], a[i][k4].y, a[i + 1][k4].y, -b[j].y);
#pragma unroll
        for (int i = 0; i < RG; i += 2)
#pragma unroll
          for (int j = 0; j < NJ; ++j)
            if (j < n8s) dmma16x8x4(im[i][j], im[i + 1][j], a[i][k4].y, a[i + 1][k4].y, b[j].x);
      }
    }
    // (not strip_row of stream_rows.cuh: the accumulators are split re / im DMMA fragments, which
    // it would take as double2 copies, and scaling happens per column pair in the store below)
    if constexpr (STRIP) {
      if (!sctx.scale) {
        // max|C|: integer scan over the accumulators, then (rarely) the values (see gett_ws.cuh)
        int hmax = 0;
#pragma unroll
        for (int i = 0; i < RG; ++i)
#pragma unroll
          for (int j = 0; j < NJ; ++j)
#pragma unroll
            for (int e = 0; e < 2; ++e)
              hmax = max(hmax, max(strip_hi(re[i][j][e]), strip_hi(im[i][j][e])));
        if (strip_hot<double2>(sctx, hmax)) {
#pragma unroll
          for (int i = 0; i < RG; ++i)
#pragma unroll
            for (int j = 0; j < NJ; ++j)
#pragma unroll
              for (int e = 0; e < 2; ++e)
                if (live[i] && j * 8 + fc + e < N) strip_track(sctx, re[i][j][e], im[i][j][e]);
        }
      }
    }
    // a lane owns columns (fc, fc+1) of fragment j in row i*8 + frow
#pragma unroll
    for (int i = 0; i < RG; ++i) {
      if (!live[i]) continue;
      double2* crow = C + oc[i];
#pragma unroll
      for (int j = 0; j < NJ; ++j) {
        const int c = j * 8 + fc;
        if (c >= N) continue;
        double2 v0 = make_double2(re[i][j][0], im[i][j][0]), v1 = make_double2(re[i][j][1], im[i][j][1]);
        if constexpr (STRIP) {
          if (sctx.scale) {
            v0 = strip_apply(sctx, v0);
            if (c + 1 < N) v1 = strip_apply(sctx, v1);
          }
        }
        if (f.pair_ok) {
          store_pair_of(crow + s.cnoff[c], v0, v1);
        } else {
          double2* p0 = crow + s.cnoff[c];
          *p0 = f.accumulate ? add_of(*p0, v0) : v0;
          if (c + 1 < N) {
            double2* p1 = crow + s.cnoff[c + 1];
            *p1 = f.accumulate ? add_of(*p1, v1) : v1;
          }
        }
      }
    }
  }
  if constexpr (STRIP) strip_end(sctx);
}
