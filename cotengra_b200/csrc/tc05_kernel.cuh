// tc05_kernel.cuh -- complex64 dense nodes on the Hopper tensor cores (wgmma kind tf32,
// accumulators in registers).  Included inside namespace ctgb, after gett_ws.cuh (mbarrier
// helpers) and tc05_policy.cuh (bprime_kernel, descriptors).
//
// A complex tile product C[128 x NT] += A[128 x 16] * B[16 x NT] runs as the real
// product C'[128 x 2NT] += A'[128 x 32] * B'[2NT x 32]^T (tc05_policy.cuh); the 3xTF32 split
// (hi*hi + lo*hi + hi*lo) takes two wgmmas per k8 because B'hi and B'lo are stacked along N.  The
// one-pass instantiation (ONE: descriptor flags bit7) takes one, A'hi x B'hi, with no lo images.
// The CTA is three warpgroups that only meet at mbarriers:
//
//   warps  8-11  producer      fetches the A tile of a k-step in A's MEMORY order into a
//                              staging ring (SA deep, 16 KB each): ONE tensor-map TMA copy
//                              (cp.async.bulk.tensor, a <= 4-D box of A's coalesced dims + an
//                              offset dim) when the tile is such a box; else TMA bulk copies of
//                              whole contiguous runs (cp.async.bulk + complete_tx) when the tile
//                              is made of runs >= 128 B, an 8-byte cp.async gather otherwise.
//                              The loads run SA steps ahead of the scatter: staging -> A'hi /
//                              A'lo in wgmma's K-major core-matrix layout (double-buffered A'
//                              images).  One thread also streams the prepared B'hi|B'lo pair
//                              of every k-step into a ring of NB slots with one TMA bulk copy
//                              (when all the B' tiles a CTA ever needs fit the ring they are
//                              loaded once and stay).
//   warps  0-3   consumer 0    rows 0-63 of the tile, warps 4-7 (consumer 1) rows 64-127: each
//                              warpgroup issues the wgmmas of a k-step into its register
//                              accumulator (2NT floats a thread: [A'hi B'hi | A'hi B'lo +
//                              A'lo B'hi]), commits a k-step and waits for the one before it, and
//                              stores the finished accumulation into C.  (ptxas serialises the
//                              wgmmas of this kernel (C7511); a setmaxnreg split that removes that
//                              spills and halved complex64 throughput on H100, so it is not used.)
//
// The scatter map (element of the staging tile -> position in the A' image) is the same for
// every stage and lives in registers.  The chunk stride (LBO) of the A' images is padded by
// D[W_LBOPAD] x 16 B, chosen by the host so that the 16 lanes of a half warp -- 16
// consecutive elements of A's memory order -- hit 16 different 8-byte bank pairs.
#pragma once

// k-steps (of 16) accumulated in ONE register accumulation: a contracted range of up to 16 steps
// (K <= 256, every dense Sycamore node) is a single accumulation.  Longer ranges are folded into C
// chunk by chunk with round-to-nearest adds; the read-modify-write of a chunk hits the C tile the
// same thread wrote a moment ago, i.e. L2.
constexpr int TC05_CHUNK = 16;
// ... balanced (17 full steps are 9 + 8), and shorter in k8 accumulations for tiles with a shorter k (12 on
// 6^n extents: 12 steps = 36 accumulations): those trees are deep chains of dependent nodes, where the
// truncating accumulation of long chunks shows in the amplitude's error
__host__ __device__ inline unsigned tc05_chunk_steps(unsigned steps, unsigned nq) {
  const unsigned cap = nq >= 4u ? (unsigned)TC05_CHUNK : 36u / (nq ? nq : 1u);
  const unsigned n = (steps + cap - 1) / cap;
  return n ? (steps + n - 1) / n : 1u;
}
// A is fetched as contiguous runs by TMA bulk copies when the descriptor says its tile is made of such
// runs (flags bit6) and A is 16-byte aligned (cp.async.bulk's source alignment); the launcher reports the
// same rule (tc05_launch_config)
__host__ __device__ inline bool tc05_bulk_a(long long flags, unsigned long long a_addr) {
  return (flags & 64) != 0 && (a_addr & 15ull) == 0;
}
// k-steps whose A base offsets are tabulated (the contracted range of one node: K <= 16384)
constexpr int TC05_KTAB = 1024;

template <int NT_, bool ONE_ = false>
struct Tc05Cfg {
  static constexpr int MT = 128, NT = NT_, KT = 16;
  static constexpr bool ONE = ONE_;                        // one tf32 pass: hi images only
  static constexpr int IMAGES = ONE ? 1 : 2;               // operand images per k-step: hi (and lo)
  static constexpr int BROWS = IMAGES * 2 * NT;            // B' rows of one chunk: 2NT hi (then 2NT lo)
  static constexpr int ACC = IMAGES * NT;                  // accumulator floats of a consumer thread
  static constexpr int SA_MAX = 8, NB_MAX = 8;             // ring depths are chosen per launch
  static constexpr int TILE_FLOATS = 8 * (2 * NT) * 4;     // floats of B'hi (or B'lo) of one k-step
  static constexpr int PAIR_BYTES = IMAGES * TILE_FLOATS * 4;  // B' of one k-step: [8 chunks][BROWS rows][4 floats]
  static constexpr int A_TILE = MT * KT;                   // float2 elements of one staged A tile
  static constexpr int LBO_BASE = MT * 16;                 // bytes between k chunks of A' (unpadded)
  static constexpr int OP_BYTES = 8 * (LBO_BASE + 64);     // one A' image with the largest padding
  static constexpr int NBARS = SA_MAX + 2 * NB_MAX + 2 + 2;
  static constexpr int THREADS = 3 * 128;
  static_assert(NT == 16 || NT == 32 || NT == 64, "wgmma N = 4NT must be 64, 128 or 256");
  static constexpr size_t fixed_bytes() {  // everything but the two rings
    return 2 * IMAGES * (size_t)OP_BYTES + 8 * (size_t)(MT + NT + TC05_KTAB + NBARS) + 128;
  }
  static constexpr size_t smem_bytes(int sa, int nb) {
    return fixed_bytes() + (size_t)sa * A_TILE * 8 + (size_t)nb * PAIR_BYTES;
  }
};

// ring position + phase bit of an mbarrier ring
struct RingPos {
  unsigned idx = 0, ph = 0;
  __device__ __forceinline__ void next(unsigned n) {
    if (++idx == n) {
      idx = 0;
      ph ^= 1;
    }
  }
};

// ---- wgmma (sm_90a): D[64 x N] (+)= A[64 x 8] * B[N x 8]^T, tf32 operands K-major in shared memory
__device__ __forceinline__ void wgmma_tf32_n32(float* d, uint64_t da, uint64_t db, unsigned acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n64(float* d, uint64_t da, uint64_t db, unsigned acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n128(float* d, uint64_t da, uint64_t db, unsigned acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
      : "l"(da), "l"(db), "r"(acc));
}
__device__ __forceinline__ void wgmma_tf32_n256(float* d, uint64_t da, uint64_t db, unsigned acc) {
  asm volatile(
      "{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %130, 0;\n\t"
      "wgmma.mma_async.sync.aligned.m64n256k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63, %64, %65, %66, %67, %68, %69, %70, %71, %72, %73, %74, %75, %76, %77, %78, %79, %80, %81, %82, %83, %84, %85, %86, %87, %88, %89, %90, %91, %92, %93, %94, %95, %96, %97, %98, %99, %100, %101, %102, %103, %104, %105, %106, %107, %108, %109, %110, %111, %112, %113, %114, %115, %116, %117, %118, %119, %120, %121, %122, %123, %124, %125, %126, %127}, %128, %129, p, 1, 1;\n\t}\n"
      : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63]), "+f"(d[64]), "+f"(d[65]), "+f"(d[66]), "+f"(d[67]), "+f"(d[68]), "+f"(d[69]), "+f"(d[70]), "+f"(d[71]), "+f"(d[72]), "+f"(d[73]), "+f"(d[74]), "+f"(d[75]), "+f"(d[76]), "+f"(d[77]), "+f"(d[78]), "+f"(d[79]), "+f"(d[80]), "+f"(d[81]), "+f"(d[82]), "+f"(d[83]), "+f"(d[84]), "+f"(d[85]), "+f"(d[86]), "+f"(d[87]), "+f"(d[88]), "+f"(d[89]), "+f"(d[90]), "+f"(d[91]), "+f"(d[92]), "+f"(d[93]), "+f"(d[94]), "+f"(d[95]), "+f"(d[96]), "+f"(d[97]), "+f"(d[98]), "+f"(d[99]), "+f"(d[100]), "+f"(d[101]), "+f"(d[102]), "+f"(d[103]), "+f"(d[104]), "+f"(d[105]), "+f"(d[106]), "+f"(d[107]), "+f"(d[108]), "+f"(d[109]), "+f"(d[110]), "+f"(d[111]), "+f"(d[112]), "+f"(d[113]), "+f"(d[114]), "+f"(d[115]), "+f"(d[116]), "+f"(d[117]), "+f"(d[118]), "+f"(d[119]), "+f"(d[120]), "+f"(d[121]), "+f"(d[122]), "+f"(d[123]), "+f"(d[124]), "+f"(d[125]), "+f"(d[126]), "+f"(d[127])
      : "l"(da), "l"(db), "r"(acc));
}
template <int N>
__device__ __forceinline__ void wgmma_tf32(float* d, uint64_t da, uint64_t db, unsigned acc) {
  if constexpr (N == 32) wgmma_tf32_n32(d, da, db, acc);
  else if constexpr (N == 64) wgmma_tf32_n64(d, da, db, acc);
  else if constexpr (N == 128) wgmma_tf32_n128(d, da, db, acc);
  else wgmma_tf32_n256(d, da, db, acc);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;\n" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;\n" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() {
  asm volatile("wgmma.wait_group.sync.aligned %0;\n" ::"n"(N) : "memory");
}
// keeps the compiler from moving accesses of an accumulator across the asynchronous wgmmas
__device__ __forceinline__ void reg_fence(float& x) { asm volatile("" : "+f"(x)::"memory"); }

// SA: depth of the A staging ring.  NB: slots of the B' ring.  b_stat: the B' tiles of this
// CTA never change (one batch, grid a multiple of tiles_n, steps_k <= NB): they are
// loaded once into slot = k-step and stay resident.
template <int NT, bool ONE = false>
__global__ void __launch_bounds__(384, 1)
tc05_kernel(const int64_t* __restrict__ D, const float2* __restrict__ A, const float* __restrict__ Bp,
            float2* __restrict__ C, const unsigned SA, const unsigned NB, const int b_stat,
            const __grid_constant__ CUtensorMap tmA, const int tm_rank) {
  using Cfg = Tc05Cfg<NT, ONE>;
  constexpr int MT = Cfg::MT, A_TILE = Cfg::A_TILE;
  constexpr int GROUP = 128;  // threads of the producer warpgroup
  extern __shared__ __align__(128) unsigned char tc05_smem[];
  unsigned char* smem_raw = tc05_smem;
  float2* stg = reinterpret_cast<float2*>(smem_raw);                  // [SA][A_TILE], memory order
  unsigned char* op = smem_raw + (size_t)SA * A_TILE * 8;             // [2 buffers][hi (| lo)][OP_BYTES]
  unsigned char* sB = op + 2 * Cfg::IMAGES * Cfg::OP_BYTES;           // [NB][PAIR_BYTES]
  long long* offMC = reinterpret_cast<long long*>(sB + (size_t)NB * Cfg::PAIR_BYTES);
  long long* offNC = offMC + MT;
  long long* kbA = offNC + NT;
  unsigned long long* stg_full = reinterpret_cast<unsigned long long*>(kbA + TC05_KTAB);
  unsigned long long* b_full = stg_full + Cfg::SA_MAX;
  unsigned long long* b_empty = b_full + Cfg::NB_MAX;
  unsigned long long* op_full = b_empty + Cfg::NB_MAX;  // [2] four producer warps
  unsigned long long* op_empty = op_full + 2;           // [2] eight consumer warps

  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;

  // ---- header ----
  const int n_tm = (int)D[W_NTM], n_tn = (int)D[W_NTN];
  const int n_gm = (int)D[W_NGM], n_gn = (int)D[W_NGN], n_gk = (int)D[W_NGK], n_gb = (int)D[W_NGB];
  const int n_lda = (int)D[W_NLDA];
  const unsigned tiles_m = (unsigned)D[W_TILES_M], tiles_n = (unsigned)D[W_TILES_N], tiles_b = (unsigned)D[W_TILES_B];
  const unsigned steps_k = (unsigned)D[W_STEPS_K], splitk = (unsigned)D[W_SPLITK];
  const bool accumulate = (D[W_FLAGS] & 1) != 0;
  const bool atomic = splitk > 1;
  const bool g_pow2 = (D[W_FLAGS] & 4) != 0;
  const unsigned run_a = (unsigned)D[W_RUNA];
  // actual tile extents: full 128 x NT x 16 on power-of-two networks; on others (PEPS bond 6) the
  // host picks exact divisors of the index extents, so every tile has the SAME smaller shape --
  // rows >= MTa and columns >= NTa of the operand images are padding that the epilogue ignores
  // (A' rows >= MTa hold whatever an earlier step left there, and bprime_kernel fills B' columns >= NTa
  // with wrapped copies of real columns: both only reach accumulator rows / columns that are never
  // stored), k >= KTa costs nothing: the wgmmas of the missing k8 groups are not issued
  const unsigned MTa = (unsigned)D[W_MTA], NTa = (unsigned)D[W_NTA], KTa = (unsigned)D[W_KTA];
  const unsigned a_elems = MTa * KTa;       // elements of one staged A tile
  const unsigned nq = KTa >> 2;             // k8 groups per k-step (KTa is a multiple of 4)
  // flags bit6: the A tile is made of contiguous runs of run_a elements (>= 128 B, even offsets)
  const bool bulk_a = tc05_bulk_a(D[W_FLAGS], reinterpret_cast<unsigned long long>(A));
  const unsigned lbo_a = (unsigned)Cfg::LBO_BASE + 16u * (unsigned)D[W_LBOPAD];
  auto digit_of = [&](unsigned idx, unsigned div, unsigned ext) -> unsigned {
    return g_pow2 ? ((idx >> (31 - __clz(div))) & (ext - 1)) : ((idx / div) % ext);
  };
  // element e of the tile in A's memory order: global offset / position in the A' image (float2 units)
  auto a_off = [&](unsigned e) -> long long {
    long long g = 0;
    for (int d = 0; d < n_lda; ++d) {
      const int64_t* L = D + OFF_LDA + d * 4;
      const unsigned ext = (unsigned)L[0];
      g += (long long)(e % ext) * L[1];
      e /= ext;
    }
    return g;
  };
  auto a_pos = [&](unsigned e) -> unsigned {
    unsigned r = 0, kk = 0;
    for (int d = 0; d < n_lda; ++d) {
      const int64_t* L = D + OFF_LDA + d * 4;
      const unsigned ext = (unsigned)L[0], dig = e % ext;
      e /= ext;
      r += dig * (unsigned)L[2];
      kk += dig * (unsigned)L[3];
    }
    return (kk >> 1) * (lbo_a >> 3) + r * 2 + (kk & 1);
  };

  // ---- one-time tables ----
  if (tid == 0) {
    for (unsigned s = 0; s < SA; ++s) mbar_init(&stg_full[s], GROUP);
    for (unsigned s = 0; s < NB; ++s) {
      mbar_init(&b_full[s], 1);
      mbar_init(&b_empty[s], 8);
    }
    mbar_init(&op_full[0], 4);
    mbar_init(&op_full[1], 4);
    mbar_init(&op_empty[0], 8);
    mbar_init(&op_empty[1], 8);
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  if (tid < 256) {
    for (int r = tid; r < MT; r += 256) {
      long long o = 0;
      unsigned e = r;
      for (int d = 0; d < n_tm; ++d) {
        const int64_t* L = D + OFF_TM + d * 3;
        const unsigned ext = (unsigned)L[0];
        o += (long long)(e % ext) * L[2];
        e /= ext;
      }
      offMC[r] = o;
    }
    for (int c = tid; c < NT; c += 256) {
      long long o = 0;
      unsigned e = c;
      for (int d = 0; d < n_tn; ++d) {
        const int64_t* L = D + OFF_TN + d * 3;
        const unsigned ext = (unsigned)L[0];
        o += (long long)(e % ext) * L[2];
        e /= ext;
      }
      offNC[c] = o;
    }
  } else {
    // A base offset of every k-step (the host guarantees steps_k <= TC05_KTAB)
    for (unsigned s = tid - 256; s < steps_k; s += GROUP) {
      long long a = 0;
      for (int j = 0; j < n_gk; ++j) {
        const int64_t* G = D + OFF_GK + j * 4;
        a += (long long)((s / (unsigned)G[1]) % (unsigned)G[0]) * G[2];
      }
      kbA[s] = a;
    }
  }
  __syncthreads();

  // the host guarantees total_work < 2^31
  const unsigned tiles_all = tiles_m * tiles_n * tiles_b;
  const unsigned total_work = tiles_all * splitk;
  const unsigned steps_per_split = (steps_k + splitk - 1) / splitk;
  const unsigned chunk = tc05_chunk_steps(steps_per_split, nq);
  const unsigned nw = blockIdx.x < total_work ? (total_work - blockIdx.x + gridDim.x - 1) / gridDim.x : 0u;
  auto work_krange = [&](unsigned j, unsigned& k0, unsigned& k1) {
    const unsigned ks = splitk > 1 ? (blockIdx.x + j * gridDim.x) / tiles_all : 0u;
    k0 = ks * steps_per_split;
    k1 = min(steps_k, k0 + steps_per_split);
  };
  // tile coordinates of work item j (n fastest: neighbouring CTAs share A tiles in L2)
  auto work_tile = [&](unsigned j, unsigned& in_, unsigned& im_, unsigned& ib_) {
    unsigned t = blockIdx.x + j * gridDim.x;
    if (splitk > 1) t %= tiles_all;
    if (g_pow2) {
      in_ = t & (tiles_n - 1);
      t >>= 31 - __clz(tiles_n);
      im_ = t & (tiles_m - 1);
      ib_ = t >> (31 - __clz(tiles_m));
    } else {
      in_ = t % tiles_n;
      t /= tiles_n;
      im_ = t % tiles_m;
      ib_ = t / tiles_m;
    }
  };
  // base offsets of work item j's tile in A and C (every lane of a converged warp)
  auto tile_bases = [&](unsigned j, long long& a, long long& c) {
    unsigned in_, im_, ib_;
    work_tile(j, in_, im_, ib_);
    a = 0;
    c = 0;
    for (int q = lane; q < n_gm; q += 32) {
      const int64_t* G = D + OFF_GM + q * 4;
      const unsigned dig = digit_of(im_, (unsigned)G[1], (unsigned)G[0]);
      a += (long long)dig * G[2];
      c += (long long)dig * G[3];
    }
    for (int q = lane; q < n_gn; q += 32) {
      const int64_t* G = D + OFF_GN + q * 4;
      c += (long long)digit_of(in_, (unsigned)G[1], (unsigned)G[0]) * G[3];
    }
    for (int q = lane; q < n_gb; q += 32) {
      const int64_t* G = D + OFF_GB + q * 5;
      const unsigned dig = digit_of(ib_, (unsigned)G[1], (unsigned)G[0]);
      a += (long long)dig * G[2];
      c += (long long)dig * G[4];
    }
    a = warp_sum_ll(a);
    c = warp_sum_ll(c);
  };

  if (warp >= 8) {
    // ===================================================== PRODUCER WARPGROUP
    const int ptid = tid - 256;
    const unsigned nruns = bulk_a ? a_elems / run_a : 0u;  // <= 128: run_a >= 16
    constexpr int NG = A_TILE / GROUP;
    long long goff[NG];  // gather mode: element ptid + i*GROUP; bulk mode: goff[0] = start of run ptid
#pragma unroll
    for (int i = 0; i < NG; ++i)
      goff[i] = (bulk_a || (unsigned)(ptid + i * GROUP) >= a_elems) ? 0ll : a_off((unsigned)(ptid + i * GROUP));
    if (bulk_a && (unsigned)ptid < nruns) goff[0] = a_off((unsigned)ptid * run_a);
    unsigned upos[NG];
#pragma unroll
    for (int i = 0; i < NG; ++i)
      upos[i] = (unsigned)(ptid + i * GROUP) < a_elems ? a_pos((unsigned)(ptid + i * GROUP)) : 0xFFFFFFFFu;

    // load cursor (A): work item lj, k-step ls of [ls, le); tile base ltA
    unsigned lj = 0, ls = 0, le = 0, issued = 0;
    bool lstart = true;
    long long ltA = 0;
    RingPos rl;
    // B' cursor: work item bj, k-step bs of [bs, be)
    unsigned bj = 0, bs = 0, be = 0, b_issued = 0;
    bool bstart = true;
    unsigned long long btile = 0;
    RingPos rbp;
    const unsigned nwb = b_stat ? min(nw, 1u) : nw;  // resident B': loaded with the first work item only
    // the pair is chunk-major (k'/4 outermost): a tile with fewer than 16 k uses a PREFIX of it, and only
    // that is fetched (12 k on 6^n extents: 24 of 32 KB)
    const unsigned pair_bytes = 2u * nq * (unsigned)Cfg::BROWS * 16u;

    RingPos rs;
    for (unsigned g = 0;; ++g) {
      // A loads run SA steps ahead: the slot of step g + SA - 1 was scattered (and released by the
      // barrier below) in iteration g - 1
      while (issued < g + SA) {
        while (ls >= le) {
          if (!lstart) ++lj;
          lstart = false;
          if (lj >= nw) break;
          work_krange(lj, ls, le);
          long long c;
          tile_bases(lj, ltA, c);
        }
        if (lj >= nw) break;
        const unsigned sa = rl.idx, step = ls;
        const float2* src = A + ltA + kbA[step];
        float2* dst = stg + (size_t)sa * A_TILE;
        const unsigned bar = (unsigned)__cvta_generic_to_shared(&stg_full[sa]);
        if (tm_rank) {
          // ONE tensor-map TMA copy per k-step: the tile is a box of up to four coalesced dims of A in
          // memory order, its position the coordinate of a fifth "offset" dim of stride 16 bytes
          // (tc05_make_tensor_map)
          const unsigned bytes = ptid == 0 ? a_elems * 8u : 0u;
          asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}\n" ::"r"(bar),
                       "r"(bytes)
                       : "memory");
          if (ptid == 0) {
            const unsigned d = (unsigned)__cvta_generic_to_shared(dst);
            const unsigned long long tm = reinterpret_cast<unsigned long long>(&tmA);
            const int c = (int)((unsigned long long)(ltA + kbA[step]) >> 1);  // 16-byte units
            if (tm_rank == 2)
              asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3}], [%4];\n" ::"r"(d), "l"(tm), "r"(0), "r"(c), "r"(bar) : "memory");
            else if (tm_rank == 3)
              asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4}], [%5];\n" ::"r"(d), "l"(tm), "r"(0), "r"(0), "r"(c), "r"(bar) : "memory");
            else if (tm_rank == 4)
              asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5}], [%6];\n" ::"r"(d), "l"(tm), "r"(0), "r"(0), "r"(0), "r"(c), "r"(bar) : "memory");
            else
              asm volatile("cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%2, %3, %4, %5, %6}], [%7];\n" ::"r"(d), "l"(tm), "r"(0), "r"(0), "r"(0), "r"(0), "r"(c), "r"(bar) : "memory");
          }
        } else if (bulk_a) {
          const bool mine = (unsigned)ptid < nruns;
          const unsigned bytes = mine ? run_a * 8u : 0u;
          asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}\n" ::"r"(bar),
                       "r"(bytes)
                       : "memory");
          if (mine) {
            const unsigned d = (unsigned)__cvta_generic_to_shared(dst + (size_t)ptid * run_a);
            asm volatile(
                "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(d),
                "l"(src + goff[0]), "r"(bytes), "r"(bar)
                : "memory");
          }
        } else {
#pragma unroll
          for (int i = 0; i < NG; ++i)
            if ((unsigned)(ptid + i * GROUP) < a_elems) cp_async_zfill<8>(dst + ptid + i * GROUP, src + goff[i], true);
          mbar_arrive_cp_async(&stg_full[sa]);
        }
        ++ls;
        ++issued;
        rl.next(SA);
      }
      if (g >= issued) break;  // every k-step of every work item is scattered

      // B' pairs: up to step g + NB - 2 (its slot was freed with step g - 2, which the scatter below
      // waits for anyway); resident B' is loaded in the first iteration
      if (ptid == 0) {
        while (b_stat ? b_issued < NB : b_issued + 1 < g + NB) {
          while (bs >= be) {
            if (!bstart) ++bj;
            bstart = false;
            if (bj >= nwb) break;
            work_krange(bj, bs, be);
            unsigned in_, im_, ib_;
            work_tile(bj, in_, im_, ib_);
            btile = (unsigned long long)ib_ * tiles_n + in_;
          }
          if (bj >= nwb) break;
          const unsigned sb = rbp.idx;
          if (!b_stat) mbar_wait(&b_empty[sb], rbp.ph ^ 1);
          const unsigned bar = (unsigned)__cvta_generic_to_shared(&b_full[sb]);
          const unsigned dst = (unsigned)__cvta_generic_to_shared(sB + (size_t)sb * Cfg::PAIR_BYTES);
          const char* src = reinterpret_cast<const char*>(Bp) + (btile * steps_k + bs) * (unsigned long long)Cfg::PAIR_BYTES;
          asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.expect_tx.shared::cta.b64 st, [%0], %1;\n\t}\n" ::"r"(bar),
                       "r"(pair_bytes)
                       : "memory");
          asm volatile(
              "cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];\n" ::"r"(dst),
              "l"(src), "r"(pair_bytes), "r"(bar)
              : "memory");
          ++bs;
          ++b_issued;
          rbp.next(NB);
        }
      }

      // scatter step g: staging -> A'hi / A'lo
      const unsigned sa = rs.idx, ob = g & 1;
      float2* hi2 = reinterpret_cast<float2*>(op + (size_t)(ob * Cfg::IMAGES) * Cfg::OP_BYTES);
      float2* lo2 = reinterpret_cast<float2*>(op + (size_t)(ob * Cfg::IMAGES + 1) * Cfg::OP_BYTES);
      const float2* src = stg + (size_t)sa * A_TILE;
      mbar_wait(&op_empty[ob], ((g >> 1) & 1) ^ 1);  // the wgmmas of step g-2 have read these images
      mbar_wait(&stg_full[sa], rs.ph);
      // all loads first: the compiler cannot prove the A' images do not alias the staging
      // tile and would otherwise serialise LDS -> STS -> LDS ...
      float2 v[NG];
#pragma unroll
      for (int i = 0; i < NG; ++i) v[i] = upos[i] != 0xFFFFFFFFu ? src[ptid + i * GROUP] : make_float2(0.f, 0.f);
      if constexpr (ONE) {
        // hi alone, rounded as in the split below (the same test finds the inputs tc05_hi must take)
        float bad = 0.f;
#pragma unroll
        for (int i = 0; i < NG; ++i) {
          if (upos[i] != 0xFFFFFFFFu) {
            const float2 h = make_float2(round_tf32(v[i].x), round_tf32(v[i].y));
            hi2[upos[i]] = h;
            bad = fmaf(v[i].x - h.x, v[i].y - h.y, bad);
          }
        }
        if (!(fabsf(bad) <= 3.402823466e38f)) {
#pragma unroll
          for (int i = 0; i < NG; ++i) {
            if (upos[i] != 0xFFFFFFFFu) {
              const float2 w = src[ptid + i * GROUP];
              hi2[upos[i]] = make_float2(tc05_hi(w.x), tc05_hi(w.y));
            }
          }
        }
      } else {
#ifdef CTGB_TC05_TRUNC_SPLIT  // A/B knob: the cheaper truncating split (biased, see tc05_policy.cuh; inf gives
                              // lo = inf - inf = NaN, so an inf operand yields NaN; not run by the test suite)
#pragma unroll
      for (int i = 0; i < NG; ++i) {
        if (upos[i] != 0xFFFFFFFFu) {
          hi2[upos[i]] = v[i];
          lo2[upos[i]] = make_float2(v[i].x - trunc_tf32(v[i].x), v[i].y - trunc_tf32(v[i].y));
        }
      }
#else
      // fast split; one FMA per element collects whether any x - hi is inf or NaN (its product with the
      // other component's is then inf or NaN, and so is the sum; a finite sum that overflows only sends
      // this thread's elements down the exact path needlessly)
      float bad = 0.f;
#pragma unroll
      for (int i = 0; i < NG; ++i) {
        if (upos[i] != 0xFFFFFFFFu) {
          const float2 h = make_float2(round_tf32(v[i].x), round_tf32(v[i].y));
          const float dx = v[i].x - h.x, dy = v[i].y - h.y;
          hi2[upos[i]] = h;
          lo2[upos[i]] = make_float2(half_up_tf32(dx), half_up_tf32(dy));
          bad = fmaf(dx, dy, bad);
        }
      }
      if (!(fabsf(bad) <= 3.402823466e38f)) {  // inf, NaN or |x| near FLT_MAX in this thread's elements (rare)
#pragma unroll
        for (int i = 0; i < NG; ++i) {
          if (upos[i] != 0xFFFFFFFFu) {
            const float2 w = src[ptid + i * GROUP];  // (re-read: v[] need not stay live past the fast loop)
            float2 h, l;
            tc05_split(w.x, h.x, l.x);
            tc05_split(w.y, h.y, l.y);
            hi2[upos[i]] = h;
            lo2[upos[i]] = l;
          }
        }
      }
#endif
      }
      // generic-proxy writes (and reads of the staging slot) -> tensor core / TMA
      asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
      __syncwarp();
      if (lane == 0) mbar_arrive(&op_full[ob]);
      named_sync<1, GROUP>();  // the staging slot is refilled in the next iteration
      rs.next(SA);
    }
    cp_async_commit();
    cp_async_wait<0>();  // do not exit with copies in flight
  } else {
    // ===================================================== CONSUMER WARPGROUPS
    const int wg = warp >> 2;
    // accumulator: [P | Q], P = A'hi B'hi (NT floats), Q = A'hi B'lo + A'lo B'hi (NT floats; not in
    // the one-pass kernel).  Thread (warp w of the group, lane l) holds rows 64wg + 16(w%4) + l/4 (+8)
    // and complex columns 4i + l%4
    constexpr int ACC = Cfg::ACC;
    float acc[ACC];
#pragma unroll
    for (int i = 0; i < ACC; ++i) acc[i] = 0.f;
    const unsigned op_base = (unsigned)__cvta_generic_to_shared(op) + (unsigned)wg * 1024u;  // 8 row groups x 128 B
    const unsigned b_base = (unsigned)__cvta_generic_to_shared(sB);
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2);
    const int cl = lane & 3;
    const bool row_ok0 = (unsigned)r0 < MTa, row_ok1 = (unsigned)(r0 + 8) < MTa;
    const long long row_off0 = row_ok0 ? offMC[r0] : 0ll, row_off1 = row_ok1 ? offMC[r0 + 8] : 0ll;
    StripCtx sctx = strip_begin(D);  // fused strip_exponent
    unsigned g = 0;
    RingPos rb;
    auto release = [&](unsigned ob, unsigned sb) {
      if (lane == 0) {
        mbar_arrive(&op_empty[ob]);
        if (!b_stat) mbar_arrive(&b_empty[sb]);
      }
    };
    for (unsigned j = 0; j < nw; ++j) {
      unsigned kb, ke;
      work_krange(j, kb, ke);
      long long a_unused, cbase;
      tile_bases(j, a_unused, cbase);
      // a contracted range longer than TC05_CHUNK k-steps (K > 256) is accumulated chunk by chunk:
      // every chunk starts a fresh accumulation, the epilogue folds it into C with round-to-nearest
      // adds (the tensor core's own accumulation truncates)
      for (unsigned k0 = kb; k0 < ke; k0 += chunk) {
        const unsigned k1 = min(ke, k0 + chunk);
        unsigned prev_ob = 0, prev_sb = 0;
        for (unsigned step = k0; step < k1; ++step, ++g, rb.next(NB)) {
          const unsigned ob = g & 1, sb = b_stat ? step : rb.idx;
          mbar_wait(&op_full[ob], (g >> 1) & 1);
          if (!b_stat) {
            mbar_wait(&b_full[sb], rb.ph);
          } else if (j == 0) {
            mbar_wait(&b_full[sb], 0);  // resident B': filled once
          }
          const unsigned a_hi = op_base + (ob * Cfg::IMAGES) * (unsigned)Cfg::OP_BYTES;
          const unsigned a_lo = a_hi + (unsigned)Cfg::OP_BYTES;
          const unsigned b_all = b_base + sb * (unsigned)Cfg::PAIR_BYTES;
#pragma unroll
          for (int i = 0; i < ACC; ++i) reg_fence(acc[i]);
          wgmma_fence();
          // Two instructions per k8 instead of three passes: B'hi and B'lo are stacked along N, so
          //   [P | Q] (4NT columns)  = A'hi x [B'hi ; B'lo]^T      (A'hi is read from shared memory once)
          //        Q  (2NT columns) += A'lo x  B'hi^T
          // and the epilogue adds the small terms Q to P.  Both corrections go to Q because the tensor
          // core truncates its accumulator after every instruction: P, the one that carries the
          // magnitude, then sees ONE truncation per k8.
#pragma unroll
          for (int q = 0; q < 4; ++q) {
            if ((unsigned)q >= nq) break;  // (uniform) a tile with fewer than 16 k
            // one wgmma eats K = 8 floats = 2 chunks; chunk stride = LBO, 8-row group stride (SBO) = 128 B
            const uint64_t d_hi = gmma_desc_kmajor(a_hi + q * 2 * lbo_a, lbo_a, 128);
            const uint64_t d_lo = gmma_desc_kmajor(a_lo + q * 2 * lbo_a, lbo_a, 128);  // (not read in one pass)
            const uint64_t d_b = gmma_desc_kmajor(b_all + q * 2 * Cfg::BROWS * 16, Cfg::BROWS * 16, 128);
            wgmma_tf32<2 * ACC>(acc, d_hi, d_b, (step != k0 || q != 0) ? 1u : 0u);
            if constexpr (!ONE) wgmma_tf32<2 * NT>(acc + NT, d_lo, d_b, 1u);
          }
          wgmma_commit();
#pragma unroll
          for (int i = 0; i < ACC; ++i) reg_fence(acc[i]);
          // the operands of the previous k-step are free once it is done
          wgmma_wait<1>();
          if (step != k0) release(prev_ob, prev_sb);
          prev_ob = ob;
          prev_sb = sb;
        }
        wgmma_wait<0>();
#pragma unroll
        for (int i = 0; i < ACC; ++i) reg_fence(acc[i]);
        release(prev_ob, prev_sb);

        // ---- epilogue: registers -> C ----
        // a later chunk of the same tile adds to what the first one stored (accumulating and split-K
        // launches add every chunk to C anyway)
        const bool fold = k0 != kb && !accumulate && !atomic;
        float2* crow0 = C + cbase + row_off0;
        float2* crow1 = C + cbase + row_off1;
#pragma unroll
        for (int i = 0; i < NT / 4; ++i) {
          const unsigned n = (unsigned)(4 * i + cl);
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            const bool ok = (h ? row_ok1 : row_ok0) && n < NTa;
            float2 val = make_float2(acc[4 * i + 2 * h], acc[4 * i + 2 * h + 1]);
            if constexpr (!ONE) {
              val.x += acc[NT + 4 * i + 2 * h];
              val.y += acc[NT + 4 * i + 2 * h + 1];
            }
            if (!ok) continue;
            if (sctx.on) {
              if (sctx.scale) {
                val = strip_apply(sctx, val);
              } else if (strip_hot<float2>(sctx, strip_hi(val))) {
                strip_track_f(sctx, val.x, val.y);
              }
            }
            float2* p = (h ? crow1 : crow0) + offNC[n];
            if (atomic) {
              atomic_add_of(p, val);
            } else if (accumulate || fold) {  // (after the strip scaling: what was stored is scaled already)
              *p = add_of(*p, val);
            } else {
              *p = val;
            }
          }
        }
      }
    }
    strip_end(sctx);
  }
}
