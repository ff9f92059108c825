// gett_ws.cuh -- warp-specialised skeleton of the permutation-fused contraction
// kernel (included from gett_kernels.cuh, after the compute policies).
//
//   producer warps (PRODUCER_THREADS, the last warps of the CTA)
//       decode tile bases, look up per-element gather offsets, issue cp.async
//       into the shared-memory ring and signal "full" mbarriers through
//       cp.async.mbarrier.arrive -- all address generation lives here;
//   consumer warps (P::THREADS, the first warps)
//       wait "full", run the policy's tile product (DMMA / FMA), release the
//       stage through the "empty" mbarrier, and store finished tiles straight
//       into the parent's index order.
//
// One CTA walks its work items (tile x k-split) as ONE stream of k-steps, so
// the ring keeps prefetching across tile boundaries and no warp ever waits at a
// CTA-wide barrier in steady state.
#pragma once
// (included inside namespace ctgb)

constexpr int KCHUNK = 128;          // k-steps whose base offsets are tabulated at once
constexpr int PRODUCER_THREADS = 128;  // one warpgroup (setmaxnreg granularity)

__device__ __forceinline__ void mbar_init(unsigned long long* bar, unsigned count) {
  unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;\n" ::"r"(a), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(unsigned long long* bar) {
  unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("{\n\t.reg .b64 st;\n\tmbarrier.arrive.shared::cta.b64 st, [%0];\n\t}\n" ::"r"(a) : "memory");
}
// arrive once all cp.async issued so far by this thread have landed
__device__ __forceinline__ void mbar_arrive_cp_async(unsigned long long* bar) {
  unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile("cp.async.mbarrier.arrive.noinc.shared::cta.b64 [%0];\n" ::"r"(a) : "memory");
}
__device__ __forceinline__ void mbar_wait(unsigned long long* bar, unsigned parity) {
  unsigned a = (unsigned)__cvta_generic_to_shared(bar);
  asm volatile(
      "{\n\t.reg .pred p;\n\t"
      "WAIT_%=:\n\t"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t"
      "@p bra DONE_%=;\n\t"
      "bra WAIT_%=;\n\t"
      "DONE_%=:\n\t}\n" ::"r"(a),
      "r"(parity)
      : "memory");
}
template <int ID, int COUNT>
__device__ __forceinline__ void named_sync() {
  asm volatile("bar.sync %0, %1;\n" ::"n"(ID), "n"(COUNT) : "memory");
}
template <int REGS>
__device__ __forceinline__ void reg_alloc() {
  asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;\n" ::"n"(REGS));
}
template <int REGS>
__device__ __forceinline__ void reg_dealloc() {
  asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;\n" ::"n"(REGS));
}

template <class P, bool HAS>
struct BCacheOf {
  struct type {};
};
template <class P>
struct BCacheOf<P, true> {
  using type = typename P::BCache;
};

// B slots of a policy: the ring's STAGES, or P::B_SLOTS where the policy declares more -- a resident
// small operand (gett_kernel's b_resident) keeps one slot per k-step of the node, so that nodes with
// more k-steps than ring stages keep it too
template <class P, class = void>
struct BSlotsOf {
  static constexpr int value = P::STAGES;
};
template <class P>
struct BSlotsOf<P, std::void_t<decltype(P::B_SLOTS)>> {
  static constexpr int value = P::B_SLOTS > P::STAGES ? P::B_SLOTS : P::STAGES;
};

template <class P>
struct GettSmem {
  static constexpr int NA = (P::A_ELEMS + PRODUCER_THREADS - 1) / PRODUCER_THREADS;
  static constexpr int NB = (P::B_ELEMS + PRODUCER_THREADS - 1) / PRODUCER_THREADS;
  // tile-info ring.  STAGES + 2 slots: the producer decodes tile j+TI right after
  // issuing tile j+TI-1, whose first stage needed the "empty" arrival of every
  // consumer warp for tile j+1 -- i.e. all of them are past the epilogue of tile
  // j, the last reader of slot j % TI.  (STAGES + 1 is one too few: the decode
  // runs BEFORE the producer waits on the stage it will fill.)
  static constexpr int TI = P::STAGES + 2;
  template <typename T>
  static constexpr size_t bytes() {
    return sizeof(T) * ((size_t)P::STAGES * P::A_ELEMS + (size_t)BSlotsOf<P>::value * P::B_ELEMS +
                        P::SCRATCH_ELEMS)                                                    // ring + scratch
           + 8 * (size_t)(NA + NB) * PRODUCER_THREADS                                      // element deltas
           + 8 * (size_t)(P::MT + P::NT)                                                   // C offsets
           + 8 * (size_t)2 * KCHUNK                                                        // k-step bases
           + 8 * (size_t)4 * TI                                                            // tile bases
           + 8 * (size_t)2 * P::STAGES                                                     // mbarriers
           + 4 * (size_t)(NA + NB) * PRODUCER_THREADS                                      // element (r, kk)
           + 4 * (size_t)KCHUNK + 4 * (size_t)2 * TI                                       // valid counts
           + 64;
  }
};

template <typename T, class P>
__global__ void __launch_bounds__(P::THREADS + PRODUCER_THREADS, P::MIN_BLOCKS)
gett_kernel(const int64_t* __restrict__ D, const T* __restrict__ A, const T* __restrict__ B, T* __restrict__ C) {
  constexpr int MT = P::MT, NT = P::NT, STAGES = P::STAGES, BSLOTS = BSlotsOf<P>::value;
  constexpr int NCONS = P::THREADS, NPROD = PRODUCER_THREADS, NTHR = NCONS + NPROD;
  constexpr int NA = GettSmem<P>::NA, NB = GettSmem<P>::NB, TI = GettSmem<P>::TI;
  extern __shared__ __align__(16) unsigned char smem_raw[];
  T* sA = reinterpret_cast<T*>(smem_raw);
  T* sB = sA + STAGES * P::A_ELEMS;
  T* scratch = sB + BSLOTS * P::B_ELEMS;
  long long* gA = reinterpret_cast<long long*>(scratch + P::SCRATCH_ELEMS);
  long long* gB = gA + NA * NPROD;
  long long* offMC = gB + NB * NPROD;
  long long* offNC = offMC + MT;
  long long* kbA = offNC + NT;
  long long* kbB = kbA + KCHUNK;
  long long* ti_base = kbB + KCHUNK;  // [TI][4]: A, B, C, -
  unsigned long long* bar_full = reinterpret_cast<unsigned long long*>(ti_base + 4 * TI);
  unsigned long long* bar_empty = bar_full + STAGES;
  unsigned* metaA = reinterpret_cast<unsigned*>(bar_empty + STAGES);
  unsigned* metaB = metaA + NA * NPROD;
  int* kval = reinterpret_cast<int*>(metaB + NB * NPROD);
  int* ti_valid = kval + KCHUNK;  // [TI][2]: m_valid, n_valid

  const int tid = threadIdx.x;
  const int lane = tid & 31;
  const bool is_producer = tid >= NCONS;
  const int ptid = tid - NCONS;  // producer-local thread id

  // ---- header (uniform loads through the read-only path) ----
  const int n_tm = (int)D[W_NTM], n_tn = (int)D[W_NTN];
  const int n_gm = (int)D[W_NGM], n_gn = (int)D[W_NGN], n_gk = (int)D[W_NGK], n_gb = (int)D[W_NGB];
  const int MTa = (int)D[W_MTA], NTa = (int)D[W_NTA], KTa = (int)D[W_KTA];
  const unsigned tiles_m = (unsigned)D[W_TILES_M], tiles_n = (unsigned)D[W_TILES_N], tiles_b = (unsigned)D[W_TILES_B];
  const unsigned steps_k = (unsigned)D[W_STEPS_K], splitk = (unsigned)D[W_SPLITK];
  const int pgm = (int)D[W_PGM], pgn = (int)D[W_PGN], pgk = (int)D[W_PGK];
  const bool accumulate = (D[W_FLAGS] & 1) != 0;
  const bool atomic = splitk > 1;
  // bit1: every pair of columns (2q, 2q+1) is adjacent in C and 32-byte aligned
  const bool pair_ok = (D[W_FLAGS] & 2) != 0 && !atomic && !accumulate && sizeof(T) == 16;
  const bool ktab = steps_k <= (unsigned)KCHUNK;
  // bit2: every tile-grid extent is a power of two -> digits by shift/mask, no idiv
  const bool g_pow2 = (D[W_FLAGS] & 4) != 0;
  auto digit_of = [&](unsigned idx, unsigned div, unsigned ext) -> unsigned {
    return g_pow2 ? ((idx >> (31 - __clz(div))) & (ext - 1)) : ((idx / div) % ext);
  };
  // no blocked (partial) dim touches the operand: every tabulated element is always valid
  const bool exactA = pgm < 0 && pgk < 0, exactB = pgn < 0 && pgk < 0;

  // k-step bases: a function of the absolute step index only
  auto kstep_bases = [&](unsigned step, long long& a, long long& b, int& kv) {
    a = 0;
    b = 0;
    kv = KTa;
    for (int j = 0; j < n_gk; ++j) {
      const int64_t* G = D + OFF_GK + j * 4;
      unsigned dig = (step / (unsigned)G[1]) % (unsigned)G[0];
      a += (long long)dig * G[2];
      b += (long long)dig * G[3];
      if (j == pgk)
        kv = (int)min((long long)D[W_KTEXT], (long long)D[W_KFULL] - (long long)dig * (long long)D[W_KTEXT]) *
             (int)D[W_KW];
    }
  };

  // ---- one-time tables (all threads) ----
  // zero the operand ring: rows/cols/k beyond the actual tile are never loaded
  for (int i = tid; i < STAGES * P::A_ELEMS + BSLOTS * P::B_ELEMS; i += NTHR) sA[i] = zero_of<T>();
  if (tid == 0) {
    for (int s = 0; s < STAGES; ++s) {
      mbar_init(&bar_full[s], NPROD);
      mbar_init(&bar_empty[s], NCONS / 32);
    }
    asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
  }
  if (is_producer) {
    // per-slot element tables, enumerated in operand-memory order for coalescing
    const int n_lda = (int)D[W_NLDA], n_ldb = (int)D[W_NLDB];
    for (int i = 0; i < NA; ++i) {
      unsigned e = ptid + i * NPROD;
      long long g = 0;
      unsigned r = 0, kk = 0xFFFFu;
      if (e < (unsigned)(MTa * KTa)) {
        kk = 0;
        for (int d = 0; d < n_lda; ++d) {
          const int64_t* L = D + OFF_LDA + d * 4;
          unsigned ext = (unsigned)L[0];
          unsigned dig = e % ext;
          e /= ext;
          g += (long long)dig * L[1];
          r += dig * (unsigned)L[2];
          kk += dig * (unsigned)L[3];
        }
      }
      gA[i * NPROD + ptid] = g;
      // exact tiles (no blocked dim): store the shared-memory index directly
      metaA[i * NPROD + ptid] = exactA ? (kk == 0xFFFFu ? 0xFFFFFFFFu : (unsigned)P::idxA((int)r, (int)kk))
                                       : (r | (kk << 16));
    }
    for (int i = 0; i < NB; ++i) {
      unsigned e = ptid + i * NPROD;
      long long g = 0;
      unsigned c = 0, kk = 0xFFFFu;
      if (e < (unsigned)(NTa * KTa)) {
        kk = 0;
        for (int d = 0; d < n_ldb; ++d) {
          const int64_t* L = D + OFF_LDB + d * 4;
          unsigned ext = (unsigned)L[0];
          unsigned dig = e % ext;
          e /= ext;
          g += (long long)dig * L[1];
          kk += dig * (unsigned)L[2];
          c += dig * (unsigned)L[3];
        }
      }
      gB[i * NPROD + ptid] = g;
      metaB[i * NPROD + ptid] = exactB ? (kk == 0xFFFFu ? 0xFFFFFFFFu : (unsigned)P::idxB((int)c, (int)kk))
                                       : (c | (kk << 16));
    }
    if (ktab) {
      for (unsigned s = ptid; s < steps_k; s += NPROD) {
        long long a, b;
        int kv;
        kstep_bases(s, a, b, kv);
        kbA[s] = a;
        kbB[s] = b;
        kval[s] = kv;
      }
    }
  } else {
    // local C offsets of every tile row / column (used by the consumers' epilogue)
    for (int r = tid; r < MT; r += NCONS) {
      long long o = 0;
      if (r < MTa) {
        unsigned e = r;
        for (int d = 0; d < n_tm; ++d) {
          const int64_t* L = D + OFF_TM + d * 3;
          unsigned ext = (unsigned)L[0];
          o += (long long)(e % ext) * L[2];
          e /= ext;
        }
      }
      offMC[r] = o;
    }
    for (int c = tid; c < NT; c += NCONS) {
      long long o = 0;
      if (c < NTa) {
        unsigned e = c;
        for (int d = 0; d < n_tn; ++d) {
          const int64_t* L = D + OFF_TN + d * 3;
          unsigned ext = (unsigned)L[0];
          o += (long long)(e % ext) * L[2];
          e /= ext;
        }
      }
      offNC[c] = o;
    }
  }
  __syncthreads();

  // the host guarantees total_work < 2^31 (lowering.py)
  const unsigned tiles_all = tiles_m * tiles_n * tiles_b;
  const unsigned total_work = tiles_all * splitk;
  const unsigned steps_per_split = (steps_k + splitk - 1) / splitk;
  const unsigned nw = blockIdx.x < total_work ? (total_work - blockIdx.x + gridDim.x - 1) / gridDim.x : 0u;

  auto work_krange = [&](unsigned j, unsigned& k0, unsigned& k1) {
    const unsigned w = blockIdx.x + j * gridDim.x;
    const unsigned ks = w / tiles_all;
    k0 = ks * steps_per_split;
    k1 = min(steps_k, k0 + steps_per_split);
  };

  // The small operand's tile of k-step s never changes when every work item of this CTA has the same n
  // tile (no batch grid, no split-K, a grid that is a multiple of tiles_n: t % tiles_n is
  // blockIdx.x % tiles_n) and every k-step has a B slot of its own: it is fetched once, into slot s,
  // with the first work item, and stays.  For a K = 64, N = 128 node that is two thirds of what the
  // producers would otherwise move per tile, all of it the same.
  const bool b_resident = splitk == 1 && n_gb == 0 && (gridDim.x % tiles_n) == 0 && steps_k <= (unsigned)BSLOTS;
  // B slot of a step: its k-step when resident, else its ring stage
  auto b_slot = [&](unsigned step, int st) -> int { return b_resident ? (int)step : st; };

  if (is_producer) {
    // ===================================================== PRODUCER WARPS
    if constexpr (P::CONSUMER_REGS > 0) reg_dealloc<P::PRODUCER_REGS>();
    unsigned ktab_base = 0;
    unsigned g = 0;  // global stage counter
    for (unsigned j = 0; j < nw; ++j) {
      unsigned k0, k1;
      work_krange(j, k0, k1);
      // ---- grid-base offsets of work item j -> tile-info slot j % TI (one lane
      // per grid dim; n fastest so neighbouring CTAs share A tiles in L2)
      const int slot = (int)(j % TI);
      if (ptid < 32) {
        unsigned t = blockIdx.x + j * gridDim.x;
        if (splitk > 1) t %= tiles_all;
        unsigned in_, im_, ib_;
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
        long long a = 0, b = 0, c = 0;
        int vm = 0, vn = 0;
        for (int q = lane; q < n_gm; q += 32) {
          const int64_t* G = D + OFF_GM + q * 4;
          unsigned dig = digit_of(im_, (unsigned)G[1], (unsigned)G[0]);
          a += (long long)dig * G[2];
          c += (long long)dig * G[3];
          if (q == pgm)
            vm = (int)min((long long)D[W_MTEXT], (long long)D[W_MFULL] - (long long)dig * (long long)D[W_MTEXT]) *
                 (int)D[W_MW];
        }
        for (int q = lane; q < n_gn; q += 32) {
          const int64_t* G = D + OFF_GN + q * 4;
          unsigned dig = digit_of(in_, (unsigned)G[1], (unsigned)G[0]);
          b += (long long)dig * G[2];
          c += (long long)dig * G[3];
          if (q == pgn)
            vn = (int)min((long long)D[W_NTEXT], (long long)D[W_NFULL] - (long long)dig * (long long)D[W_NTEXT]) *
                 (int)D[W_NW];
        }
        for (int q = lane; q < n_gb; q += 32) {
          const int64_t* G = D + OFF_GB + q * 5;
          unsigned dig = digit_of(ib_, (unsigned)G[1], (unsigned)G[0]);
          a += (long long)dig * G[2];
          b += (long long)dig * G[3];
          c += (long long)dig * G[4];
        }
        a = warp_sum_ll(a);
        b = warp_sum_ll(b);
        c = warp_sum_ll(c);
        vm = warp_sum_i(vm);
        vn = warp_sum_i(vn);
        if (lane == 0) {
          ti_base[slot * 4 + 0] = a;
          ti_base[slot * 4 + 1] = b;
          ti_base[slot * 4 + 2] = c;
          ti_valid[slot * 2 + 0] = pgm < 0 ? MTa : vm;
          ti_valid[slot * 2 + 1] = pgn < 0 ? NTa : vn;
          __threadfence_block();
        }
      }
      named_sync<1, NPROD>();
      const long long tA = ti_base[slot * 4 + 0], tB = ti_base[slot * 4 + 1];
      const unsigned m_valid = (unsigned)ti_valid[slot * 2 + 0], n_valid = (unsigned)ti_valid[slot * 2 + 1];

      for (unsigned step = k0; step < k1; ++step, ++g) {
        if (!ktab && (step == k0 || step >= ktab_base + KCHUNK)) {
          // long contracted ranges: the k table is a window of KCHUNK steps
          named_sync<1, NPROD>();  // every producer is done reading the old window
          ktab_base = step;
          for (unsigned s = ptid; s < (unsigned)KCHUNK && step + s < k1; s += NPROD) {
            long long a, b;
            int kv;
            kstep_bases(step + s, a, b, kv);
            kbA[s] = a;
            kbB[s] = b;
            kval[s] = kv;
          }
          named_sync<1, NPROD>();
        }
        const int st = (int)(g % STAGES);
        mbar_wait(&bar_empty[st], ((g / STAGES) & 1) ^ 1);
        T* dA = sA + st * P::A_ELEMS;
        T* dB = sB + b_slot(step, st) * P::B_ELEMS;
        const unsigned ti = step - ktab_base;
        const T* srcA = A + tA + kbA[ti];
        const T* srcB = B + tB + kbB[ti];
        const unsigned kv = (unsigned)kval[ti];
        if (exactA) {
#pragma unroll
          for (int i = 0; i < NA; ++i) {
            const unsigned meta = metaA[i * NPROD + ptid];
            if (meta != 0xFFFFFFFFu) cp_async_zfill<sizeof(T)>(dA + meta, srcA + gA[i * NPROD + ptid], true);
          }
        } else {
#pragma unroll
          for (int i = 0; i < NA; ++i) {
            const unsigned meta = metaA[i * NPROD + ptid];
            const unsigned r = meta & 0xFFFFu, kk = meta >> 16;
            if (kk != 0xFFFFu) {
              const bool ok = (r < m_valid) && (kk < kv);
              cp_async_zfill<sizeof(T)>(dA + P::idxA(r, kk), ok ? (srcA + gA[i * NPROD + ptid]) : A, ok);
            }
          }
        }
        if (b_resident && g >= steps_k) {
          // (slot `step` already holds the tile: the first work item, k-steps 0 .. steps_k - 1, filled it)
        } else if (exactB) {
#pragma unroll
          for (int i = 0; i < NB; ++i) {
            const unsigned meta = metaB[i * NPROD + ptid];
            if (meta != 0xFFFFFFFFu) cp_async_zfill<sizeof(T)>(dB + meta, srcB + gB[i * NPROD + ptid], true);
          }
        } else {
#pragma unroll
          for (int i = 0; i < NB; ++i) {
            const unsigned meta = metaB[i * NPROD + ptid];
            const unsigned c = meta & 0xFFFFu, kk = meta >> 16;
            if (kk != 0xFFFFu) {
              const bool ok = (c < n_valid) && (kk < kv);
              cp_async_zfill<sizeof(T)>(dB + P::idxB(c, kk), ok ? (srcB + gB[i * NPROD + ptid]) : B, ok);
            }
          }
        }
        mbar_arrive_cp_async(&bar_full[st]);
      }
    }
    cp_async_commit();
    cp_async_wait<0>();  // do not exit with copies in flight
  } else {
    // ===================================================== CONSUMER WARPS
    if constexpr (P::CONSUMER_REGS > 0) reg_alloc<P::CONSUMER_REGS>();
    // valid k of a step: only a blocked (partial) k dim can shorten it
    const unsigned pk_div = pgk >= 0 ? (unsigned)D[OFF_GK + pgk * 4 + 1] : 1u;
    const unsigned pk_ext = pgk >= 0 ? (unsigned)D[OFF_GK + pgk * 4 + 0] : 1u;
    const int ktext = (int)D[W_KTEXT], kfull = (int)D[W_KFULL], kw = (int)D[W_KW];
    typename P::Acc acc;
    P::clear(acc);
    StripCtx sctx = strip_begin(D);  // fused strip_exponent (off: one uniform branch per tile)
    unsigned g = 0;
    // the small operand's tile is identical for every work item of this launch
    [[maybe_unused]] const bool b_invariant = steps_k == 1 && n_gn == 0 && n_gb == 0;
    [[maybe_unused]] bool b_loaded = false;
    [[maybe_unused]] typename BCacheOf<P, P::HAS_BCACHE>::type bcache;
    for (unsigned j = 0; j < nw; ++j) {
      unsigned k0, k1;
      work_krange(j, k0, k1);
      for (unsigned step = k0; step < k1; ++step, ++g) {
        const int st = (int)(g % STAGES);
        int kv = KTa;
        if (pgk >= 0) {
          const int dig = (int)((step / pk_div) % pk_ext);
          kv = min(ktext, kfull - dig * ktext) * kw;
        }
        mbar_wait(&bar_full[st], (g / STAGES) & 1);
        if constexpr (P::HAS_BCACHE) {
          if (b_invariant) {
            if (!b_loaded) {
              P::load_b(sB + b_slot(step, st) * P::B_ELEMS, bcache);
              b_loaded = true;
            }
            P::compute_cached(sA + st * P::A_ELEMS, bcache, acc, kv, NTa);
          } else {
            P::compute(sA + st * P::A_ELEMS, sB + b_slot(step, st) * P::B_ELEMS, acc, kv, NTa);
          }
        } else
          P::compute(sA + st * P::A_ELEMS, sB + b_slot(step, st) * P::B_ELEMS, acc, kv, NTa);
        __syncwarp();
        if (lane == 0) mbar_arrive(&bar_empty[st]);
      }
      // ---- epilogue of tile j: store in the parent's index order (strided C)
      const int slot = (int)(j % TI);
      const long long baseC = ti_base[slot * 4 + 2];
      const int m_valid = ti_valid[slot * 2 + 0], n_valid = ti_valid[slot * 2 + 1];
      // One straight-line copy of the policy's epilogue per store mode: with the mode tested
      // inside every fragment the executed instructions were islands between dead branches
      // and the warps sat in instruction-fetch stalls (ncu: 42 % of the epilogue samples of a
      // K=16 node were no_inst, the epilogue 30 % of the consumers' time).
      T* const ctile = C + baseC;
      P::finalize(acc);
      bool strip_store = false;
      if (sctx.on) {
        if (sctx.scale || !P::SCAN_OK) {
          // both operands large (no pre-scaled copy of the small one): scale by 1/(fA fB) and track
          // in the store pass itself (rare: dot-type nodes, whose results are tiny)
          strip_store = true;
        } else {
          // strip_exponent, the usual case: max|C| of the tile.  A branch-free integer scan over the
          // accumulators (two ALU ops per component) finds the leading bit pattern of the largest
          // component; only if that can raise this thread's running maximum does the cold block look
          // at the values themselves.  The stores below are the ordinary ones.
          int hmax = 0;
          P::epilogue(
              acc, scratch, [&](int, int, T v) { hmax = max(hmax, strip_hi(v)); },
              [&](int, int, T v0, T v1) { hmax = max(hmax, max(strip_hi(v0), strip_hi(v1))); }, pair_ok, n_valid);
          if (strip_hot<T>(sctx, hmax)) {
            P::epilogue(
                acc, scratch,
                [&](int r, int c, T v) {
                  if (r < m_valid && c < n_valid) strip_note(sctx, v);
                },
                [&](int r, int c, T v0, T v1) {
                  if (r < m_valid && c < n_valid) {
                    strip_note(sctx, v0);
                    strip_note(sctx, v1);
                  }
                },
                pair_ok, n_valid);
          }
        }
      }
      if (strip_store) {
        P::epilogue(
            acc, scratch,
            [&](int r, int c, T v) {
              if (r < m_valid && c < n_valid) {
                v = strip_apply(sctx, v);
                T* p = ctile + offMC[r] + offNC[c];
                if (atomic) {
                  atomic_add_of(p, v);
                } else if (accumulate) {
                  *p = add_of(*p, v);
                } else {
                  *p = v;
                }
              }
            },
            [&](int, int, T, T) {}, false, n_valid);
      } else if (pair_ok && m_valid == MT && n_valid == NT) {
        P::epilogue(
            acc, scratch, [&](int r, int c, T v) { ctile[offMC[r] + offNC[c]] = v; },
            [&](int r, int c, T v0, T v1) { store_pair_of(ctile + offMC[r] + offNC[c], v0, v1); }, true, n_valid);
      } else if (pair_ok) {
        // (only taken when pair_ok: columns c, c+1 are adjacent and 32-byte aligned)
        P::epilogue(
            acc, scratch,
            [&](int r, int c, T v) {
              if (r < m_valid && c < n_valid) ctile[offMC[r] + offNC[c]] = v;
            },
            [&](int r, int c, T v0, T v1) {
              if (r < m_valid && c < n_valid) store_pair_of(ctile + offMC[r] + offNC[c], v0, v1);
            },
            true, n_valid);
      } else if (atomic) {
        P::epilogue(
            acc, scratch,
            [&](int r, int c, T v) {
              if (r < m_valid && c < n_valid) atomic_add_of(ctile + offMC[r] + offNC[c], v);
            },
            [&](int, int, T, T) {}, false, n_valid);
      } else if (accumulate) {
        P::epilogue(
            acc, scratch,
            [&](int r, int c, T v) {
              if (r < m_valid && c < n_valid) {
                T* p = ctile + offMC[r] + offNC[c];
                *p = add_of(*p, v);
              }
            },
            [&](int, int, T, T) {}, false, n_valid);
      } else {
        P::epilogue(
            acc, scratch,
            [&](int r, int c, T v) {
              if (r < m_valid && c < n_valid) ctile[offMC[r] + offNC[c]] = v;
            },
            [&](int, int, T, T) {}, false, n_valid);
      }
      P::clear(acc);
    }
    strip_end(sctx);
  }
}

