// ctg_b200.cu -- C-ABI implementation (include/ctg_b200.h): kernel dispatch, the
// per-slice node loop and the slice loop, all on the device stream.
//
// Reference path replaced:
//   Contractor.__call__ node loop ........ cotengra/contract.py:791-832
//   ContractionTree.contract slice loop .. cotengra/core.py:4015-4030
//   slice_key / slice_arrays ............. cotengra/core.py:3775-3819
//   gather_slices (sum and stack) ........ cotengra/core.py:3825-3882
//   contract_mpi round robin ............. cotengra/core.py:4070
#include <cuda.h>  // CUtensorMap (types only: the encoder is fetched through cudaGetDriverEntryPoint)
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <type_traits>
#include <string>
#include <vector>

#include "../../include/ctg_b200.h"
#include "gett_desc.h"
#include "gett_kernels.cuh"
#include "probe.cuh"

using namespace ctgb;

namespace {

thread_local std::string g_err;
std::atomic<int64_t> g_launches{0};

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}
#define CUDA_TRY(expr)                                                                       \
  do {                                                                                       \
    cudaError_t _e = (expr);                                                                 \
    if (_e != cudaSuccess)                                                                   \
      return fail(CTGB_E_CUDA, std::string(#expr) + ": " + cudaGetErrorString(_e));          \
  } while (0)

struct DevInfo {
  bool ok = false;
  int sms = 0, major = 0, minor = 0;
  size_t smem_optin = 0;
};
DevInfo& devinfo() {
  static thread_local DevInfo d;
  static thread_local int cached_dev = -1;
  int dev = -1;
  if (cudaGetDevice(&dev) != cudaSuccess) {
    d.ok = false;
    return d;
  }
  if (dev != cached_dev) {
    cudaDeviceProp p;
    if (cudaGetDeviceProperties(&p, dev) == cudaSuccess) {
      d.ok = true;
      d.sms = p.multiProcessorCount;
      d.major = p.major;
      d.minor = p.minor;
      d.smem_optin = p.sharedMemPerBlockOptin;
      cached_dev = dev;
      // the wgmma launches take their B' scratch from the stream-ordered pool: keep freed
      // blocks cached across synchronisation points instead of returning them to the driver
      cudaMemPool_t pool;
      if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
        uint64_t keep = UINT64_MAX;
        cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
      }
    } else {
      d.ok = false;
    }
  }
  return d;
}

size_t elem_size(int dtype) {
  switch (dtype) {
    case CTGB_F32: return 4;
    case CTGB_F64: return 8;
    case CTGB_C64: return 8;
    case CTGB_C128: return 16;
  }
  return 0;
}

// ---------------------------------------------------------------- dispatch
template <typename T, class P>
int launch_gett_policy(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st) {
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  constexpr size_t smem = GettSmem<P>::template bytes<T>();
  if (smem > di.smem_optin) return fail(CTGB_E_CUDA, "kernel variant needs more shared memory than the device offers");
  static thread_local int attr_dev = -1;
  int dev;
  cudaGetDevice(&dev);
  if (attr_dev != dev) {
    CUDA_TRY(cudaFuncSetAttribute(gett_kernel<T, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_dev = dev;
  }
  if constexpr (P::CONSUMER_REGS > 0) {
    // setmaxnreg safety: the re-partitioned registers must fit the pool the CTA
    // was launched with (regs/thread chosen by ptxas x block size), otherwise
    // setmaxnreg.inc would block forever
    static thread_local int checked = 0;
    if (!checked) {
      cudaFuncAttributes fa;
      CUDA_TRY(cudaFuncGetAttributes(&fa, gett_kernel<T, P>));
      const long pool = (long)fa.numRegs * (P::THREADS + PRODUCER_THREADS);
      const long want = (long)P::CONSUMER_REGS * P::THREADS + (long)P::PRODUCER_REGS * PRODUCER_THREADS;
      if (want > pool) return fail(CTGB_E_CUDA, "setmaxnreg budget exceeds the launch register pool");
      checked = 1;
    }
  }
  static thread_local int occ = 0;
  if (occ == 0) {
    CUDA_TRY(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, gett_kernel<T, P>, P::THREADS + PRODUCER_THREADS, smem));
    if (occ < 1) occ = 1;
  }
  const uint64_t work = (uint64_t)h[W_TILES_M] * (uint64_t)h[W_TILES_N] * (uint64_t)h[W_TILES_B] * (uint64_t)h[W_SPLITK];
  if (work == 0) return CTGB_OK;
  if (work >= (1ull << 31)) return fail(CTGB_E_VALUE, "too many tiles for one launch");
  uint64_t grid = (uint64_t)di.sms * occ;
  if (grid > work) grid = work;
  if (h[W_SPLITK] > 1 && !(h[W_FLAGS] & 1)) {
    if (h[W_CELEMS] <= 0) return fail(CTGB_E_VALUE, "split-K into a strided C needs accumulate");
    CUDA_TRY(cudaMemsetAsync(C, 0, (size_t)h[W_CELEMS] * sizeof(T), st));
  }
  gett_kernel<T, P><<<(unsigned)grid, P::THREADS + PRODUCER_THREADS, smem, st>>>(d, (const T*)A, (const T*)B, (T*)C);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

unsigned long long stream_row_count(const int64_t* h) {
  return (unsigned long long)h[W_MTA] * (unsigned long long)h[W_TILES_M];
}
// What the row-stream and DMMA stream kernels take (stream_rows.cuh): N <= nmax, K <= kmax,
// one n tile, one batch tile, one k-step and no split-K, whole m blocks, no blocked n or k dim,
// and fewer than 2^32 rows (a row index is 32 bits wide)
bool stream_desc_fits(const int64_t* h, int nmax, int kmax) {
  return h[W_NTA] <= nmax && h[W_KTA] <= kmax && h[W_TILES_N] == 1 && h[W_TILES_B] == 1 && h[W_STEPS_K] == 1 &&
         h[W_SPLITK] == 1 && !(h[W_PGM] >= 0 && (h[W_MFULL] % h[W_MTEXT]) != 0) && h[W_PGN] < 0 && h[W_PGK] < 0 &&
         stream_row_count(h) < (1ull << 32);
}
// fused strip_exponent (scale the product or measure C's factor): the STRIP instantiations
bool desc_stripped(const int64_t* h) { return h[W_SCALE_A] != 0 || h[W_FACTOR_C] != 0; }

// A2, B2 non-null: the two-term form C (+)= A.B + A2.B2 (stream_rows.cuh)
template <typename T>
int launch_rowstream(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st,
                     const void* A2 = nullptr, const void* B2 = nullptr) {
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  const int N = (int)h[W_NTA], K = (int)h[W_KTA];
  if (!stream_desc_fits(h, 8, 8)) return fail(CTGB_E_VALUE, "descriptor does not fit the row-stream kernel");
  const unsigned long long M = stream_row_count(h);
  unsigned long long blocks = (M + 255) / 256;
  const unsigned long long cap = (unsigned long long)di.sms * 8;
  if (blocks > cap) blocks = cap;
  if (blocks == 0) return CTGB_OK;
  const T* a = (const T*)A;
  const T* b = (const T*)B;
  T* c = (T*)C;
  const bool strip = desc_stripped(h);
  if (A2) {
    const T* a2 = (const T*)A2;
    const T* b2 = (const T*)B2;
    if (N <= 4 && K <= 4) rowstream_kernel<T, 4, 4, false, false, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, a2, b2);
    else if (N <= 2) rowstream_kernel<T, 2, 8, false, false, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, a2, b2);
    else rowstream_kernel<T, 8, 8, false, false, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, a2, b2);
  } else if (N <= 4 && K <= 4) {
    if (strip) rowstream_kernel<T, 4, 4, true, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, nullptr, nullptr);
    else rowstream_kernel<T, 4, 4, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, nullptr, nullptr);
  } else if (N <= 2) {  // (B from shared memory: in registers it costs 154 registers = one block / SM)
    if (strip) rowstream_kernel<T, 2, 8, sizeof(T) < 16, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, nullptr, nullptr);
    else rowstream_kernel<T, 2, 8, sizeof(T) < 16><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, nullptr, nullptr);
  } else {
    if (strip) rowstream_kernel<T, 8, 8, false, true><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, nullptr, nullptr);
    else rowstream_kernel<T, 8, 8, false><<<(unsigned)blocks, 256, 0, st>>>(d, a, b, c, nullptr, nullptr);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

template <typename T>
int launch_rowstream_longk(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st,
                           const void* A2 = nullptr, const void* B2 = nullptr) {
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  if constexpr (sizeof(T) > 8) {
    return fail(CTGB_E_VALUE, "the long-k row stream takes 8-byte and narrower element types");
  } else {
    const int K = (int)h[W_KTA];
    if (!stream_desc_fits(h, RSK_NMAX, RSK_KMAX))
      return fail(CTGB_E_VALUE, "descriptor does not fit the long-k row-stream kernel");
    // offset(k) must decompose as chunk_base[k / 8] + in_chunk[k % 8]
    auto koff = [&](long long e) {
      long long o = 0;
      for (int i = 0; i < (int)h[W_NTK]; ++i) {
        o += (e % h[OFF_TK + 3 * i]) * h[OFF_TK + 3 * i + 1];
        e /= h[OFF_TK + 3 * i];
      }
      return o;
    };
    for (long long e = 0; e < K; ++e)
      if (koff(e) != koff(e - e % 8) + koff(e % 8)) return fail(CTGB_E_VALUE, "k offsets do not split into chunks of 8");
    const unsigned long long M = stream_row_count(h);
    unsigned long long blocks = (M + 511) / 512;
    const unsigned long long cap = (unsigned long long)di.sms * 6;
    if (blocks > cap) blocks = cap;
    if (blocks == 0) return CTGB_OK;
    if (A2)
      rowstream_longk_kernel<T, false, true><<<(unsigned)blocks, 256, 0, st>>>(d, (const T*)A, (const T*)B, (T*)C,
                                                                             (const T*)A2, (const T*)B2);
    else if (desc_stripped(h))
      rowstream_longk_kernel<T, true><<<(unsigned)blocks, 256, 0, st>>>(d, (const T*)A, (const T*)B, (T*)C, nullptr,
                                                                       nullptr);
    else
      rowstream_longk_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(d, (const T*)A, (const T*)B, (T*)C, nullptr, nullptr);
    g_launches.fetch_add(1, std::memory_order_relaxed);
    CUDA_TRY(cudaGetLastError());
    return CTGB_OK;
  }
}

// flags bit8: C is the wide type (double for float32, complex128 for complex64) and the dot-stream
// kernels sum in it; set on the dot-stream roots of accumulate="double" plans only
constexpr int64_t FLAG_WIDE_C = 256;

// (CT: the type of C and of the sums, T or WideOf<T>)
template <typename T, typename CT>
int launch_dotstream(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st) {
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  const bool mn = h[W_VARIANT] == VAR_DOTSTREAM4;
  const int lim = mn ? DOT4_MN : 1, kt = mn ? dot4_kt<T>() : DOT_KT;
  if (h[W_MTA] > lim || h[W_NTA] > lim || h[W_TILES_M] != 1 || h[W_TILES_N] != 1 || h[W_TILES_B] != 1 ||
      h[W_KTA] > kt || h[W_NGK] > 64 || h[W_STEPS_K] >= (1ll << 31) || h[W_PGM] >= 0 || h[W_PGN] >= 0 ||
      (h[W_PGK] >= 0 && (h[W_KFULL] % h[W_KTEXT]) != 0))
    return fail(CTGB_E_VALUE, "descriptor does not fit the dot-stream kernel");
  if (h[W_STEPS_K] == 0) return CTGB_OK;
  if (!(h[W_FLAGS] & 1)) {
    // block partial sums are added atomically: a dense result is zeroed first
    const long long celems = h[W_MTA] * h[W_NTA];
    if (celems > 1 && h[W_CELEMS] != celems) return fail(CTGB_E_VALUE, "dot-stream into a strided C needs accumulate");
    CUDA_TRY(cudaMemsetAsync(C, 0, (size_t)celems * sizeof(CT), st));
  }
  unsigned long long blocks = (unsigned long long)h[W_STEPS_K];
  // one wave: two resident blocks per SM (one for the 16-accumulator variant)
  const unsigned long long cap = (unsigned long long)di.sms * (mn ? 1 : 2);
  if (blocks > cap) blocks = cap;
  if (mn)
    dotstream_kernel<T, DOT4_MN, DOT4_MN, dot4_u<T>(), CT><<<(unsigned)blocks, DOT_THREADS, 0, st>>>(d, (const T*)A, (const T*)B, (CT*)C);
  else
    dotstream_kernel<T, 1, 1, DOT_U, CT><<<(unsigned)blocks, DOT_THREADS, 0, st>>>(d, (const T*)A, (const T*)B, (CT*)C);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

// The DMMA stream kernel's instantiation and grid for a descriptor: pure host code, so
// ctgb_dmmastream_launch_config reports exactly what launch_dmmastream runs.
struct DsLaunch {
  int nj = 0;                       // column fragments (N <= 8*nj)
  int rows = 0;                     // rows of one warp block (8 per row group)
  unsigned long long blocks = 0;    // CTAs (0: nothing to launch)
};

// (two: the two-term form, whose k range is ds_two_kb)
int dmmastream_launch_config(const int64_t* h, int sms, DsLaunch& lc, bool two = false) {
  const int N = (int)h[W_NTA];
  // 64 accumulator doubles per lane at most: 32-row warp blocks up to N = 32, 16-row ones beyond
  lc.nj = N <= 8 ? 1 : N <= 16 ? 2 : N <= 32 ? 4 : 8;
  const int kmax = two ? ds_two_kb(lc.nj) : N <= 32 ? DS_KMAX : DS_KMAX_WIDE;
  if (h[W_DTYPE] != CTGB_C128 || !stream_desc_fits(h, 64, kmax))
    return fail(CTGB_E_VALUE, two ? "descriptor does not fit the two-term DMMA stream kernel"
                                  : "descriptor does not fit the DMMA stream kernel");
  const unsigned long long M = stream_row_count(h);
  lc.rows = lc.nj <= 4 ? 32 : 16;
  const unsigned long long per = 4ull * lc.rows;  // 4 warps per block and pass
  lc.blocks = (M + per - 1) / per;
  const unsigned long long cap = (unsigned long long)sms * 12;
  if (lc.blocks > cap) lc.blocks = cap;
  return CTGB_OK;
}

template <int NJ, int RG>
void dmmastream_launch(bool strip, unsigned blocks, const int64_t* d, const double2* a, const double2* b, double2* c,
                       const double2* a2, const double2* b2, cudaStream_t st) {
  if (a2) dmmastream_kernel<NJ, RG, false, true><<<blocks, 128, 0, st>>>(d, a, b, c, a2, b2);
  else if (strip) dmmastream_kernel<NJ, RG, true><<<blocks, 128, 0, st>>>(d, a, b, c, nullptr, nullptr);
  else dmmastream_kernel<NJ, RG><<<blocks, 128, 0, st>>>(d, a, b, c, nullptr, nullptr);
}

int launch_dmmastream(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st,
                      const void* A2 = nullptr, const void* B2 = nullptr) {
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  DsLaunch lc;
  if (int rc = dmmastream_launch_config(h, di.sms, lc, A2 != nullptr)) return rc;
  if (lc.blocks == 0) return CTGB_OK;
  const bool strip = desc_stripped(h);
  const double2 *a = (const double2*)A, *b = (const double2*)B, *a2 = (const double2*)A2, *b2 = (const double2*)B2;
  double2* c = (double2*)C;
  const unsigned blocks = (unsigned)lc.blocks;
  switch (lc.nj) {
    case 1: dmmastream_launch<1, 4>(strip, blocks, d, a, b, c, a2, b2, st); break;
    case 2: dmmastream_launch<2, 4>(strip, blocks, d, a, b, c, a2, b2, st); break;
    case 4: dmmastream_launch<4, 4>(strip, blocks, d, a, b, c, a2, b2, st); break;
    default: dmmastream_launch<8, 2>(strip, blocks, d, a, b, c, a2, b2, st); break;
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

// absorb-root node (absorbdot.cuh): one CTA per SM at most, each taking an even share of the k' units
int launch_absorb_root(const int64_t* h, const int64_t* d, const void* A, const void* Bs, const void* V, void* C,
                       cudaStream_t st) {
  if (h[W_DTYPE] != CTGB_C128) return fail(CTGB_E_VALUE, "the absorb-root kernel is complex128 only");
  if (h[AB_M] < 1 || h[AB_M] > 32 || h[AB_N] < 1 || h[AB_N] > 32 || h[AB_K] < 1 || h[AB_K] > 16 || h[AB_C] < 1 ||
      h[AB_C] > h[AB_CCP] || h[AB_CCP] % 32 || h[AB_CCP] > 128 || (h[AB_KL] != 1 && h[AB_KL] != 2) || h[AB_NG] < 0 || h[AB_NG] > AB_MAXG || h[AB_UNITS] < 1 || h[AB_UNITS] >= (1ll << 32) ||
      h[AB_GRID] < 1 || h[AB_GRID] > h[AB_UNITS] || h[AB_GRID] > (1 << 20))
    return fail(CTGB_E_VALUE, "absorb-root descriptor out of range");
  for (int mb = 0; mb < 4; ++mb)
    if (h[AB_TBCK + mb] < 0 || (h[AB_TBCK + mb] + 1) * h[AB_CCP] > 128)
      return fail(CTGB_E_VALUE, "absorb-root descriptor out of range");
  if (!(h[W_FLAGS] & 1)) {
    if (h[W_CELEMS] <= 0) return fail(CTGB_E_VALUE, "absorb-root into a strided C needs accumulate");
    CUDA_TRY(cudaMemsetAsync(C, 0, (size_t)h[W_CELEMS] * sizeof(double2), st));
  }
  // A8: every row is one of the first 8 A rows again (one block per kept Bs column), so a stage
  // holds 8 A rows; one quarter of c: the Bs fragments stay in registers
  bool a8 = true;
  for (int r = 8; r < 32; ++r)
    if (h[AB_TMC + r] >= 0 && (h[AB_TMC + r % 8] < 0 || h[AB_TMA + r] != h[AB_TMA + r % 8])) a8 = false;
  const bool breg = h[AB_CCP] == 32;
  using Kern = void (*)(const int64_t*, const double2*, const double2*, const double2*, double2*);
  const Kern kern = a8 ? (breg ? absorbdot_kernel<true, true> : absorbdot_kernel<true, false>)
                    : (breg ? absorbdot_kernel<false, true> : absorbdot_kernel<false, false>);
  const size_t smem = a8 ? AbRing<true>::SMEM : AbRing<false>::SMEM;
  static bool attr[4] = {};
  if (!attr[2 * a8 + breg]) {
    CUDA_TRY(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr[2 * a8 + breg] = true;
  }
  kern<<<(unsigned)h[AB_GRID], AB_THREADS, smem, st>>>(d, (const double2*)A, (const double2*)Bs, (const double2*)V,
                                                       (double2*)C);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

std::atomic<int64_t> g_tmap_launches{0};

// Tensor map for the A tile of the wgmma kernel.  The tile is described in A's memory order by
// the descriptor's load list (ext, stride), smallest stride first; adjacent entries that continue
// each other coalesce into box dims.  If at most four box dims remain, the innermost is contiguous
// and everything is 16-byte granular, ONE cp.async.bulk.tensor fetches the tile: dims 0..n-1 are
// the box (coordinates 0), and one more dim of stride 16 bytes carries the tile's base offset as
// its coordinate (tensor-map strides need not nest).
//
// tc05_tensor_map_box derives the box (pure host code, no CUDA calls) and returns the rank of the
// tensor map it describes (2..5), or 0 when the tile is not such a box.
struct Tc05Box {
  int nb = 0;  // box dims (the rank is nb + 1)
  struct Dim { uint64_t ext, stride; } dim[8];
};
int tc05_tensor_map_box(const int64_t* h, uint64_t a_addr, Tc05Box& bx) {
  if (a_addr & 15u) return 0;
  auto& box = bx.dim;
  int& nb = bx.nb;
  nb = 0;
  const int n_lda = (int)h[W_NLDA];
  for (int i = 0; i < n_lda; ++i) {
    const uint64_t ext = (uint64_t)h[OFF_LDA + 4 * i], st = (uint64_t)h[OFF_LDA + 4 * i + 1];
    if (h[OFF_LDA + 4 * i + 1] <= 0) return 0;
    if (nb && st == box[nb - 1].stride * box[nb - 1].ext) {
      box[nb - 1].ext *= ext;
    } else {
      if (nb == 4) return 0;
      box[nb].ext = ext;
      box[nb].stride = st;
      ++nb;
    }
  }
  // a box dim holds at most 256 elements: split longer (contiguous) ones
  for (int i = 0; i < nb; ++i) {
    while (box[i].ext > 256) {
      uint64_t f = 256;
      while (f > 1 && box[i].ext % f) --f;
      if (f < 2 || nb == 4) return 0;
      for (int j = nb; j > i + 1; --j) box[j] = box[j - 1];
      box[i + 1].ext = box[i].ext / f;
      box[i + 1].stride = box[i].stride * f;
      box[i].ext = f;
      ++nb;
    }
  }
  if (nb == 0 || box[0].stride != 1 || (box[0].ext & 1)) return 0;
  uint64_t prod = 1;
  for (int i = 0; i < nb; ++i) {
    if (box[i].ext > 256 || (i && (box[i].stride & 1))) return 0;
    prod *= box[i].ext;
  }
  if (prod != (uint64_t)(h[W_MTA] * h[W_KTA])) return 0;
  // base offsets of the tiles: sums of grid-dim digits times even strides, below 2^32 elements
  uint64_t reach = 0;
  auto grid = [&](int off, int n, int width, int col) -> bool {
    for (int i = 0; i < n; ++i) {
      const int64_t e = h[off + i * width], st = h[off + i * width + col];
      if (st < 0 || (st & 1)) return false;
      reach += (uint64_t)(e - 1) * (uint64_t)st;
    }
    return true;
  };
  if (!grid(OFF_GM, (int)h[W_NGM], 4, 2) || !grid(OFF_GK, (int)h[W_NGK], 4, 2) || !grid(OFF_GB, (int)h[W_NGB], 5, 2))
    return 0;
  if (reach >= (1ull << 32)) return 0;
  return nb + 1;
}

// Encodes the tensor map of tc05_tensor_map_box.  Returns its rank, or 0 when the tile is not a
// box, the driver has no encoder or the encode fails.
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
int tc05_make_tensor_map(const int64_t* h, const void* A, CUtensorMap* tm) {
  Tc05Box bx;
  if (!tc05_tensor_map_box(h, (uint64_t)(uintptr_t)A, bx)) return 0;
  static EncodeTiledFn encode = nullptr;
  static bool tried = false;
  if (!tried) {
    tried = true;
    void* fn = nullptr;
    cudaDriverEntryPointQueryResult qres;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres) == cudaSuccess &&
        qres == cudaDriverEntryPointSuccess)
      encode = (EncodeTiledFn)fn;
    else
      cudaGetLastError();
  }
  if (!encode) return 0;
  const int nb = bx.nb;
  cuuint64_t gdim[5], gstr[4];
  cuuint32_t bdim[5], estr[5];
  for (int i = 0; i < nb; ++i) {
    gdim[i] = bx.dim[i].ext;
    bdim[i] = (cuuint32_t)bx.dim[i].ext;
    estr[i] = 1;
    if (i) gstr[i - 1] = bx.dim[i].stride * 8;
  }
  gdim[nb] = 1ull << 31;  // offset dim: coordinate = base offset in 16-byte units
  bdim[nb] = 1;
  estr[nb] = 1;
  gstr[nb - 1] = 16;
  const CUresult rc = encode(tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, (cuuint32_t)(nb + 1), const_cast<void*>(A), gdim, gstr,
                             bdim, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE,
                             CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  return rc == CUDA_SUCCESS ? nb + 1 : 0;
}

// Launch-time choices of the wgmma kernel, from the descriptor, the A pointer and the device's SM
// count and opt-in shared memory.  tc05_launch_config is pure host code (no CUDA calls), so
// ctgb_tc05_launch_config reports exactly what launch_tc05 runs.
struct Tc05Launch {
  int b_stat = 0;        // B' resident (one slot per k-step, loaded once) instead of a ring
  long long nb = 0;      // B' slots
  long long sa = 0;      // A staging depth
  uint64_t grid = 0;     // CTAs (0: nothing to do)
  size_t smem = 0;       // dynamic shared memory of one CTA
  int tm_rank = 0;       // rank of the A tensor map tc05_tensor_map_box describes, 0 if none
  int bulk = 0;          // A runs fetched by bulk copies (tc05_bulk_a)
  unsigned chunk = 0;    // k-steps per register accumulation (tc05_chunk_steps)
  unsigned chunks = 0;   // accumulations of the longest contracted range of a work item
};

// (ONE: the one-pass kernel, whose B' k-steps and A' images are half the size)
template <int NT, bool ONE>
int tc05_launch_config(const int64_t* h, uint64_t a_addr, int sms, uint64_t smem_optin, Tc05Launch& lc) {
  using Cfg = Tc05Cfg<NT, ONE>;
  lc = Tc05Launch();
  auto exact = [&](int pg, int full, int text) { return h[pg] < 0 || (h[full] % h[text]) == 0; };
  // every tile has the same shape: the full 128 x NT x 16, or exact divisors of the index extents
  // (MTa <= 128 rows, NTa <= NT columns, KTa a multiple of 4 up to 16)
  if (h[W_DTYPE] != CTGB_C64 || h[W_MTA] < 1 || h[W_MTA] > 128 || h[W_NTA] < 1 || h[W_NTA] > NT || h[W_KTA] < 4 ||
      h[W_KTA] > 16 || (h[W_KTA] & 3) ||
      !exact(W_PGM, W_MFULL, W_MTEXT) || !exact(W_PGN, W_NFULL, W_NTEXT) || !exact(W_PGK, W_KFULL, W_KTEXT) ||
      h[W_STEPS_K] > TC05_KTAB || h[W_LBOPAD] < 0 || h[W_LBOPAD] > 4 ||
      ((h[W_FLAGS] & 64) && (h[W_RUNA] < 16 || (h[W_MTA] * h[W_KTA]) % h[W_RUNA] != 0)))
    return fail(CTGB_E_VALUE, "descriptor does not fit the wgmma kernel");
  const uint64_t work = (uint64_t)h[W_TILES_M] * (uint64_t)h[W_TILES_N] * (uint64_t)h[W_TILES_B] * (uint64_t)h[W_SPLITK];
  if (work == 0) return CTGB_OK;
  if (work >= (1ull << 31)) return fail(CTGB_E_VALUE, "too many tiles for one launch");
  // ring depths: B' resident (one slot per k-step) when this CTA's B' tiles never change and
  // still leave room for >= 3 A stages; otherwise a 3-slot B' ring.  A gets the rest.
  const long long pool = (long long)smem_optin - 1024 /* static + slack */ - (long long)Cfg::fixed_bytes();
  const long long steps_k = h[W_STEPS_K], tiles_n = h[W_TILES_N];
  uint64_t grid = (uint64_t)sms;
  int b_stat = 0;
  long long nb = 3;
  if (h[W_TILES_B] == 1 && h[W_SPLITK] == 1 && steps_k <= Cfg::NB_MAX && tiles_n <= (long long)sms &&
      pool - steps_k * Cfg::PAIR_BYTES >= 3ll * Cfg::A_TILE * 8) {
    b_stat = 1;
    nb = steps_k;
    grid = (grid / (uint64_t)tiles_n) * (uint64_t)tiles_n;  // t % tiles_n is the same for every work item of a CTA
  }
  long long sa = (pool - nb * Cfg::PAIR_BYTES) / ((long long)Cfg::A_TILE * 8);
  if (sa > Cfg::SA_MAX) sa = Cfg::SA_MAX;
  if (sa < 2) return fail(CTGB_E_CUDA, "wgmma kernel needs more shared memory than the device offers");
  // (a resident B' keeps grid a multiple of tiles_n here too: it needs one batch and no split-K, so
  // work = tiles_m * tiles_n)
  if (grid > work) grid = work;
  const size_t smem = Cfg::smem_bytes((int)sa, (int)nb);
  if (smem + 1024 > smem_optin)
    return fail(CTGB_E_CUDA, "wgmma kernel needs more shared memory than the device offers");
  const unsigned steps_per_split = (unsigned)((steps_k + h[W_SPLITK] - 1) / h[W_SPLITK]);
  Tc05Box bx;
  lc.b_stat = b_stat;
  lc.nb = nb;
  lc.sa = sa;
  lc.grid = grid;
  lc.smem = smem;
  lc.tm_rank = tc05_tensor_map_box(h, a_addr, bx);
  lc.bulk = tc05_bulk_a(h[W_FLAGS], a_addr);
  lc.chunk = tc05_chunk_steps(steps_per_split, (unsigned)(h[W_KTA] >> 2));
  lc.chunks = (steps_per_split + lc.chunk - 1) / lc.chunk;
  return CTGB_OK;
}

// complex64 on wgmma: prepare B' (hi/lo, tile order) once, then the warp-specialised kernel
template <int NT, bool ONE>
int launch_tc05(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st) {
  using Cfg = Tc05Cfg<NT, ONE>;
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  Tc05Launch lc;
  if (int rc = tc05_launch_config<NT, ONE>(h, (uint64_t)(uintptr_t)A, di.sms, di.smem_optin, lc)) return rc;
  if (lc.grid == 0) return CTGB_OK;
  static thread_local int attr_dev = -1;
  int dev;
  cudaGetDevice(&dev);
  if (attr_dev != dev) {
    CUDA_TRY(cudaFuncSetAttribute(tc05_kernel<NT, ONE>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                  (int)di.smem_optin - 1024));
    attr_dev = dev;
  }

  const unsigned long long tiles = (unsigned long long)h[W_TILES_B] * h[W_TILES_N] * h[W_STEPS_K];
  const size_t bytes = (size_t)tiles * Cfg::PAIR_BYTES;
  float* Bp = nullptr;
  CUDA_TRY(cudaMallocAsync((void**)&Bp, bytes, st));
  const unsigned long long total = tiles * Cfg::TILE_FLOATS;
  unsigned long long blocks = (total + 255) / 256;
  if (blocks > (unsigned long long)di.sms * 8) blocks = (unsigned long long)di.sms * 8;
  bprime_kernel<NT, ONE><<<(unsigned)blocks, 256, 0, st>>>(d, (const float2*)B, Bp);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  if (h[W_SPLITK] > 1 && !(h[W_FLAGS] & 1)) {
    if (h[W_CELEMS] <= 0) {
      cudaFreeAsync(Bp, st);
      return fail(CTGB_E_VALUE, "split-K into a strided C needs accumulate");
    }
    CUDA_TRY(cudaMemsetAsync(C, 0, (size_t)h[W_CELEMS] * sizeof(float2), st));
  }
  CUtensorMap tm;
  memset(&tm, 0, sizeof(tm));
  // (CTGB_NO_TENSOR_MAP=1 is a measurement knob: bulk-copy / gather staging only)
  static const bool tm_off = getenv("CTGB_NO_TENSOR_MAP") != nullptr;
  const int tm_rank = tm_off ? 0 : tc05_make_tensor_map(h, A, &tm);
  if (tm_rank) g_tmap_launches.fetch_add(1, std::memory_order_relaxed);
  tc05_kernel<NT, ONE><<<(unsigned)lc.grid, Cfg::THREADS, lc.smem, st>>>(d, (const float2*)A, Bp, (float2*)C,
                                                                         (unsigned)lc.sa, (unsigned)lc.nb, lc.b_stat,
                                                                         tm, tm_rank);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  cudaError_t e = cudaGetLastError();
  cudaFreeAsync(Bp, st);
  if (e != cudaSuccess) return fail(CTGB_E_CUDA, cudaGetErrorString(e));
  return CTGB_OK;
}

// flags bit7: float32 / complex64 tensor-core variants run one tf32 pass instead of three
constexpr int64_t FLAG_TF32_ONE_PASS = 128;

template <typename T>
int launch_gett_typed(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st) {
  const int variant = (int)h[W_VARIANT];
  const bool one = (h[W_FLAGS] & FLAG_TF32_ONE_PASS) != 0;
  if (variant == VAR_ROWSTREAM) return launch_rowstream<T>(h, d, A, B, C, st);
  if (variant == VAR_ROWSTREAM_K) return launch_rowstream_longk<T>(h, d, A, B, C, st);
  if (variant == VAR_DMMASTREAM) return launch_dmmastream(h, d, A, B, C, st);
  if (h[W_FLAGS] & FLAG_WIDE_C) {
    using Wide = typename WideOf<T>::type;
    if (std::is_same<Wide, T>::value || (variant != VAR_DOTSTREAM && variant != VAR_DOTSTREAM4))
      return fail(CTGB_E_VALUE, "a wide C belongs to float32 / complex64 dot-stream nodes");
    return launch_dotstream<T, Wide>(h, d, A, B, C, st);
  }
  if (variant == VAR_DOTSTREAM || variant == VAR_DOTSTREAM4) return launch_dotstream<T, T>(h, d, A, B, C, st);
  if constexpr (std::is_same<T, float2>::value) {
    if (variant == VAR_TC05_128x64) return one ? launch_tc05<64, true>(h, d, A, B, C, st) : launch_tc05<64, false>(h, d, A, B, C, st);
    if (variant == VAR_TC05_128x32) return one ? launch_tc05<32, true>(h, d, A, B, C, st) : launch_tc05<32, false>(h, d, A, B, C, st);
    if (variant == VAR_TC05_128x16) return one ? launch_tc05<16, true>(h, d, A, B, C, st) : launch_tc05<16, false>(h, d, A, B, C, st);
  }
  switch (variant) {
    case VAR_SIMT_64x64: return launch_gett_policy<T, SimtPolicy<T, 64, 64, 8, 3>>(h, d, A, B, C, st);
    case VAR_KRED: return launch_gett_policy<T, KredPolicy<T, 1, 1, 512, 6>>(h, d, A, B, C, st);
    case VAR_ROW_128x8: return launch_gett_policy<T, RowPolicy<T, 256, 8, 4, 3>>(h, d, A, B, C, st);
    case VAR_ROW_256x4: return launch_gett_policy<T, RowPolicy<T, 256, 4, 4, 3>>(h, d, A, B, C, st);
    default: break;
  }
  if constexpr (sizeof(T) == 16 || (sizeof(T) == 8 && std::is_same<T, double>::value)) {
    switch (variant) {
      // (B slots: K = 64 keeps the small operand resident -- four k-steps of 16, eight of 8)
      case VAR_DMMA_128x64: return launch_gett_policy<T, DmmaPolicy<T, 4, 2, 4, 4, 16, 3, false, 4>>(h, d, A, B, C, st);
      case VAR_DMMA_64x128: return launch_gett_policy<T, DmmaPolicy<T, 2, 4, 4, 4, 16, 3, false, 4>>(h, d, A, B, C, st);
      case VAR_DMMA_256x32: return launch_gett_policy<T, DmmaPolicy<T, 8, 1, 4, 4, 8, 4, false, 8>>(h, d, A, B, C, st);
      case VAR_DMMA_256x16: return launch_gett_policy<T, DmmaPolicy<T, 8, 1, 4, 2, 8, 5>>(h, d, A, B, C, st);
      // (K 16 x 4 stages = 80 KB per CTA: with K 32 x 3 stages -- 122 KB -- only ONE CTA fitted an SM,
      // four consumer warps, tensor pipe 72 % under ncu)
      case VAR_DMMA_32x32: return launch_gett_policy<T, DmmaPolicy<T, 2, 2, 2, 2, 16, 4>>(h, d, A, B, C, st);
      default: break;
    }
  }
  if constexpr (sizeof(T) == 16) {
    switch (variant) {
      case VAR_DMMA3M_128x32: return launch_gett_policy<T, DmmaPolicy<T, 4, 2, 4, 2, 16, 4, true>>(h, d, A, B, C, st);
      case VAR_DMMA3M_256x16: return launch_gett_policy<T, DmmaPolicy<T, 8, 1, 4, 2, 8, 5, true>>(h, d, A, B, C, st);
      default: break;
    }
  }
  if constexpr (std::is_same<T, float>::value || std::is_same<T, float2>::value) {
    // single precision on the tensor pipe: 3xTF32 mma.sync (one pass with flags bit7), same tile shapes
    switch (variant) {
#define CTGB_TF32(...)                                                                             \
  return one ? launch_gett_policy<T, Tf32Policy<T, __VA_ARGS__, true>>(h, d, A, B, C, st)           \
             : launch_gett_policy<T, Tf32Policy<T, __VA_ARGS__>>(h, d, A, B, C, st)
      case VAR_DMMA_128x64: CTGB_TF32(4, 2, 2, 4, 16, 3);
      case VAR_DMMA_64x128: CTGB_TF32(2, 4, 2, 4, 16, 3);
      case VAR_DMMA_256x32: CTGB_TF32(8, 1, 2, 4, 8, 3);
      case VAR_DMMA_256x16: CTGB_TF32(8, 1, 2, 2, 8, 3);
      // DMMA_32x32's geometry: one 32 x 32 tile, four warps, the contracted range split over the SMs
      case VAR_TF32_32x32: CTGB_TF32(2, 2, 1, 2, 16, 4);
#undef CTGB_TF32
      default: break;
    }
  }
  return fail(CTGB_E_VALUE, "unknown kernel variant for this dtype");
}

int launch_gett(const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st) {
  if (h[W_MAGIC] != DESC_MAGIC) return fail(CTGB_E_VALUE, "bad pair descriptor magic");
  if (h[W_VARIANT] == VAR_ABSORB_ROOT) return fail(CTGB_E_VALUE, "an absorb-root node has three operands (ctgb_absorb_root)");
  switch ((int)h[W_DTYPE]) {
    case CTGB_F32: return launch_gett_typed<float>(h, d, A, B, C, st);
    case CTGB_F64: return launch_gett_typed<double>(h, d, A, B, C, st);
    case CTGB_C64: return launch_gett_typed<float2>(h, d, A, B, C, st);
    case CTGB_C128: return launch_gett_typed<double2>(h, d, A, B, C, st);
  }
  return fail(CTGB_E_VALUE, "bad dtype");
}

// The two-term node C (+)= A.B + A2.B2 (A2 laid out as A, B2 as B) in one launch: the row-stream and
// DMMA stream kernels only, with C of the plan dtype.  Scale words (W_SCALE_A / W_SCALE_B, both) make
// it C (+)= (A.B + A2.B2) / (fA fB), B and B2 scaled as they are staged; it never measures a factor
template <typename T>
int launch_gett2_typed(const int64_t* h, const int64_t* d, const void* A, const void* B, const void* A2,
                       const void* B2, void* C, cudaStream_t st) {
  const int variant = (int)h[W_VARIANT];
  if (variant == VAR_ROWSTREAM) return launch_rowstream<T>(h, d, A, B, C, st, A2, B2);
  if (variant == VAR_ROWSTREAM_K) return launch_rowstream_longk<T>(h, d, A, B, C, st, A2, B2);
  if (variant == VAR_DMMASTREAM) return launch_dmmastream(h, d, A, B, C, st, A2, B2);
  return fail(CTGB_E_VALUE, "the two-term form runs on the row-stream and DMMA stream kernels only");
}

int launch_gett2(const int64_t* h, const int64_t* d, const void* A, const void* B, const void* A2, const void* B2,
                 void* C, cudaStream_t st) {
  if (h[W_MAGIC] != DESC_MAGIC) return fail(CTGB_E_VALUE, "bad pair descriptor magic");
  if (!A2 || !B2) return fail(CTGB_E_VALUE, "the two-term form needs both A2 and B2");
  if (h[W_FACTOR_C] != 0) return fail(CTGB_E_VALUE, "the two-term form measures no factor of C (W_FACTOR_C)");
  if ((h[W_SCALE_A] == 0) != (h[W_SCALE_B] == 0))
    return fail(CTGB_E_VALUE, "the two-term form takes both scale words or neither");
  if (h[W_FLAGS] & FLAG_WIDE_C) return fail(CTGB_E_VALUE, "the two-term form has no wide C");
  switch ((int)h[W_DTYPE]) {
    case CTGB_F32: return launch_gett2_typed<float>(h, d, A, B, A2, B2, C, st);
    case CTGB_F64: return launch_gett2_typed<double>(h, d, A, B, A2, B2, C, st);
    case CTGB_C64: return launch_gett2_typed<float2>(h, d, A, B, A2, B2, C, st);
    case CTGB_C128: return launch_gett2_typed<double2>(h, d, A, B, A2, B2, C, st);
  }
  return fail(CTGB_E_VALUE, "bad dtype");
}

template <typename T>
int launch_single_typed(const int64_t* h, const int64_t* d, const void* X, void* out, cudaStream_t st) {
  long long n = h[S_OUT_ELEMS];
  if (n <= 0) return CTGB_OK;
  const long long cap = (long long)(devinfo().ok ? devinfo().sms : 132) * 16;
  long long blocks = (n + 255) / 256;
  if (blocks > cap) blocks = cap;
  if (h[S_SUM_ELEMS] >= 1024 && n <= cap) {
    // few outputs over a long summed range: one block per output element
    single_reduce_kernel<T><<<(unsigned)n, 256, 0, st>>>(d, (const T*)X, (T*)out);
  } else {
    single_kernel<T><<<(unsigned)blocks, 256, 0, st>>>(d, (const T*)X, (T*)out);
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}
int launch_single(const int64_t* h, const int64_t* d, const void* X, void* out, cudaStream_t st) {
  if (h[S_MAGIC] != SDESC_MAGIC) return fail(CTGB_E_VALUE, "bad single descriptor magic");
  switch ((int)h[S_DTYPE]) {
    case CTGB_F32: return launch_single_typed<float>(h, d, X, out, st);
    case CTGB_F64: return launch_single_typed<double>(h, d, X, out, st);
    case CTGB_C64: return launch_single_typed<float2>(h, d, X, out, st);
    case CTGB_C128: return launch_single_typed<double2>(h, d, X, out, st);
  }
  return fail(CTGB_E_VALUE, "bad dtype");
}

unsigned flat_grid(long long n) {
  const long long cap = (long long)(devinfo().ok ? devinfo().sms : 132) * 8;
  long long b = (n + 255) / 256;
  if (b > cap) b = cap;
  if (b < 1) b = 1;
  return (unsigned)b;
}

template <typename T>
int scale_copy_typed(const void* src, void* dst, long long n, const double* fa, const double* fb, cudaStream_t st) {
  scale_copy_kernel<T><<<flat_grid(n), 256, 0, st>>>((const T*)src, (T*)dst, n, fa, fb);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}
int scale_copy(int dtype, const void* src, void* dst, long long n, const double* fa, const double* fb, cudaStream_t st) {
  switch (dtype) {
    case CTGB_F32: return scale_copy_typed<float>(src, dst, n, fa, fb, st);
    case CTGB_F64: return scale_copy_typed<double>(src, dst, n, fa, fb, st);
    case CTGB_C64: return scale_copy_typed<float2>(src, dst, n, fa, fb, st);
    case CTGB_C128: return scale_copy_typed<double2>(src, dst, n, fa, fb, st);
  }
  return fail(CTGB_E_VALUE, "bad dtype");
}

// max|C| of a node whose own epilogue cannot measure it (split-K / block partial sums)
template <typename T>
int absmax_typed(const void* p, long long n, unsigned long long* slot, cudaStream_t st) {
  absmax_kernel<T><<<flat_grid(n), 256, 0, st>>>((const T*)p, n, slot);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}
int absmax_into(int dtype, const void* p, long long n, unsigned long long* slot, cudaStream_t st) {
  switch (dtype) {
    case CTGB_F32: return absmax_typed<float>(p, n, slot, st);
    case CTGB_F64: return absmax_typed<double>(p, n, slot, st);
    case CTGB_C64: return absmax_typed<float2>(p, n, slot, st);
    case CTGB_C128: return absmax_typed<double2>(p, n, slot, st);
  }
  return fail(CTGB_E_VALUE, "bad dtype");
}

int wide_dtype(int dtype) { return dtype == CTGB_F32 ? CTGB_F64 : dtype == CTGB_C64 ? CTGB_C128 : dtype; }

// The root's tangent of a stripped forward-mode plan rides along (StripTangent: the tangent output,
// its chunk, the dense raw tangent root, the tangent's running exponent Et and e'_s, the slice exponent
// without the root's factor); the same three launches fold both.  (O: the type of the output
// accumulator, T or WideOf<T>)
struct StripTangent {
  void* tout = nullptr;
  void* tchunk = nullptr;
  const void* tm = nullptr;
  double* Et = nullptr;
  const double* es_t = nullptr;
};
template <typename T, typename O>
int accum_stripped_typed(const int64_t* dchunk, const int64_t* hchunk, void* out, void* chunk, long long out_elems,
                         const void* m, double* E, const double* es, const double* froot, const StripTangent& tg,
                         cudaStream_t st) {
  rescale_out_kernel<T, O><<<flat_grid(out_elems), 256, 0, st>>>((O*)out, out_elems, E, es, (O*)tg.tout, tg.Et,
                                                                  tg.es_t);
  add_chunk_kernel<T, O><<<flat_grid(hchunk[S_OUT_ELEMS]), 256, 0, st>>>(dchunk, (O*)chunk, (const T*)m, E, es, froot,
                                                                         (O*)tg.tchunk, (const T*)tg.tm, tg.Et,
                                                                         tg.es_t);
  commit_exponent_kernel<<<1, 1, 0, st>>>(E, es, tg.Et, tg.es_t);
  g_launches.fetch_add(3, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}
int accum_stripped(int dtype, bool wide, const int64_t* dchunk, const int64_t* hchunk, void* out, void* chunk,
                   long long out_elems, const void* m, double* E, const double* es, const double* froot,
                   const StripTangent& tg, cudaStream_t st) {
  switch (dtype) {
    case CTGB_F32:
      return wide ? accum_stripped_typed<float, double>(dchunk, hchunk, out, chunk, out_elems, m, E, es, froot, tg, st)
                  : accum_stripped_typed<float, float>(dchunk, hchunk, out, chunk, out_elems, m, E, es, froot, tg, st);
    case CTGB_F64:
      return accum_stripped_typed<double, double>(dchunk, hchunk, out, chunk, out_elems, m, E, es, froot, tg, st);
    case CTGB_C64:
      return wide ? accum_stripped_typed<float2, double2>(dchunk, hchunk, out, chunk, out_elems, m, E, es, froot, tg, st)
                  : accum_stripped_typed<float2, float2>(dchunk, hchunk, out, chunk, out_elems, m, E, es, froot, tg, st);
    case CTGB_C128:
      return accum_stripped_typed<double2, double2>(dchunk, hchunk, out, chunk, out_elems, m, E, es, froot, tg, st);
  }
  return fail(CTGB_E_VALUE, "bad dtype");
}

// stripped forward mode, once per call: the tangent output from its own running exponent to the
// mantissa's (tangent_to_exponent_kernel); `dtype` is the accumulator's
int tangent_to_exponent(int dtype, void* tout, long long n, const double* Et, const double* E, cudaStream_t st) {
  const unsigned grid = flat_grid(n);
  switch (dtype) {
    case CTGB_F32: tangent_to_exponent_kernel<float><<<grid, 256, 0, st>>>((float*)tout, n, Et, E); break;
    case CTGB_F64: tangent_to_exponent_kernel<double><<<grid, 256, 0, st>>>((double*)tout, n, Et, E); break;
    case CTGB_C64: tangent_to_exponent_kernel<float2><<<grid, 256, 0, st>>>((float2*)tout, n, Et, E); break;
    case CTGB_C128: tangent_to_exponent_kernel<double2><<<grid, 256, 0, st>>>((double2*)tout, n, Et, E); break;
    default: return fail(CTGB_E_VALUE, "bad dtype");
  }
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

// the dense float32 / complex64 root result of one slice, added into its chunk of the double output
int add_chunk_wide(int dtype, const int64_t* dchunk, const int64_t* hchunk, void* chunk, const void* m, cudaStream_t st) {
  const unsigned grid = flat_grid(hchunk[S_OUT_ELEMS]);
  if (dtype == CTGB_F32) add_chunk_wide_kernel<float, double><<<grid, 256, 0, st>>>(dchunk, (double*)chunk, (const float*)m);
  else if (dtype == CTGB_C64) add_chunk_wide_kernel<float2, double2><<<grid, 256, 0, st>>>(dchunk, (double2*)chunk, (const float2*)m);
  else return fail(CTGB_E_VALUE, "a wide accumulator belongs to float32 / complex64 plans");
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}

template <typename T>
int conj_typed(void* p, long long n, cudaStream_t st) {
  conj_kernel<T><<<flat_grid(n), 256, 0, st>>>((T*)p, n);
  g_launches.fetch_add(1, std::memory_order_relaxed);
  CUDA_TRY(cudaGetLastError());
  return CTGB_OK;
}
// in-place conjugate of n elements (nothing to do for real dtypes)
int conj_inplace(int dtype, void* p, long long n, cudaStream_t st) {
  if (n <= 0) return CTGB_OK;
  if (dtype == CTGB_C64) return conj_typed<float2>(p, n, st);
  if (dtype == CTGB_C128) return conj_typed<double2>(p, n, st);
  return CTGB_OK;
}

int launch_node(int kind, const int64_t* h, const int64_t* d, const void* A, const void* B, void* C, cudaStream_t st) {
  return kind == 0 ? launch_gett(h, d, A, B, C, st) : launch_single(h, d, A, C, st);
}

}  // namespace

// ================================================================== plans
// A tensor slot (ctgb_tensor) as the library keeps it.
struct ctgb_tensor_rec {
  int kind, input_index;
  int64_t offset, nbytes;
  std::vector<int32_t> slice_pos;
  std::vector<int64_t> slice_stride;
};

// The memory tensor slots resolve to while one slice runs.
struct ctgb_slice_mem {
  const void* const* inputs = nullptr;  // kind 0
  void* const* grads = nullptr;         // kind 5
  const void* const* tangents = nullptr;  // kind 7
  char* tout = nullptr;                 // kind 8
  char* persistent = nullptr;           // kinds 2, 6
  char* scratch = nullptr;              // kind 1
  char* out = nullptr;                  // kind 3
  const char* cot = nullptr;            // kind 4
  size_t es = 0;
  size_t out_es = 0;                    // element size of the output accumulator (kind 3)
  const int64_t* digits = nullptr;
};

static char* resolve_tensor(const ctgb_tensor_rec& q, const ctgb_slice_mem& m, int64_t out_off) {
  auto sliced = [&](const void* base) {
    int64_t off = 0;
    for (size_t j = 0; j < q.slice_pos.size(); ++j) off += m.digits[q.slice_pos[j]] * q.slice_stride[j];
    return (char*)base + off * (int64_t)m.es;
  };
  switch (q.kind) {
    case 0: return sliced(m.inputs[q.input_index]);
    case 1: return m.scratch + q.offset;
    case 2:
    case 6: return m.persistent + q.offset;
    case 4: return (char*)m.cot + out_off * (int64_t)m.es;
    case 5: return sliced(m.grads[q.input_index]);
    case 7: return sliced(m.tangents[q.input_index]);
    case 8: return m.tout + out_off * (int64_t)m.out_es;
    default: return m.out + out_off * (int64_t)m.out_es;
  }
}

// slice id -> digits, most significant first (core.py:3775-3800); returns the element offset of the
// slice's output view (sum of digit * out_stride)
static int64_t decode_slice(int64_t id, const std::vector<int64_t>& radix, const std::vector<int64_t>& project,
                            const std::vector<int64_t>& out_stride, std::vector<int64_t>& digits) {
  // least-significant digit first: the same digits as i // stride_j % radix_j,
  // without forming the strides (their product overflows 64 bits for trees
  // with more than 63 binary sliced indices; ids themselves are < 2^63)
  const int ns = (int)radix.size();
  int64_t rem = id;
  for (int j = ns - 1; j >= 0; --j) {
    if (project[j] >= 0) {
      digits[j] = project[j];
    } else {
      digits[j] = rem % radix[j];
      rem /= radix[j];
    }
  }
  int64_t out_off = 0;
  for (int j = 0; j < ns; ++j) out_off += digits[j] * out_stride[j];
  return out_off;
}

// copies a ctgb_tensor array into records, checking input and slice references
static int copy_tensors(const ctgb_tensor* ts, int n, int n_inputs, int n_sliced, std::vector<ctgb_tensor_rec>& out) {
  out.resize(n);
  for (int i = 0; i < n; ++i) {
    const ctgb_tensor& t = ts[i];
    auto& q = out[i];
    q.kind = t.kind;
    q.input_index = t.input_index;
    q.offset = t.offset;
    q.nbytes = t.nbytes;
    if ((t.kind == 0 || t.kind == 5 || t.kind == 7) && (t.input_index < 0 || t.input_index >= n_inputs))
      return fail(CTGB_E_VALUE, "tensor refers to a missing input");
    for (int j = 0; j < t.n_sliced; ++j) {
      if (t.slice_pos[j] < 0 || t.slice_pos[j] >= n_sliced) return fail(CTGB_E_VALUE, "slice position out of range");
      q.slice_pos.push_back(t.slice_pos[j]);
      q.slice_stride.push_back(t.slice_stride[j]);
    }
  }
  return CTGB_OK;
}

// A forward plan runs phases 0 and 1.  A reverse-mode plan (cotengra_b200/vjp.py plans it) also runs
// phases 2 and 3: it propagates H = conj(cotangent), for which the adjoint of a contraction needs no
// conjugation, so every backward node is an ordinary pairwise or single-operand descriptor and only the
// cotangent's copy and the finished input gradients are conjugated (complex dtypes).
struct ctgb_plan {
  int dtype = 0;
  int n_inputs = 0;
  using Tensor = ctgb_tensor_rec;
  struct Node {
    int kind, a, b, c, phase, zero_fill, is_root;
    int a2 = -1, b2 = -1;  // two-term node (kind 2): the slots of A' and B'
    size_t desc_off;  // word offset into descs
    int64_t c_elems;  // dense elements of the result (strip_exponent)
    int measure_after = 0;  // strip_exponent: max|C| needs its own pass (split-K / block partial sums)
    int prescale_b = 0;     // strip_exponent: the small operand is copied, scaled by 1/(fA fB), first
    int prescale_a = 0;     // stripped reverse mode: a single-operand node reads a copy of A scaled by 1/fA
    int fa = -1, fb = -1;   // strip_exponent: the factor slots fA, fB it divides by (-1: 1.0)
    int tangent = 0;        // stripped forward mode: a tangent record (divides by fA, fB, measures nothing)
    int bscale_reuse = 0;   // ... whose small operand's scaled copy the node before it has just made
  };
  std::vector<Tensor> tensors;
  std::vector<Node> nodes;
  std::vector<int64_t> descs;  // host copy of every descriptor, concatenated
  int64_t* d_descs = nullptr;
  std::vector<int64_t> radix, project, out_stride;
  int64_t out_elements = 0, workspace_bytes = 0, persistent_bytes = 0;
  int strip_exponent = 0;
  // dtype of the output accumulator (ctgb_plan_set_accumulator): the plan's, or its double counterpart.
  // A wide forward plan either has a flagged dot-stream root that adds into `out` in double, or a
  // root that stores its slice densely in the plan dtype (as stripped plans do), folded afterwards.
  int acc_dtype = 0;
  bool wide_desc = false;           // a descriptor carries FLAG_WIDE_C: runs only with a wide accumulator
  int root = -1;                    // the node that writes the output
  bool backward = false;            // phase 2/3 nodes: needs a cotangent and the gradient buffers
  // forward-mode plans (tangent slots, two-term nodes): run by ctgb_plan_execute_jvp
  bool jvp = false;
  int troot = -1;                   // a node that writes the root's tangent (is_root = 2)
  std::vector<char> needs_tangent;  // per input: a kind-7 slot reads its tangent
  int64_t cot_offset = -1;          // conjugated cotangent copy in the persistent arena
  std::vector<int64_t> grad_elems;  // per input: elements of its gradient (0: not differentiated)
  int64_t launches_per_slice = 0;
  // strip_exponent scratch (device): [1] slice exponent, [2] invariant exponent
  double* d_scalars = nullptr;
  // fused strip_exponent: one factor slot per tensor (1.0 for inputs and single-operand results,
  // max|C| for pairwise results) and the slots to reset / sum per pass; then slot n_tensors, the
  // root's seed divisor of a stripped reverse-mode plan, and slot n_tensors + 1, a constant 1.0
  double* d_factors = nullptr;
  bool scale_pending = false;   // stripped reverse mode: waits for ctgb_plan_set_scale_slots
  char* d_bscale = nullptr;     // scaled copy of the current node's small operand
  size_t bscale_bytes = 0;
  int* d_slot_lists = nullptr;  // [variant slots..., invariant slots...]
  int n_var_slots = 0, n_inv_slots = 0;
  // chunk descriptor for stripped accumulation (host + device), built at create
  std::vector<int64_t> chunk_desc;
  int64_t* d_chunk_desc = nullptr;
  int device = -1;
  // optional per-node timing (bench.py roofline): events around every node launch
  bool profile = false;
  std::vector<cudaEvent_t> ev0, ev1;
  // pinned staging block of ctgb_plan_execute_host (all inputs in one H2D copy)
  char* h_stage = nullptr;
  size_t h_stage_bytes = 0;
};

// Factor slots of a strip_exponent plan and the descriptor words that point into them.  A forward
// plan divides every pairwise node by the factors of its own operands (slot_a = slot_b = null).  A
// stripped reverse-mode plan names the slots node by node (ctgb_plan_set_scale_slots): its phase 0/1
// nodes measure max|C| into their own slot as the forward does; a recomputed forward node (phase 2)
// divides by the phase-1 factors of the values it recomputes and measures nothing, so that it forms
// the same quotient as phase 1; a backward node divides by f_p and f_r (the seed at the root) and
// measures nothing.  A stripped forward-mode plan (ctgb_plan_set_tangent_scale_slots) marks its
// tangent records (`tangent`): each divides by its primal node's two factor slots and measures nothing,
// a two-term one through its scale words (the kernel scales B and B' as it stages them), and a
// one-term one whose small operand the node before it has just copied, scaled alike, reads that copy.
static cudaError_t strip_setup(ctgb_plan* p, const int32_t* slot_a, const int32_t* slot_b,
                               const int32_t* tangent = nullptr) {
  const size_t nt = p->tensors.size();
  std::vector<double> ones(nt + 2, 1.0);
  cudaError_t e = cudaMalloc((void**)&p->d_factors, (nt + 2) * sizeof(double));
  if (e == cudaSuccess) e = cudaMemcpy(p->d_factors, ones.data(), (nt + 2) * sizeof(double), cudaMemcpyHostToDevice);
  std::vector<int> var_slots, inv_slots;
  for (size_t i = 0; i < p->nodes.size(); ++i) {
    auto& n = p->nodes[i];
    n.fa = slot_a ? slot_a[i] : n.a;
    n.fb = slot_b ? slot_b[i] : n.b;
    n.tangent = tangent != nullptr && tangent[i] != 0;
    const bool measures = n.phase <= 1 && !n.tangent;
    if (n.kind == 2) {
      int64_t* w = p->descs.data() + n.desc_off;
      w[W_SCALE_A] = (int64_t)(uintptr_t)(p->d_factors + n.fa);
      w[W_SCALE_B] = (int64_t)(uintptr_t)(p->d_factors + n.fb);
      continue;
    }
    if (n.kind != 0) {
      // (a reverse-mode plan whose root is a single-operand node: its adjoint reads the seeded cotangent)
      n.prescale_a = slot_a != nullptr && n.fa >= 0;
      if (n.prescale_a && (size_t)p->tensors[n.a].nbytes > p->bscale_bytes) p->bscale_bytes = (size_t)p->tensors[n.a].nbytes;
      continue;
    }
    if (!measures) n.measure_after = 0;
    int64_t* w = p->descs.data() + n.desc_off;
    // small second operand (the usual case on a stem): scale a copy of it instead of every
    // output element; otherwise the epilogue multiplies by 1/(fA fB)
    const int64_t bbytes = p->tensors[n.b].nbytes;
    n.prescale_b = bbytes > 0 && bbytes <= (16ll << 20) && p->tensors[n.b].kind != 3;
    if (n.prescale_b && n.tangent && i > 0) {
      const auto& prev = p->nodes[i - 1];
      n.bscale_reuse = prev.kind == 0 && prev.prescale_b && prev.b == n.b && prev.fa == n.fa && prev.fb == n.fb &&
                       prev.phase == n.phase;
    }
    if (n.prescale_b) {
      if ((size_t)bbytes > p->bscale_bytes) p->bscale_bytes = (size_t)bbytes;
    } else {
      w[W_SCALE_A] = (int64_t)(uintptr_t)(p->d_factors + n.fa);
      w[W_SCALE_B] = (int64_t)(uintptr_t)(p->d_factors + n.fb);
    }
    w[W_FACTOR_C] = (n.measure_after || !measures) ? 0 : (int64_t)(uintptr_t)(p->d_factors + n.c);
    if (measures) (n.phase == 0 ? inv_slots : var_slots).push_back(n.c);
  }
  p->n_var_slots = (int)var_slots.size();
  p->n_inv_slots = (int)inv_slots.size();
  var_slots.insert(var_slots.end(), inv_slots.begin(), inv_slots.end());
  if (e == cudaSuccess && p->bscale_bytes) e = cudaMalloc((void**)&p->d_bscale, p->bscale_bytes + 256);
  if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_slot_lists, (var_slots.size() + 1) * sizeof(int));
  if (e == cudaSuccess && !var_slots.empty())
    e = cudaMemcpy(p->d_slot_lists, var_slots.data(), var_slots.size() * sizeof(int), cudaMemcpyHostToDevice);
  if (e == cudaSuccess)
    e = cudaMemcpy(p->d_descs, p->descs.data(), p->descs.size() * sizeof(int64_t), cudaMemcpyHostToDevice);
  return e;
}

extern "C" {

int ctgb_abi_version(void) { return CTGB_ABI_VERSION; }
int ctgb_desc_words(void) { return DESC_WORDS; }
int ctgb_single_desc_words(void) { return SDESC_WORDS; }
const char* ctgb_last_error(void) { return g_err.c_str(); }
int64_t ctgb_launch_count(void) { return g_launches.load(); }
int64_t ctgb_tensor_map_launches(void) { return g_tmap_launches.load(); }

int ctgb_tc05_launch_config(const int64_t* words, uint64_t a_addr, int sms, uint64_t smem_optin, int64_t* out,
                            int n_out) {
  if (!words || !out) return fail(CTGB_E_VALUE, "null argument");
  if (words[W_MAGIC] != DESC_MAGIC) return fail(CTGB_E_VALUE, "bad descriptor");
  if (n_out < 9) return fail(CTGB_E_VALUE, "ctgb_tc05_launch_config writes 9 words");
  if (sms < 1) return fail(CTGB_E_VALUE, "sms must be positive");
  Tc05Launch lc;
  int rc;
  const bool one = (words[W_FLAGS] & FLAG_TF32_ONE_PASS) != 0;
  switch (words[W_VARIANT]) {
    case VAR_TC05_128x64:
      rc = one ? tc05_launch_config<64, true>(words, a_addr, sms, smem_optin, lc)
               : tc05_launch_config<64, false>(words, a_addr, sms, smem_optin, lc);
      break;
    case VAR_TC05_128x32:
      rc = one ? tc05_launch_config<32, true>(words, a_addr, sms, smem_optin, lc)
               : tc05_launch_config<32, false>(words, a_addr, sms, smem_optin, lc);
      break;
    case VAR_TC05_128x16:
      rc = one ? tc05_launch_config<16, true>(words, a_addr, sms, smem_optin, lc)
               : tc05_launch_config<16, false>(words, a_addr, sms, smem_optin, lc);
      break;
    default: return fail(CTGB_E_VALUE, "not a wgmma descriptor");
  }
  if (rc) return rc;
  const int64_t v[9] = {lc.b_stat, lc.nb, lc.sa, (int64_t)lc.grid, (int64_t)lc.smem, lc.tm_rank, lc.bulk,
                        (int64_t)lc.chunk, (int64_t)lc.chunks};
  for (int i = 0; i < 9; ++i) out[i] = v[i];
  return CTGB_OK;
}

int ctgb_dmmastream_launch_config(const int64_t* words, int sms, int64_t* out, int n_out) {
  if (!words || !out) return fail(CTGB_E_VALUE, "null argument");
  if (words[W_MAGIC] != DESC_MAGIC) return fail(CTGB_E_VALUE, "bad descriptor");
  if (n_out < 3) return fail(CTGB_E_VALUE, "ctgb_dmmastream_launch_config writes 3 words");
  if (sms < 1) return fail(CTGB_E_VALUE, "sms must be positive");
  if (words[W_VARIANT] != VAR_DMMASTREAM) return fail(CTGB_E_VALUE, "not a DMMA stream descriptor");
  DsLaunch lc;
  if (int rc = dmmastream_launch_config(words, sms, lc)) return rc;
  out[0] = lc.nj;
  out[1] = lc.rows;
  out[2] = (int64_t)lc.blocks;
  return CTGB_OK;
}

int ctgb_device_info(int* sm_count, int* cc_major, int* cc_minor, size_t* smem_optin_bytes) {
  DevInfo& d = devinfo();
  if (!d.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  if (sm_count) *sm_count = d.sms;
  if (cc_major) *cc_major = d.major;
  if (cc_minor) *cc_minor = d.minor;
  if (smem_optin_bytes) *smem_optin_bytes = d.smem_optin;
  return CTGB_OK;
}

int ctgb_probe_fp64_peaks(double* dmma_tflops, double* dfma_tflops, void* stream) {
  DevInfo& di = devinfo();
  if (!di.ok) return fail(CTGB_E_CUDA, "no CUDA device");
  cudaStream_t st = (cudaStream_t)stream;
  double* sink = nullptr;
  CUDA_TRY(cudaMalloc((void**)&sink, 64));
  cudaEvent_t e0, e1;
  CUDA_TRY(cudaEventCreate(&e0));
  CUDA_TRY(cudaEventCreate(&e1));
  const int blocks = di.sms * 8, iters = 4096;
  auto timed = [&](int which, double flop_per_thread_iter, double* out) -> int {
    float best = 1e30f;
    for (int rep = 0; rep < 4; ++rep) {
      CUDA_TRY(cudaEventRecord(e0, st));
      if (which == 0) probe_dmma_kernel<<<blocks, 256, 0, st>>>(sink, iters);
      else probe_dfma_kernel<<<blocks, 256, 0, st>>>(sink, iters);
      CUDA_TRY(cudaEventRecord(e1, st));
      CUDA_TRY(cudaEventSynchronize(e1));
      float ms = 0.f;
      CUDA_TRY(cudaEventElapsedTime(&ms, e0, e1));
      if (rep > 0 && ms < best) best = ms;
    }
    g_launches.fetch_add(4, std::memory_order_relaxed);
    *out = flop_per_thread_iter * iters * 256.0 * blocks / (best * 1e-3) / 1e12;
    return CTGB_OK;
  };
  int rc = CTGB_OK;
  // one DMMA = 16*8*4 MACs per warp = 1024 flop / 32 lanes; 8 per iteration
  if (dmma_tflops) rc = timed(0, 8 * 1024.0 / 32.0, dmma_tflops);
  if (!rc && dfma_tflops) rc = timed(1, 8 * 2.0, dfma_tflops);
  cudaEventDestroy(e0);
  cudaEventDestroy(e1);
  cudaFree(sink);
  return rc;
}

int ctgb_contract_pair(const int64_t* desc, const void* A, const void* B, void* C, void* stream) {
  if (!desc) return fail(CTGB_E_VALUE, "null descriptor");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* d = nullptr;
  CUDA_TRY(cudaMallocAsync((void**)&d, DESC_WORDS * sizeof(int64_t), st));
  CUDA_TRY(cudaMemcpyAsync(d, desc, DESC_WORDS * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  int rc = launch_gett(desc, d, A, B, C, st);
  cudaFreeAsync(d, st);
  return rc;
}

int ctgb_contract_pair2(const int64_t* desc, const void* A, const void* B, const void* A2, const void* B2, void* C,
                        void* stream) {
  if (!desc) return fail(CTGB_E_VALUE, "null descriptor");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* d = nullptr;
  CUDA_TRY(cudaMallocAsync((void**)&d, DESC_WORDS * sizeof(int64_t), st));
  CUDA_TRY(cudaMemcpyAsync(d, desc, DESC_WORDS * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  int rc = launch_gett2(desc, d, A, B, A2, B2, C, st);
  cudaFreeAsync(d, st);
  return rc;
}

int ctgb_absorb_root(const int64_t* desc, const void* A, const void* Bs, const void* V, void* C, void* stream) {
  if (!desc || desc[0] != DESC_MAGIC || desc[W_VARIANT] != VAR_ABSORB_ROOT)
    return fail(CTGB_E_VALUE, "not an absorb-root descriptor");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* d = nullptr;
  CUDA_TRY(cudaMallocAsync((void**)&d, DESC_WORDS * sizeof(int64_t), st));
  CUDA_TRY(cudaMemcpyAsync(d, desc, DESC_WORDS * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  int rc = launch_absorb_root(desc, d, A, Bs, V, C, st);
  cudaFreeAsync(d, st);
  return rc;
}

int ctgb_reduce_single(const int64_t* desc, const void* X, void* out, void* stream) {
  if (!desc) return fail(CTGB_E_VALUE, "null descriptor");
  cudaStream_t st = (cudaStream_t)stream;
  int64_t* d = nullptr;
  CUDA_TRY(cudaMallocAsync((void**)&d, SDESC_WORDS * sizeof(int64_t), st));
  CUDA_TRY(cudaMemcpyAsync(d, desc, SDESC_WORDS * sizeof(int64_t), cudaMemcpyHostToDevice, st));
  int rc = launch_single(desc, d, X, out, st);
  cudaFreeAsync(d, st);
  return rc;
}

int ctgb_plan_create(const ctgb_plan_desc* pd, ctgb_plan** out) {
  if (!pd || !out) return fail(CTGB_E_VALUE, "null argument");
  const size_t es = elem_size(pd->dtype);
  if (es == 0) return fail(CTGB_E_VALUE, "bad dtype");
  ctgb_plan* p = new ctgb_plan();
  auto refuse = [&](const char* msg) {
    delete p;
    return fail(CTGB_E_VALUE, msg);
  };
  p->dtype = p->acc_dtype = pd->dtype;
  p->n_inputs = pd->n_inputs;
  if (int rc = copy_tensors(pd->tensors, pd->n_tensors, pd->n_inputs, pd->n_sliced, p->tensors)) {
    delete p;
    return rc;
  }
  p->nodes.resize(pd->n_nodes);
  int64_t per_slice = 0;
  for (int i = 0; i < pd->n_nodes; ++i) {
    const ctgb_node& n = pd->nodes[i];
    auto& q = p->nodes[i];
    q.kind = n.kind;
    q.a = n.a;
    q.b = n.b;
    q.c = n.c;
    q.phase = n.phase;
    q.zero_fill = n.zero_fill;
    q.is_root = n.is_root;
    // (a two-term node: the pair words, then the slots of A' and B')
    const int words = n.kind == 0 ? (int)DESC_WORDS : n.kind == 2 ? (int)DESC_WORDS + 2 : (int)SDESC_WORDS;
    const int64_t magic = n.kind == 1 ? SDESC_MAGIC : DESC_MAGIC;
    if (n.kind < 0 || n.kind > 2 || !n.desc || n.desc[0] != magic) return refuse("bad node descriptor");
    if (n.phase < 0 || n.phase > 3) return refuse("bad node phase");
    if (n.is_root < 0 || n.is_root > 2) return refuse("bad node root mark");
    auto bad = [&](int t) { return t < 0 || t >= pd->n_tensors; };
    if (bad(n.a) || bad(n.c) || (n.kind != 1 && bad(n.b))) return refuse("node refers to a missing tensor");
    if (n.kind == 2) {
      const int64_t v = n.desc[W_VARIANT];
      if (v != VAR_ROWSTREAM && v != VAR_ROWSTREAM_K && v != VAR_DMMASTREAM)
        return refuse("a two-term node runs on the row-stream and DMMA stream kernels only");
      if (bad((int)n.desc[DESC_WORDS]) || bad((int)n.desc[DESC_WORDS + 1])) return refuse("node refers to a missing tensor");
      q.a2 = (int)n.desc[DESC_WORDS];
      q.b2 = (int)n.desc[DESC_WORDS + 1];
    }
    p->jvp |= n.kind == 2 || n.is_root == 2;
    if (n.kind == 0 && n.desc[W_VARIANT] == VAR_ABSORB_ROOT) {
      if (bad((int)n.desc[AB_BS_SLOT])) return refuse("node refers to a missing tensor");
      if (pd->strip_exponent) return refuse("an absorb-root node runs in unstripped plans only");
    }
    p->backward |= n.phase >= 2;
    if (n.is_root == 1) p->root = i;
    if (n.is_root == 2) p->troot = i;
    if (n.kind == 0 && (n.desc[W_FLAGS] & FLAG_WIDE_C)) {
      if (!n.is_root || pd->strip_exponent) return refuse("a wide C belongs to the root of an unstripped plan");
      p->wide_desc = true;
    }
    q.desc_off = p->descs.size();
    p->descs.insert(p->descs.end(), n.desc, n.desc + words);
    q.c_elems = p->tensors[n.c].nbytes / (int64_t)es;
    if (pd->strip_exponent && n.kind == 0) {
      const int64_t* w = n.desc;
      q.measure_after = w[W_SPLITK] > 1 || w[W_VARIANT] == VAR_DOTSTREAM || w[W_VARIANT] == VAR_DOTSTREAM4;
      // (the block-reduction epilogue of KRED runs once: its result is measured afterwards as well;
      // so is a wgmma node whose contracted range is folded into C chunk by chunk)
      q.measure_after |= w[W_VARIANT] == VAR_KRED;
      q.measure_after |= (w[W_VARIANT] == VAR_TC05_128x64 || w[W_VARIANT] == VAR_TC05_128x32 ||
                          w[W_VARIANT] == VAR_TC05_128x16) &&
                         tc05_chunk_steps((unsigned)((w[W_STEPS_K] + w[W_SPLITK] - 1) / w[W_SPLITK]),
                                          (unsigned)(w[W_KTA] >> 2)) < (unsigned)w[W_STEPS_K];
    }
    if (n.phase == 1 || n.phase == 2) per_slice += 1 + q.measure_after + (pd->strip_exponent && n.kind == 0 ? 1 : 0);
  }
  // kind 3 (the output) belongs to forward plans, kinds 4-6 (cotangent, gradients, H accumulators) to
  // reverse-mode ones: execute checks exactly the buffers the plan's kind needs
  for (const auto& q : p->tensors) p->jvp |= q.kind >= 7;
  // (stripped derivative plans get their factor slots from ctgb_plan_set_scale_slots or, forward
  // mode, ctgb_plan_set_tangent_scale_slots)
  p->scale_pending = pd->strip_exponent && (p->backward || p->jvp);
  p->grad_elems.assign(pd->n_inputs, 0);
  p->needs_tangent.assign(pd->n_inputs, 0);
  if (p->jvp && p->backward) return refuse("a forward-mode plan has phases 0 and 1");
  for (const auto& q : p->tensors) {
    const bool rev = q.kind >= 4 && q.kind <= 6, fwd = q.kind >= 7;
    if (q.kind < 0 || q.kind > 8 || (q.kind == 3 && p->backward) || (rev && !p->backward) || (fwd && !p->jvp))
      return refuse("bad tensor kind for the plan's phases");
    if (q.kind == 5) p->grad_elems[q.input_index] = q.nbytes / (int64_t)es;
    if (q.kind == 7) p->needs_tangent[q.input_index] = 1;
  }
  const bool cplx = pd->dtype == CTGB_C64 || pd->dtype == CTGB_C128;
  if (cplx && p->backward && pd->cotangent_offset < 0)
    return refuse("a complex reverse-mode plan needs room for the conjugated cotangent");
  p->cot_offset = cplx ? pd->cotangent_offset : -1;
  if (p->cot_offset >= 0 && p->cot_offset + pd->out_elements * (int64_t)es > pd->persistent_bytes)
    return refuse("the conjugated cotangent does not fit the persistent arena");
  if (pd->strip_exponent) per_slice += 5;  // reset slots, sum of logs, rescale/add/commit
  p->launches_per_slice = per_slice;
  p->radix.assign(pd->slice_radix, pd->slice_radix + pd->n_sliced);
  p->project.assign(pd->slice_project, pd->slice_project + pd->n_sliced);
  p->out_stride.assign(pd->slice_out_stride, pd->slice_out_stride + pd->n_sliced);
  p->out_elements = pd->out_elements;
  p->workspace_bytes = pd->workspace_bytes;
  p->persistent_bytes = pd->persistent_bytes;
  p->strip_exponent = pd->strip_exponent;

  if (cudaGetDevice(&p->device) != cudaSuccess) {
    delete p;
    return fail(CTGB_E_CUDA, "no CUDA device");
  }
  cudaError_t e = cudaMalloc((void**)&p->d_descs, p->descs.size() * sizeof(int64_t) + 8);
  if (e == cudaSuccess)
    e = cudaMemcpy(p->d_descs, p->descs.data(), p->descs.size() * sizeof(int64_t), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMalloc((void**)&p->d_scalars, 8 * sizeof(double));
  if (e == cudaSuccess) e = cudaMemset(p->d_scalars, 0, 8 * sizeof(double));
  // (stripped derivative plans get their factor slots from a setter)
  if (e == cudaSuccess && p->strip_exponent && !p->scale_pending) e = strip_setup(p, nullptr, nullptr);
  if (e != cudaSuccess) {
    std::string msg = cudaGetErrorString(e);
    ctgb_plan_destroy(p);
    return fail(CTGB_E_CUDA, "plan upload: " + msg);
  }
  *out = p;
  return CTGB_OK;
}

int ctgb_plan_profile(ctgb_plan* p, int enable) {
  if (!p) return fail(CTGB_E_VALUE, "null plan");
  if (enable && p->ev0.empty()) {
    p->ev0.resize(p->nodes.size());
    p->ev1.resize(p->nodes.size());
    for (size_t i = 0; i < p->nodes.size(); ++i) {
      CUDA_TRY(cudaEventCreate(&p->ev0[i]));
      CUDA_TRY(cudaEventCreate(&p->ev1[i]));
    }
  }
  p->profile = enable != 0;
  return CTGB_OK;
}

int ctgb_plan_profile_read(ctgb_plan* p, float* ms, int n_nodes) {
  if (!p || !ms) return fail(CTGB_E_VALUE, "null argument");
  if (p->ev0.empty()) return fail(CTGB_E_VALUE, "profiling was never enabled");
  if (n_nodes != (int)p->nodes.size()) return fail(CTGB_E_VALUE, "node count mismatch");
  for (int i = 0; i < n_nodes; ++i) {
    ms[i] = -1.f;
    if (cudaEventQuery(p->ev1[i]) == cudaErrorInvalidResourceHandle) continue;
    cudaError_t e = cudaEventSynchronize(p->ev1[i]);
    if (e != cudaSuccess) { cudaGetLastError(); continue; }
    float t = 0.f;
    if (cudaEventElapsedTime(&t, p->ev0[i], p->ev1[i]) == cudaSuccess) ms[i] = t; else cudaGetLastError();
  }
  return CTGB_OK;
}

void ctgb_plan_destroy(ctgb_plan* p) {
  if (!p) return;
  for (auto e : p->ev0) cudaEventDestroy(e);
  for (auto e : p->ev1) cudaEventDestroy(e);
  if (p->d_descs) cudaFree(p->d_descs);
  if (p->d_scalars) cudaFree(p->d_scalars);
  if (p->d_factors) cudaFree(p->d_factors);
  if (p->d_bscale) cudaFree(p->d_bscale);
  if (p->d_slot_lists) cudaFree(p->d_slot_lists);
  if (p->d_chunk_desc) cudaFree(p->d_chunk_desc);
  if (p->h_stage) cudaFreeHost(p->h_stage);
  delete p;
}

size_t ctgb_plan_workspace_bytes(const ctgb_plan* p) {
  return p ? (size_t)(p->workspace_bytes + p->persistent_bytes) : 0;
}
int64_t ctgb_plan_launches_per_slice(const ctgb_plan* p) { return p ? p->launches_per_slice : 0; }
int ctgb_plan_strip_modes(const ctgb_plan* p, int32_t* prescale_b, int32_t* measure_after, int n) {
  if (!p || n < (int)p->nodes.size() || !prescale_b || !measure_after) return fail(CTGB_E_VALUE, "bad arguments");
  for (size_t i = 0; i < p->nodes.size(); ++i) {
    const auto& q = p->nodes[i];
    prescale_b[i] = q.kind == 0 ? q.prescale_b : -1;
    measure_after[i] = q.measure_after;
  }
  return CTGB_OK;
}

// Install the (single-operand style) descriptor that maps the dense root result
// of one slice onto its chunk of the full output; only used with strip_exponent.
int ctgb_plan_set_chunk_desc(ctgb_plan* p, const int64_t* desc) {
  if (!p || !desc || desc[0] != SDESC_MAGIC) return fail(CTGB_E_VALUE, "bad chunk descriptor");
  p->chunk_desc.assign(desc, desc + SDESC_WORDS);
  if (!p->d_chunk_desc) CUDA_TRY(cudaMalloc((void**)&p->d_chunk_desc, SDESC_WORDS * sizeof(int64_t)));
  CUDA_TRY(cudaMemcpy(p->d_chunk_desc, desc, SDESC_WORDS * sizeof(int64_t), cudaMemcpyHostToDevice));
  return CTGB_OK;
}

int ctgb_plan_set_accumulator(ctgb_plan* p, int32_t dtype) {
  if (!p) return fail(CTGB_E_VALUE, "null plan");
  if (dtype != p->dtype && dtype != wide_dtype(p->dtype))
    return fail(CTGB_E_VALUE, "the accumulator has the plan's dtype or its double counterpart");
  const bool wide = dtype != p->dtype;
  if (wide && p->backward) return fail(CTGB_E_VALUE, "a wide accumulator belongs to forward plans");
  if (wide && !p->strip_exponent) {
    // the root adds into the double output itself (a flagged dot-stream node) or leaves its slice in
    // the per-slice workspace for add_chunk_wide
    if (p->root < 0) return fail(CTGB_E_VALUE, "plan has no root node");
    const int ckind = p->tensors[p->nodes[p->root].c].kind;
    if (ckind != (p->wide_desc ? 3 : 1)) return fail(CTGB_E_VALUE, "root slot does not match the wide accumulator");
    if (!p->wide_desc && p->acc_dtype == p->dtype) p->launches_per_slice += p->troot >= 0 ? 2 : 1;
  } else if (p->wide_desc) {
    return fail(CTGB_E_VALUE, "the plan's root descriptor needs a wide accumulator");
  }
  p->acc_dtype = dtype;
  return CTGB_OK;
}

int ctgb_plan_set_scale_slots(ctgb_plan* p, const int32_t* slot_a, const int32_t* slot_b, int n) {
  if (!p || !slot_a || !slot_b) return fail(CTGB_E_VALUE, "null argument");
  if (!p->scale_pending || p->jvp) return fail(CTGB_E_VALUE, "scale slots belong to stripped reverse-mode plans, once");
  if (n != (int)p->nodes.size()) return fail(CTGB_E_VALUE, "node count mismatch");
  const int seed = (int)p->tensors.size();
  for (int i = 0; i < n; ++i) {
    const bool pair = p->nodes[i].kind == 0;
    if (slot_a[i] < (pair ? 0 : -1) || slot_a[i] > seed || slot_b[i] < (pair ? 0 : -1) || slot_b[i] > seed)
      return fail(CTGB_E_VALUE, "scale slot out of range");
  }
  CUDA_TRY(strip_setup(p, slot_a, slot_b));
  p->scale_pending = false;
  int64_t per_slice = 3;  // reset slots, sum of logs, seed
  for (const auto& q : p->nodes)
    if (q.phase == 1 || q.phase == 2) per_slice += 1 + q.measure_after + q.prescale_b + q.prescale_a;
  p->launches_per_slice = per_slice;
  return CTGB_OK;
}

int ctgb_plan_set_tangent_scale_slots(ctgb_plan* p, const int32_t* slot_a, const int32_t* slot_b,
                                      const int32_t* tangent, int n) {
  if (!p || !slot_a || !slot_b || !tangent) return fail(CTGB_E_VALUE, "null argument");
  if (!p->scale_pending || !p->jvp)
    return fail(CTGB_E_VALUE, "tangent scale slots belong to stripped forward-mode plans, once");
  if (n != (int)p->nodes.size()) return fail(CTGB_E_VALUE, "node count mismatch");
  const int nt = (int)p->tensors.size();
  for (int i = 0; i < n; ++i) {
    const auto& q = p->nodes[i];
    if (tangent[i] != 0 && tangent[i] != 1) return fail(CTGB_E_VALUE, "tangent marks are 0 or 1");
    if (q.kind == 1) {
      if (slot_a[i] != -1 || slot_b[i] != -1) return fail(CTGB_E_VALUE, "a single-operand node divides by nothing");
      continue;
    }
    if (slot_a[i] < 0 || slot_a[i] >= nt || slot_b[i] < 0 || slot_b[i] >= nt)
      return fail(CTGB_E_VALUE, "scale slot out of range");
    // (a primal record is the forward plan's node: it divides by its own operands' factors)
    if (!tangent[i] && (q.kind != 0 || slot_a[i] != q.a || slot_b[i] != q.b))
      return fail(CTGB_E_VALUE, "a primal record divides by its own operands' factor slots");
    if (tangent[i] && q.is_root == 1) return fail(CTGB_E_VALUE, "the primal root is not a tangent record");
  }
  CUDA_TRY(strip_setup(p, slot_a, slot_b, tangent));
  p->scale_pending = false;
  int64_t per_slice = 5;  // reset slots, sum of logs, rescale / add / commit
  for (const auto& q : p->nodes)
    if (q.phase == 1) per_slice += 1 + q.measure_after + (q.prescale_b && !q.bscale_reuse);
  p->launches_per_slice = per_slice;
  return CTGB_OK;
}

}  // extern "C"

// ctgb_plan_execute and ctgb_plan_execute_jvp: `tangents` and `tangent_out` belong to forward-mode
// plans, whose primal root is skipped when `out` is null
static int plan_run(ctgb_plan* p, const void* const* inputs, const void* const* tangents, void* out,
                    void* tangent_out, double* exponent_dev, const void* cotangent, void* const* grads,
                    void* workspace, size_t workspace_bytes, int64_t slice_begin, int64_t slice_step,
                    int64_t slice_count, void* stream) {
  if (workspace_bytes < (size_t)(p->workspace_bytes + p->persistent_bytes))
    return fail(CTGB_E_MEMORY, "workspace too small");
  if (!inputs) return fail(CTGB_E_VALUE, "null inputs");
  if (p->strip_exponent && !p->backward && (!exponent_dev || p->chunk_desc.empty()))
    return fail(CTGB_E_VALUE, "strip_exponent needs an exponent buffer and a chunk descriptor");
  const bool wide = p->acc_dtype != p->dtype;
  if (p->wide_desc && !wide) return fail(CTGB_E_VALUE, "the plan's root descriptor needs a wide accumulator");
  const bool wide_fold = wide && !p->strip_exponent && !p->wide_desc;  // dense root + add_chunk_wide
  if (wide_fold && p->chunk_desc.empty()) return fail(CTGB_E_VALUE, "a wide accumulator needs a chunk descriptor");
  if (p->strip_exponent && !p->backward && p->root < 0) return fail(CTGB_E_VALUE, "plan has no root node");
  // a stripped reverse-mode plan reads the exponent of the forward call it differentiates
  if (p->strip_exponent && p->backward && (!exponent_dev || p->scale_pending))
    return fail(CTGB_E_VALUE, "a stripped reverse-mode plan needs the forward's exponent and its scale slots");
  // a stripped forward-mode plan always runs its primal root: its factor sets the slice exponent
  if (p->strip_exponent && p->jvp && (p->scale_pending || !out || p->troot < 0))
    return fail(CTGB_E_VALUE, "a stripped forward-mode plan needs its scale slots, the output and a tangent root");
  if ((p->backward || p->cot_offset >= 0) && !cotangent) return fail(CTGB_E_VALUE, "the plan needs a cotangent");
  for (int i = 0; i < p->n_inputs; ++i)
    if (p->grad_elems[i] > 0 && (!grads || !grads[i]))
      return fail(CTGB_E_VALUE, "missing gradient buffer of a differentiated input");
  for (int i = 0; i < p->n_inputs; ++i)
    if (p->needs_tangent[i] && (!tangents || !tangents[i]))
      return fail(CTGB_E_VALUE, "missing tangent of an input the plan differentiates");
  if (p->jvp && !tangent_out) return fail(CTGB_E_VALUE, "a forward-mode plan needs a tangent output");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t es = elem_size(p->dtype);
  char* persistent = (char*)workspace;
  char* scratch = persistent + p->persistent_bytes;
  std::vector<int64_t> digits(p->radix.size(), 0);

  double* d_slice_exp = p->d_scalars + 1;
  double* d_inv_exp = p->d_scalars + 2;
  double* d_slice_exp_t = p->d_scalars + 3;  // stripped forward mode: e'_s, without the root's factor
  double* d_tangent_exp = p->d_scalars + 4;  // ... and the tangent's running exponent Et
  // (stripped forward mode: the slot of the root's factor, kept out of e'_s; -1 for a single-operand root)
  const int root_slot = p->strip_exponent && p->jvp && p->nodes[p->root].kind == 0 ? p->nodes[p->root].c : -1;

  ctgb_slice_mem mem;
  mem.inputs = inputs;
  mem.grads = grads;
  mem.tangents = tangents;
  mem.tout = (char*)tangent_out;
  mem.persistent = persistent;
  mem.scratch = scratch;
  mem.out = (char*)out;
  mem.cot = (const char*)cotangent;
  mem.es = es;
  mem.out_es = elem_size(p->acc_dtype);
  mem.digits = digits.data();
  auto resolve = [&](int t, int64_t out_off) -> char* { return resolve_tensor(p->tensors[t], mem, out_off); };
  int rc;

  if (p->cot_offset >= 0) {
    // H of the root = conj(cotangent): conjugate a copy, the caller's tensor stays as it is
    char* copy = persistent + p->cot_offset;
    CUDA_TRY(cudaMemcpyAsync(copy, cotangent, (size_t)p->out_elements * es, cudaMemcpyDeviceToDevice, st));
    if ((rc = conj_inplace(p->dtype, copy, p->out_elements, st))) return rc;
    mem.cot = copy;
  }

  auto run_phase = [&](int phase, int64_t out_off) -> int {
    for (size_t ni = 0; ni < p->nodes.size(); ++ni) {
      const auto& n = p->nodes[ni];
      if (n.phase != phase) continue;
      if (n.is_root == 1 && p->jvp && !out) continue;  // forward mode without the primal
      if (p->profile) cudaEventRecord(p->ev0[ni], st);
      const int64_t* h = p->descs.data() + n.desc_off;
      const int64_t* d = p->d_descs + n.desc_off;
      char* A = resolve(n.a, out_off);
      char* B = n.kind != 1 ? resolve(n.b, out_off) : nullptr;  // (pairwise and two-term nodes)
      char* C = resolve(n.c, out_off);
      if (n.zero_fill) CUDA_TRY(cudaMemsetAsync(C, 0, (size_t)p->tensors[n.c].nbytes, st));
      // the whole underlying buffer of an operand (a sliced input, or the cotangent's slice view,
      // keeps its base offset into a copy)
      auto under = [&](const ctgb_plan::Tensor& t) -> char* {
        if (t.kind == 0) return (char*)inputs[t.input_index];
        if (t.kind == 7) return (char*)tangents[t.input_index];
        if (t.kind == 4) return (char*)mem.cot;
        return (t.kind == 1 ? scratch : persistent) + t.offset;
      };
      if (n.prescale_b) {
        // the small operand, scaled by 1/(fA fB) read from the factor slots on the device (a tangent
        // record right after its primal node may find that copy made already)
        const ctgb_plan::Tensor& tb = p->tensors[n.b];
        char* base = under(tb);
        if (!n.bscale_reuse) {
          if (int r = scale_copy(p->dtype, base, p->d_bscale, tb.nbytes / (int64_t)es, p->d_factors + n.fa,
                                 p->d_factors + n.fb, st))
            return r;
        }
        B = p->d_bscale + (B - base);
      }
      if (n.prescale_a) {
        const ctgb_plan::Tensor& ta = p->tensors[n.a];
        char* base = under(ta);
        const double* one = p->d_factors + p->tensors.size() + 1;
        if (int r = scale_copy(p->dtype, base, p->d_bscale, ta.nbytes / (int64_t)es, p->d_factors + n.fa,
                               n.fb >= 0 ? p->d_factors + n.fb : one, st))
          return r;
        A = p->d_bscale + (A - base);
      }
      if (n.kind == 2) {
        if (int r = launch_gett2(h, d, A, B, resolve(n.a2, out_off), resolve(n.b2, out_off), C, st)) return r;
      } else if (n.kind == 0 && h[W_VARIANT] == VAR_ABSORB_ROOT) {
        if (int r = launch_absorb_root(h, d, A, resolve((int)h[AB_BS_SLOT], out_off), B, C, st)) return r;
      } else if (int r = launch_node(n.kind, h, d, A, B, C, st)) {
        return r;
      }
      // contract.py:816-829 strips after every *pairwise* node (single-operand preprocessing
      // steps `continue` before reaching it, :792-796).  The kernels do it in their epilogues
      // (scale by the operands' factors, record max|C|: gett_kernels.cuh StripCtx); only nodes
      // that add partial sums atomically need max|C| measured in a pass of its own.
      if (n.measure_after) {
        if (int r = absmax_into(p->dtype, C, n.c_elems, (unsigned long long*)(p->d_factors + n.c), st)) return r;
      }
      if (p->profile) cudaEventRecord(p->ev1[ni], st);
    }
    return CTGB_OK;
  };

  // stripped forward mode: the tangent output holds the tangent relative to the entry exponent, so its
  // running exponent starts there
  const bool strip_jvp = p->strip_exponent && p->jvp;
  if (strip_jvp)
    CUDA_TRY(cudaMemcpyAsync(d_tangent_exp, exponent_dev, sizeof(double), cudaMemcpyDeviceToDevice, st));
  // slice-invariant subtrees: once per execute call, kept in the persistent arena
  if (p->strip_exponent && p->n_inv_slots > 0) {
    reset_slots_kernel<<<1, 256, 0, st>>>(p->d_factors, p->d_slot_lists + p->n_var_slots, p->n_inv_slots);
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  if ((rc = run_phase(0, 0))) return rc;
  if (p->strip_exponent) {
    // exponent of the slice-invariant part: sum of log10(factor) over the hoisted pairwise nodes
    sum_log_kernel<<<1, 256, 0, st>>>(p->d_factors, p->d_slot_lists + p->n_var_slots, p->n_inv_slots, d_inv_exp,
                                      nullptr);
    g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  // H accumulators of slice-invariant tensors collect every slice of the call
  for (const auto& q : p->tensors)
    if (q.kind == 6) CUDA_TRY(cudaMemsetAsync(persistent + q.offset, 0, (size_t)q.nbytes, st));

  for (int64_t k = 0; k < slice_count; ++k) {
    const int64_t out_off = decode_slice(slice_begin + k * slice_step, p->radix, p->project, p->out_stride, digits);
    if (p->strip_exponent && p->n_var_slots > 0) {
      reset_slots_kernel<<<1, 256, 0, st>>>(p->d_factors, p->d_slot_lists, p->n_var_slots);
      g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    if ((rc = run_phase(1, out_off))) return rc;
    if (p->strip_exponent) {
      sum_log_kernel<<<1, 256, 0, st>>>(p->d_factors, p->d_slot_lists, p->n_var_slots, d_slice_exp, d_inv_exp,
                                        p->jvp ? d_slice_exp_t : nullptr, root_slot);
      g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    if (p->strip_exponent && p->backward) {
      // the root is not run: d_slice_exp is the slice's exponent without the root's own factor, and
      // the backward steps next to the root divide by the seed 10^(e - e'_s)
      strip_seed_kernel<<<1, 1, 0, st>>>(p->d_factors + p->tensors.size(), exponent_dev, d_slice_exp);
      g_launches.fetch_add(1, std::memory_order_relaxed);
    }
    if ((rc = run_phase(2, out_off))) return rc;
    if (p->strip_exponent && !p->backward) {
      // the root wrote a dense mantissa into its workspace slot; fold it into the
      // output against the running exponent (core.py:163-170, 3856-3861)
      const ctgb_plan::Node& root = p->nodes[p->root];
      char* m = resolve(root.c, 0);
      // (the stored root is the raw product: its own factor divides it here)
      const double* froot = root.kind == 0 ? p->d_factors + root.c : nullptr;
      StripTangent tg;
      if (p->jvp) {
        // the raw tangent root, stored densely as the root is, follows into the tangent output
        tg.tout = tangent_out;
        tg.tchunk = (char*)tangent_out + out_off * (int64_t)mem.out_es;
        tg.tm = resolve(p->nodes[p->troot].c, 0);
        tg.Et = d_tangent_exp;
        tg.es_t = d_slice_exp_t;
      }
      rc = accum_stripped(p->dtype, wide, p->d_chunk_desc, p->chunk_desc.data(), out,
                          (char*)out + out_off * (int64_t)mem.out_es, p->out_elements, m, exponent_dev, d_slice_exp,
                          froot, tg, st);
      if (rc) return rc;
    }
    if (wide_fold && out) {
      rc = add_chunk_wide(p->dtype, p->d_chunk_desc, p->chunk_desc.data(), (char*)out + out_off * (int64_t)mem.out_es,
                          resolve(p->nodes[p->root].c, 0), st);
      if (rc) return rc;
    }
    if (wide_fold && p->troot >= 0) {
      // the root's tangent, stored densely as the root is, into its chunk of the tangent output
      rc = add_chunk_wide(p->dtype, p->d_chunk_desc, p->chunk_desc.data(),
                          (char*)tangent_out + out_off * (int64_t)mem.out_es, resolve(p->nodes[p->troot].c, 0), st);
      if (rc) return rc;
    }
  }
  if (strip_jvp && (rc = tangent_to_exponent(p->acc_dtype, tangent_out, p->out_elements, d_tangent_exp, exponent_dev, st)))
    return rc;
  // the invariant subtrees are differentiated once, from the accumulated H
  std::fill(digits.begin(), digits.end(), 0);
  if ((rc = run_phase(3, 0))) return rc;
  for (int i = 0; i < p->n_inputs; ++i)
    if (p->grad_elems[i] > 0 && (rc = conj_inplace(p->dtype, grads[i], p->grad_elems[i], st))) return rc;
  return CTGB_OK;
}

extern "C" {

int ctgb_plan_execute(ctgb_plan* p, const void* const* inputs, void* out, double* exponent_dev,
                      const void* cotangent, void* const* grads, void* workspace, size_t workspace_bytes,
                      int64_t slice_begin, int64_t slice_step, int64_t slice_count, void* stream) {
  if (!p) return fail(CTGB_E_VALUE, "null plan");
  if (p->jvp) return fail(CTGB_E_VALUE, "a forward-mode plan runs through ctgb_plan_execute_jvp");
  return plan_run(p, inputs, nullptr, out, nullptr, exponent_dev, cotangent, grads, workspace, workspace_bytes,
                  slice_begin, slice_step, slice_count, stream);
}

int ctgb_plan_execute_jvp(ctgb_plan* p, const void* const* inputs, const void* const* tangents, void* out,
                          void* tangent_out, void* workspace, size_t workspace_bytes, int64_t slice_begin,
                          int64_t slice_step, int64_t slice_count, void* stream) {
  if (!p) return fail(CTGB_E_VALUE, "null plan");
  if (!p->jvp) return fail(CTGB_E_VALUE, "not a forward-mode plan");
  return plan_run(p, inputs, tangents, out, tangent_out, nullptr, nullptr, nullptr, workspace, workspace_bytes,
                  slice_begin, slice_step, slice_count, stream);
}

int ctgb_plan_execute_jvp_stripped(ctgb_plan* p, const void* const* inputs, const void* const* tangents, void* out,
                                   void* tangent_out, double* exponent_dev, void* workspace, size_t workspace_bytes,
                                   int64_t slice_begin, int64_t slice_step, int64_t slice_count, void* stream) {
  if (!p) return fail(CTGB_E_VALUE, "null plan");
  if (!p->jvp || !p->strip_exponent) return fail(CTGB_E_VALUE, "not a stripped forward-mode plan");
  return plan_run(p, inputs, tangents, out, tangent_out, exponent_dev, nullptr, nullptr, workspace, workspace_bytes,
                  slice_begin, slice_step, slice_count, stream);
}

int ctgb_plan_execute_host(ctgb_plan* p, const void* const* host_inputs, const int64_t* input_nbytes, void* host_out,
                           double* host_exponent, void* workspace, size_t workspace_bytes, int64_t slice_begin,
                           int64_t slice_step, int64_t slice_count, void* stream) {
  if (!p) return fail(CTGB_E_VALUE, "null plan");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t es = elem_size(p->acc_dtype);  // (of the output: the inputs come with their byte counts)
  const size_t core = (size_t)(p->workspace_bytes + p->persistent_bytes);
  // staging area at the tail of the workspace: inputs, output, exponent
  size_t need = core;
  auto align = [](size_t x) { return (x + 255) & ~(size_t)255; };
  need = align(need);
  std::vector<size_t> in_off(p->n_inputs);
  for (int i = 0; i < p->n_inputs; ++i) {
    in_off[i] = need;
    need = align(need + (size_t)input_nbytes[i]);
  }
  const size_t out_off = need;
  need = align(need + (size_t)p->out_elements * es);
  const size_t exp_off = need;
  need += 256;
  if (workspace_bytes < need) return fail(CTGB_E_MEMORY, "workspace too small for host staging");
  char* ws = (char*)workspace;
  std::vector<const void*> dev_inputs(p->n_inputs);
  // ONE host->device copy for all inputs (a Sycamore network has 381 tensors of 16-256 bytes:
  // 381 separate copies cost more than the bytes): pack them into the plan's pinned staging
  // block at their device offsets, then copy the block
  const size_t in_base = p->n_inputs ? in_off[0] : out_off, in_span = out_off - in_base;
  if (in_span <= ((size_t)64 << 20)) {
    if (p->h_stage_bytes < in_span) {
      if (p->h_stage) cudaFreeHost(p->h_stage);
      p->h_stage = nullptr;
      p->h_stage_bytes = 0;
      CUDA_TRY(cudaHostAlloc((void**)&p->h_stage, in_span ? in_span : 1, cudaHostAllocDefault));
      p->h_stage_bytes = in_span;
    } else {
      // the previous call's copy out of this block has completed (each call ends synchronised)
    }
    for (int i = 0; i < p->n_inputs; ++i) {
      memcpy(p->h_stage + (in_off[i] - in_base), host_inputs[i], (size_t)input_nbytes[i]);
      dev_inputs[i] = ws + in_off[i];
    }
    if (in_span) CUDA_TRY(cudaMemcpyAsync(ws + in_base, p->h_stage, in_span, cudaMemcpyHostToDevice, st));
  } else {
    for (int i = 0; i < p->n_inputs; ++i) {
      CUDA_TRY(cudaMemcpyAsync(ws + in_off[i], host_inputs[i], (size_t)input_nbytes[i], cudaMemcpyHostToDevice, st));
      dev_inputs[i] = ws + in_off[i];
    }
  }
  CUDA_TRY(cudaMemsetAsync(ws + out_off, 0, (size_t)p->out_elements * es, st));
  double* d_exp = (double*)(ws + exp_off);
  if (p->strip_exponent) {
    // running exponent starts at -inf so that the first slice sets it
    const double ninf = -__builtin_huge_val();
    CUDA_TRY(cudaMemcpyAsync(d_exp, &ninf, sizeof(double), cudaMemcpyHostToDevice, st));
  }
  int rc = ctgb_plan_execute(p, dev_inputs.data(), ws + out_off, d_exp, nullptr, nullptr, workspace, core, slice_begin,
                             slice_step, slice_count, stream);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(host_out, ws + out_off, (size_t)p->out_elements * es, cudaMemcpyDeviceToHost, st));
  if (p->strip_exponent && host_exponent)
    CUDA_TRY(cudaMemcpyAsync(host_exponent, d_exp, sizeof(double), cudaMemcpyDeviceToHost, st));
  CUDA_TRY(cudaStreamSynchronize(st));
  return CTGB_OK;
}

}  // extern "C"

