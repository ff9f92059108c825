// gett_desc.h -- word layout of a pairwise-contraction ("GETT") descriptor.
//
// A descriptor is a flat array of int64 words produced on the host by
// cotengra_b200/lowering.py and consumed by the kernels in gett_kernels.cuh.
// It describes  C[b,m,n] (+)= sum_k A[b,m,k] * B[b,k,n]  where every one of the
// four index classes (cotengra/contract.py:226-243: bat / a_keep / b_keep / con)
// is a LIST of dims, each with its own stride in A, B and C, so that no operand
// is ever permuted in memory (the reference materialises the permutation at
// contract.py:380-396).
//
// Each class is split by the host into TILE dims (iterated inside a CTA tile;
// local index = sum digit_j * w_j, dim 0 fastest, an optional PARTIAL dim last)
// and GRID dims (iterated across tiles / k-steps).
#pragma once
#include <stdint.h>

namespace ctgb {

constexpr int MAX_T = 12;   // tile dims per class
constexpr int MAX_G = 40;   // grid dims per class
constexpr int MAX_GB = 12;  // batch grid dims
constexpr int MAX_LD = 24;  // tile dims of one operand (= MAX_T * 2)

enum : int {
  W_MAGIC = 0,
  W_DTYPE = 1,
  W_NTM = 2, W_NTN = 3, W_NTK = 4,
  W_NGM = 5, W_NGN = 6, W_NGK = 7, W_NGB = 8,
  W_MTA = 9, W_NTA = 10, W_KTA = 11,          // actual tile sizes
  W_TILES_M = 12, W_TILES_N = 13, W_TILES_B = 14, W_STEPS_K = 15,
  W_SPLITK = 16,
  // partial (blocked) dim of each class: index into the GRID list of the block
  // counter (-1: none), full extent, tile extent, weight of the partial dim in
  // the local index (valid local indices are < w * min(text, full - blk*text))
  W_PGM = 17, W_MFULL = 18, W_MTEXT = 19, W_MW = 20,
  W_PGN = 21, W_NFULL = 22, W_NTEXT = 23, W_NW = 24,
  W_PGK = 25, W_KFULL = 26, W_KTEXT = 27, W_KW = 28,
  W_NLDA = 29, W_NLDB = 30,
  W_FLAGS = 31,        // bit0: accumulate into C; bit1: column pairs adjacent+aligned in C;
                       // bit2: tile-grid extents are powers of two; bit3: all m dims are powers of two;
                       // bit4/5: column quads/pairs of 8-byte elements adjacent+aligned in C;
                       // bit6: wgmma A tile made of contiguous runs; bit7: float32/complex64
                       // tensor-core variants run ONE round-to-nearest tf32 pass (precision="tf32");
                       // bit8: C is the wide type (double / complex128 for float32 / complex64) and the
                       // sums are formed in it -- dot-stream roots of accumulate="double" plans only
  W_VARIANT = 32,      // kernel variant chosen by the host
  W_CELEMS = 33,       // elements of a dense C (memset before split-K atomics); 0: strided C
  W_RUNA = 34,         // wgmma: elements of the contiguous runs the A tile is made of (flags bit6)
  W_LBOPAD = 35,       // wgmma: chunk-stride padding of the A' images, x16 bytes (bank spreading)
  // fused strip_exponent (contract.py:816-829), patched into the plan's device copy of the
  // descriptor by ctgb_plan_create; 0 = off.  Device addresses of doubles:
  W_SCALE_A = 36,      //   max|A| of operand A as stored (A is a lazily-normalised intermediate) or 1.0
  W_SCALE_B = 37,      //   same for B; the epilogue multiplies by 1/(fA*fB)
  W_FACTOR_C = 38,     //   slot receiving max|product| of this launch, as scaled (atomicMax of the double's bits);
                       //   an accumulating launch adds C0 after it is measured, so it is max|C| only without C0
  W_HDR = 40,
  // arrays
  OFF_TM = W_HDR,                 // MAX_T x (ext, sA, sC)
  OFF_TN = OFF_TM + MAX_T * 3,    // MAX_T x (ext, sB, sC)
  OFF_TK = OFF_TN + MAX_T * 3,    // MAX_T x (ext, sA, sB)
  OFF_GM = OFF_TK + MAX_T * 3,    // MAX_G x (ext, div, sA, sC)
  OFF_GN = OFF_GM + MAX_G * 4,    // MAX_G x (ext, div, sB, sC)
  OFF_GK = OFF_GN + MAX_G * 4,    // MAX_G x (ext, div, sA, sB)
  OFF_GB = OFF_GK + MAX_G * 4,    // MAX_GB x (ext, div, sA, sB, sC)
  OFF_LDA = OFF_GB + MAX_GB * 5,  // MAX_LD x (ext, sA, w_r, w_k)  A-memory order
  OFF_LDB = OFF_LDA + MAX_LD * 4, // MAX_LD x (ext, sB, w_k, w_c)  B-memory order
  DESC_WORDS = OFF_LDB + MAX_LD * 4
};

constexpr int64_t DESC_MAGIC = 0x43544742'32303031LL;  // "CTGB2001"

// kernel variants (W_VARIANT)
enum : int {
  VAR_SIMT_64x64 = 0,  // generic FMA tile kernel, any dtype / any extents
  VAR_KRED = 1,        // tiny M x N, huge K: per-thread k partial sums
  VAR_DMMA_128x64 = 2, // fp64 tensor-core (mma.sync m16n8k4) tile kernel
  VAR_DMMA_64x128 = 3,
  VAR_DMMA_256x32 = 4,
  VAR_DMMA_256x16 = 5,
  VAR_ROW_128x8 = 6,   // one output row per thread (HBM-bound skinny nodes), N <= 8
  VAR_ROW_256x4 = 7,   // same, N <= 4 (fewer registers -> more resident CTAs)
  VAR_ROWSTREAM = 8,   // N, K <= 8, exact tiles, no batch: thread-per-row straight from global memory
  VAR_TC05_128x64 = 9, // complex64, exact 128 x 64 x 16 tiles: wgmma tf32 (3 passes), register accumulators
  VAR_TC05_128x32 = 10,
  VAR_TC05_128x16 = 11,
  VAR_DMMA3M_128x32 = 12,  // complex128, 3M complex product (three DMMAs per fragment pair)
  VAR_DMMA3M_256x16 = 13,
  VAR_DOTSTREAM = 15,      // M = N = 1: the final inner product, operands straight from global memory
  VAR_DMMASTREAM = 14,     // complex128, N <= 32 with K <= 64, N <= 64 with K <= 32: DMMA fragments straight from global memory
  VAR_DOTSTREAM4 = 16,     // M, N <= 4 over a huge contracted range: a peeled stem tail times the other stem
  // (17: a DMMA-fragments-from-global variant of the next one, measured slower -- 11.1 vs 10.1 ms on
  //  the M = N = 32, K = 2^25 node -- and removed)
  VAR_ROWSTREAM_K = 19,    // N <= 8, 8 < K <= 64, 8-byte and narrower types: the row stream in chunks of 8 k
  VAR_DMMA_32x32 = 18,     // fp64 DMMA, one 32 x 32 tile with split-K over all SMs, two CTAs per SM: a few
                           // peeled stem tails times the other stem (M, N <= 32 over K ~ 2^25)
  VAR_TF32_32x32 = 20,     // its float32 / complex64 counterpart (3xTF32 mma.sync); chosen by VJP plans only,
                           // for the small-result backward nodes of stem absorptions
  VAR_ABSORB_ROOT = 21     // complex128: a stem absorption X = A.Bs folded into the DMMA_32x32 product R = X.V
                           // that is X's only reader (absorbdot.cuh); three operands, its own word layout below
};

// ---- absorb-root descriptor (VAR_ABSORB_ROOT) --------------------------------
// R[m,n] (+)= sum_{k',c} (sum_k A[m,k',k] Bs[k,c]) V[k',c,n].  Same size and magic as a pair
// descriptor; W_DTYPE, W_FLAGS (bit0: accumulate into C), W_VARIANT and W_CELEMS keep their meaning.
constexpr int AB_MAXG = 32;  // grid k' dims (one lane each)
enum : int {
  AB_M = 2, AB_N = 3, AB_K = 4, AB_C = 5,  // row slots, N <= 32, K <= 16, contracted c (CC)
  AB_KL = 6,                               // extent of the tile k' dim (1 or 2)
  AB_NG = 7,                               // grid k' dims
  AB_UNITS = 8,                            // k' units (product of the grid extents)
  AB_KLA = 9, AB_KLV = 10,                 // strides of the tile k' dim in A and V
  AB_GRID = 11,                            // CTAs (units split evenly among them)
  AB_BS_SLOT = 12,                         // in a plan: the tensor slot of Bs (the node's a, b, c are A, V, C)
  AB_CCP = 13,                             // CC rounded up to 32; Bs column of (ck, cc) is ck * CCP + cc, <= 128
  // R's row r = mb * 8 + g (8-row block mb) is an A row and a kept column ck(mb) of Bs (one per block)
  AB_TMA = W_HDR,             // 32: A offset of row r      AB_TMC: C offset of row r (-1: no row)
  AB_TMC = AB_TMA + 32,
  AB_TNV = AB_TMC + 32,       // 32: V offset of column n   AB_TNC: C offset of column n
  AB_TNC = AB_TNV + 32,
  AB_TKA = AB_TNC + 32,       // 16: A offset of k          AB_TKB: Bs offset of k
  AB_TKB = AB_TKA + 16,
  AB_TCB = AB_TKB + 16,       // 128: Bs offset of column ck * CCP + cc (-1: none)   AB_TCV: V offset of cc
  AB_TCV = AB_TCB + 128,
  AB_G = AB_TCV + 128,        // AB_MAXG x (ext, div, sA, sV), unit digit = u / div % ext
  AB_TBCK = AB_G + AB_MAXG * 4,  // 4: ck of row block mb
  AB_WORDS = AB_TBCK + 4
};
static_assert(AB_WORDS <= DESC_WORDS, "absorb-root words fit a pair descriptor");

// ---- single-operand descriptor (cotengra/contract.py:332-361) -------------
// out[o] = sum_s X[off_o(o) + off_s(s)], out written at its own strides.
constexpr int MAX_S = 40;
enum : int {
  S_MAGIC = 0, S_DTYPE = 1, S_NO = 2, S_NS = 3, S_OUT_ELEMS = 4, S_SUM_ELEMS = 5,
  S_FLAGS = 6,
  S_HDR = 8,
  OFF_SO = S_HDR,                 // MAX_S x (ext, sX, sOut)
  OFF_SS = OFF_SO + MAX_S * 3,    // MAX_S x (ext, sX)
  SDESC_WORDS = OFF_SS + MAX_S * 2
};
constexpr int64_t SDESC_MAGIC = 0x43544742'53303031LL;

}  // namespace ctgb
