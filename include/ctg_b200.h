/*
 * ctg_b200.h -- C-ABI of the B200-native sliced contraction-tree executor.
 *
 * This is the drop-in boundary for cotengra's execution path.  cotengra is pure
 * Python and has no FFI of its own; these entry points are what a binding for
 * that path would call (see INTEGRATION.md for the ctypes stub and the three
 * lines that install it through cotengra's `implementation=` hook).
 *
 * Reference interfaces replaced (paths relative to jcmgray/cotengra @ 2182a79):
 *
 *   ctgb_contract_pair ....... cotengra/contract.py:414 `einsum(eq, a, b)` and
 *                              :521 `tensordot(a, b, axes)` -- one pairwise node,
 *                              lowered there to transpose+reshape -> matmul
 *                              (:364-411); here ONE kernel launch with the index
 *                              permutations folded into the tile loads/stores.
 *   ctgb_reduce_single ....... cotengra/contract.py:332 `_einsum_single` (diag /
 *                              sum / transpose of one operand; preprocessing
 *                              steps :792-796 and single-input trees :797-803).
 *   ctgb_plan_create/execute . cotengra/contract.py:654-837 `Contractor.__call__`
 *                              (the node loop, strip_exponent :816-829) together
 *                              with cotengra/core.py:3943-4030
 *                              `ContractionTree.contract` (slice loop),
 *                              :3775-3819 `slice_key`/`slice_arrays` and
 *                              :3825-3882 `gather_slices` (sum / stack);
 *                              slice_begin/slice_step reproduce the round-robin
 *                              of `contract_mpi` (core.py:4070).
 *
 * Conventions
 *   - All tensors are dense arrays addressed as base + sum(digit * stride), with
 *     strides in ELEMENTS; the caller (host side, cotengra_b200/lowering.py)
 *     turns index labels into strides, so transposes, diagonals (summed strides),
 *     broadcasts (stride 0) and slicing (base offsets) need no data movement.
 *   - Device buffers and the CUDA stream are owned by the caller; the library
 *     owns only immutable plans (plus a small internal descriptor arena).
 *   - Every function returns 0 on success or a CTGB_E_* code; the message is
 *     available from ctgb_last_error() (thread local).
 *   - No CPU fallback exists: without a CUDA device every compute entry point
 *     fails with CTGB_E_CUDA.
 */
#ifndef CTG_B200_H
#define CTG_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define CTGB_ABI_VERSION 2

/* element types (output dtype == input dtype, no casting on the path:
 * cotengra/contract.py has none either) */
enum {
  CTGB_F32 = 0,
  CTGB_F64 = 1,
  CTGB_C64 = 2,
  CTGB_C128 = 3
};

/* status codes; mapped by the Python host to the exceptions the reference raises */
enum {
  CTGB_OK = 0,
  CTGB_E_VALUE = 1,    /* -> ValueError   (bad shapes / descriptor)          */
  CTGB_E_NOTIMPL = 2,  /* -> NotImplementedError                             */
  CTGB_E_CUDA = 3,     /* -> RuntimeError (CUDA failure, or no device)       */
  CTGB_E_MEMORY = 4    /* -> MemoryError  (workspace too small)              */
};

/* Number of int64 words in one pairwise-contraction descriptor.  The word
 * layout is defined in cotengra_b200/csrc/gett_desc.h and mirrored by
 * cotengra_b200/lowering.py (checked at import through ctgb_desc_words()). */
int ctgb_abi_version(void);
int ctgb_desc_words(void);
int ctgb_single_desc_words(void);
const char* ctgb_last_error(void);

/* Device properties the host-side planner sizes grids with. */
int ctgb_device_info(int* sm_count, int* cc_major, int* cc_minor,
                     size_t* smem_optin_bytes);

/* One pairwise node: C = sum_k A * B with arbitrary index placement.
 * `desc` is a host array of ctgb_desc_words() int64 words.  A, B, C are device
 * pointers; `stream` is a cudaStream_t (0 = default stream). */
int ctgb_contract_pair(const int64_t* desc, const void* A, const void* B,
                       void* C, void* stream);

/* The two-term form of one pairwise node: C (+)= A.B + A2.B2 in one launch, where
 * A2 has A's index structure and strides and B2 has B's, so the same descriptor
 * describes both products and C is stored once (accumulated when the descriptor
 * says so).  Runs on the row-stream and DMMA stream kernels (variants 8, 19 and
 * 14).  A descriptor with both scale words (W_SCALE_A, W_SCALE_B: device doubles
 * fA, fB) forms C (+)= (A.B + A2.B2) / (fA fB), a zero factor scaling by 0; one
 * with a factor slot of C (W_FACTOR_C), one scale word alone, a wide C or any
 * other variant fails with CTGB_E_VALUE before any launch.
 * The DMMA stream kernel's two-term form takes K <= 64 for N <= 16, K <= 32 for
 * N <= 32 and K <= 16 beyond. */
int ctgb_contract_pair2(const int64_t* desc, const void* A, const void* B,
                        const void* A2, const void* B2, void* C, void* stream);

/* One absorb-root node (variant 21, complex128):
 * C[m,n] (+)= sum_{k',c} (sum_k A[m,k',k] Bs[k,c]) V[k',c,n], the result of the
 * absorption A.Bs never formed.  `desc` is a pair-sized word array in the
 * absorb-root layout (cotengra_b200/csrc/gett_desc.h). */
int ctgb_absorb_root(const int64_t* desc, const void* A, const void* Bs,
                     const void* V, void* C, void* stream);

/* One single-operand node: out = diag/sum/transpose of X. */
int ctgb_reduce_single(const int64_t* desc, const void* X, void* out,
                       void* stream);

/* ---- whole-tree plans ---------------------------------------------------- */

typedef struct ctgb_plan ctgb_plan;

/* A tensor slot of the plan.  kind:
 *   0 = network input `input_index` (device pointer supplied at execute time;
 *       for sliced inputs the per-slice element offset is
 *       sum(digit[slice_pos[j]] * slice_stride[j])),
 *   1 = per-slice workspace at byte offset `offset`,
 *   2 = persistent (slice-invariant) workspace at byte offset `offset`,
 *   3 = the output accumulator (at the slice's output view, slice_out_stride),
 *   4 = the cotangent's view of the slice (element offset as kind 3),
 *   5 = the gradient of network input `input_index` (slice offset as kind 0),
 *   6 = a persistent accumulator at byte offset `offset` of the persistent
 *       arena, zeroed before the slice loop (H of a slice-invariant tensor),
 *   7 = the tangent of network input `input_index` (slice offset as kind 0),
 *   8 = the tangent output accumulator (at the slice's view, as kind 3).
 * Kinds 4-6 belong to reverse-mode plans, kind 3 to forward ones, and kinds 7-8
 * to forward-mode plans (ctgb_plan_execute_jvp), which may also hold kind 3. */
typedef struct {
  int32_t kind;
  int32_t input_index;
  int64_t offset;
  int64_t nbytes;
  int32_t n_sliced;         /* sliced indices carried by this input      */
  const int32_t* slice_pos; /* position in the plan's slice-digit list   */
  const int64_t* slice_stride;
} ctgb_tensor;

/* A node of the linear program (cotengra/contract.py:573-651 IR, lowered).
 * A forward plan has phases 0 and 1 only.  A reverse-mode plan propagates
 * H = conj(cotangent) from the root to the inputs through phases 2 and 3; every
 * backward step is an ordinary pairwise or single-operand descriptor.  Phase 2
 * may also hold forward nodes: a plan under a workspace budget recomputes
 * per-slice values there, right before the backward steps that read them.
 * Each phase runs its nodes in list order, so this needs nothing new here. */
typedef struct {
  int32_t kind;       /* 0 = pairwise (desc = pair words), 1 = single-operand,
                         2 = two-term pairwise (desc = pair words followed by the
                         slots of A2 and B2: ctgb_contract_pair2's form)        */
  int32_t a, b, c;    /* tensor slots (b unused for kind 1)                     */
  int32_t phase;      /* 0 invariant forward (once), 1 variant forward, 2 variant
                         backward (per slice), 3 invariant backward (once, last) */
  int32_t zero_fill;  /* 1: zero tensor c (nbytes) before the launch           */
  int32_t is_root;    /* 1: writes the output (accumulated over slices); 2: writes
                         the tangent of the output (forward-mode plans)         */
  const int64_t* desc;
} ctgb_node;

typedef struct {
  int32_t dtype;
  int32_t n_inputs;
  int32_t n_tensors;
  const ctgb_tensor* tensors;
  int32_t n_nodes;
  const ctgb_node* nodes;
  /* slicing: mixed-radix digits, most significant first, exactly
   * cotengra/core.py:114-122 + 3775-3800; radix 1 + project >= 0 encodes a
   * projected index (it consumes no digit of the slice id). */
  int32_t n_sliced;
  const int64_t* slice_radix;
  const int64_t* slice_project; /* -1 = sliced normally */
  /* the root's output view: element offset into `out` contributed by the
   * digits of sliced indices that are also OUTPUT indices (gather_slices'
   * stack, core.py:3865-3876); 0 stride for inner sliced indices. */
  const int64_t* slice_out_stride;
  int64_t out_elements;       /* elements of the full output (or cotangent)  */
  int64_t workspace_bytes;    /* per-slice arena                              */
  int64_t persistent_bytes;   /* arena kept over the whole call               */
  int32_t strip_exponent;     /* contract.py:816-829 semantics (reverse mode:
                                 ctgb_plan_set_scale_slots)                   */
  int64_t cotangent_offset;   /* complex reverse-mode plans: byte offset of the
                                 conjugated cotangent copy in the persistent
                                 arena; -1 = no copy                          */
} ctgb_plan_desc;

/* strip_exponent together with phase 2/3 nodes makes a stripped reverse-mode
 * plan, which runs only after ctgb_plan_set_scale_slots; together with tangent
 * slots (kinds 7, 8) a stripped forward-mode plan, which runs only after
 * ctgb_plan_set_tangent_scale_slots. */
int ctgb_plan_create(const ctgb_plan_desc* desc, ctgb_plan** plan);
/* strip_exponent plans, and plans with a wide accumulator whose root is not a
 * dot-stream node: the single-operand descriptor (ctgb_single_desc_words()
 * words) that maps the dense root result of one slice onto its chunk of the
 * output tensor (identity layout when no sliced index is an output index). */
int ctgb_plan_set_chunk_desc(ctgb_plan* plan, const int64_t* desc);
/* Stripped reverse-mode plans, once before the first execute: the factor slots
 * each of the n (= n_nodes) nodes divides its product by, in desc->nodes order.
 * A slot is a tensor slot index, whose factor is max|value| for a pairwise
 * result formed in phase 0 or 1 and 1.0 otherwise, or n_tensors: the root's
 * seed 10^(e - e'_s), formed per slice after phase 1 from the forward's exponent
 * e and the slice's exponent e'_s without the root's factor.  A pairwise node
 * divides by slot_a[i] * slot_b[i] (its descriptor's A and B operands); a
 * single-operand node by slot_a[i] * slot_b[i] when slot_a[i] >= 0, a missing
 * slot_b (-1) counting as 1.0, and not at all when slot_a[i] is -1.  Phase 0/1
 * pairwise nodes record max|C| in slot c as in a forward plan; phase 2/3 nodes
 * record nothing.  The gradient is that of m = amp * 10^-e with e held constant. */
int ctgb_plan_set_scale_slots(ctgb_plan* plan, const int32_t* slot_a,
                              const int32_t* slot_b, int n);
/* Stripped forward-mode plans, once before the first execute: tangent[i] = 1 marks
 * the tangent records among the n (= n_nodes) nodes.  A primal record (0) is the
 * forward plan's node and divides by its own operands' factors (slot_a[i], slot_b[i]
 * = its a and b; -1, -1 for a single-operand node).  A pairwise or two-term tangent
 * record divides by the two tensor slots named (its primal node's operands) and
 * records no factor: T_p = (T_l S_r + S_l T_r) / (f_l f_r), the scale of the primal
 * value S_p, so that tangents of intermediates are never normalised on their own. */
int ctgb_plan_set_tangent_scale_slots(ctgb_plan* plan, const int32_t* slot_a,
                                      const int32_t* slot_b,
                                      const int32_t* tangent, int n);
/* Forward plans, once after ctgb_plan_create: the dtype of the output accumulator,
 * the plan's dtype (the default) or its double counterpart (CTGB_F64 for CTGB_F32,
 * CTGB_C128 for CTGB_C64); anything else fails with CTGB_E_VALUE.  With the double
 * counterpart every slice is added to `out` in double precision.  The root of such a
 * plan is either a dot-stream node whose descriptor has flags bit 8 set (C is the
 * wide type: the kernel forms products and sums in double and adds them into the
 * output tensor slot, kind 3), or any other node that stores its slice densely in a
 * workspace slot (kind 1) in the plan dtype; ctgb_plan_set_chunk_desc then maps that
 * slot onto its chunk of the output, one extra launch per slice.  With
 * strip_exponent the mantissa of a slice stays in the plan dtype and the running
 * mantissa in `out` is double. */
int ctgb_plan_set_accumulator(ctgb_plan* plan, int32_t dtype);
void ctgb_plan_destroy(ctgb_plan* plan);
size_t ctgb_plan_workspace_bytes(const ctgb_plan* plan);
int64_t ctgb_plan_launches_per_slice(const ctgb_plan* plan);
/* strip_exponent plans: how each node (in desc->nodes order, n entries) applies the 1/(fA fB) of its
 * operands' factors.  prescale_b[i] = 1: a scaled copy of the B operand is made first (operands of at
 * most 16 MiB); 0: the kernel's epilogue multiplies (and may take the float, double or two-factor
 * route); -1: a single-operand node.  measure_after[i] = 1: max|C| is measured by a pass after the
 * launch (split-K, dot-type, KRED and chunked wgmma nodes). */
int ctgb_plan_strip_modes(const ctgb_plan* plan, int32_t* prescale_b, int32_t* measure_after, int n);

/* Run slices slice_begin, slice_begin + slice_step, ... (slice_count of them).
 * `inputs` is a host array of n_inputs DEVICE pointers to the unsliced,
 * C-contiguous input arrays.  `workspace` must hold ctgb_plan_workspace_bytes()
 * bytes.  A smaller one fails with CTGB_E_MEMORY, and a missing buffer the plan
 * needs with CTGB_E_VALUE, before any launch.
 *
 * A forward plan ACCUMULATES the slices' contributions into `out` (device,
 * out_elements of the accumulator dtype -- the plan dtype unless
 * ctgb_plan_set_accumulator chose its double counterpart; the caller zeroes it
 * before the first call).
 * With strip_exponent the mantissa is accumulated against the running base-10
 * exponent stored in exponent_dev[0] (device double; core.py:163-170).
 * `cotangent` and `grads` may be null.
 *
 * A reverse-mode plan forms the input gradients of the sum of the slices for
 * the output cotangent `cotangent` (device, out_elements).  `grads` is a host
 * array of n_inputs device pointers, null for inputs that are not
 * differentiated; the caller zeroes the buffers (the final conjugation of
 * complex gradients acts on the whole buffer), and on return they hold the
 * finished gradients in torch's convention (grad_x = sum over outputs of
 * grad_out * conj(d out / d x)).  `out` may be null, and so may `exponent_dev`
 * except for a stripped plan, which reads from it the exponent e of the forward
 * result (m, e) whose mantissa's cotangent `cotangent` is.
 *
 * Order: conjugated cotangent copy; phase 0; H accumulators zeroed; per slice
 * phases 1 and 2 (and the stripped accumulation); phase 3; conjugated
 * gradients.  Asynchronous on `stream`. */
int ctgb_plan_execute(ctgb_plan* plan, const void* const* inputs, void* out,
                      double* exponent_dev, const void* cotangent,
                      void* const* grads, void* workspace,
                      size_t workspace_bytes, int64_t slice_begin,
                      int64_t slice_step, int64_t slice_count, void* stream);

/* Forward mode: a plan with tangent slots (kinds 7, 8) forms, for the slices
 * slice_begin, slice_begin + slice_step, ... (slice_count of them), the tangent
 * of the sum of the slices for the input tangents `tangents` (a host array of
 * n_inputs device pointers laid out as the inputs, null for inputs the plan does
 * not differentiate) and accumulates it into `tangent_out` (device, out_elements
 * of the accumulator dtype, zeroed by the caller).  `out` receives the primal
 * result as ctgb_plan_execute does; it may be null, and the primal root is then
 * not run.  The workspace rules are ctgb_plan_execute's.  Asynchronous. */
int ctgb_plan_execute_jvp(ctgb_plan* plan, const void* const* inputs,
                          const void* const* tangents, void* out,
                          void* tangent_out, void* workspace,
                          size_t workspace_bytes, int64_t slice_begin,
                          int64_t slice_step, int64_t slice_count,
                          void* stream);
/* Forward mode of a strip_exponent plan: `out` and exponent_dev[0] receive the
 * stripped result (m, e) as ctgb_plan_execute does (neither may be null: the
 * primal root always runs, its factor sets each slice's exponent), and
 * `tangent_out` the tangent of the mantissa with the exponent held constant,
 * dm = 10^-e d(amp); on entry `tangent_out` holds a tangent relative to
 * exponent_dev[0] as `out` does (zeros with -inf).  The root's raw tangent is
 * folded against a running exponent of its own, Et' = max(Et, e'_s):
 * tout = tout 10^(Et - Et') + T_s 10^(e'_s - Et'), e'_s being the slice's
 * exponent without the root's factor, and one launch after the slices brings
 * tout to the final e.  So a slice whose amplitude is exactly zero keeps its
 * tangent in any slice order.  A slice with a zero factor below its root adds
 * nothing; a zero result (e = -inf) gives a zero tangent; a NaN exponent, NaN. */
int ctgb_plan_execute_jvp_stripped(ctgb_plan* plan, const void* const* inputs,
                                   const void* const* tangents, void* out,
                                   void* tangent_out, double* exponent_dev,
                                   void* workspace, size_t workspace_bytes,
                                   int64_t slice_begin, int64_t slice_step,
                                   int64_t slice_count, void* stream);

/* Same job for a forward plan with HOST buffers: copies the inputs
 * host->device, runs the slices, copies the accumulated output (out_elements of the
 * accumulator dtype) and the exponent back, synchronises.  This is the end-to-end call bench.py times as `e2e`.  `workspace` stays a device buffer
 * (it is scratch); input staging memory is taken from its tail. */
int ctgb_plan_execute_host(ctgb_plan* plan, const void* const* host_inputs,
                           const int64_t* input_nbytes, void* host_out,
                           double* host_exponent, void* workspace,
                           size_t workspace_bytes, int64_t slice_begin,
                           int64_t slice_step, int64_t slice_count,
                           void* stream);

/* Per-node device timing for roofline reporting: when enabled, CUDA events are
 * recorded on the execute stream around every node; ctgb_plan_profile_read
 * synchronises and returns the milliseconds of each of the plan's n_nodes
 * nodes for the LAST slice executed (-1 for nodes that did not run). */
int ctgb_plan_profile(ctgb_plan* plan, int enable);
int ctgb_plan_profile_read(ctgb_plan* plan, float* ms, int n_nodes);

/* Measured fp64 tensor-core (DMMA m16n8k4) and fp64 FMA peaks of the current
 * device in TFLOP/s, from a register-resident microbenchmark kernel: the
 * denominators bench.py uses for the fp64 roofline (MEASURED_PEAKS.json holds
 * only HBM and bf16 numbers). */
int ctgb_probe_fp64_peaks(double* dmma_tflops, double* dfma_tflops, void* stream);

/* Number of kernels this library has launched since load (bench.py's
 * `gpu_launches`). */
int64_t ctgb_launch_count(void);
/* ... of which wgmma launches whose A tiles are fetched by tensor-map TMA (cp.async.bulk.tensor). */
int64_t ctgb_tensor_map_launches(void);

/* The launch-time choices ctgb_contract_pair makes for a wgmma (complex64) descriptor whose A
 * operand starts at device address a_addr, on a device with `sms` SMs and `smem_optin` bytes of
 * opt-in shared memory per block.  Touches no device.  Writes n_out >= 9 words:
 *   out[0] 1: B' resident (one slot per k-step, loaded once per CTA), 0: a B' ring
 *   out[1] B' slots           out[2] A staging depth
 *   out[3] CTAs (0: nothing to launch)
 *   out[4] dynamic shared memory of one CTA, bytes
 *   out[5] rank of the A tensor map (2..5), 0: no tensor map
 *   out[6] 1: A fetched as contiguous runs by bulk copies (when out[5] is 0)
 *   out[7] k-steps per register accumulation
 *   out[8] accumulations (chunks) of the longest contracted range of one work item
 * A descriptor the kernel does not take fails as ctgb_contract_pair would. */
int ctgb_tc05_launch_config(const int64_t* words, uint64_t a_addr, int sms,
                            uint64_t smem_optin, int64_t* out, int n_out);

/* The instantiation and grid ctgb_contract_pair launches for a DMMA stream (complex128)
 * descriptor on a device with `sms` SMs.  Touches no device.  Writes n_out >= 3 words:
 *   out[0] column fragments of 8 (N <= 8*out[0])
 *   out[1] rows of one warp block (32, or 16 for N > 32)
 *   out[2] CTAs (0: nothing to launch)
 * A descriptor the kernel does not take fails as ctgb_contract_pair would. */
int ctgb_dmmastream_launch_config(const int64_t* words, int sms, int64_t* out, int n_out);

#ifdef __cplusplus
}
#endif
#endif /* CTG_B200_H */
