/*
 * exl3b200 -- Hopper-native (sm_90a) EXL3 quantized-GEMM path, C ABI.
 *
 * Drop-in boundary for the hot path of turboderp-org/exllamav3 (reference paths are relative to the
 * exllamav3 package directory of its checkout).  Every entry point replaces one pybind11 binding of the reference's
 * `exllamav3_ext` module; the reference-side shim a maintainer would add is shown in INTEGRATION.md and is
 * implemented in exllamav3_b200/ext.py (ctypes).
 *
 * Conventions
 *   - plain pointers and sizes only: no torch / ATen types cross this boundary.
 *   - every `const void*` / `void*` tensor argument is a DEVICE pointer on the current CUDA device unless the
 *     name ends in `_host`.  `stream` is a `cudaStream_t` passed as `void*` (NULL = legacy default stream).
 *   - the caller owns all buffers.  The library allocates its per-device scratch (split-K partials, tile counters,
 *     transformed-activation buffers for in_features <= 65536) with cudaMalloc ONCE, on the first call on a device, like the
 *     reference's DevCtx (exllamav3_ext/quant/exl3_devctx.cu:24-70); exl3b_moe and exl3b_quantize_tiles add their own fixed work
 *     areas on their first call on a device.  Scratch is never freed, moved or grown afterwards, so a
 *     CUDA graph captured over these entry points stays valid, and no entry point allocates or synchronises once the device
 *     context exists (make the first call on a device OUTSIDE stream capture).
 *   - Threading / streams: the scratch is per DEVICE and shared by all streams; launches rotate through 8 scratch slots, so
 *     the supported pattern is one in-order stream of qgemm launches per device at a time (what the reference supports as
 *     well: one lock buffer per device, exl3_devctx.cuh:35, ops called with the GIL held).  Calls from several host threads
 *     are safe as far as the slot rotation goes (atomic), but more than 8 launches in flight on one device across streams
 *     may share split-K scratch and is undefined.  In-kernel watchdogs (4 s split-K, 20 s tensor-parallel exchange) print
 *     and trap instead of hanging the GPU; a trap is a sticky CUDA error like the reference's exit-on-error (util.cuh:92-100).
 *   - return value: >= 0 on success (exl3b_gemm / exl3b_mgemm return a kernel-path tag like the reference's
 *     exl3_gemm, exllamav3_ext/quant/exl3_gemm.cu:234,247,308), < 0 = -(enum exl3b_status).  On error nothing was launched
 *     and exl3b_last_error() describes the problem (the reference raises via TORCH_CHECK, exllamav3_ext/util.h:24-37;
 *     exllamav3_b200/ext.py turns negative codes into RuntimeError with the same wording family).
 *   - there is NO CPU fallback: without a CUDA device every compute entry point returns -EXL3B_ERR_CUDA.
 *   - cb (codebook): 0 = 3INST (default), 1 = MCG, 2 = MUL1   (exllamav3_ext/quant/exl3_gemm.cu:173-176).
 *   - trellis layout: (k/16, n/16, 16*K) uint16, exactly the on-disk / reference layout (exllamav3_ext/quant/exl3_gemm.cu:27).
 */
#ifndef EXL3B200_H
#define EXL3B200_H

#include <stdint.h>
#include <stddef.h>

#ifdef __cplusplus
extern "C" {
#endif

#define EXL3B_ABI_VERSION 1

enum exl3b_status
{
    EXL3B_OK = 0,
    EXL3B_ERR_SHAPE = 1,      /* dimension / divisibility violation                      */
    EXL3B_ERR_ARG = 2,        /* null pointer, bad K / cb / flag                         */
    EXL3B_ERR_CUDA = 3,       /* CUDA runtime error (message has cudaGetErrorString)     */
    EXL3B_ERR_UNSUPPORTED = 4 /* valid in the reference but not implemented here         */
};

/* Kernel-path tags returned by exl3b_gemm / exl3b_mgemm */
#define EXL3B_TAG_NOP 0        /* empty problem                                            */
#define EXL3B_TAG_SIMT 100     /* CUDA-core bring-up kernel                                */
#define EXL3B_TAG_TC 200       /* wgmma decode-GEMM, bit-exact fp16 weights                */
#define EXL3B_TAG_TC_I8 210    /* wgmma u8 x s8 codebook path: mul1, m <= 4 (auto); m <= 8 with m*k <= 32768 when forced */
#define EXL3B_TAG_TC_I8_ROUTED 212 /* routed / weighted exl3b_mgemm (MoE decode) on the kind::i8 kernel: mul1, m <= 4 (auto) */
#define EXL3B_TAG_TC_I8_CHAIN 220 /* persistent multi-GEMM kernel (exl3b_chain_*; exl3b_gemm when forced): mul1, m <= 4 */
#define EXL3B_TAG_TC_I8_AR 211 /* the same kernel with the tensor-parallel sum fused into its epilogue (exl3b_gemm_allreduce) */
#define EXL3B_TAG_TC_MOE 230   /* fused routed-expert MLP (exl3b_moe) on the exact wgmma decode-GEMM                          */

int exl3b_abi_version(void);

/* Thread-local description of the last error returned on this thread ("" if none). */
const char* exl3b_last_error(void);

/* Device introspection -- replaces ext.g_get_num_sms / ext.g_get_cc (exllamav3_ext/bindings.cpp:130-131).
   Return the value, or a negative status. */
int exl3b_num_sms(int device);
int exl3b_cc(int device);

/* Force a kernel path for exl3b_gemm on this process: 0 = auto, EXL3B_TAG_SIMT, EXL3B_TAG_TC, EXL3B_TAG_TC_I8;
   EXL3B_TAG_TC_I8_ROUTED: exl3b_gemm as auto, exl3b_mgemm with indices / weights on the tensor-core path where eligible.
   (The reference exposes force_shape_idx / force_num_sms per call for the same purpose.) Returns previous value. */
int exl3b_set_gemm_path(int tag);

/*
 * Launch-geometry introspection -- the counterpart of ext.exl3_gemm_num_kernel_shapes / ext.exl3_gemm_shape_compat
 * (exllamav3_ext/bindings.cpp:128-129, exllamav3_ext/quant/exl3_kernel_map.cu:23-75): which kernel path a call takes and with
 * what persistent grid and shared-memory ring, computed by the same host functions the launchers use.  Pure
 * host arithmetic: needs no device (num_sms is an argument), so shapes can be vetted without a GPU.
 * exl3b_plan_unit_range / exl3b_plan_cta_of_unit expose the stream-K partition of `units` 128x128 work units (k fastest)
 * over `grid` CTAs: CTA c owns [units*c/grid, units*(c+1)/grid).
 */
struct exl3b_plan
{
    int32_t path;        /* EXL3B_TAG_*                                                                  */
    int32_t passes;      /* launches of the GEMM kernel (exact path: ceil(m / 128))                      */
    int32_t rows;        /* rows the kernel variant is built for (i8 path: 4 or 8; exact path: m rounded up to 16) */
    int32_t grid;        /* CTAs                                                                         */
    int32_t stages;      /* shared-memory ring depth                                                     */
    int32_t smem_bytes;  /* dynamic shared memory per CTA                                                */
    int32_t a_stages, d_bufs, tmem_cols;     /* operand stages / accumulator buffers / tensor-memory columns: on sm_90a
                                                a_stages = tmem_cols = 0, d_bufs = accumulator hand-off buffers */
    int32_t reserved;
    int64_t units;       /* 128 x 128 work units                                                         */
};
int exl3b_gemm_plan(int m, int k, int n, int K, int cb, int num_sms, int force_num_sms, struct exl3b_plan* out);
int exl3b_plan_unit_range(int64_t units, int grid, int cta, int64_t* begin, int64_t* end);
int exl3b_plan_cta_of_unit(int64_t units, int grid, int64_t unit);

/*
 * exl3b_gemm -- replaces ext.exl3_gemm (exllamav3_ext/bindings.cpp:126, exllamav3_ext/quant/exl3_gemm.cuh:21-33,
 * implementation exllamav3_ext/quant/exl3_gemm.cu:110-309).
 *
 *   C[m,n] = had128( had128(A[m,k] * suh) @ W_hat[k,n] ) * svh
 *
 *   A      (m, k) fp16, contiguous rows
 *   B      trellis (k/16, n/16, 16*K) uint16
 *   C      (m, n) fp16 (c_fp32 = 0) or fp32 (c_fp32 = 1); overwritten, need not be zeroed
 *   suh    (k) fp16 or NULL (NULL: A is already in the rotated basis, no input transform)
 *   A_had  (m, k) fp16 scratch for the transformed input; may alias A; may be NULL (library scratch is used)
 *   svh    (n) fp16 or NULL (NULL: no output transform)
 *   k % 128 == 0, n % 128 == 0, 1 <= K <= 8.
 *   force_shape_idx (exl3_gemm.cuh:28): <= 0 automatic; 1 = CUDA-core twin, 2 = exact tensor-core kernel for THIS call (what
 *   science/qgemm_benchmark.py uses to time every kernel "shape"); larger values are an error.
 *   force_num_sms (exl3_gemm.cuh:32): > 0 caps the persistent grid.
 */
int exl3b_gemm(void* stream,
               const void* A, const void* B, void* C,
               const void* suh, void* A_had, const void* svh,
               int m, int k, int n, int K, int cb, int c_fp32,
               int force_shape_idx, int force_num_sms);

/*
 * exl3b_act_mul -- replaces ext.silu_mul / gelu_mul / relu2_mul (exllamav3_ext/activation.cu).
 *
 *   a[i] = fp16( act(g[i]) * u[i] ),   act = 0 SiLU g / (1 + exp(-g)), 1 GELU (tanh form), 2 ReLU^2 max(g, 0)^2
 *   act_limit != 0: u is clamped to [-act_limit, act_limit] and act(g) from above at act_limit first.
 *
 *   g, u   numel elements, fp16 (in_fp32 = 0) or fp32 (in_fp32 = 1), contiguous; a numel fp16, may alias g or u.
 *   Computed in fp32 and rounded once (the reference's fp16-input kernel computes in half arithmetic).  Returns 0.
 */
int exl3b_act_mul(void* stream, const void* g, const void* u, void* a, int64_t numel, int in_fp32, int act, float act_limit);

/*
 * ---- RMSNorm ------------------------------------------------------------------------------------------------------------
 *
 * exl3b_rms_norm -- replaces ext.rms_norm and ext.rms_norm_res_in (exllamav3_ext/bindings.cpp:84-85, exllamav3_ext/norm.cu).
 * Over each of `rows` rows of `dim` elements, in fp32:
 *   rmf = rsqrt(sum(x^2) / dim + eps) * constant_scale,   v = (x * (w + constant_bias)) * rmf   (v = x * rmf when w is NULL)
 *   res_mode EXL3B_RES_NONE   y = v
 *            EXL3B_RES_POST   y = y + v, added in fp32 and rounded once
 *            EXL3B_RES_IN     r = (x + r) rounded to r's dtype and written back; v is then taken of that r instead of x
 *   x      fp16 (clamped to +-65504 where read) or fp32;  w  (dim) fp16 or bf16, or NULL;  y  fp16 or fp32, may alias x
 *   r      (rows, dim) fp16 or fp32, EXL3B_RES_IN only (y fp16 there); ignored otherwise
 *   dtype codes EXL3B_DTYPE_*; w_dtype is ignored when w is NULL, r_dtype unless EXL3B_RES_IN.  All tensors contiguous.
 *   dim % 4 == 0 and dim <= 16384; the tensors 16-byte aligned, or, when dim % 8 != 0, aligned to 4 of their elements.
 *   rows = 0 or dim = 0 launches nothing.  Deterministic: a row's result depends on its own values only.  Returns 0.
 *
 * exl3b_gated_rms_norm -- replaces ext.gated_rms_norm (bindings.cpp:86):
 *   s = silu(g),  gate_first = 0:  y = ((x * (w + constant_bias)) * rmf) * s,  rmf = rsqrt(sum(x^2) / dim + eps)
 *                 gate_first = 1:  the same with x * s in place of x, and no factor s afterwards
 *   x bf16 (x_dtype must say so);  w (w_groups, dim) fp32 or bf16, row i uses w row i % w_groups;  g (rows, dim) bf16 or fp32;
 *   y fp16 or fp32.  Sizes and alignment as exl3b_rms_norm, w_groups >= 1.  Returns 0.
 */
#define EXL3B_DTYPE_FP16 0
#define EXL3B_DTYPE_FP32 1
#define EXL3B_DTYPE_BF16 2
#define EXL3B_RES_NONE 0
#define EXL3B_RES_POST 1
#define EXL3B_RES_IN 2
int exl3b_rms_norm(void* stream, const void* x, const void* w, void* y, void* r, int64_t rows, int dim,
                   int x_dtype, int w_dtype, int y_dtype, int r_dtype, int res_mode,
                   float eps, float constant_bias, float constant_scale);
int exl3b_gated_rms_norm(void* stream, const void* x, const void* w, void* y, const void* g, int64_t rows, int dim,
                         int x_dtype, int w_dtype, int y_dtype, int g_dtype, int w_groups, int gate_first,
                         float eps, float constant_bias);

/*
 * exl3b_gemm_gated -- exl3b_gemm(exl3b_act_mul(G, U), B, ...) with the activation applied where the GEMM reads its input: the
 * down projection of a gated MLP block without the intermediate tensor.  Bit-identical to exl3b_act_mul into a buffer followed by
 * exl3b_gemm on it, with the same path and grid.
 *
 *   G, U   (m, k) fp16 (gu_fp32 = 0, 8-byte aligned) or fp32 (gu_fp32 = 1, 16-byte aligned), contiguous; e.g. the gate and up
 *          rows of an exl3b_mgemm output (2, m, k)
 *   B, C, suh, svh, K, cb, c_fp32, force_num_sms   as exl3b_gemm;  act, act_limit   as exl3b_act_mul
 *   Paths: the one exl3b_gemm selects for (m, k, n, K, cb) under exl3b_set_gemm_path, when it is EXL3B_TAG_TC_I8 at m <= 4 or
 *   EXL3B_TAG_TC at m <= 8.  Any other selection, and m > 8, returns -EXL3B_ERR_UNSUPPORTED.  Returns the path tag.
 */
int exl3b_gemm_gated(void* stream, const void* G, const void* U, const void* B, void* C, const void* suh, const void* svh,
                     int m, int k, int n, int K, int cb, int c_fp32, int gu_fp32, int act, float act_limit, int force_num_sms);

/*
 * exl3b_mgemm -- replaces ext.exl3_mgemm (exllamav3_ext/bindings.cpp:146, exllamav3_ext/quant/exl3_gemm.cuh:58-78; semantics
 * exllamav3_ext/quant/exl3_gemm.cu:341-381).
 *
 *   A         (bszm_in, m, k) fp16
 *   B_ptrs, suh_ptrs, svh_ptrs : device arrays of device addresses, one per quantized matrix
 *   C         (bszm_out, m, n) fp16|fp32
 *   A_had     fp16 scratch, at least max(bszm_in, bszm_out) * m * k elements (exl3_gemm.cu:452-453)
 *   indices   device int64 [num_indices] or NULL; negative entries skip the slot
 *   weights   device fp16 [num_indices] or NULL; if given every result is scaled and groups of
 *             (slots / num_tokens) are summed into C[t]
 *   min_index/max_index : expert-range filter with rebasing (min_index < 0 = off)
 *   size_n_list (device int32, per matrix) + c_ptrs (device addresses, per matrix): per-matrix output widths
 *             (NULL = uniform n, outputs in C); num_c_ptrs = number of entries.
 */
int exl3b_mgemm(void* stream,
                const void* A, const uint64_t* B_ptrs, void* C,
                const uint64_t* suh_ptrs, void* A_had, const uint64_t* svh_ptrs,
                const int64_t* indices, int num_indices, const void* weights,
                int bszm_in, int bszm_out, int m, int k, int n, int K, int cb, int c_fp32,
                int min_index, int max_index, int num_tokens,
                const int32_t* size_n_list, const uint64_t* c_ptrs, int num_c_ptrs,
                int force_shape_idx, int force_num_sms);

/*
 * Fan-out launches (exl3_mgemm with size_n_list / c_ptrs: several projections of the same input with different widths in one
 * launch, as the reference's fused attention does, exllamav3_ext/libtorch/dsv4_attn.cpp:88-99).  The reference's operator hands
 * over the widths as a DEVICE tensor only; the tensor-core path needs them on the host to lay out the launch (CTA groups
 * proportional to the matrices' sizes, the packed tensors' row pitch).  A caller that keeps the list unchanged registers a host
 * copy once:
 *   exl3b_register_widths(size_n_list (device address, the key), host_widths, count)     count = 0 forgets the entry
 * exl3b_mgemm then runs registered fan-outs (mul1, <= 4 rows, widths multiples of 128, <= 8 matrices, no indices) as ONE
 * launch of the wgmma int8 kernel; unregistered lists, or shapes outside that envelope, take the generic path as before.
 * The entry is the caller's promise about the memory at that address: withdraw or renew it when the tensor is rewritten or
 * freed (a recycled address would otherwise inherit the old widths; the shim in ext.py ties the entry to the tensor object and
 * its version counter and withdraws it when the object dies).
 * exl3b_plan_fanout: the CTA-group boundaries the launch would use (cta0[count + 1]); returns the grid size, 0 = not eligible.
 */
int exl3b_register_widths(const int32_t* size_n_list, const int32_t* host_widths, int count);
int exl3b_plan_fanout(int k, const int32_t* host_widths, int count, int num_sms, int32_t* cta0);

/*
 * ---- GEMM chains: one persistent launch for the quantized linears of a decode block ------------------------------------
 *
 * The reference runs the linears of a block as separate graph nodes of its C++ block modules: BC_GatedMLP issues
 * exl3_mgemm(gate, up) -> silu_mul -> exl3_gemm(down) (exllamav3_ext/libtorch/mlp.cpp:14-91), BC_Attention the q / k / v
 * projections and, after attention, o (exllamav3_ext/libtorch/attention.cpp:286-365).  A chain is the drop-in for those
 * launch sequences: a list of exl3_gemm-shaped ops executed by ONE persistent kernel whose weight stream does not stop at a
 * GEMM boundary (chain_i8.cu).  Ops are grouped into stages: an op with new_stage != 0 starts a stage whose inputs may be
 * outputs of earlier ops of the chain (a grid-wide dependency inside the kernel); ops of one stage are independent.
 *   A / A2 / in_mode   0: A = (m, k) fp16 input rows;  1: input = silu(A) * A2 with A = gate, A2 = up outputs, fp32 (m, k);
 *                      2: the same with fp16 gate / up  (the activation the reference applies between gate/up and down,
 *                      activation_kernels.cuh:144-240, folded into down's input stage; result rounded to fp16 as there)
 *   B, suh, svh, C, m, k, n, K, cb, c_fp32   as exl3b_gemm (no A_had: the transform runs inside the kernel)
 * Eligibility per op: mul1 codebook, 1 <= m <= 4, k % 128 == n % 128 == 0; otherwise -EXL3B_ERR_UNSUPPORTED from create.
 * Alignment per op (the kernel reads and writes these by 8- and 16-byte vectors): A 8 bytes (in_mode 0: 16 bytes lets the rows
 * be staged in shared memory by one bulk copy, 8 runs uncached), gate / up 16 bytes (fp32) or 8 bytes (fp16), suh and svh 8 bytes
 * (suh at 16 bytes is staged by a bulk copy), C 16 bytes (fp32) or 8 bytes (fp16); otherwise -EXL3B_ERR_ARG.  A contiguous view at
 * an element offset, e.g. buf[1:].view(m, k), can miss these.
 * exl3b_chain_create copies the op table to the device (synchronous: call it outside stream capture, once per block, like the
 * reference constructs its BC_* modules once); exl3b_chain_run is one asynchronous launch, capturable in a CUDA graph;
 * returns EXL3B_TAG_TC_I8_CHAIN.  One chain runs at a time per device (stream order).
 * exl3b_chain_plan: host-only introspection (stages, persistent grid, ring depth, shared memory) for tests.
 */
struct exl3b_chain_op
{
    const void* A; const void* A2; const void* B; const void* suh; const void* svh; void* C;
    int m, k, n, K, cb, c_fp32;
    int in_mode;
    int new_stage;
};
struct exl3b_chain_plan
{
    int stages, grid, ring_stages, smem_bytes, cache_bytes;
    int64_t units;
};
int exl3b_chain_plan(const struct exl3b_chain_op* ops, int n_ops, int num_sms, struct exl3b_chain_plan* out);
/* tests: replay CTA `cta`'s walk over its units with the kernel's own cursor; 8 int32 per unit: stage, op, strip, kb, seq,
   run_begin, run_end, chunk_begin * 65536 + chunk_len.  Returns the number of units of that CTA (may exceed max_units). */
int exl3b_chain_walk(const struct exl3b_chain_op* ops, int n_ops, int num_sms, int cta, int32_t* out, int max_units);
int exl3b_chain_create(const struct exl3b_chain_op* ops, int n_ops, void** chain);
int exl3b_chain_run(void* stream, void* chain);
int exl3b_chain_destroy(void* chain);

/*
 * exl3b_moe -- replaces ext.exl3_moe (exllamav3_ext/bindings.cpp:209, exllamav3_ext/quant/exl3_moe.cu): the routed experts'
 * gated MLP of a mixture-of-experts block in one call.  E = num_experts experts; expert e owns positions [s_e, s_e + c_e) of
 * token_sorted / weight_sorted, s_e = sum of expert_count[0..e), c_e = expert_count[e] (expert_count has E + 1 entries, the
 * last one is ignored).  Experts with 0 < c_e <= max_tokens are processed; for each of their positions j, t = token_sorted[j]:
 *   g = gate_e(x_t), u = up_e(x_t)            as exl3b_gemm with fp16 output (act_function 2: no gate GEMM)
 *   h = fp16(act(g) * u)                      act 0 = SiLU, 1 = tanh-GELU, 2 = ReLU^2 of u (h = relu(u) * u)
 *                                             act_limit != 0: u clamped to [-L, L], act(g) <= L
 *   output_state[t] += weight_sorted[j] * down_e(h)     fp32, added in ascending j: the result is deterministic
 * Other rows of output_state keep their bits.
 *   hidden_state (bsz, hidden) fp16 (8-byte aligned), output_state (bsz, hidden) fp32 (16-byte aligned), expert_count (E + 1)
 *   int64, token_sorted and weight_sorted (num_positions) int64 / fp16; the nine tables: E device addresses each; cb 1 = mcg or
 *   2 = mul1 for all three; hidden % 128 == intermediate % 128 == 0, K_* in 1..8, E <= 2048, concurrency * 8 <= num_sms,
 *   num_positions and bsz <= 2^20.  The caller's temp buffers are not needed.  The first call on a device allocates the
 *   operator's fixed work area (about 256 MB: the work list of up to 2^20 positions and a 240 MB row region); it is never
 *   grown, so make that first call outside stream capture, like the first call of any entry point.  Calls whose processed rows
 *   do not fit the row region at once run in several chunks of passes, with the same result bit for bit.
 *   num_active = 0: nothing is launched (EXL3B_TAG_NOP).  Returns EXL3B_TAG_TC_MOE.
 * exl3b_moe_max_concurrency(device) = num_sms / 8, as the reference (callers size their temp buffers from it).
 * exl3b_moe_plan: host-only introspection of the work list the route kernel derives on the device from the same counts, by
 * the same code: the passes (up to 128 consecutive positions of one processed expert, rows padded to 16) packed in order into
 * chunks of at most chunk_rows rows, written as int32 (expert, pos0, rows, row0, chunk) quintuples to passes_out (NULL = not
 * written; room for max_passes), and every position's code (128 * pass + row in pass, -1 = not processed) to pos_code_out
 * (num_positions entries, or NULL).  units_*: work items (pass, 128-column strip) of the gate / up and the down GEMMs.
 */
struct exl3b_moe_plan
{
    int32_t passes, chunks;          /* passes and chunks of the call                                        */
    int32_t rows, chunk_rows;        /* most rows any chunk uses, rows one chunk may hold                      */
    int32_t max_passes, max_chunks;  /* the launcher's bounds from sizes alone (grids, chunk launches)         */
    int64_t units_gate_up, units_down;
};
int exl3b_moe(void* stream,
              const void* hidden_state, void* output_state,
              const int64_t* expert_count, const int64_t* token_sorted, const void* weight_sorted,
              int bsz, int hidden, int intermediate, int num_experts, int num_positions, int max_tokens, int concurrency,
              int act_function, int K_gate, int K_up, int K_down,
              const uint64_t* gate_trellis, const uint64_t* gate_suh, const uint64_t* gate_svh,
              const uint64_t* up_trellis, const uint64_t* up_suh, const uint64_t* up_svh,
              const uint64_t* down_trellis, const uint64_t* down_suh, const uint64_t* down_svh,
              int gate_mcg, int gate_mul1, int up_mcg, int up_mul1, int down_mcg, int down_mul1,
              float act_limit, int num_active);
int exl3b_moe_max_concurrency(int device);
int exl3b_moe_plan(const int64_t* expert_count_host, int num_experts, int max_tokens, int num_positions, int hidden,
                   int intermediate, struct exl3b_moe_plan* out, int32_t* passes_out, int32_t* pos_code_out);

/*
 * exl3b_reconstruct -- replaces ext.reconstruct / ext.reconstruct_slice (exllamav3_ext/bindings.cpp:122-123,
 * exllamav3_ext/quant/reconstruct.cu:98-144,375-386):  trellis -> W_hat fp16, bit-exact.
 *   unpacked (k, n_out) fp16 contiguous; packed (k/16, packed_tiles_n, 16*K) uint16; columns
 *   [n_offset, n_offset + n_out) of the packed tensor are decoded.  n_out % 128 == 0, n_offset % 128 == 0.
 */
int exl3b_reconstruct(void* stream, void* unpacked, const void* packed,
                      int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset);

/*
 * exl3b_reconstruct_had -- replaces ext.reconstruct_had_slice (exllamav3_ext/bindings.cpp:124, exllamav3_ext/quant/reconstruct.cu:324-373):
 *   unpacked = diag(suh) . H128 . W_hat . H128 . diag(svh)  (original-basis weights), k % 128 == 0, n_out % 128 == 0;
 *   svh is pre-offset by the caller (points at the first emitted column), suh has k entries.
 */
int exl3b_reconstruct_had(void* stream, void* unpacked, const void* packed,
                          const void* suh, const void* svh,
                          int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset);

/*
 * exl3b_had_r_128 -- replaces ext.had_r_128 (exllamav3_ext/bindings.cpp:125, exllamav3_ext/quant/hadamard.cu:88-173):
 *   out = (in.view(-1,128) @ H128) * scale / sqrt(128), optional per-column fp16 pre_scale OR post_scale
 *   (pre_scale wins if both given, as in the reference).  is_fp32 selects fp32 in/out, else fp16.  In place OK.
 */
int exl3b_had_r_128(void* stream, const void* in, void* out,
                    const void* pre_scale, const void* post_scale, float scale,
                    int rows, int cols, int is_fp32);

/*
 * exl3b_hgemm -- replaces ext.hgemm (exllamav3_ext/bindings.cpp:147, exllamav3_ext/hgemm.cu:19-102): row-major c = a @ b,
 * a (m,k) fp16, b (k,n) fp16, c (m,n) fp16|fp32 with row stride c_stride (elements), fp32 accumulate.
 */
int exl3b_hgemm(void* stream, const void* a, const void* b, void* c,
                int m, int k, int n, int c_fp32, int64_t c_stride);

/*
 * Host-buffer convenience used by the end-to-end benchmark leg and by non-torch integrations:
 * copies A_host (pinned or pageable, m*k fp16) to the device, runs exl3b_gemm against device-resident weights,
 * copies C back to C_host and synchronises the stream.  d_A / d_C / d_A_had are caller-provided device staging
 * buffers of the same sizes.
 */
int exl3b_gemm_host(void* stream,
                    const void* A_host, void* C_host,
                    void* d_A, void* d_C, void* d_A_had,
                    const void* B, const void* suh, const void* svh,
                    int m, int k, int n, int K, int cb, int c_fp32);

/*
 * ---- tensor-parallel row-parallel output: GEMM + sum over ranks in ONE kernel (NVLink peer memory) ----------------------
 *
 * Replaces, for the row-parallel linears (o_proj, down_proj) of the reference's tensor-parallel mode, the pair
 *     ext.exl3_gemm(...)                      exllamav3_ext/bindings.cpp:126
 *     backend.all_reduce(y)                   exllamav3/model/model_tp_backend.py:119-126 (one NCCL launch per output),
 * issued by exllamav3/modules/mlp.py:769-770 and exllamav3/modules/attn.py:546-547.
 *
 * One process per GPU.  Setup, once per process:
 *   1. exl3b_tp_alloc(rank, world, max_elems, handle)   allocate this rank's receive buffer on the current device
 *                                                       (max_elems >= m * n of the largest row-parallel output, multiple
 *                                                       of 128) and get its 64-byte CUDA IPC handle
 *   2. the ranks exchange the handles (any transport: the reference-side shim uses torch.distributed.all_gather_object)
 *   3. exl3b_tp_attach(handles, world)                  handles = world x EXL3B_TP_HANDLE_BYTES in rank order
 * Then exl3b_gemm_allreduce(...) = exl3b_gemm(...) followed by a sum over the ranks, every rank receiving the bit-identical
 * result (partials are added in rank order).  Every rank must issue the same sequence of exl3b_gemm_allreduce calls.
 * Eligibility: mul1 codebook, 1 <= m <= 4, m * n <= max_elems, world <= 8; otherwise -EXL3B_ERR_UNSUPPORTED and nothing is
 * launched (the caller falls back to exl3b_gemm + its own all-reduce).  Returns EXL3B_TAG_TC_I8_AR.
 * exl3b_tp_attach_loopback(): single-process bring-up -- "peer" buffers are local allocations, peer partials are supplied
 * with exl3b_tp_debug_inject (tests only).
 * Tests: tests/test_tp_fused.py (one GPU: loop-back protocol; -m multigpu: two GPUs).
 */
#define EXL3B_TP_HANDLE_BYTES 64
int exl3b_tp_alloc(int rank, int world, int64_t max_elems, void* handle_out);
int exl3b_tp_attach(const void* handles, int world);
int exl3b_tp_attach_loopback(void);
int exl3b_tp_info(int* rank, int* world, int64_t* max_elems, int* attached);
int exl3b_tp_free(void);
int exl3b_gemm_allreduce(void* stream,
                         const void* A, const void* B, void* C,
                         const void* suh, void* A_had, const void* svh,
                         int m, int k, int n, int K, int cb, int c_fp32);
/* 0 if a call with these sizes can take the fused path on a group of `world` ranks with `max_elems` slots, else
   -EXL3B_ERR_UNSUPPORTED with the reason in exl3b_last_error().  Pure host logic: needs no device. */
int exl3b_gemm_allreduce_check(int m, int k, int n, int K, int cb, int world, int64_t max_elems);
/* bring-up / tests: write a peer's partial (count fp32 words, device pointer) into this rank's receive buffer for the NEXT
   exl3b_gemm_allreduce on `stream`; copy (slot, src_rank) of rank `buffer_rank`'s buffer to the host; read the epoch. */
int exl3b_tp_debug_inject(void* stream, int src_rank, const void* partial, int64_t count);
int exl3b_tp_debug_peek(int buffer_rank, int slot, int src_rank, void* host_out, int64_t count);
int64_t exl3b_tp_debug_epoch(void);

/*
 * ---- trellis encoder (conversion) ---------------------------------------------------------------------------------------
 *
 * exl3b_quantize_tiles -- replaces ext.quantize_tiles (exllamav3_ext/bindings.cpp:116, quant/quantize.cu): for each of
 * num_tiles rows of 256 fp32 values `in` (one 16x16 tile in trellis position order), the tail-biting state sequence
 * s[0..255] of minimum squared error against the codebook cb, found by Viterbi with fp32 path costs.  Writes the states
 * (uint16, num_tiles x 256) to out_idx and their codebook values as fp32 to out_tiles.  The wrap overlap s[0] >> K is
 * chosen like the reference does (best unconstrained path started at position 128); the sequence is the exact minimum
 * for that overlap.  Deterministic; a tile's result does not depend on the other tiles of the call.  The first call on
 * a device allocates a fixed backpointer scratch of 2 MB per SM (make it outside stream capture).
 *
 * exl3b_pack_trellis -- replaces ext.pack_trellis (bindings.cpp:119, quant/pack.cu:9-57): unpacked (num_tiles x 256
 * uint16 states) -> packed (num_tiles x 16K uint16), the low K bits of each state MSB first, 16-bit words swapped
 * pairwise per 32-bit word: the trellis layout every GEMM entry point reads.
 */
int exl3b_quantize_tiles(void* stream, const void* in, void* out_tiles, void* out_idx, int64_t num_tiles, int K, int cb);
int exl3b_pack_trellis(void* stream, void* packed, const void* unpacked, int64_t num_tiles, int K);

/* Count of kernels launched by this library in this process (for bench.py's gpu_launches claim). */
int64_t exl3b_launch_count(void);

#ifdef __cplusplus
}
#endif
#endif /* EXL3B200_H */
