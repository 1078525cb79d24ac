// Shared host/device helpers for the exl3b200 library.
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <stdarg.h>
#include <atomic>
#include "../../include/exl3b200.h"

namespace exl3b {

constexpr float R_SCALE = 0.088388347648f;      // 1/sqrt(128), same literal as the reference (hadamard.cu:112)

// ---- error plumbing ---------------------------------------------------------------------------------------
void set_error(const char* fmt, ...);
int fail(int status, const char* fmt, ...);
#define EXL3B_CHECK(cond, status, ...) do { if (!(cond)) return ::exl3b::fail(status, __VA_ARGS__); } while (0)
#define EXL3B_CUDA(call) do { cudaError_t e__ = (call); if (e__ != cudaSuccess) \
    return ::exl3b::fail(EXL3B_ERR_CUDA, "%s: %s", #call, cudaGetErrorString(e__)); } while (0)

void count_launch(int n = 1);

// Per-launch table of active matrix slots for mgemm (device memory, owned by DevCtx).
struct MSlotTable
{
    static constexpr int MAX_SLOTS = 128;       // same capacity as the reference's v_indices (exl3_gemm_kernel.cuh:82-85)
    int n_active;
    int mat[MAX_SLOTS];
    half weight[MAX_SLOTS];
};

// ---- per-device context -----------------------------------------------------------------------------------
// Split-K partial sums and tile counters.  Launches rotate through NUM_SLOTS independent regions so that
// consecutive (PDL-overlapped) launches on one stream never share counters; counters are self-resetting.
struct DevCtx
{
    static constexpr int NUM_SLOTS = 8;
    static constexpr size_t WS_BYTES_PER_SLOT = 40u << 20;    // fp32 split-K partials (2 x up to 160 CTAs x 256 rows x 128 cols)
    static constexpr int COUNTERS_PER_SLOT = 32768;
    int device = -1;
    int num_sms = 0;
    int cc = 0;
    float* ws = nullptr;          // NUM_SLOTS * WS_BYTES_PER_SLOT
    int* counters = nullptr;      // NUM_SLOTS * COUNTERS_PER_SLOT, zero-initialised once
    MSlotTable* tabs = nullptr;   // NUM_SLOTS mgemm slot tables
    static constexpr int XH_SLOTS = 4;
    static constexpr int XH_MAX_K = 65536;  // largest in_features the fixed activation scratch below is sized for
    uint8_t* xh_tiled = nullptr;  // XH_SLOTS tiled activation buffers for the tensor-core path (256 rows x XH_MAX_K fp16 each), allocated once
    size_t xh_tiled_slot_bytes = 0;
    half* xh_scratch = nullptr;   // input-transform scratch when the caller passes A_had = NULL (256 x XH_MAX_K), allocated once
    size_t xh_scratch_elems = 0;
    uint8_t* tmap_slots = nullptr;   // NUM_SLOTS x TMAP_SLOTS x 128 B: per-CTA patched tensor maps of multi-matrix launches
    static constexpr int TMAP_SLOTS = 256;
    uint8_t* tmap_slot(int s) { return tmap_slots + (size_t) s * TMAP_SLOTS * 128; }
    // i8 path split-K exchange: NUM_SLOTS x I8_PART_CTAS slots of up to 8 x 128 fp32, all-ones (sentinel) whenever no launch is
    // in flight: contributors overwrite, the strip's reducer reads and restores the sentinel
    float* i8_parts = nullptr;
    static constexpr int I8_PART_CTAS = 256;
    float* i8_parts_slot(int s) { return i8_parts + (size_t) s * I8_PART_CTAS * 1024; }
    // chain kernel (chain_i8.cu): stage counters + exit ticket (zero between launches) and its split-K exchange
    // [2][I8_PART_CTAS][4 x 128] (sentinel between launches); shared by all chains of the device (one in-order stream)
    unsigned int* chain_ctr = nullptr;
    float* chain_parts = nullptr;
    // Launch slots rotate per device, not per stream: launches issued concurrently on two streams of one device (or from two
    // host threads: ctypes releases the GIL) get distinct slots from this atomic counter, but more than NUM_SLOTS launches in
    // flight on one device would share split-K scratch -- the library supports ONE in-order stream of qgemm launches per
    // device at a time, like the reference (single DevCtx lock buffer, exl3_devctx.cuh:35; include/exl3b200.h "Threading").
    std::atomic<uint64_t> launch_seq{0};
    int next_slot() { return (int) (launch_seq.fetch_add(1, std::memory_order_relaxed) % NUM_SLOTS); }
    float* ws_slot(int s) { return (float*) ((char*) ws + (size_t) s * WS_BYTES_PER_SLOT); }
    int* counter_slot(int s) { return counters + (size_t) s * COUNTERS_PER_SLOT; }
    MSlotTable* tab_slot(int s) { return tabs + s; }
};
int get_ctx(DevCtx** out);       // context of the current device (lazy init), status code
int ensure_xh_scratch(DevCtx* ctx, size_t elems);
int ensure_xh_tiled(DevCtx* ctx, size_t bytes_per_slot);

// ---- launchers implemented in the .cu files ------------------------------------------------------------------
int launch_had_r_128(cudaStream_t stream, const void* in, void* out, const half* pre, const half* post,
                     float scale, int rows, int cols, bool fp32);
int launch_reconstruct(cudaStream_t stream, half* unpacked, const uint16_t* packed, int k, int n_out,
                       int packed_tiles_n, int K, int cb, int64_t n_offset);
int launch_reconstruct_had(cudaStream_t stream, half* unpacked, const uint16_t* packed, const half* suh,
                           const half* svh, int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset);
// tensor-core variant (reconstruct_tc.cu): both Hadamards as wgmma GEMMs; the default unless EXL3B_RECONSTRUCT_HAD=simt
bool reconstruct_had_tc_enabled();
void reconstruct_had_set_mode(int mode);
int launch_reconstruct_had_tc(cudaStream_t stream, half* unpacked, const uint16_t* packed, const half* suh, const half* svh,
                              int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset, int num_sms);

struct GemmArgs
{
    const half* A;           // raw input (m, k)
    const half* suh;         // may be null: no input transform
    half* A_had;             // caller scratch for the transformed input (may be null / alias A)
    const uint32_t* B;
    void* C;
    const half* svh;         // may be null
    int m, k, n, K, cb;
    bool c_fp32;
    float out_scale;         // extra factor folded into the output transform (mgemm weights), 1.0f otherwise
    int max_ctas;            // 0 = all SMs
};
// Launch geometry of one tensor-core kernel launch: computed by the SAME functions the launchers use (plan_gemm_tc_i8 in
// gemm_tc_i8.cu, plan_gemm_tc in gemm_tc.cu), pure host arithmetic -- exposed through exl3b_gemm_plan so that the CPU tests
// can check budgets and the stream-K partition for shapes no GPU test runs.  Returns 0 or a negative status.
struct TcPlan
{
    int rows;            // activation rows the kernel variant is built for: MR (i8 path) or NT (exact path)
    int stages;          // shared-memory ring depth
    int b_bytes;         // activation bytes reserved per stage
    int b_load_bytes;    // i8: activation-cache bytes (0 = recompute per unit); exact: activation bytes copied per unit
    int smem_total;      // dynamic shared memory of the launch
    int grid;            // CTAs (single-matrix launch)
    long long units;     // 128 x 128 work units
    int d_bufs;          // accumulator hand-off buffers
};
int plan_gemm_tc_i8(int m, int k, int n, int K, int num_sms, int max_ctas, TcPlan* pl);
int plan_gemm_tc(int m, int k, int n, int K, int num_sms, int max_ctas, TcPlan* pl);     // m <= 256: one pass

int launch_gemm_simt(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a);
// gate != null (exl3b_gemm_gated, act.cuh): the kernel's rows are fp16(act(G) * U) instead of a.A
struct GateIn;
int launch_gemm_tc(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a, const GateIn* gate = nullptr);
bool gemm_tc_supported(const GemmArgs& a);
int launch_gemm_tc_i8(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a, const GateIn* gate = nullptr);
struct MGemmArgs;
bool mgemm_tc_i8_supported(const DevCtx* ctx, const MGemmArgs& a);
int launch_mgemm_tc_i8(cudaStream_t stream, DevCtx* ctx, const MGemmArgs& a);
bool gemm_tc_i8_supported(const GemmArgs& a);
// The int8 decode-GEMM's shape rule (gemm_tc_i8.cu), for every launch of its kernels: the mul1 codebook, 1..4 rows (5..8 too
// when rows8 and the activation fits the shared-memory cache), K in 1..8, k and n multiples of 128.  nullptr = supported,
// else the reason, which exl3b_gemm_allreduce_check and exl3_chain show to users.
const char* i8_shape_unsupported(int m, int k, int n, int K, int cb, bool rows8);

// tensor-parallel row-parallel GEMM with the sum over ranks fused into the epilogue (gemm_tc_i8_ar.cu)
int launch_gemm_tc_i8_ar(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a);
const char* gemm_tc_i8_ar_unsupported(int m, int k, int n, int K, int cb, int world, long long slot_elems);
int tp_alloc(int rank, int world, long long max_elems, void* handle_out);
int tp_attach(const void* handles, int world);
int tp_attach_loopback();
int tp_info(int* rank, int* world, long long* max_elems, int* attached);
int tp_free();
int tp_debug_inject(cudaStream_t stream, int src_rank, const void* partial, long long count);
int tp_debug_peek(int buffer_rank, int slot, int src_rank, void* host_out, long long count);
long long tp_debug_epoch();

struct MGemmArgs
{
    const half* A; const uint64_t* B_ptrs; void* C; const uint64_t* suh_ptrs; half* A_had; const uint64_t* svh_ptrs;
    const int64_t* indices; int num_indices; const half* weights;
    int bszm_in, bszm_out, m, k, n, K, cb; bool c_fp32;
    int min_index, max_index, num_tokens;
    const int32_t* size_n_list; const uint64_t* c_ptrs; int num_c_ptrs;
    const int32_t* size_n_host;          // host copy of size_n_list if the caller registered one (exl3b_register_widths), else null
};
// fan-out launches (per-matrix widths) on the wgmma int8 path: CTA group boundaries proportional to the matrices' unit counts
// (host + tests: the partition the kernel is given); returns the grid size, 0 if the shapes do not fit
int plan_fanout_groups(int k, const int32_t* widths, int mats, int num_sms, int* cta0 /* mats + 1 */);
int launch_mgemm(cudaStream_t stream, DevCtx* ctx, const MGemmArgs& a);

// persistent multi-GEMM kernel (chain_i8.cu)
bool gemm_chain_supported(const GemmArgs& a);
int launch_gemm_chain(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a);
int chain_plan(const exl3b_chain_op* in, int n_ops, int num_sms, struct exl3b_chain_plan* out);
int chain_walk(const exl3b_chain_op* in, int n_ops, int num_sms, int cta, int32_t* out, int max_units);
int chain_create(DevCtx* ctx, const exl3b_chain_op* in, int n_ops, void** out);
int chain_run(cudaStream_t stream, void* chain);
int chain_destroy(void* chain);
int launch_mgemm_resolve(cudaStream_t stream, MSlotTable* tab, const MGemmArgs& a, int bszm);
int launch_mgemm_reduce(cudaStream_t stream, DevCtx* ctx, const MSlotTable* tab, const MGemmArgs& a);
// routed / weighted exl3_mgemm (MoE decode) on the wgmma int8 path (gemm_tc_i8_routed.cu): opt-in, tag EXL3B_TAG_TC_I8_ROUTED
bool mgemm_tc_i8_routed_supported(const DevCtx* ctx, const MGemmArgs& a);
int launch_mgemm_tc_i8_routed(cudaStream_t stream, DevCtx* ctx, const MGemmArgs& a);

// standalone gated activation (act.cu): a = fp16(act(g) * u) elementwise
int launch_act_mul(cudaStream_t stream, const void* g, const void* u, half* a, long long numel, bool in_fp32, int act, float limit);

// RMSNorm operators (norm.cu); the entry points in api.cu check the arguments and pick e
constexpr int NORM_MAX_DIM = 16384;    // longest row: it is held in registers from its load to its store
struct NormArgs
{
    const void* x; const void* w; void* y; void* r; const void* g;     // w may be NULL (rms_norm); r: RES_IN only; g: gated only
    long long rows; int dim;
    int x_dtype, w_dtype, y_dtype, r_dtype, g_dtype;                    // EXL3B_DTYPE_*
    int res_mode;                                                       // EXL3B_RES_*
    float eps, bias, scale;
    int w_groups, gate_first;
    int e;                                                              // elements per load unit: 8 (16-byte loads of fp16) or 4
};
int launch_rms_norm(cudaStream_t stream, const NormArgs& a);
int launch_gated_rms_norm(cudaStream_t stream, const NormArgs& a);

int launch_hgemm(cudaStream_t stream, const half* a, const half* b, void* c, int m, int k, int n, bool c_fp32,
                 int64_t c_stride);

// fused routed-expert MLP (moe_tc.cu, tag EXL3B_TAG_TC_MOE)
constexpr int MOE_MAX_EXPERTS = 2048;
// one pass: up to F16_MAX_ROWS (f16_pipeline.cuh) consecutive positions of one expert; row0 = its first row in chunk `chunk`
// of the work area
struct MoePass { int expert, pos0, rows, row0, chunk; };
struct MoeArgs
{
    const half* hidden_state; float* output_state;
    const int64_t* expert_count; const int64_t* token_sorted; const half* weight_sorted;
    int bsz, hidden, inter, num_experts, num_positions, max_tokens;
    int act; float act_limit;
    int K_gate, K_up, K_down, cb;
    const uint64_t *gate_trellis, *gate_suh, *gate_svh, *up_trellis, *up_suh, *up_svh, *down_trellis, *down_suh, *down_svh;
    int num_active;
};
int launch_moe(cudaStream_t stream, DevCtx* ctx, const MoeArgs& a);
int moe_plan_host(const int64_t* count, int E, int T, int N, int hidden, int inter, struct exl3b_moe_plan* out, int32_t* passes_out,
                  int32_t* pos_code_out);

// trellis encoder (encode.cu): tail-biting Viterbi per 256-value tile, and the K-bit packer
int launch_quantize_tiles(cudaStream_t stream, DevCtx* ctx, const float* in, float* out_values, uint16_t* out_states,
                          int64_t num_tiles, int K, int cb);
int launch_pack_trellis(cudaStream_t stream, uint16_t* packed, const uint16_t* unpacked, int64_t num_tiles, int K);

// ---- (K, cb) template dispatch ---------------------------------------------------------------------------------
#define EXL3B_DISPATCH_K_CB(FN, K, cb, ...)                                                        \
    do { switch ((cb) * 8 + (K) - 1) {                                                             \
        case  0: FN<1, 0>(__VA_ARGS__); break; case  1: FN<2, 0>(__VA_ARGS__); break;              \
        case  2: FN<3, 0>(__VA_ARGS__); break; case  3: FN<4, 0>(__VA_ARGS__); break;              \
        case  4: FN<5, 0>(__VA_ARGS__); break; case  5: FN<6, 0>(__VA_ARGS__); break;              \
        case  6: FN<7, 0>(__VA_ARGS__); break; case  7: FN<8, 0>(__VA_ARGS__); break;              \
        case  8: FN<1, 1>(__VA_ARGS__); break; case  9: FN<2, 1>(__VA_ARGS__); break;              \
        case 10: FN<3, 1>(__VA_ARGS__); break; case 11: FN<4, 1>(__VA_ARGS__); break;              \
        case 12: FN<5, 1>(__VA_ARGS__); break; case 13: FN<6, 1>(__VA_ARGS__); break;              \
        case 14: FN<7, 1>(__VA_ARGS__); break; case 15: FN<8, 1>(__VA_ARGS__); break;              \
        case 16: FN<1, 2>(__VA_ARGS__); break; case 17: FN<2, 2>(__VA_ARGS__); break;              \
        case 18: FN<3, 2>(__VA_ARGS__); break; case 19: FN<4, 2>(__VA_ARGS__); break;              \
        case 20: FN<5, 2>(__VA_ARGS__); break; case 21: FN<6, 2>(__VA_ARGS__); break;              \
        case 22: FN<7, 2>(__VA_ARGS__); break; case 23: FN<8, 2>(__VA_ARGS__); break;              \
    } } while (0)
// K-only dispatch: runs the statement(s) with the compile-time constant KK = K (1..8)
#define EXL3B_DISPATCH_K(K, ...)                                                                   \
    do { switch (K) {                                                                              \
        case 1: { constexpr int KK = 1; __VA_ARGS__; } break; case 2: { constexpr int KK = 2; __VA_ARGS__; } break; \
        case 3: { constexpr int KK = 3; __VA_ARGS__; } break; case 4: { constexpr int KK = 4; __VA_ARGS__; } break; \
        case 5: { constexpr int KK = 5; __VA_ARGS__; } break; case 6: { constexpr int KK = 6; __VA_ARGS__; } break; \
        case 7: { constexpr int KK = 7; __VA_ARGS__; } break; case 8: { constexpr int KK = 8; __VA_ARGS__; } break; \
    } } while (0)

// ---- kernel launch helpers ------------------------------------------------------------------------------------
// Raise KERNEL's dynamic shared-memory limit to `bytes`, once per device (the attribute belongs to the kernel on each device).
template <auto KERNEL>
cudaError_t set_max_smem_once(int bytes)
{
    static bool done[32] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (done[dev & 31]) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(KERNEL, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes);
    if (e == cudaSuccess) done[dev & 31] = true;
    return e;
}
// Launch a kernel of up to 220 KiB dynamic shared memory with programmatic stream serialization (PDL): it may start while
// the previous kernel of the stream finishes, so it must pdl_wait() before it reads that kernel's results.  Only a launch
// beyond the default 48 KiB raises the kernel's limit: a kernel with large static shared memory could not take the raise.
template <auto KERNEL, typename... Args>
cudaError_t launch_pdl(cudaStream_t stream, dim3 grid, int threads, int smem_bytes, const Args&... args)
{
    if (smem_bytes > 48 * 1024)
    {
        const cudaError_t e = set_max_smem_once<KERNEL>(220 * 1024);
        if (e != cudaSuccess) return e;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = grid; cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, KERNEL, args...);
}

// ---- device helpers -----------------------------------------------------------------------------------------
#ifdef __CUDACC__

// 128-point Sylvester Hadamard across one warp, 4 consecutive elements per lane, fp32.  Performs exactly the
// additions of the reference's had_*_r_128_inner (hadamard_inner.cuh:118-131, 14-41): in-lane 4-point, then
// xor-shuffle stages 1..16 with new = (lane & i ? -own : own) + partner.
__device__ __forceinline__ void had128_warp_tail(float& h0, float& h1, float& h2, float& h3, int lane);
__device__ __forceinline__ void had128_warp(float& h0, float& h1, float& h2, float& h3, int lane)
{
    float s0 = h0 + h1, d0 = h0 - h1, s1 = h2 + h3, d1 = h2 - h3;
    h0 = s0 + s1; h1 = d0 + d1; h2 = s0 - s1; h3 = d0 - d1;
    had128_warp_tail(h0, h1, h2, h3, lane);
}
// the five cross-lane stages (the in-lane 4-point stage already applied)
__device__ __forceinline__ void had128_warp_tail(float& h0, float& h1, float& h2, float& h3, int lane)
{
    #pragma unroll
    for (int i = 1; i < 32; i <<= 1)
    {
        float p0 = __shfl_xor_sync(0xffffffffu, h0, i);
        float p1 = __shfl_xor_sync(0xffffffffu, h1, i);
        float p2 = __shfl_xor_sync(0xffffffffu, h2, i);
        float p3 = __shfl_xor_sync(0xffffffffu, h3, i);
        bool neg = (lane & i) != 0;
        h0 = (neg ? -h0 : h0) + p0;
        h1 = (neg ? -h1 : h1) + p1;
        h2 = (neg ? -h2 : h2) + p2;
        h3 = (neg ? -h3 : h3) + p3;
    }
}

// The input transform of lane's four values k = 4 lane .. 4 lane + 3 of one 128-k block (fp16 pairs in `raw`, one block per
// warp), as the reference's A_had: x * suh in fp16 (`scb`: lane's four suh scales; null when x already carries them), the
// 128-point Hadamard in fp32, then * 1/sqrt(128) rounded once to fp16.  Returns the two fp16 pairs.
__device__ __forceinline__ uint2 had128_fp16(uint2 raw, const uint2* scb, int lane)
{
    half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
    if (scb)
    {
        a = __hmul2(a, *reinterpret_cast<const half2*>(&scb->x));
        b = __hmul2(b, *reinterpret_cast<const half2*>(&scb->y));
    }
    float v0 = __low2float(a), v1 = __high2float(a), v2 = __low2float(b), v3 = __high2float(b);
    had128_warp(v0, v1, v2, v3, lane);
    a = __floats2half2_rn(v0 * R_SCALE, v1 * R_SCALE);
    b = __floats2half2_rn(v2 * R_SCALE, v3 * R_SCALE);
    uint2 o; o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
    return o;
}

__device__ __forceinline__ uint32_t pack_half2(half a, half b)
{
    return (uint32_t) __half_as_ushort(a) | ((uint32_t) __half_as_ushort(b) << 16);
}

#endif  // __CUDACC__

}  // namespace exl3b
