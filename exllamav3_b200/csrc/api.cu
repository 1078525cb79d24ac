// C ABI of libexl3b200.so (declared in include/exl3b200.h): argument validation mirroring the reference's
// TORCH_CHECKs, per-device context, kernel-path selection.  No torch types, no CPU fallback.
#include "common.cuh"
#include "epilogue.cuh"
#include "tc_common.cuh"
#include "act.cuh"
#include <mutex>
#include <unordered_map>
#include <vector>
#include <string>
#include <atomic>
#include <cstring>
#include <cstdlib>

namespace exl3b {

static thread_local std::string g_err;
static std::atomic<int64_t> g_launches{0};
static std::atomic<int> g_force_path{0};

void set_error(const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_err = buf;
}

int fail(int status, const char* fmt, ...)
{
    char buf[512];
    va_list ap; va_start(ap, fmt); vsnprintf(buf, sizeof(buf), fmt, ap); va_end(ap);
    g_err = buf;
    return -status;
}

void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

static constexpr int MAX_DEVICES = 32;
static DevCtx g_ctx[MAX_DEVICES];
static std::mutex g_ctx_mutex;

int get_ctx(DevCtx** out)
{
    int dev = -1;
    EXL3B_CUDA(cudaGetDevice(&dev));
    EXL3B_CHECK(dev >= 0 && dev < MAX_DEVICES, EXL3B_ERR_CUDA, "device index %d out of range", dev);
    std::lock_guard<std::mutex> lock(g_ctx_mutex);
    DevCtx& c = g_ctx[dev];
    if (c.device < 0)
    {
        cudaDeviceProp prop;
        EXL3B_CUDA(cudaGetDeviceProperties(&prop, dev));
        EXL3B_CHECK(prop.major == 9 && prop.minor == 0, EXL3B_ERR_CUDA,
                    "exl3b200 is built for sm_90a only; device %d is sm_%d%d (no fallback path exists)",
                    dev, prop.major, prop.minor);
        c.num_sms = prop.multiProcessorCount;
        c.cc = prop.major * 10 + prop.minor;
        EXL3B_CUDA(cudaMalloc(&c.ws, DevCtx::NUM_SLOTS * DevCtx::WS_BYTES_PER_SLOT));
        EXL3B_CUDA(cudaMalloc(&c.counters, sizeof(int) * DevCtx::NUM_SLOTS * DevCtx::COUNTERS_PER_SLOT));
        EXL3B_CUDA(cudaMemset(c.counters, 0, sizeof(int) * DevCtx::NUM_SLOTS * DevCtx::COUNTERS_PER_SLOT));
        EXL3B_CUDA(cudaMalloc(&c.tabs, sizeof(MSlotTable) * DevCtx::NUM_SLOTS));
        EXL3B_CUDA(cudaMalloc(&c.tmap_slots, (size_t) DevCtx::NUM_SLOTS * DevCtx::TMAP_SLOTS * 128));
        EXL3B_CUDA(cudaMalloc(&c.i8_parts, (size_t) DevCtx::NUM_SLOTS * DevCtx::I8_PART_CTAS * 1024 * sizeof(float)));
        EXL3B_CUDA(cudaMemset(c.i8_parts, 0xff, (size_t) DevCtx::NUM_SLOTS * DevCtx::I8_PART_CTAS * 1024 * sizeof(float)));
        // tiled / plain transformed activations: one pass of the exact path is <= 128 rows (gemm_tc.cu); sized for 256
        c.xh_tiled_slot_bytes = (size_t) 2 * 256 * DevCtx::XH_MAX_K;
        EXL3B_CUDA(cudaMalloc(&c.xh_tiled, c.xh_tiled_slot_bytes * DevCtx::XH_SLOTS));
        EXL3B_CUDA(cudaMemset(c.xh_tiled, 0, c.xh_tiled_slot_bytes * DevCtx::XH_SLOTS));
        EXL3B_CUDA(cudaMalloc(&c.chain_ctr, 256 * sizeof(unsigned int)));
        EXL3B_CUDA(cudaMemset(c.chain_ctr, 0, 256 * sizeof(unsigned int)));
        EXL3B_CUDA(cudaMalloc(&c.chain_parts, (size_t) 2 * DevCtx::I8_PART_CTAS * 512 * sizeof(float)));
        EXL3B_CUDA(cudaMemset(c.chain_parts, 0xff, (size_t) 2 * DevCtx::I8_PART_CTAS * 512 * sizeof(float)));
        c.xh_scratch_elems = (size_t) 256 * DevCtx::XH_MAX_K;
        EXL3B_CUDA(cudaMalloc(&c.xh_scratch, c.xh_scratch_elems * sizeof(half)));
        EXL3B_CUDA(cudaDeviceSynchronize());
        c.device = dev;
    }
    *out = &c;
    return 0;
}

// Library scratch is allocated ONCE per device (get_ctx) at a fixed worst-case size and never freed or moved: a CUDA graph
// captured earlier keeps replaying with these addresses, and nothing here may synchronise or allocate inside a launch path
// (the reference has the same rule for its workspaces, exl3_gemv_int8.cu:93-99).  A call that needs more than the fixed
// size is refused (EXL3B_ERR_UNSUPPORTED); exl3_gemm callers that pass their own A_had never touch xh_scratch.
int ensure_xh_scratch(DevCtx* ctx, size_t elems)
{
    EXL3B_CHECK(elems <= ctx->xh_scratch_elems, EXL3B_ERR_UNSUPPORTED,
                "exl3_gemm: A_had = NULL needs %zu scratch elements, the library holds %zu (pass A_had)", elems, ctx->xh_scratch_elems);
    return 0;
}

int ensure_xh_tiled(DevCtx* ctx, size_t bytes_per_slot)
{
    EXL3B_CHECK(bytes_per_slot <= ctx->xh_tiled_slot_bytes, EXL3B_ERR_UNSUPPORTED,
                "exl3_gemm: %zu bytes of tiled activations per pass exceed the library's fixed buffer (%zu: 256 rows x k <= %d)",
                bytes_per_slot, ctx->xh_tiled_slot_bytes, DevCtx::XH_MAX_K);
    return 0;
}

}  // namespace exl3b

namespace exl3b { void tc_set_debug_buffer(unsigned long long* d); }
using namespace exl3b;

extern "C" {

int exl3b_abi_version(void) { return EXL3B_ABI_VERSION; }

const char* exl3b_last_error(void) { return g_err.c_str(); }

int64_t exl3b_launch_count(void) { return g_launches.load(); }

int exl3b_set_gemm_path(int tag) { return g_force_path.exchange(tag); }

// bring-up aid (not in the public header): per-CTA %globaltimer stamps of the tensor-core kernels, 16 x u64 per CTA
void exl3b_debug_tc_timeline(void* dev_buf) { exl3b::tc_set_debug_buffer((unsigned long long*) dev_buf); }
void exl3b_debug_reconstruct_had(int mode) { exl3b::reconstruct_had_set_mode(mode); }

int exl3b_num_sms(int device)
{
    cudaDeviceProp prop;
    EXL3B_CUDA(cudaGetDeviceProperties(&prop, device));
    return prop.multiProcessorCount;
}

int exl3b_cc(int device)
{
    cudaDeviceProp prop;
    EXL3B_CUDA(cudaGetDeviceProperties(&prop, device));
    return prop.major * 10 + prop.minor;
}

static int check_kcb(int K, int cb)
{
    EXL3B_CHECK(K >= 1 && K <= 8, EXL3B_ERR_ARG, "K must be 1..8, got %d", K);
    EXL3B_CHECK(cb >= 0 && cb <= 2, EXL3B_ERR_ARG, "cb must be 0 (3inst), 1 (mcg) or 2 (mul1), got %d", cb);
    return 0;
}

// The size checks of the GEMM entries, after the entry's own argument checks: the entry's lower bounds (m >= m_min, k and
// n >= kn_min, else the message `bounds`), then k and n multiples of 128 (messages prefixed with `who`).  Fills the shape
// fields of *g; the caller sets the pointers.
static int gemm_args(const char* who, const char* bounds, int m_min, int kn_min, int m, int k, int n, int K, int cb, int c_fp32,
                     int force_num_sms, GemmArgs* g)
{
    EXL3B_CHECK(m >= m_min && k >= kn_min && n >= kn_min, EXL3B_ERR_SHAPE, "%s", bounds);
    EXL3B_CHECK(k % 128 == 0, EXL3B_ERR_SHAPE, "%s: k (%d) must be divisible by 128", who, k);
    EXL3B_CHECK(n % 128 == 0, EXL3B_ERR_SHAPE, "%s: n (%d) must be divisible by 128", who, n);
    *g = GemmArgs{};
    g->m = m; g->k = k; g->n = n; g->K = K; g->cb = cb; g->c_fp32 = c_fp32 != 0; g->out_scale = 1.0f;
    g->max_ctas = force_num_sms > 0 ? force_num_sms : 0;
    return 0;
}

int exl3b_had_r_128(void* stream, const void* in, void* out, const void* pre_scale, const void* post_scale,
                    float scale, int rows, int cols, int is_fp32)
{
    EXL3B_CHECK(rows >= 0 && cols >= 0, EXL3B_ERR_SHAPE, "had_r_128: negative size");
    EXL3B_CHECK(cols % 128 == 0, EXL3B_ERR_SHAPE, "had_r_128: dim 1 (%d) must be divisible by 128", cols);
    if (rows == 0 || cols == 0) return 0;
    EXL3B_CHECK(in && out, EXL3B_ERR_ARG, "had_r_128: null tensor");
    DevCtx* ctx; int r = get_ctx(&ctx); if (r) return r;
    return launch_had_r_128((cudaStream_t) stream, in, out, (const half*) pre_scale, (const half*) post_scale,
                            scale, rows, cols, is_fp32 != 0);
}

int exl3b_reconstruct(void* stream, void* unpacked, const void* packed, int k, int n_out, int packed_tiles_n,
                      int K, int cb, int64_t n_offset)
{
    int r = check_kcb(K, cb); if (r) return r;
    EXL3B_CHECK(k >= 0 && k % 16 == 0, EXL3B_ERR_SHAPE, "reconstruct: K dimension (%d) must be divisible by 16", k);
    if (k == 0 || n_out == 0) return 0;
    EXL3B_CHECK(n_out % 128 == 0, EXL3B_ERR_SHAPE, "unpacked N dimension must be divisible by 128");
    EXL3B_CHECK(n_offset % 128 == 0, EXL3B_ERR_SHAPE, "n_offset must be divisible by 128");
    EXL3B_CHECK(n_offset >= 0, EXL3B_ERR_SHAPE, "n_offset must be non-negative");
    EXL3B_CHECK(n_offset + n_out <= (int64_t) packed_tiles_n * 16, EXL3B_ERR_SHAPE,
                "reconstruct slice exceeds packed tensor bounds");
    EXL3B_CHECK(unpacked && packed, EXL3B_ERR_ARG, "reconstruct: null tensor");
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    return launch_reconstruct((cudaStream_t) stream, (half*) unpacked, (const uint16_t*) packed, k, n_out,
                              packed_tiles_n, K, cb, n_offset);
}

int exl3b_reconstruct_had(void* stream, void* unpacked, const void* packed, const void* suh, const void* svh,
                          int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset)
{
    int r = check_kcb(K, cb); if (r) return r;
    if (k == 0 || n_out == 0) return 0;
    EXL3B_CHECK(k % 128 == 0, EXL3B_ERR_SHAPE, "reconstruct_had: K dimension must be divisible by 128");
    EXL3B_CHECK(n_out % 128 == 0, EXL3B_ERR_SHAPE, "reconstruct_had: N dimension must be divisible by 128");
    EXL3B_CHECK(n_offset % 128 == 0, EXL3B_ERR_SHAPE, "n_offset must be divisible by 128");
    EXL3B_CHECK(n_offset >= 0, EXL3B_ERR_SHAPE, "n_offset must be non-negative");
    EXL3B_CHECK(n_offset + n_out <= (int64_t) packed_tiles_n * 16, EXL3B_ERR_SHAPE,
                "reconstruct slice exceeds packed tensor bounds");
    EXL3B_CHECK(unpacked && packed && suh && svh, EXL3B_ERR_ARG, "reconstruct_had: null tensor");
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    if (reconstruct_had_tc_enabled())
        return launch_reconstruct_had_tc((cudaStream_t) stream, (half*) unpacked, (const uint16_t*) packed, (const half*) suh,
                                         (const half*) svh, k, n_out, packed_tiles_n, K, cb, n_offset, ctx->num_sms);
    return launch_reconstruct_had((cudaStream_t) stream, (half*) unpacked, (const uint16_t*) packed,
                                  (const half*) suh, (const half*) svh, k, n_out, packed_tiles_n, K, cb, n_offset);
}

// Path selection: auto = int8 tensor-core codebook path for mul1 at m <= 4 (like the reference, whose default for mul1 at
// m <= 2 is its int8 GEMV, exl3_gemm.cu:182-186), else the bit-exact tensor-core path; exl3b_set_gemm_path overrides.
// Rows 5..8 exist on the int8 path (forced) but are not selected automatically: its two per-unit digit warps quantise
// every row of every unit, a cost that grows with m while the exact path's per-unit work does not.
static int select_gemm_path(const GemmArgs& g, int force_shape_idx = -1)
{
    int path = g_force_path.load();
    if (path == EXL3B_TAG_TC_I8_ROUTED) path = 0;            // only concerns exl3b_mgemm
    // per-call kernel choice, the role of the reference's force_shape_idx (exl3_gemm.cuh:28; science/qgemm_benchmark.py times
    // every "shape" 1..exl3_gemm_num_kernel_shapes() this way): 1 = CUDA-core twin, 2 = exact tensor-core kernel; <= 0 = automatic
    if (force_shape_idx > 0)
    {
        EXL3B_CHECK(force_shape_idx <= 2, EXL3B_ERR_ARG, "exl3_gemm: force_shape_idx %d out of range (1 = CUDA-core, 2 = tensor-core)", force_shape_idx);
        path = force_shape_idx == 1 ? EXL3B_TAG_SIMT : EXL3B_TAG_TC;
    }
    if (path == EXL3B_TAG_TC_I8_CHAIN)
    {
        EXL3B_CHECK(gemm_chain_supported(g), EXL3B_ERR_UNSUPPORTED, "exl3_gemm: chain kernel forced but unsupported (needs mul1, m <= 4)");
        return EXL3B_TAG_TC_I8_CHAIN;
    }
    if (path == EXL3B_TAG_TC_I8)
        EXL3B_CHECK(gemm_tc_i8_supported(g), EXL3B_ERR_UNSUPPORTED, "exl3_gemm: int8 tensor-core path forced but unsupported (needs mul1, m <= 4, or m <= 8 with m * k <= 32768)");
    if (path == EXL3B_TAG_TC)
        EXL3B_CHECK(gemm_tc_supported(g), EXL3B_ERR_UNSUPPORTED, "exl3_gemm: tensor-core path forced but shape unsupported");
    if ((path == EXL3B_TAG_TC_I8 || (path == 0 && g.m <= 4)) && gemm_tc_i8_supported(g)) return EXL3B_TAG_TC_I8;
    if (path != EXL3B_TAG_SIMT && gemm_tc_supported(g)) return EXL3B_TAG_TC;
    return EXL3B_TAG_SIMT;
}

int exl3b_gemm_plan(int m, int k, int n, int K, int cb, int num_sms, int force_num_sms, struct exl3b_plan* out)
{
    int r = check_kcb(K, cb); if (r) return r;
    EXL3B_CHECK(out, EXL3B_ERR_ARG, "exl3_gemm_plan: null output");
    GemmArgs g;
    r = gemm_args("exl3_gemm", "exl3_gemm_plan: empty problem", 1, 128, m, k, n, K, cb, 0, force_num_sms, &g); if (r) return r;
    EXL3B_CHECK(num_sms >= 1, EXL3B_ERR_ARG, "exl3_gemm_plan: num_sms must be positive");
    const int path = select_gemm_path(g);
    if (path < 0) return path;
    memset(out, 0, sizeof(*out));
    out->path = path;
    if (path == EXL3B_TAG_SIMT) return 0;
    TcPlan pl{};
    const int m_pass = path == EXL3B_TAG_TC && m > 128 ? 128 : m;
    r = path == EXL3B_TAG_TC_I8 ? plan_gemm_tc_i8(m, k, n, K, num_sms, g.max_ctas, &pl)
                                : plan_gemm_tc(m_pass, k, n, K, num_sms, g.max_ctas, &pl);
    if (r) return r;
    out->passes = path == EXL3B_TAG_TC ? (m + 127) / 128 : 1;
    out->rows = pl.rows; out->grid = pl.grid; out->stages = pl.stages; out->smem_bytes = pl.smem_total;
    out->d_bufs = pl.d_bufs; out->units = pl.units;
    return 0;
}

int exl3b_plan_unit_range(int64_t units, int grid, int cta, int64_t* begin, int64_t* end)
{
    EXL3B_CHECK(units >= 1 && grid >= 1 && grid <= units && partition_fits(units, grid) && cta >= 0 && cta < grid && begin && end, EXL3B_ERR_ARG, "exl3_plan_unit_range: bad argument");
    *begin = unit_begin((int) units, grid, cta); *end = unit_begin((int) units, grid, cta + 1);
    return 0;
}

int exl3b_plan_cta_of_unit(int64_t units, int grid, int64_t unit)
{
    EXL3B_CHECK(units >= 1 && grid >= 1 && grid <= units && partition_fits(units, grid) && unit >= 0 && unit < units, EXL3B_ERR_ARG, "exl3_plan_cta_of_unit: bad argument");
    return cta_of_unit((int) units, grid, (int) unit);
}

int exl3b_gemm(void* stream_, const void* A, const void* B, void* C, const void* suh, void* A_had, const void* svh,
               int m, int k, int n, int K, int cb, int c_fp32, int force_shape_idx, int force_num_sms)
{
    cudaStream_t stream = (cudaStream_t) stream_;
    int r = check_kcb(K, cb); if (r) return r;
    EXL3B_CHECK(force_shape_idx <= 2, EXL3B_ERR_ARG, "exl3_gemm: force_shape_idx %d out of range (1 = CUDA-core, 2 = tensor-core)", force_shape_idx);
    GemmArgs g;
    r = gemm_args("exl3_gemm", "exl3_gemm: negative size", 0, 0, m, k, n, K, cb, c_fp32, force_num_sms, &g); if (r) return r;
    if (m == 0 || n == 0) return EXL3B_TAG_NOP;
    EXL3B_CHECK(A && B && C, EXL3B_ERR_ARG, "exl3_gemm: null tensor");
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    g.A = (const half*) A; g.suh = (const half*) suh; g.A_had = (half*) A_had; g.B = (const uint32_t*) B; g.C = C; g.svh = (const half*) svh;

    int path = select_gemm_path(g, force_shape_idx);
    if (path < 0) return path;
    if (path == EXL3B_TAG_TC_I8_CHAIN) return launch_gemm_chain(stream, ctx, g);
    if (path == EXL3B_TAG_TC_I8) return launch_gemm_tc_i8(stream, ctx, g);
    if (path == EXL3B_TAG_TC) return launch_gemm_tc(stream, ctx, g);
    return launch_gemm_simt(stream, ctx, g);
}

int exl3b_act_mul(void* stream, const void* g, const void* u, void* a, int64_t numel, int in_fp32, int act, float act_limit)
{
    EXL3B_CHECK(act >= ACT_SILU && act <= ACT_RELU2, EXL3B_ERR_ARG, "act_mul: act must be 0 (SiLU), 1 (GELU) or 2 (ReLU^2), got %d", act);
    EXL3B_CHECK(numel >= 0, EXL3B_ERR_SHAPE, "act_mul: negative size");
    if (numel == 0) return 0;
    EXL3B_CHECK(g && u && a, EXL3B_ERR_ARG, "act_mul: null tensor");
    DevCtx* ctx; int r = get_ctx(&ctx); if (r) return r;
    return launch_act_mul((cudaStream_t) stream, g, u, (half*) a, (long long) numel, in_fp32 != 0, act, act_limit);
}

// Elements per load unit of the norm kernels: 8 (16-byte vectors) when dim allows it and every tensor is 16-byte aligned, else 4,
// which needs 4-element alignment (8 bytes for 16-bit types, 16 for fp32); 0 = misaligned
static int norm_unit(int dim, const void* const* ptrs, const int* dtypes, int n)
{
    bool e8 = dim % 8 == 0, e4 = true;
    for (int i = 0; i < n; ++i)
    {
        if (!ptrs[i]) continue;
        const uintptr_t p = (uintptr_t) ptrs[i];
        e8 = e8 && p % 16 == 0;
        e4 = e4 && p % (dtypes[i] == EXL3B_DTYPE_FP32 ? 16 : 8) == 0;
    }
    return e8 ? 8 : (e4 ? 4 : 0);
}

int exl3b_rms_norm(void* stream, const void* x, const void* w, void* y, void* r, int64_t rows, int dim,
                   int x_dtype, int w_dtype, int y_dtype, int r_dtype, int res_mode,
                   float eps, float constant_bias, float constant_scale)
{
    EXL3B_CHECK(res_mode >= EXL3B_RES_NONE && res_mode <= EXL3B_RES_IN, EXL3B_ERR_ARG, "rms_norm: res_mode must be 0 (none), 1 (post) or 2 (in), got %d", res_mode);
    EXL3B_CHECK(rows >= 0 && dim >= 0, EXL3B_ERR_SHAPE, "rms_norm: negative size");
    EXL3B_CHECK(dim % 4 == 0, EXL3B_ERR_SHAPE, "x dimension -1 must be divisible by 4");
    if (!w) w_dtype = EXL3B_DTYPE_FP16;
    if (res_mode != EXL3B_RES_IN) r_dtype = x_dtype;
    // the reference's table: x fp16 / fp32, w fp16 / bf16, y fp16 / fp32 (fp16 in RES_IN), r fp16 / fp32 (RES_IN) or x's type
    EXL3B_CHECK((x_dtype == EXL3B_DTYPE_FP16 || x_dtype == EXL3B_DTYPE_FP32) && (w_dtype == EXL3B_DTYPE_FP16 || w_dtype == EXL3B_DTYPE_BF16)
                && (y_dtype == EXL3B_DTYPE_FP16 || (y_dtype == EXL3B_DTYPE_FP32 && res_mode != EXL3B_RES_IN))
                && (r_dtype == EXL3B_DTYPE_FP16 || r_dtype == EXL3B_DTYPE_FP32), EXL3B_ERR_ARG, "rms_norm: Invalid datatypes for input/output");
    if (rows == 0 || dim == 0) return 0;
    EXL3B_CHECK(dim <= NORM_MAX_DIM, EXL3B_ERR_UNSUPPORTED, "rms_norm: dim %d exceeds the %d elements a row may have", dim, NORM_MAX_DIM);
    EXL3B_CHECK(res_mode != EXL3B_RES_IN || r, EXL3B_ERR_ARG, "rms_norm: res_mode RES_IN requires residual tensor");
    EXL3B_CHECK(x && y, EXL3B_ERR_ARG, "rms_norm: null tensor");
    const void* ptrs[4] = {x, w, y, res_mode == EXL3B_RES_IN ? r : nullptr};
    const int dts[4] = {x_dtype, w_dtype, y_dtype, r_dtype};
    const int e = norm_unit(dim, ptrs, dts, 4);
    EXL3B_CHECK(e, EXL3B_ERR_ARG, "rms_norm: x, w, y and r must be aligned to 4 of their elements");
    NormArgs a{};
    a.x = x; a.w = w; a.y = y; a.r = res_mode == EXL3B_RES_IN ? r : nullptr; a.rows = rows; a.dim = dim;
    a.x_dtype = x_dtype; a.w_dtype = w_dtype; a.y_dtype = y_dtype; a.r_dtype = r_dtype; a.res_mode = res_mode;
    a.eps = eps; a.bias = constant_bias; a.scale = constant_scale; a.e = e;
    DevCtx* ctx; int rc = get_ctx(&ctx); if (rc) return rc;
    return launch_rms_norm((cudaStream_t) stream, a);
}

int exl3b_gated_rms_norm(void* stream, const void* x, const void* w, void* y, const void* g, int64_t rows, int dim,
                         int x_dtype, int w_dtype, int y_dtype, int g_dtype, int w_groups, int gate_first,
                         float eps, float constant_bias)
{
    EXL3B_CHECK(rows >= 0 && dim >= 0, EXL3B_ERR_SHAPE, "gated_rms_norm: negative size");
    EXL3B_CHECK(dim % 4 == 0, EXL3B_ERR_SHAPE, "x dimension -1 must be divisible by 4");
    EXL3B_CHECK(w_groups >= 1, EXL3B_ERR_ARG, "gated_rms_norm: w_groups must be positive, got %d", w_groups);
    EXL3B_CHECK(x_dtype == EXL3B_DTYPE_BF16 && (w_dtype == EXL3B_DTYPE_FP32 || w_dtype == EXL3B_DTYPE_BF16)
                && (y_dtype == EXL3B_DTYPE_FP16 || y_dtype == EXL3B_DTYPE_FP32) && (g_dtype == EXL3B_DTYPE_FP32 || g_dtype == EXL3B_DTYPE_BF16),
                EXL3B_ERR_ARG, "gated_rms_norm: Invalid datatypes for input/output");
    if (rows == 0 || dim == 0) return 0;
    EXL3B_CHECK(dim <= NORM_MAX_DIM, EXL3B_ERR_UNSUPPORTED, "gated_rms_norm: dim %d exceeds the %d elements a row may have", dim, NORM_MAX_DIM);
    EXL3B_CHECK(x && w && y && g, EXL3B_ERR_ARG, "gated_rms_norm: null tensor");
    const void* ptrs[4] = {x, w, y, g};
    const int dts[4] = {x_dtype, w_dtype, y_dtype, g_dtype};
    const int e = norm_unit(dim, ptrs, dts, 4);
    EXL3B_CHECK(e, EXL3B_ERR_ARG, "gated_rms_norm: x, w, y and g must be aligned to 4 of their elements");
    NormArgs a{};
    a.x = x; a.w = w; a.y = y; a.g = g; a.rows = rows; a.dim = dim;
    a.x_dtype = x_dtype; a.w_dtype = w_dtype; a.y_dtype = y_dtype; a.g_dtype = g_dtype;
    a.eps = eps; a.bias = constant_bias; a.w_groups = w_groups; a.gate_first = gate_first != 0; a.e = e;
    DevCtx* ctx; int rc = get_ctx(&ctx); if (rc) return rc;
    return launch_gated_rms_norm((cudaStream_t) stream, a);
}

// exl3b_gemm on the rows fp16(act(G) * U): the path exl3b_gemm takes for (m, k, n, K, cb), restricted to the two kernels with a
// gated input stage (tag 210 at m <= 4, tag 200 at m <= 8); any other choice is refused, never replaced
int exl3b_gemm_gated(void* stream, const void* G, const void* U, const void* B, void* C, const void* suh, const void* svh,
                     int m, int k, int n, int K, int cb, int c_fp32, int gu_fp32, int act, float act_limit, int force_num_sms)
{
    int r = check_kcb(K, cb); if (r) return r;
    EXL3B_CHECK(act >= ACT_SILU && act <= ACT_RELU2, EXL3B_ERR_ARG, "exl3_gemm_gated: act must be 0 (SiLU), 1 (GELU) or 2 (ReLU^2), got %d", act);
    GemmArgs g;
    r = gemm_args("exl3_gemm_gated", "exl3_gemm_gated: negative size", 0, 0, m, k, n, K, cb, c_fp32, force_num_sms, &g); if (r) return r;
    if (m == 0 || n == 0) return EXL3B_TAG_NOP;
    EXL3B_CHECK(m <= 8, EXL3B_ERR_UNSUPPORTED, "exl3_gemm_gated: gated input is implemented for 1..8 rows, got %d", m);
    EXL3B_CHECK(G && U && B && C, EXL3B_ERR_ARG, "exl3_gemm_gated: null tensor");
    const uintptr_t align = gu_fp32 ? 16 : 8;
    EXL3B_CHECK((uintptr_t) G % align == 0 && (uintptr_t) U % align == 0, EXL3B_ERR_ARG,
                "exl3_gemm_gated: G and U must be %d-byte aligned", (int) align);
    g.suh = (const half*) suh; g.B = (const uint32_t*) B; g.C = C; g.svh = (const half*) svh;
    const int path = select_gemm_path(g);
    if (path < 0) return path;
    EXL3B_CHECK(path == EXL3B_TAG_TC || (path == EXL3B_TAG_TC_I8 && m <= 4), EXL3B_ERR_UNSUPPORTED,
                "exl3_gemm_gated: the call selects path %d at m = %d; gated input exists on paths 210 (m <= 4) and 200", path, m);
    GateIn gate{G, U, gu_fp32 != 0, act, act_limit};
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    if (path == EXL3B_TAG_TC_I8) return launch_gemm_tc_i8((cudaStream_t) stream, ctx, g, &gate);
    return launch_gemm_tc((cudaStream_t) stream, ctx, g, &gate);
}

int exl3b_gemm_allreduce(void* stream_, const void* A, const void* B, void* C, const void* suh, void* A_had, const void* svh,
                         int m, int k, int n, int K, int cb, int c_fp32)
{
    (void) A_had;                                   // the transform runs inside the kernel (m <= 4): no scratch is written
    int r = check_kcb(K, cb); if (r) return r;
    GemmArgs g;
    r = gemm_args("exl3_gemm_allreduce", "exl3_gemm_allreduce: bad size", 1, 0, m, k, n, K, cb, c_fp32, 0, &g); if (r) return r;
    EXL3B_CHECK(A && B && C, EXL3B_ERR_ARG, "exl3_gemm_allreduce: null tensor");
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    g.A = (const half*) A; g.suh = (const half*) suh; g.B = (const uint32_t*) B; g.C = C; g.svh = (const half*) svh;
    return launch_gemm_tc_i8_ar((cudaStream_t) stream_, ctx, g);
}

int exl3b_gemm_allreduce_check(int m, int k, int n, int K, int cb, int world, int64_t max_elems)
{
    const char* why = gemm_tc_i8_ar_unsupported(m, k, n, K, cb, world, (long long) max_elems);
    EXL3B_CHECK(!why, EXL3B_ERR_UNSUPPORTED, "exl3_gemm_allreduce: %s", why ? why : "");
    return 0;
}

int exl3b_tp_alloc(int rank, int world, int64_t max_elems, void* handle_out) { return tp_alloc(rank, world, (long long) max_elems, handle_out); }
int exl3b_tp_attach(const void* handles, int world) { return tp_attach(handles, world); }
int exl3b_tp_attach_loopback(void) { return tp_attach_loopback(); }
int exl3b_tp_info(int* rank, int* world, int64_t* max_elems, int* attached)
{
    long long me = 0;
    int r = tp_info(rank, world, &me, attached);
    if (max_elems) *max_elems = me;
    return r;
}
int exl3b_tp_free(void) { return tp_free(); }
int exl3b_tp_debug_inject(void* stream, int src_rank, const void* partial, int64_t count) { return tp_debug_inject((cudaStream_t) stream, src_rank, partial, (long long) count); }
int exl3b_tp_debug_peek(int buffer_rank, int slot, int src_rank, void* host_out, int64_t count) { return tp_debug_peek(buffer_rank, slot, src_rank, host_out, (long long) count); }
int64_t exl3b_tp_debug_epoch(void) { return tp_debug_epoch(); }

// Host copies of size_n_list tensors (device int32) the caller vouches for: the fan-out launch geometry (CTA groups, row pitch)
// depends on the widths, and the reference's operator only hands over the device tensor.  Keyed by the device address.
static std::mutex g_widths_mu;
static std::unordered_map<const void*, std::vector<int32_t>> g_widths;

int exl3b_register_widths(const int32_t* size_n_list, const int32_t* host_widths, int count)
{
    EXL3B_CHECK(size_n_list, EXL3B_ERR_ARG, "register_widths: null device pointer");
    EXL3B_CHECK(count >= 0 && (count == 0 || host_widths), EXL3B_ERR_ARG, "register_widths: bad host list");
    std::lock_guard<std::mutex> lock(g_widths_mu);
    if (count == 0) g_widths.erase(size_n_list);
    else g_widths[size_n_list] = std::vector<int32_t>(host_widths, host_widths + count);
    return 0;
}

int exl3b_plan_fanout(int k, const int32_t* host_widths, int count, int num_sms, int32_t* cta0)
{
    EXL3B_CHECK(host_widths && cta0 && num_sms >= 1, EXL3B_ERR_ARG, "plan_fanout: bad argument");
    return plan_fanout_groups(k, host_widths, count, num_sms, cta0);
}

int exl3b_mgemm(void* stream, const void* A, const uint64_t* B_ptrs, void* C, const uint64_t* suh_ptrs, void* A_had,
                const uint64_t* svh_ptrs, const int64_t* indices, int num_indices, const void* weights,
                int bszm_in, int bszm_out, int m, int k, int n, int K, int cb, int c_fp32,
                int min_index, int max_index, int num_tokens,
                const int32_t* size_n_list, const uint64_t* c_ptrs, int num_c_ptrs,
                int force_shape_idx, int force_num_sms)
{
    (void) force_shape_idx; (void) force_num_sms;
    int r = check_kcb(K, cb); if (r) return r;
    EXL3B_CHECK(num_tokens == 1 || min_index < 0, EXL3B_ERR_ARG,
                "exl3_mgemm: multi-token reduction (num_tokens > 1) is not compatible with expert-range "
                "filtering (min_index >= 0); TP-sharded experts must use num_tokens == 1");
    EXL3B_CHECK(num_tokens >= 1, EXL3B_ERR_ARG, "exl3_mgemm: num_tokens must be >= 1");
    EXL3B_CHECK(k % 128 == 0, EXL3B_ERR_SHAPE, "exl3_mgemm: k (%d) must be divisible by 128", k);
    EXL3B_CHECK(n % 128 == 0, EXL3B_ERR_SHAPE, "exl3_mgemm: n (%d) must be divisible by 128", n);
    if (size_n_list)
    {
        EXL3B_CHECK(c_ptrs, EXL3B_ERR_ARG, "exl3_mgemm: size_n_list requires c_ptrs");
        EXL3B_CHECK(num_tokens == 1 && min_index < 0 && !weights, EXL3B_ERR_ARG,
                    "exl3_mgemm: per-matrix widths incompatible with multi-token/filtering/weights");
        bszm_out = num_c_ptrs;
    }
    EXL3B_CHECK(min_index < 0 || indices, EXL3B_ERR_ARG, "exl3_mgemm: expert-range filtering requires indices");
    EXL3B_CHECK(!weights || indices, EXL3B_ERR_ARG, "exl3_mgemm: weights require indices");
    if (indices)
        EXL3B_CHECK(num_indices <= bszm_in || num_indices <= bszm_out, EXL3B_ERR_SHAPE,
                    "mgemm: too many indices for tensor batch");
    EXL3B_CHECK(A && B_ptrs && C && suh_ptrs && A_had && svh_ptrs, EXL3B_ERR_ARG, "exl3_mgemm: null tensor");
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    MGemmArgs a{};
    a.A = (const half*) A; a.B_ptrs = B_ptrs; a.C = C; a.suh_ptrs = suh_ptrs; a.A_had = (half*) A_had;
    a.svh_ptrs = svh_ptrs; a.indices = indices; a.num_indices = num_indices; a.weights = (const half*) weights;
    a.bszm_in = bszm_in; a.bszm_out = bszm_out; a.m = m; a.k = k; a.n = n; a.K = K; a.cb = cb;
    a.c_fp32 = c_fp32 != 0; a.min_index = min_index; a.max_index = max_index; a.num_tokens = num_tokens;
    a.size_n_list = size_n_list; a.c_ptrs = c_ptrs; a.num_c_ptrs = num_c_ptrs;
    std::vector<int32_t> widths;                    // copy: the registry may change under another thread
    if (size_n_list)
    {
        std::lock_guard<std::mutex> lock(g_widths_mu);
        auto it = g_widths.find(size_n_list);
        if (it != g_widths.end() && (int) it->second.size() == num_c_ptrs) { widths = it->second; a.size_n_host = widths.data(); }
    }
    const int path = g_force_path.load();
    if ((path == EXL3B_TAG_TC_I8 || path == EXL3B_TAG_TC_I8_ROUTED || (path == 0 && m <= 4)) && mgemm_tc_i8_supported(ctx, a))
        return launch_mgemm_tc_i8((cudaStream_t) stream, ctx, a);
    // routed / weighted calls (MoE decode: indices, weights, expert-range filter) with mul1 at <= 4 rows: the tensor-core
    // kernel with one CTA group per active slot (EXL3B_TAG_SIMT still forces the CUDA-core twin)
    if ((path == 0 || path == EXL3B_TAG_TC_I8 || path == EXL3B_TAG_TC_I8_ROUTED) && (a.indices || a.weights || a.min_index >= 0)
        && mgemm_tc_i8_routed_supported(ctx, a))
        return launch_mgemm_tc_i8_routed((cudaStream_t) stream, ctx, a);
    return launch_mgemm((cudaStream_t) stream, ctx, a);
}

int exl3b_chain_plan(const struct exl3b_chain_op* ops, int n_ops, int num_sms, struct exl3b_chain_plan* out)
{
    EXL3B_CHECK(out && num_sms >= 1, EXL3B_ERR_ARG, "exl3_chain_plan: bad argument");
    return chain_plan(ops, n_ops, num_sms, out);
}

int exl3b_chain_walk(const struct exl3b_chain_op* ops, int n_ops, int num_sms, int cta, int32_t* out, int max_units)
{
    return chain_walk(ops, n_ops, num_sms, cta, out, max_units);
}

int exl3b_chain_create(const struct exl3b_chain_op* ops, int n_ops, void** chain)
{
    DevCtx* ctx; int r = get_ctx(&ctx); if (r) return r;
    return chain_create(ctx, ops, n_ops, chain);
}

int exl3b_chain_run(void* stream, void* chain) { return chain_run((cudaStream_t) stream, chain); }

int exl3b_chain_destroy(void* chain) { return chain_destroy(chain); }

int exl3b_moe_max_concurrency(int device)
{
    const int sms = exl3b_num_sms(device);
    return sms < 0 ? sms : sms / 8;
}

int exl3b_moe_plan(const int64_t* expert_count_host, int num_experts, int max_tokens, int num_positions, int hidden,
                   int intermediate, struct exl3b_moe_plan* out, int32_t* passes_out, int32_t* pos_code_out)
{
    return moe_plan_host(expert_count_host, num_experts, max_tokens, num_positions, hidden, intermediate, out, passes_out,
                         pos_code_out);
}

// validation of exllamav3_ext/quant/exl3_moe.cu:143-200 that needs no tensor types, plus this library's own limits
int exl3b_moe(void* stream, const void* hidden_state, void* output_state,
              const int64_t* expert_count, const int64_t* token_sorted, const void* weight_sorted,
              int bsz, int hidden, int intermediate, int num_experts, int num_positions, int max_tokens, int concurrency,
              int act_function, int K_gate, int K_up, int K_down,
              const uint64_t* gate_trellis, const uint64_t* gate_suh, const uint64_t* gate_svh,
              const uint64_t* up_trellis, const uint64_t* up_suh, const uint64_t* up_svh,
              const uint64_t* down_trellis, const uint64_t* down_suh, const uint64_t* down_svh,
              int gate_mcg, int gate_mul1, int up_mcg, int up_mul1, int down_mcg, int down_mul1,
              float act_limit, int num_active)
{
    if (num_active == 0) return EXL3B_TAG_NOP;
    EXL3B_CHECK(gate_mcg == up_mcg && up_mcg == down_mcg && gate_mul1 == up_mul1 && up_mul1 == down_mul1, EXL3B_ERR_ARG,
                "MoE kernel: gate/up/down must share the same codebook");
    EXL3B_CHECK((gate_mcg != 0) != (gate_mul1 != 0), EXL3B_ERR_ARG, "MoE kernel: Only mcg and mul1 codebooks are supported");
    EXL3B_CHECK(act_function >= 0 && act_function <= 2, EXL3B_ERR_ARG, "exl3_moe: act_function must be 0 (SiLU), 1 (GELU) or 2 (ReLU^2), got %d", act_function);
    for (int K : {K_gate, K_up, K_down}) EXL3B_CHECK(K >= 1 && K <= 8, EXL3B_ERR_ARG, "K must be 1..8, got %d", K);
    EXL3B_CHECK(bsz >= 0 && num_positions >= 0 && max_tokens >= 1 && concurrency >= 1, EXL3B_ERR_SHAPE, "exl3_moe: bad sizes");
    EXL3B_CHECK(hidden >= 128 && hidden % 128 == 0, EXL3B_ERR_SHAPE, "exl3_moe: hidden size (%d) must be divisible by 128", hidden);
    EXL3B_CHECK(intermediate >= 128 && intermediate % 128 == 0, EXL3B_ERR_SHAPE,
                "exl3_moe: intermediate size (%d) must be divisible by 128", intermediate);
    EXL3B_CHECK(num_experts >= 1 && num_experts <= MOE_MAX_EXPERTS, EXL3B_ERR_UNSUPPORTED,
                "exl3_moe: 1..%d experts supported, got %d", MOE_MAX_EXPERTS, num_experts);
    EXL3B_CHECK(hidden_state && output_state && expert_count && token_sorted && weight_sorted && gate_trellis && gate_suh
                && gate_svh && up_trellis && up_suh && up_svh && down_trellis && down_suh && down_svh, EXL3B_ERR_ARG,
                "exl3_moe: null tensor");
    EXL3B_CHECK(((uintptr_t) hidden_state & 7) == 0 && ((uintptr_t) output_state & 15) == 0, EXL3B_ERR_ARG,
                "exl3_moe: hidden_state must be 8-byte and output_state 16-byte aligned");
    DevCtx* ctx; int r = get_ctx(&ctx); if (r) return r;
    EXL3B_CHECK((long long) concurrency * 8 <= ctx->num_sms, EXL3B_ERR_ARG, "Concurrency too high for device num_sms");
    if (bsz == 0 || num_positions == 0) return EXL3B_TAG_NOP;
    MoeArgs a{};
    a.hidden_state = (const half*) hidden_state; a.output_state = (float*) output_state;
    a.expert_count = expert_count; a.token_sorted = token_sorted; a.weight_sorted = (const half*) weight_sorted;
    a.bsz = bsz; a.hidden = hidden; a.inter = intermediate; a.num_experts = num_experts; a.num_positions = num_positions;
    a.max_tokens = max_tokens; a.act = act_function; a.act_limit = act_limit;
    a.K_gate = K_gate; a.K_up = K_up; a.K_down = K_down; a.cb = gate_mul1 ? 2 : 1;
    a.gate_trellis = gate_trellis; a.gate_suh = gate_suh; a.gate_svh = gate_svh;
    a.up_trellis = up_trellis; a.up_suh = up_suh; a.up_svh = up_svh;
    a.down_trellis = down_trellis; a.down_suh = down_suh; a.down_svh = down_svh;
    a.num_active = num_active;
    return launch_moe((cudaStream_t) stream, ctx, a);
}

int exl3b_quantize_tiles(void* stream, const void* in, void* out_tiles, void* out_idx, int64_t num_tiles, int K, int cb)
{
    int r = check_kcb(K, cb); if (r) return r;
    EXL3B_CHECK(num_tiles >= 0, EXL3B_ERR_SHAPE, "quantize_tiles: negative number of tiles");
    if (num_tiles == 0) return 0;
    EXL3B_CHECK(in && out_tiles && out_idx, EXL3B_ERR_ARG, "quantize_tiles: null tensor");
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;
    return launch_quantize_tiles((cudaStream_t) stream, ctx, (const float*) in, (float*) out_tiles, (uint16_t*) out_idx,
                                 num_tiles, K, cb);
}

int exl3b_pack_trellis(void* stream, void* packed, const void* unpacked, int64_t num_tiles, int K)
{
    EXL3B_CHECK(K >= 1 && K <= 8, EXL3B_ERR_ARG, "K must be 1..8, got %d", K);
    EXL3B_CHECK(num_tiles >= 0, EXL3B_ERR_SHAPE, "pack_trellis: negative number of tiles");
    if (num_tiles == 0) return 0;
    EXL3B_CHECK(packed && unpacked, EXL3B_ERR_ARG, "pack_trellis: null tensor");
    DevCtx* ctx; int r = get_ctx(&ctx); if (r) return r;
    return launch_pack_trellis((cudaStream_t) stream, (uint16_t*) packed, (const uint16_t*) unpacked, num_tiles, K);
}

int exl3b_hgemm(void* stream, const void* a, const void* b, void* c, int m, int k, int n, int c_fp32,
                int64_t c_stride)
{
    EXL3B_CHECK(m >= 0 && k >= 0 && n >= 0, EXL3B_ERR_SHAPE, "hgemm: negative size");
    if (m == 0 || n == 0) return 0;
    EXL3B_CHECK(a && b && c, EXL3B_ERR_ARG, "hgemm: null tensor");
    EXL3B_CHECK(c_stride >= n, EXL3B_ERR_SHAPE, "c row stride is too small");
    DevCtx* ctx; int r = get_ctx(&ctx); if (r) return r;
    return launch_hgemm((cudaStream_t) stream, (const half*) a, (const half*) b, c, m, k, n, c_fp32 != 0, c_stride);
}

int exl3b_gemm_host(void* stream_, const void* A_host, void* C_host, void* d_A, void* d_C, void* d_A_had,
                    const void* B, const void* suh, const void* svh, int m, int k, int n, int K, int cb, int c_fp32)
{
    cudaStream_t stream = (cudaStream_t) stream_;
    EXL3B_CHECK(A_host && C_host && d_A && d_C, EXL3B_ERR_ARG, "exl3_gemm_host: null buffer");
    EXL3B_CUDA(cudaMemcpyAsync(d_A, A_host, (size_t) m * k * sizeof(half), cudaMemcpyHostToDevice, stream));
    int r = exl3b_gemm(stream_, d_A, B, d_C, suh, d_A_had, svh, m, k, n, K, cb, c_fp32, -1, 0);
    if (r < 0) return r;
    EXL3B_CUDA(cudaMemcpyAsync(C_host, d_C, (size_t) m * n * (c_fp32 ? 4 : 2), cudaMemcpyDeviceToHost, stream));
    EXL3B_CUDA(cudaStreamSynchronize(stream));
    return r;
}

}  // extern "C"
