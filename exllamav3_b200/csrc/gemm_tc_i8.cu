// The kernel entries and the shared host side of the wgmma u8 x s8 EXL3 decode-GEMM: shape rule, launch geometry, launch
// parameters and the launch itself, for the plain and gated (tag 210), row-parallel (tag 211, gemm_tc_i8_ar.cu) and routed
// (tag 212, gemm_tc_i8_routed.cu) calls.  The kernel body is in gemm_tc_i8_body.cuh.
#include "gemm_tc_i8_body.cuh"

namespace exl3b {

template <int K, int MR>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_i8_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w)
{
    gemm_tc_i8_body<K, MR, false>(p, &tmap_w, nullptr);
}

// gated input (exl3b_gemm_gated): the rows are fp16(act(G) * U), formed in the prologue; one rows variant (MR = 4), the activation
// kind and the input dtype are warp-uniform values of `gate`
template <int K, int MR>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_i8_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w, const GateIn gate)
{
    gemm_tc_i8_body<K, MR, false, false, true>(p, &tmap_w, nullptr, nullptr, &gate);
}
template <int K, int MR> constexpr void (*i8_plain_kernel)(const TcParams, const CUtensorMap) = gemm_tc_i8_kernel<K, MR>;
template <int K> constexpr void (*i8_gated_kernel)(const TcParams, const CUtensorMap, const GateIn) = gemm_tc_i8_kernel<K, 4>;

// row-parallel: the epilogue sums the ranks' partial outputs over NVLink peer memory (gemm_tc_i8_ar.cu)
template <int K>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_i8_ar_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ ArArgs ar)
{
    gemm_tc_i8_body<K, 4, true>(p, &tmap_w, &ar);
}

// routed: one CTA group per active slot of the call (gemm_tc_i8_routed.cu)
template <int K>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_i8_routed_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ RouteArgs route)
{
    gemm_tc_i8_body<K, 4, false, true>(p, &tmap_w, nullptr, &route);
}

// ---- host side -------------------------------------------------------------------------------------------------------

// the kernel entry of a launch: row-parallel (ar), routed (route), gated rows (gate) or plain rows
template <int K>
static cudaError_t i8_kernel(cudaStream_t stream, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap,
                             const GateIn* gate, const ArArgs* ar, const RouteArgs* route)
{
    const dim3 g(grid);
    if (ar) return launch_pdl<gemm_tc_i8_ar_kernel<K>>(stream, g, TC_THREADS, smem_bytes, p, tmap, *ar);
    if (route) return launch_pdl<gemm_tc_i8_routed_kernel<K>>(stream, g, TC_THREADS, smem_bytes, p, tmap, *route);
    if (gate) return launch_pdl<i8_gated_kernel<K>>(stream, g, TC_THREADS, smem_bytes, p, tmap, *gate);
    return p.m <= 4 ? launch_pdl<i8_plain_kernel<K, 4>>(stream, g, TC_THREADS, smem_bytes, p, tmap)
                    : launch_pdl<i8_plain_kernel<K, 8>>(stream, g, TC_THREADS, smem_bytes, p, tmap);
}

int i8_launch(cudaStream_t stream, int K, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap, const GateIn* gate,
              const ArArgs* ar, const RouteArgs* route)
{
    cudaError_t err = cudaSuccess;
    EXL3B_DISPATCH_K(K, err = i8_kernel<KK>(stream, grid, smem_bytes, p, tmap, gate, ar, route));
    count_launch();
    EXL3B_CUDA(err);
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

TcParams i8_params(DevCtx* ctx, int slot, const TcPlan& pl, const GemmArgs& a)
{
    TcParams p{};
    p.A_raw = a.A; p.suh = a.suh; p.B = a.B; p.svh = a.svh; p.C = a.C;
    p.m = a.m; p.k = a.k; p.n = a.n; p.NT = I8_NT; p.c_fp32 = a.c_fp32; p.out_scale = a.out_scale;
    p.ws = ctx->ws_slot(slot); p.counters = ctx->counter_slot(slot); p.parts = ctx->i8_parts_slot(slot); p.dbg = g_tc_dbg;
    p.stages = pl.stages; p.b_bytes = pl.b_bytes; p.b_load_bytes = pl.b_load_bytes;
    return p;
}

TcParams i8_params(DevCtx* ctx, int slot, const TcPlan& pl, const MGemmArgs& a, int mats)
{
    GemmArgs g{};
    g.A = a.A; g.C = a.C; g.m = a.m; g.k = a.k; g.n = a.n; g.c_fp32 = a.c_fp32; g.out_scale = 1.f;
    TcParams p = i8_params(ctx, slot, pl, g);
    p.num_mats = mats;                           // > 0 selects the table-driven path in the kernel
    p.B_ptrs = a.B_ptrs; p.suh_ptrs = a.suh_ptrs; p.svh_ptrs = a.svh_ptrs;
    p.a_mat_stride = a.bszm_in == 1 ? 0 : (long long) a.m * a.k;
    p.c_mat_stride = (long long) a.m * a.n * (a.c_fp32 ? 4 : 2);
    p.tmap_slots = ctx->tmap_slot(slot);
    return p;
}

const char* i8_shape_unsupported(int m, int k, int n, int K, int cb, bool rows8)
{
    // rows 5..8 need the whole transformed activation cached in shared memory (the per-unit digit warps cannot afford eight
    // Hadamards)
    const bool rows_ok = m >= 1 && (m <= 4 || (rows8 && m <= I8_MAX_M && (size_t) m * k * 2 <= I8_CACHE_MAX_BYTES));
    if (cb != 2) return "needs the mul1 codebook";
    if (!rows_ok) return rows8 ? "needs 1 <= m <= 4, or m <= 8 with m * k <= 32768" : "needs 1 <= m <= 4";
    if (K < 1 || K > 8) return "K out of range";
    if (k < 128 || n < 128 || k % 128 || n % 128) return "k and n must be multiples of 128";
    return nullptr;
}

bool gemm_tc_i8_supported(const GemmArgs& a) { return !i8_shape_unsupported(a.m, a.k, a.n, a.K, a.cb, true); }

// rows variant, ring depth, activation cache and shared memory of a launch (single- and multi-matrix alike)
static int plan_i8_smem(int m, int k, int K, TcPlan* pl)
{
    const int MR = m <= 4 ? 4 : 8;
    const int stage_bytes = 2048 * K + i8_b_stage(MR);
    int cache_bytes = m * k * 2;
    cache_bytes = (cache_bytes + 127) / 128 * 128;
    if (cache_bytes > I8_CACHE_MAX_BYTES) cache_bytes = 0;
    int stages = (200 * 1024 - i8_d_bytes(MR) - cache_bytes) / stage_bytes;
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages < 2) stages = 2;
    const TcSmemLayout L = i8_smem_layout(K, MR, stages, cache_bytes);
    EXL3B_CHECK(L.total <= 220 * 1024, EXL3B_ERR_UNSUPPORTED, "exl3_gemm (i8): shared-memory budget exceeded");
    pl->rows = MR; pl->stages = stages; pl->b_bytes = i8_b_stage(MR); pl->b_load_bytes = cache_bytes; pl->smem_total = L.total;
    return 0;
}

// launch geometry (also behind exl3b_gemm_plan): rows variant, ring depth, activation cache, grid
int plan_gemm_tc_i8(int m, int k, int n, int K, int num_sms, int max_ctas, TcPlan* pl)
{
    { int r = plan_i8_smem(m, k, K, pl); if (r) return r; }
    const long long U = (long long) (k / 128) * (n / 128);
    int grid = num_sms;
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    if (grid > U) grid = (int) U;
    EXL3B_CHECK(n / 128 <= DevCtx::COUNTERS_PER_SLOT, EXL3B_ERR_UNSUPPORTED, "exl3_gemm: too many column strips");
    EXL3B_CHECK(grid <= DevCtx::I8_PART_CTAS, EXL3B_ERR_UNSUPPORTED, "exl3_gemm (i8): grid exceeds the split-K exchange buffer");
    EXL3B_CHECK(partition_fits(U, grid), EXL3B_ERR_UNSUPPORTED, "exl3_gemm (i8): too many units for the 32-bit stream-K partition");
    pl->grid = grid; pl->units = U; pl->d_bufs = 2;
    return 0;
}

int launch_gemm_tc_i8(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a, const GateIn* gate)
{
    EXL3B_CHECK(!gate || a.m <= 4, EXL3B_ERR_UNSUPPORTED, "exl3_gemm_gated (i8): gated input needs m <= 4");
    CUtensorMap tmap;
    { int r = get_weight_tmap(a.B, a.k, a.n, a.K, &tmap); if (r) return r; }
    TcPlan pl;
    { int r = plan_gemm_tc_i8(a.m, a.k, a.n, a.K, ctx->num_sms, a.max_ctas, &pl); if (r) return r; }
    const TcParams p = i8_params(ctx, ctx->next_slot(), pl, a);
    { int r = i8_launch(stream, a.K, pl.grid, pl.smem_total, p, tmap, gate); if (r) return r; }
    return EXL3B_TAG_TC_I8;
}

// Fan-out partition: matrix j gets a share of the persistent grid proportional to its units (k/128 x n_j/128), at least one CTA
// and at most one CTA per unit; the shares are handed out left to right from what is left, so they always sum to the grid.
int plan_fanout_groups(int k, const int32_t* widths, int mats, int num_sms, int* cta0)
{
    if (mats < 1 || mats > TC_RAG_MAX_MATS || mats > num_sms) return 0;
    long long U[TC_RAG_MAX_MATS], Utot = 0;
    for (int j = 0; j < mats; ++j)
    {
        if (widths[j] < 128 || widths[j] % 128) return 0;
        U[j] = (long long) (k / 128) * (widths[j] / 128); Utot += U[j];
        if (!partition_fits(U[j], num_sms)) return 0;
    }
    int grid = num_sms; if (grid > Utot) grid = (int) Utot;
    long long Urem = Utot; int Grem = grid; cta0[0] = 0;
    for (int j = 0; j < mats; ++j)
    {
        const int after = mats - 1 - j;                                        // matrices still to be served: one CTA each at least
        long long g = (Grem * U[j] + Urem / 2) / Urem;
        if (g < 1) g = 1;
        if (g > Grem - after) g = Grem - after;
        if (g > U[j]) g = U[j];
        cta0[j + 1] = cta0[j] + (int) g;
        Grem -= (int) g; Urem -= U[j];
    }
    return cta0[mats];
}

bool mgemm_tc_i8_supported(const DevCtx* ctx, const MGemmArgs& a)
{
    // dense case only: one output per matrix, shared or per-matrix input, no routing / weighting; per-matrix widths (fan-out) only
    // when the caller registered a host copy of the width list (the launch geometry depends on it, and checks the widths)
    if (i8_shape_unsupported(a.m, a.k, a.size_n_list ? 128 : a.n, a.K, a.cb, true)) return false;
    if (a.indices || a.weights || a.min_index >= 0 || a.num_tokens != 1) return false;
    if (a.size_n_list)
    {
        if (!a.size_n_host || !a.c_ptrs) return false;
        if (!(a.bszm_in == 1 || a.bszm_in == a.bszm_out)) return false;
        int cta0[TC_RAG_MAX_MATS + 1];
        return plan_fanout_groups(a.k, a.size_n_host, a.bszm_out, ctx->num_sms, cta0) > 0;
    }
    if (a.bszm_out < 1 || !(a.bszm_in == 1 || a.bszm_in == a.bszm_out)) return false;
    if (a.bszm_out > ctx->num_sms || a.bszm_out > DevCtx::TMAP_SLOTS) return false;
    if ((long long) a.bszm_out * (a.n / 128) > DevCtx::COUNTERS_PER_SLOT) return false;
    return true;
}

// exl3_mgemm, dense case, as ONE launch: the persistent grid is split into bszm_out groups of CTAs, one group per matrix.
// Replaces exl3_mgemm_kernel for the reference's fused k+v and gate+up projections (modules/attn.py:603-631,
// modules/mlp.py:726-760).  The weight tensor map is patched per CTA on the device (the pointer table is device memory).
int launch_mgemm_tc_i8(cudaStream_t stream, DevCtx* ctx, const MGemmArgs& a)
{
    const int mats = a.bszm_out;
    CUtensorMap tmap;
    { int r = get_weight_tmap(ctx->ws, a.k, a.size_n_list ? 128 : a.n, a.K, &tmap); if (r) return r; }     // template: address patched per CTA (unused by fan-out launches)
    const int slot = ctx->next_slot();
    TcPlan pl;
    { int r = plan_i8_smem(a.m, a.k, a.K, &pl); if (r) return r; }
    TcParams p = i8_params(ctx, slot, pl, a, mats);
    const long long U = (long long) (a.k / 128) * (a.n / 128);
    int gpm = ctx->num_sms / mats;
    if (gpm > U) gpm = (int) U;
    EXL3B_CHECK(partition_fits(U, gpm), EXL3B_ERR_UNSUPPORTED, "exl3_mgemm (i8): too many units for the 32-bit stream-K partition");
    p.g_per_mat = gpm;
    int grid = gpm * mats;
    if (a.size_n_list)
    {
        // fan-out: per-matrix widths and output pointers (exl3_gemm_kernel.cuh:172-181); the weights arrive as row copies, no tensor map
        p.rag = 1; p.c_ptrs = a.c_ptrs;
        grid = plan_fanout_groups(a.k, a.size_n_host, mats, ctx->num_sms, p.rag_cta0);
        EXL3B_CHECK(grid > 0, EXL3B_ERR_UNSUPPORTED, "exl3_mgemm (i8): fan-out widths not supported");
        for (int j = 0; j < mats; ++j) p.rag_n[j] = a.size_n_host[j];
    }
    { int r = i8_launch(stream, a.K, grid, pl.smem_total, p, tmap); if (r) return r; }
    return EXL3B_TAG_TC_I8;
}

}  // namespace exl3b
