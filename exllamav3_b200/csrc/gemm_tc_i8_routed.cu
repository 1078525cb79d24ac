// Routed / weighted exl3_mgemm (the reference's MoE decode calls, modules/block_sparse_mlp.py:1362-1421,1435-1493: gate and up
// with `indices` = the token's selected experts and one broadcast input, down with per-slot inputs and `weights`, optionally an
// expert-range filter for expert-parallel shards) on the wgmma u8 x s8 decode-GEMM (tag 212).
//
//   launch 1   mgemm_resolve_kernel (gemm_simt.cu): indices / filter -> table of active slots {matrix, weight}
//   launch 2   gemm_tc_i8_body<K, 4, false, ROUTED = true>: one CTA group per SLOT; group z runs matrix tab.mat[z] on input
//              A[z] (or the shared A[0]) into C[z], scaled by tab.weight[z]; groups of inactive slots exit at once
//   launch 3   mgemm_reduce_kernel (weights only): C[t] = sum of the token's slots, in C's dtype, as the reference does
//              (exl3_gemm_kernel.cuh:238-291)
// It replaces the CUDA-core contraction that the default path (launch_mgemm, tag 100) runs between the same two bookkeeping
// kernels; semantics are those of exl3_gemm.cu:341-381.
//
// Tests: tests/test_moe_routed.py (five routing modes vs the oracle and vs the CUDA-core twin,
// Mixtral expert shapes); selected automatically for routed mul1 calls at <= 4 rows, the CUDA-core kernels take the rest.
#include "gemm_tc_i8_body.cuh"

namespace exl3b {

template <int K>
__global__ void __launch_bounds__(TC_THREADS, 1)
gemm_tc_i8_routed_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w, const __grid_constant__ RouteArgs route)
{
    gemm_tc_i8_body<K, 4, false, true>(p, &tmap_w, nullptr, &route);
}

static int routed_slots(const MGemmArgs& a)
{
    int bszm_in = a.bszm_in, bszm_out = a.bszm_out;
    if (a.indices)
    {
        if (bszm_in > a.num_indices) bszm_in = a.num_indices;
        if (bszm_out > a.num_indices) bszm_out = a.num_indices;
    }
    return bszm_in > bszm_out ? bszm_in : bszm_out;          // as launch_mgemm / the reference (exl3_gemm.cu:476-489)
}

bool mgemm_tc_i8_routed_supported(const DevCtx* ctx, const MGemmArgs& a)
{
    if (a.cb != 2 || a.m < 1 || a.m > 4) return false;
    if (a.size_n_list || a.c_ptrs) return false;                        // ragged widths stay on the SIMT path
    if (a.k < 128 || a.n < 128 || a.k % 128 || a.n % 128) return false;
    const int bszm = routed_slots(a);
    if (bszm < 1 || bszm > ctx->num_sms || bszm > DevCtx::TMAP_SLOTS || bszm > MSlotTable::MAX_SLOTS) return false;
    if (!(a.bszm_in == 1 || a.bszm_in >= bszm)) return false;           // shared input or one input per slot
    if ((long long) bszm * (a.n / 128) > DevCtx::COUNTERS_PER_SLOT) return false;
    return true;
}

template <int K>
static cudaError_t i8_routed_launch(cudaStream_t stream, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap, const RouteArgs& route)
{
    static bool attr_set[32] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (!attr_set[dev & 31])
    {
        cudaError_t e = cudaFuncSetAttribute(gemm_tc_i8_routed_kernel<K>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 31] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, gemm_tc_i8_routed_kernel<K>, p, tmap, route);
}

int launch_mgemm_tc_i8_routed(cudaStream_t stream, DevCtx* ctx, const MGemmArgs& a)
{
    const int bszm = routed_slots(a);
    if (bszm == 0 || a.m == 0) return EXL3B_TAG_NOP;
    CUtensorMap tmap;
    { int r = get_weight_tmap(ctx->ws, a.k, a.n, a.K, &tmap); if (r) return r; }     // shape template: address patched per CTA
    // geometry of ONE slot's group: the single-matrix plan on num_sms / bszm CTAs
    const int gpm_max = ctx->num_sms / bszm;
    TcPlan pl;
    { int r = plan_gemm_tc_i8(a.m, a.k, a.n, a.K, gpm_max, 0, &pl); if (r) return r; }
    const int slot = ctx->next_slot();
    MSlotTable* tab = ctx->tab_slot(slot);
    { int r = launch_mgemm_resolve(stream, tab, a, bszm); if (r) return r; }

    TcParams p{};
    p.C = a.C; p.m = a.m; p.k = a.k; p.n = a.n; p.NT = I8_NT; p.c_fp32 = a.c_fp32;
    p.out_scale = 1.f; p.ws = ctx->ws_slot(slot); p.counters = ctx->counter_slot(slot);
    p.A_raw = a.A; p.dbg = g_tc_dbg; p.knob_ = g_tc_knob;
    p.num_mats = bszm;
    p.B_ptrs = a.B_ptrs; p.suh_ptrs = a.suh_ptrs; p.svh_ptrs = a.svh_ptrs;
    p.a_mat_stride = a.bszm_in == 1 ? 0 : (long long) a.m * a.k;
    p.c_mat_stride = (long long) a.m * a.n * (a.c_fp32 ? 4 : 2);
    p.tmap_slots = ctx->tmap_slot(slot);
    p.parts = ctx->i8_parts_slot(slot);
    p.stages = pl.stages; p.b_bytes = pl.b_bytes; p.b_load_bytes = pl.b_load_bytes;
    p.g_per_mat = pl.grid;
    const int grid = pl.grid * bszm;
    EXL3B_CHECK(grid <= DevCtx::I8_PART_CTAS && grid <= DevCtx::TMAP_SLOTS, EXL3B_ERR_UNSUPPORTED, "exl3_mgemm (routed i8): grid too large");
    RouteArgs route{tab, a.weights != nullptr ? 1 : 0};
    cudaError_t err = cudaSuccess;
    switch (a.K)
    {
        case 1: err = i8_routed_launch<1>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 2: err = i8_routed_launch<2>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 3: err = i8_routed_launch<3>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 4: err = i8_routed_launch<4>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 5: err = i8_routed_launch<5>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 6: err = i8_routed_launch<6>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 7: err = i8_routed_launch<7>(stream, grid, pl.smem_total, p, tmap, route); break;
        case 8: err = i8_routed_launch<8>(stream, grid, pl.smem_total, p, tmap, route); break;
    }
    count_launch();
    EXL3B_CUDA(err);
    if (a.weights)
    {
        int r = launch_mgemm_reduce(stream, ctx, tab, a); if (r) return r;
    }
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC_I8_ROUTED;
}

}  // namespace exl3b
