// Routed / weighted exl3_mgemm (the reference's MoE decode calls, modules/block_sparse_mlp.py:1362-1421,1435-1493: gate and up
// with `indices` = the token's selected experts and one broadcast input, down with per-slot inputs and `weights`, optionally an
// expert-range filter for expert-parallel shards) on the wgmma u8 x s8 decode-GEMM (tag 212).
//
//   launch 1   mgemm_resolve_kernel (gemm_simt.cu): indices / filter -> table of active slots {matrix, weight}
//   launch 2   gemm_tc_i8_body<K, 4, false, ROUTED = true> (entry in gemm_tc_i8.cu): one CTA group per SLOT; group z runs matrix tab.mat[z] on input
//              A[z] (or the shared A[0]) into C[z], scaled by tab.weight[z]; groups of inactive slots exit at once
//   launch 3   mgemm_reduce_kernel (weights only): C[t] = sum of the token's slots, in C's dtype, as the reference does
//              (exl3_gemm_kernel.cuh:238-291)
// It replaces the CUDA-core contraction that the default path (launch_mgemm, tag 100) runs between the same two bookkeeping
// kernels; semantics are those of exl3_gemm.cu:341-381.
//
// Tests: tests/test_moe_routed.py (five routing modes vs the oracle and vs the CUDA-core twin, Mixtral expert shapes) and
// tests/test_moe_routed_exact.py (every slot vs the exact int8 model and bit for bit vs tag 210, the reduce bit for bit at
// num_tokens >= 1, shards, 1..128 slots, graph replay); selected automatically for routed mul1 calls at <= 4 rows, the
// CUDA-core kernels take the rest.
#include "tc_common.cuh"

namespace exl3b {

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
    if (i8_shape_unsupported(a.m, a.k, a.n, a.K, a.cb, false)) return false;
    if (a.size_n_list || a.c_ptrs) return false;                        // ragged widths stay on the SIMT path
    const int bszm = routed_slots(a);
    if (bszm < 1 || bszm > ctx->num_sms || bszm > DevCtx::TMAP_SLOTS || bszm > MSlotTable::MAX_SLOTS) return false;
    if (!(a.bszm_in == 1 || a.bszm_in >= bszm)) return false;           // shared input or one input per slot
    if ((long long) bszm * (a.n / 128) > DevCtx::COUNTERS_PER_SLOT) return false;
    return true;
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

    TcParams p = i8_params(ctx, slot, pl, a, bszm);
    p.g_per_mat = pl.grid;
    const int grid = pl.grid * bszm;
    EXL3B_CHECK(grid <= DevCtx::I8_PART_CTAS && grid <= DevCtx::TMAP_SLOTS, EXL3B_ERR_UNSUPPORTED, "exl3_mgemm (routed i8): grid too large");
    const RouteArgs route{tab, a.weights != nullptr ? 1 : 0};
    { int r = i8_launch(stream, a.K, grid, pl.smem_total, p, tmap, nullptr, nullptr, &route); if (r) return r; }
    if (a.weights)
    {
        int r = launch_mgemm_reduce(stream, ctx, tab, a); if (r) return r;
    }
    return EXL3B_TAG_TC_I8_ROUTED;
}

}  // namespace exl3b
