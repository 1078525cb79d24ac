// CUDA-core EXL3 GEMM ("SIMT path", tag 100): bring-up / fallback-free correctness path for every (K, cb, m) and the
// home of the mgemm semantics.  Same thread->column decomposition, split-K protocol and output-transform epilogue as
// the tensor-core path (gemm_tc.cu); only the contraction differs (fp32 FMA per thread instead of wgmma).
//
// Reference behaviour restated: exllamav3_ext/quant/exl3_gemm_kernel.cuh:8-50 (gemm), :88-292 (mgemm),
// exl3_gemm_inner.cuh:426-480 (output transform), exl3_gemm.cu:341-381 (mgemm semantics).
#include "common.cuh"
#include "decode.cuh"
#include "epilogue.cuh"

namespace exl3b {

constexpr int SIMT_MAXM = 16;

struct SimtParams
{
    const half* xh;            // (slots, m_total, k) transformed input; slot stride = m_total * k
    const uint32_t* B;         // single-matrix mode
    void* C;
    const half* svh;
    int m;                     // rows in this launch (<= SIMT_MAXM)
    int m_total;               // rows of the whole problem (slot strides)
    int m0;                    // first row of this launch
    int k, n;
    int c_fp32;
    int splits;
    float out_scale;
    float* ws;
    int* counters;
    // multi-matrix mode (tab != nullptr)
    const MSlotTable* tab;
    const uint64_t* B_ptrs;
    const uint64_t* svh_ptrs;
    const uint64_t* c_ptrs;
    const int32_t* size_n_list;
    int has_weights;
};

template <int K, int cb>
__global__ void __launch_bounds__(128)
gemm_simt_kernel(const SimtParams p)
{
    __shared__ __align__(16) half xs[SIMT_MAXM][128];
    __shared__ __align__(16) float tile[SIMT_MAXM][128];
    __shared__ int s_last;

    const int q = threadIdx.x >> 5, i = threadIdx.x & 31;
    const int strip = blockIdx.x, split = blockIdx.y, z = blockIdx.z;

    const uint32_t* B = p.B;
    const half* svh = p.svh;
    char* C = (char*) p.C;
    int n = p.n;
    float out_scale = p.out_scale;
    const size_t esz = p.c_fp32 ? 4 : 2;
    if (p.tab)
    {
        if (z >= p.tab->n_active) return;
        int mat = p.tab->mat[z];
        if (mat < 0) return;
        B = (const uint32_t*) p.B_ptrs[mat];
        svh = (const half*) p.svh_ptrs[mat];
        if (p.size_n_list) n = p.size_n_list[mat];
        if (strip * 128 >= n) return;
        C = p.c_ptrs ? (char*) p.c_ptrs[mat] : C + (size_t) z * p.m_total * p.n * esz;
        if (p.has_weights) out_scale = __half2float(p.tab->weight[z]);
    }
    const half* xh = p.xh + ((size_t) z * p.m_total + p.m0) * p.k;
    C += (size_t) p.m0 * n * esz;

    const int tiles_n = n / 16;
    const int kb_total = p.k / 128;
    const int kb0 = (int) ((long) kb_total * split / p.splits);
    const int kb1 = (int) ((long) kb_total * (split + 1) / p.splits);
    const int tl = strip_tile(q, i);
    const int chunk = i & 7;

    float acc[SIMT_MAXM];
    #pragma unroll
    for (int r = 0; r < SIMT_MAXM; ++r) acc[r] = 0.f;

    for (int kb = kb0; kb < kb1; ++kb)
    {
        __syncthreads();
        for (int e = threadIdx.x; e < p.m * 16; e += 128)       // m rows x 16 uint4
        {
            int r = e >> 4, c = e & 15;
            *reinterpret_cast<uint4*>(&xs[r][c * 8]) =
                *reinterpret_cast<const uint4*>(xh + (size_t) r * p.k + kb * 128 + c * 8);
        }
        __syncthreads();
        #pragma unroll 1
        for (int t = 0; t < 8; ++t)
        {
            const uint32_t* tp = B + ((size_t) (kb * 8 + t) * tiles_n + strip * 8 + tl) * (8 * K);
            uint32_t w[K + 1], o[8];
            load_chunk<K>(tp, chunk, w);
            if (q & 1) decode16<K, cb, 1>(w, o); else decode16<K, cb, 0>(w, o);
            float wf[16];
            #pragma unroll
            for (int j = 0; j < 8; ++j)
            {
                half2 h = *reinterpret_cast<half2*>(&o[j]);
                wf[2 * j] = __low2float(h); wf[2 * j + 1] = __high2float(h);
            }
            for (int r = 0; r < p.m; ++r)
            {
                float a = acc[r];
                #pragma unroll
                for (int j = 0; j < 16; ++j) a = fmaf(__half2float(xs[r][t * 16 + j]), wf[j], a);
                acc[r] = a;
            }
        }
    }

    // ---- split-K combine + output transform ----
    const int col = strip_col(q, i);
    const int tile_id = z * (p.n / 128) + strip;
    bool last = true;
    if (p.splits > 1)
    {
        float* wsp = p.ws + ((size_t) tile_id * p.splits + split) * (SIMT_MAXM * 128);
        for (int r = 0; r < p.m; ++r) wsp[r * 128 + col] = acc[r];
        __threadfence();
        __syncthreads();
        if (threadIdx.x == 0)
        {
            int old = atomicAdd(&p.counters[tile_id], 1);
            s_last = (old == p.splits - 1);
            if (s_last) p.counters[tile_id] = 0;       // self-reset for the next launch using this slot
        }
        __syncthreads();
        last = s_last != 0;
        if (last)
        {
            __threadfence();
            const float* wsb = p.ws + (size_t) tile_id * p.splits * (SIMT_MAXM * 128);
            for (int r = 0; r < p.m; ++r)
            {
                float s = 0.f;
                for (int sidx = 0; sidx < p.splits; ++sidx)          // fixed order: deterministic
                    s += __ldcg(wsb + (size_t) sidx * (SIMT_MAXM * 128) + r * 128 + col);
                acc[r] = s;
            }
        }
    }
    if (!last) return;
    for (int r = 0; r < p.m; ++r) tile[r][col] = acc[r];
    __syncthreads();
    for (int r = q; r < p.m; r += 4)
        output_row_128(&tile[r][0], C, (size_t) r * n + strip * 128, svh ? svh + strip * 128 : nullptr,
                       out_scale, p.c_fp32 != 0, i);
}

template <int K, int cb>
static void simt_launch(cudaStream_t stream, dim3 grid, const SimtParams& p)
{
    gemm_simt_kernel<K, cb><<<grid, 128, 0, stream>>>(p);
}

static int pick_splits(DevCtx* ctx, int k, int n, int slots)
{
    int strips = n / 128 * slots;
    int kb_total = k / 128;
    int splits = 1;
    // aim for ~4 CTAs per SM, bounded by the k-blocks, the workspace and the counter region
    while (splits * 2 <= kb_total && strips * splits * 2 <= ctx->num_sms * 4) splits *= 2;
    while (splits > 1 && (size_t) strips * splits * SIMT_MAXM * 128 * 4 > DevCtx::WS_BYTES_PER_SLOT) splits /= 2;
    if (strips > DevCtx::COUNTERS_PER_SLOT) splits = 1;
    return splits;
}

int launch_gemm_simt(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a)
{
    int slot = ctx->next_slot();
    const half* xh = a.A;
    if (a.suh)
    {
        half* dst = a.A_had;
        if (!dst)
        {
            int r = ensure_xh_scratch(ctx, (size_t) a.m * a.k); if (r) return r;
            dst = ctx->xh_scratch;
        }
        int r = launch_had_r_128(stream, a.A, dst, a.suh, nullptr, 1.0f, a.m, a.k, false); if (r) return r;
        xh = dst;
    }
    SimtParams p{};
    p.xh = xh; p.B = a.B; p.C = a.C; p.svh = a.svh; p.k = a.k; p.n = a.n; p.c_fp32 = a.c_fp32;
    p.m_total = a.m; p.out_scale = a.out_scale;
    p.splits = pick_splits(ctx, a.k, a.n, 1);
    p.ws = ctx->ws_slot(slot); p.counters = ctx->counter_slot(slot);
    for (int m0 = 0; m0 < a.m; m0 += SIMT_MAXM)
    {
        p.m0 = m0; p.m = a.m - m0 < SIMT_MAXM ? a.m - m0 : SIMT_MAXM;
        dim3 grid(a.n / 128, p.splits, 1);
        EXL3B_DISPATCH_K_CB(simt_launch, a.K, a.cb, stream, grid, p);
        count_launch();
    }
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_SIMT;
}

// ==================================================================================================================
// mgemm
// ==================================================================================================================

// Resolve the active slots exactly like the reference kernel prologue (exl3_gemm_kernel.cuh:101-128,132-146).
__global__ void mgemm_resolve_kernel(MSlotTable* tab, const int64_t* indices, const half* weights, int bszm,
                                     int min_index, int max_index)
{
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    if (min_index >= 0)
    {
        int j = 0;
        for (int s = 0; s < bszm; ++s)
        {
            int idx = (int) indices[s];
            if (idx >= min_index && idx < max_index)
            {
                tab->mat[j] = idx - min_index;
                if (weights) tab->weight[j] = weights[s];
                j++;
            }
        }
        tab->n_active = j;
    }
    else
    {
        for (int s = 0; s < bszm; ++s)
        {
            tab->mat[s] = indices ? (int) indices[s] : s;
            if (weights) tab->weight[s] = weights[s];
        }
        tab->n_active = bszm;
    }
}

// Input transform for every active slot: A_had[j] = had128(A[j or 0] * suh[mat]).
__global__ void __launch_bounds__(128)
mgemm_had_kernel(const half* __restrict__ A, half* __restrict__ A_had, const uint64_t* __restrict__ suh_ptrs,
                 const MSlotTable* __restrict__ tab, int bszm_in, int m, int k)
{
    const int z = blockIdx.y;
    if (z >= tab->n_active) return;
    const int mat = tab->mat[z];
    if (mat < 0) return;
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int bpr = k / 128;
    if (warp >= m * bpr) return;
    const half* suh = (const half*) suh_ptrs[mat];
    const half* src = (bszm_in == 1 ? A : A + (size_t) z * m * k) + (size_t) warp * 128 + lane * 4;
    half* dst = A_had + (size_t) z * m * k + (size_t) warp * 128 + lane * 4;
    const uint2 raw = *reinterpret_cast<const uint2*>(src);
    const uint2 scb = *reinterpret_cast<const uint2*>(suh + (warp % bpr) * 128 + lane * 4);
    *reinterpret_cast<uint2*>(dst) = had128_fp16(raw, &scb, lane);
}

// Weighted-MoE reduction: groups of (n_active / num_tokens) slots are summed into C[t] in C's dtype
// (exl3_gemm_kernel.cuh:238-291).
__global__ void mgemm_reduce_kernel(void* C, const MSlotTable* tab, int m, int n, int c_fp32, int num_tokens)
{
    const int bszm = tab->n_active;
    const int stride = bszm / num_tokens;
    const size_t mn = (size_t) m * n;
    for (size_t col = (size_t) blockIdx.x * blockDim.x + threadIdx.x; col < mn; col += (size_t) gridDim.x * blockDim.x)
    {
        for (int t = 0; t < num_tokens; ++t)
        {
            if (c_fp32)
            {
                const float* src = (const float*) C + (size_t) t * stride * mn + col;
                float s = 0.f;
                for (int j = 0; j < stride; ++j) s += src[(size_t) j * mn];
                ((float*) C)[(size_t) t * mn + col] = s;
            }
            else
            {
                const half* src = (const half*) C + (size_t) t * stride * mn + col;
                half s = __float2half(0.f);
                for (int j = 0; j < stride; ++j) s = __hadd(s, src[(size_t) j * mn]);
                ((half*) C)[(size_t) t * mn + col] = s;
            }
        }
    }
}

// The two bookkeeping stages of exl3_mgemm as stand-alone launches, for the tensor-core routed path (gemm_tc_i8_routed.cu), which
// replaces only the contraction in between.
int launch_mgemm_resolve(cudaStream_t stream, MSlotTable* tab, const MGemmArgs& a, int bszm)
{
    mgemm_resolve_kernel<<<1, 32, 0, stream>>>(tab, a.indices, a.weights, bszm, a.min_index, a.max_index);
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

int launch_mgemm_reduce(cudaStream_t stream, DevCtx* ctx, const MSlotTable* tab, const MGemmArgs& a)
{
    size_t mn = (size_t) a.m * a.n;
    int grid = (int) ((mn + 255) / 256);
    if (grid > 4 * ctx->num_sms) grid = 4 * ctx->num_sms;
    mgemm_reduce_kernel<<<grid, 256, 0, stream>>>(a.C, tab, a.m, a.n, a.c_fp32, a.num_tokens);
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

int launch_mgemm(cudaStream_t stream, DevCtx* ctx, const MGemmArgs& a)
{
    int bszm_in = a.bszm_in, bszm_out = a.bszm_out;
    if (a.indices)
    {
        if (bszm_in > a.num_indices) bszm_in = a.num_indices;
        if (bszm_out > a.num_indices) bszm_out = a.num_indices;
    }
    int bszm = bszm_in > bszm_out ? bszm_in : bszm_out;
    if (bszm == 0 || a.m == 0) return EXL3B_TAG_NOP;
    EXL3B_CHECK(bszm <= MSlotTable::MAX_SLOTS, EXL3B_ERR_UNSUPPORTED, "exl3_mgemm: more than %d slots", MSlotTable::MAX_SLOTS);

    int slot = ctx->next_slot();
    MSlotTable* tab = ctx->tab_slot(slot);
    mgemm_resolve_kernel<<<1, 32, 0, stream>>>(tab, a.indices, a.weights, bszm, a.min_index, a.max_index);
    {
        int warps = a.m * (a.k / 128);
        dim3 grid((warps + 3) / 4, bszm);
        mgemm_had_kernel<<<grid, 128, 0, stream>>>(a.A, a.A_had, a.suh_ptrs, tab, a.bszm_in, a.m, a.k);
    }
    count_launch(2);

    SimtParams p{};
    p.xh = a.A_had; p.C = a.C; p.k = a.k; p.n = a.n; p.c_fp32 = a.c_fp32; p.m_total = a.m; p.out_scale = 1.f;
    p.splits = pick_splits(ctx, a.k, a.n, bszm);
    p.ws = ctx->ws_slot(slot); p.counters = ctx->counter_slot(slot);
    p.tab = tab; p.B_ptrs = a.B_ptrs; p.svh_ptrs = a.svh_ptrs; p.c_ptrs = a.c_ptrs; p.size_n_list = a.size_n_list;
    p.has_weights = a.weights != nullptr;
    for (int m0 = 0; m0 < a.m; m0 += SIMT_MAXM)
    {
        p.m0 = m0; p.m = a.m - m0 < SIMT_MAXM ? a.m - m0 : SIMT_MAXM;
        dim3 grid(a.n / 128, p.splits, bszm);
        EXL3B_DISPATCH_K_CB(simt_launch, a.K, a.cb, stream, grid, p);
        count_launch();
    }
    if (a.weights)
    {
        size_t mn = (size_t) a.m * a.n;
        int grid = (int) ((mn + 255) / 256);
        if (grid > 4 * ctx->num_sms) grid = 4 * ctx->num_sms;
        mgemm_reduce_kernel<<<grid, 256, 0, stream>>>(a.C, tab, a.m, a.n, a.c_fp32, a.num_tokens);
        count_launch();
    }
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_SIMT;
}

}  // namespace exl3b
