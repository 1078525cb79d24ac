// wgmma EXL3 decode-GEMM for sm_90a ("TC path", tag 200).
//
//   C[m, n] = had128( xh[m, k] @ W_hat[k, n] ) * svh,      xh = fp16( had128(A * suh) / sqrt(128) )
//
// Design:
//   * swap-AB: the decoded weights are the M operand of wgmma (one 128-column strip of W_hat^T, two M = 64 halves), the
//     activations are the N = 16..128 operand, so the weight stream is decoded exactly ONCE for any m <= 128 per pass
//     (the reference re-streams and re-decodes B per 16-row slab, exl3_gemm_kernel.cuh:37-50).
//   * persistent stream-K over work units of 128(k) x 128(n) weights: CTA c owns units [U*c/G, U*(c+1)/G), k fastest.
//   * warp-specialised, 384 threads:
//        warp 0      producer: TMA of the raw trellis rows + the activation tile into an mbarrier ring (weights prefetch
//                    starts BEFORE griddepcontrol.wait: PDL overlap with the previous kernel's tail); warps 1-3 idle
//        warpgroups 1-2  decode + MMA + epilogue: warpgroup h owns output columns 64 h .. 64 h + 63 of the strip.  Each unit
//                    is decoded straight into wgmma A fragments (f16_pipeline.cuh), so decoded weights never touch shared
//                    memory.  fp32 accumulators stay in registers over a k-segment, then go through shared memory into the
//                    split-K combine (global workspace, last arriver reduces in fixed order => deterministic), output
//                    Hadamard + svh, store.
//   * activations arrive pre-tiled in the no-swizzle K-major core-matrix layout wgmma reads, written by the input-transform
//     kernel (fused suh scale + 128-point Hadamard), so the B tile is one contiguous bulk copy.
//
// Reference behaviour being replaced: exllamav3_ext/quant/exl3_gemm_kernel.cuh:8-50, exl3_gemm_inner.cuh:22-733.
#include "common.cuh"
#include "decode.cuh"
#include "epilogue.cuh"
#include "f16_pipeline.cuh"
#include "act.cuh"
#include <unordered_map>
#include <mutex>

namespace exl3b {

using namespace ptx;

// ---- input transform into the tiled activation layout (xt_tile_offset, tc_common.cuh) -------------------------
template <bool HAD>
__global__ void __launch_bounds__(128)
had_tiled_kernel(const half* __restrict__ A, uint8_t* __restrict__ out, const half* __restrict__ suh,
                 int m, int k, int NT)
{
    pdl_launch_dependents();
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int bpr = k / 128;
    if (warp >= m * bpr) return;
    const int r = warp / bpr, kb = warp % bpr;
    uint2 raw = *reinterpret_cast<const uint2*>(A + (size_t) r * k + kb * 128 + lane * 4);
    if constexpr (HAD) raw = xt_transform(raw, suh + kb * 128 + lane * 4, lane);
    store_tile_pair(out + (size_t) kb * NT * 256 + xt_tile_offset(r, lane), raw);
}

// gated variant (exl3b_gemm_gated): the row is fp16(act(G) * U) (act.cuh), then the same transform and tile store
template <bool HAD>
__global__ void __launch_bounds__(128)
had_tiled_gated_kernel(const GateIn gate, uint8_t* __restrict__ out, const half* __restrict__ suh, int m, int k, int NT)
{
    pdl_launch_dependents();
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int bpr = k / 128;
    if (warp >= m * bpr) return;
    const int r = warp / bpr, kb = warp % bpr;
    uint2 raw = gated_load4(gate, (size_t) r * k + kb * 128 + lane * 4);
    if constexpr (HAD) raw = xt_transform(raw, suh + kb * 128 + lane * 4, lane);
    store_tile_pair(out + (size_t) kb * NT * 256 + xt_tile_offset(r, lane), raw);
}

// ---- the kernel -------------------------------------------------------------------------------------------------
template <int K, int cb>
__global__ void __launch_bounds__(F16_THREADS, 1)
gemm_tc_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    // the activation stage size comes from the plan (NT * 256): derived from NT in the kernel, it makes ptxas schedule the
    // 3inst / mcg decode of the unit loop differently (slower, see f16_pipeline.cuh)
    const TcSmemLayout L = f16_smem_layout(K, p.b_bytes, p.stages, p.NT);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = p.stages;

    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    // barrier map: [0,S) w_full  [S,2S) w_empty  [2S,3S) x_full
    const uint32_t bar0 = smem_u32(bars);
    auto W_FULL = [&](int s) { return bar0 + 8u * s; };
    auto W_EMPTY = [&](int s) { return bar0 + 8u * (S + s); };
    auto X_FULL = [&](int s) { return bar0 + 8u * (2 * S + s); };
    int* s_flag = reinterpret_cast<int*>(smem + L.off_bars + 8 * (3 * TC_MAX_STAGES + 20));

    if (threadIdx.x == 0) tc_stamp(p.dbg, 0);
    pdl_launch_dependents();

    if (warp == 0)
    {
        // W_EMPTY: the eight consumer warps, after their MMAs have read the stage
        for (int s = lane; s < S; s += 32) { mbar_init(W_FULL(s), 1); mbar_init(X_FULL(s), 1); mbar_init(W_EMPTY(s), F16_CONS_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) tc_stamp(p.dbg, 1);

    // ---- this CTA's unit range ----
    const int KB = p.k / 128;
    const int strips = p.n / 128;
    const int U = KB * strips;
    const int G = gridDim.x;
    const int ubeg = unit_begin(U, G, blockIdx.x), uend = unit_begin(U, G, blockIdx.x + 1);
    const int n_units = uend - ubeg;

    if (warp == 0)
    {
        // =========================== producer ===========================
        // whole warp runs the loop (uniform control flow -> uniform-register operands); one elected lane issues
        if (elect_one()) prefetch_tmap(&tmap_w);
        const uint64_t pol_w = policy_evict_first(), pol_x = policy_evict_last();
        const uint32_t w_smem0 = smem_u32(smem), x_smem0 = smem_u32(smem + L.off_b);
        auto issue_w = [&](int s, int strip, int kb)
        {
            if (elect_one())
            {
                mbar_arrive_expect_tx(W_FULL(s), (uint32_t) L.w_bytes);
                // one 2-D TMA box per unit: 8 tile-rows x (256*K bytes = 32*K uint64) of the trellis
                tma_load_2d(w_smem0 + s * L.w_bytes, &tmap_w, strip * (32 * K), kb * 8, W_FULL(s), pol_w);
            }
        };
        auto issue_x = [&](int s, int kb)
        {
            if (elect_one())
            {
                mbar_arrive_expect_tx(X_FULL(s), (uint32_t) p.b_load_bytes);
                bulk_g2s(x_smem0 + s * L.b_bytes, p.xh_tiled + (size_t) kb * p.NT * 256,
                         (uint32_t) p.b_load_bytes, X_FULL(s), pol_x);
            }
        };
        const int pre = n_units < S ? n_units : S;
        const int strip0 = ubeg / KB, kb0 = ubeg % KB;
        int strip = strip0, kb = kb0;
        auto next_unit = [&] { if (++kb == KB) { kb = 0; ++strip; } };
        for (int u = 0; u < pre; ++u) { issue_w(u, strip, kb); next_unit(); }   // weights never depend on the previous kernel
        pdl_wait();                                                              // activations do
        { int kbx = kb0; for (int u = 0; u < pre; ++u) { issue_x(u, kbx); if (++kbx == KB) kbx = 0; } }
        if (lane == 0) tc_stamp(p.dbg, 2);
        int s = (pre == S) ? 0 : pre, ph = (pre == S) ? 1 : 0;                   // ring position of unit `pre`
        for (int u = pre; u < n_units; ++u)
        {
            mbar_wait<64>(W_EMPTY(s), ph ^ 1);
            issue_w(s, strip, kb);
            issue_x(s, kb);
            next_unit();
            if (++s == S) { s = 0; ph ^= 1; }
        }
        __syncwarp();
    }
    else if (warp >= F16_CONS_WARP0)
    {
        // =========================== decode + MMA + epilogue (two warpgroups) ===========================
        const int ct = threadIdx.x - F16_CONS_WARP0 * 32;            // 0..255
        const int cw = ct >> 5;                                      // consumer warp 0..7
        const int h = cw >> 2, wq = cw & 3;
        const int tl = 4 * h + wq;                                   // tile column of the strip owned by this warp
        const int chunk = lane >> 2, c = lane & 3;                   // computed once: derived from lane in each helper, the
                                                                     // 3inst / mcg decode loop gets other registers, ~4 % slower
        const int nchunks = p.NT / 16;
        float* tile = reinterpret_cast<float*>(smem + L.off_tile);   // [NT][128] fp32: one strip's k-segment sums
        auto cons_bar = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };
        const int part_stride = p.NT * 128;
        const uint64_t desc0 = f16_tile_desc(smem + L.off_b);
        pdl_wait();                                                  // no global write before the previous grid has completed

        float acc[F16_MAX_ROWS / 16][8];
        f16_zero(acc);

        // all rows of one strip: tile (fp32 sums) -> output transform -> C
        auto emit_rows = [&](int strip)
        {
            cons_bar();
            for (int j = cw; j < p.m; j += F16_CONS_WARPS)
                output_row_128(tile + j * 128, (char*) p.C, (size_t) j * p.n + strip * 128,
                               p.svh ? p.svh + strip * 128 : nullptr, p.out_scale, p.c_fp32 != 0, lane);
            cons_bar();
        };

        int s = 0, sph = 0;
        int u = 0;
        while (u < n_units)
        {
            const int g = ubeg + u;
            const int strip = g / KB, kb = g % KB;
            const int to_strip_end = KB - kb;
            const int seg = (n_units - u) < to_strip_end ? (n_units - u) : to_strip_end;
            const int gs = strip * KB;
            const int c_a = cta_of_unit(U, G, gs), c_b = cta_of_unit(U, G, gs + KB - 1);
            const int n_contrib = c_b - c_a + 1;
            const bool full = n_contrib == 1;
            float* my_part = p.ws + (size_t) (2 * blockIdx.x + (ubeg >= gs ? 0 : 1)) * part_stride;

            for (int i = 0; i < seg; ++i)
            {
                mbar_wait<32>(W_FULL(s), sph);
                if (u + i == 0 && ct == 0) tc_stamp(p.dbg, 3);
                uint32_t w[2][K + 1];
                f16_load_unit<K>(reinterpret_cast<const uint32_t*>(smem + s * L.w_bytes), tl, chunk, c, w);
                mbar_wait(X_FULL(s), sph);
                const uint64_t desc_s = desc0 + (uint64_t) ((s * L.b_bytes) >> 4);
                #pragma unroll
                for (int r = 0; r < 2; ++r)
                {
                    uint32_t o0[8], o1[8];
                    decode16<K, cb, 0>(w[r], o0);
                    decode16<K, cb, 1>(w[r], o1);
                    #pragma unroll
                    for (int ii = 0; ii < F16_MAX_ROWS / 16; ++ii)
                        #pragma unroll
                        for (int e = 0; e < 8; ++e) reg_fence(acc[ii][e]);
                    wgmma_fence();
                    #pragma unroll
                    for (int j = 0; j < 4; ++j)
                    {
                        // instruction 4 r + j: K-chunks 2 (4 r + j), +1;  N-chunk ii: row groups 2 ii, 2 ii + 1
                        #pragma unroll
                        for (int ii = 0; ii < F16_MAX_ROWS / 16; ++ii)
                            if (ii < nchunks)
                                wgmma_f16_n16(acc[ii], o0[2 * j], o1[2 * j], o0[2 * j + 1], o1[2 * j + 1],
                                              desc_s + (uint64_t) (16 * (4 * r + j) + 256 * ii));
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    #pragma unroll
                    for (int e = 0; e < 8; ++e) { reg_fence(o0[e]); reg_fence(o1[e]); }
                    #pragma unroll
                    for (int ii = 0; ii < F16_MAX_ROWS / 16; ++ii)
                        #pragma unroll
                        for (int e = 0; e < 8; ++e) reg_fence(acc[ii][e]);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(W_EMPTY(s));
                if (++s == S) { s = 0; sph ^= 1; }
            }

            cons_bar();                                              // the previous segment's readers of the tile are done
            f16_store_tile(tile, acc, tl, chunk, c, nchunks);
            f16_zero(acc);
            if (u + seg >= n_units && ct == 0) tc_stamp(p.dbg, 7);
            if (full) emit_rows(strip);
            else
            {
                cons_bar();
                for (int idx = ct; idx < p.m * 128; idx += 256) my_part[idx] = tile[idx];
                cons_bar();                                   // all partial stores of this CTA are ordered before ...
                if (ct == 0)
                {
                    __threadfence();                          // ... this single gpu-scope fence + the arrival count (cumulativity)
                    const int old = atomicAdd(&p.counters[strip], 1);
                    const int last = old == n_contrib - 1;
                    if (last) { p.counters[strip] = 0; __threadfence(); }          // self-reset for the next launch using this slot
                    *s_flag = last;
                }
                cons_bar();
                if (*s_flag)
                {
                    const int which_a = unit_begin(U, G, c_a) >= gs ? 0 : 1;       // only c_a can have started in an earlier strip
                    for (int idx = ct; idx < p.m * 128; idx += 256)
                    {
                        float a = 0.f;
                        for (int cc = c_a; cc <= c_b; ++cc)                        // fixed order: deterministic
                            a += __ldcg(p.ws + (size_t) (2 * cc + (cc == c_a ? which_a : 0)) * part_stride + idx);
                        tile[idx] = a;
                    }
                    emit_rows(strip);
                }
            }
            u += seg;
        }
        if (ct == 0) tc_stamp(p.dbg, 8);
    }

    // ---- teardown ----
    __syncthreads();
    if (threadIdx.x == 0) tc_stamp(p.dbg, 9);
}

// ---- host side -------------------------------------------------------------------------------------------------------

// ---- tensor map for the trellis: 2-D view [k/16 rows][n/16 * 32K bytes] in uint64 elements, box = 8 rows x 256K bytes ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int get_weight_tmap(const void* B, int k, int n, int K, CUtensorMap* out)
{
    static PFN_encodeTiled encode = nullptr;
    static std::mutex mu;
    struct Key { const void* p; int k, n, K; bool operator==(const Key& o) const { return p == o.p && k == o.k && n == o.n && K == o.K; } };
    struct Hash { size_t operator()(const Key& x) const { return std::hash<const void*>()(x.p) ^ ((size_t) x.k * 1315423911u) ^ ((size_t) x.n << 20) ^ (size_t) x.K; } };
    static std::unordered_map<Key, CUtensorMap, Hash> cache;
    std::lock_guard<std::mutex> lock(mu);
    if (!encode)
    {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        EXL3B_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        EXL3B_CHECK(fn && qres == cudaDriverEntryPointSuccess, EXL3B_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
        encode = (PFN_encodeTiled) fn;
    }
    Key key{B, k, n, K};
    auto it = cache.find(key);
    if (it == cache.end())
    {
        CUtensorMap tm;
        const cuuint64_t row_bytes = (cuuint64_t) (n / 16) * 32 * K;
        const cuuint64_t rows = (cuuint64_t) (k / 16);
        cuuint64_t gdim[2] = { row_bytes / 8, rows };
        cuuint64_t gstride[1] = { row_bytes };
        cuuint32_t box[2] = { (cuuint32_t) (32 * K), 8 };
        cuuint32_t estr[2] = { 1, 1 };
        CUresult r = encode(&tm, CU_TENSOR_MAP_DATA_TYPE_UINT64, 2, const_cast<void*>(B), gdim, gstride, box, estr,
                            CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                            CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        EXL3B_CHECK(r == CUDA_SUCCESS, EXL3B_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) for trellis %p k=%d n=%d K=%d", (int) r, B, k, n, K);
        if (cache.size() > 65536) cache.clear();
        it = cache.emplace(key, tm).first;
    }
    *out = it->second;
    return 0;
}

template <int K, int cb>
static void tc_launch_v(cudaStream_t stream, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap,
                        cudaError_t* err)
{
    *err = launch_pdl<gemm_tc_kernel<K, cb>>(stream, dim3(grid), F16_THREADS, smem_bytes, p, tmap);
}

unsigned long long* g_tc_dbg = nullptr;
// bring-up hooks: live only in the EXL3B_TC_DEBUG build (libexl3b200_dbg.so); the production library ignores them, so no
// exported call can change what its kernels compute
#ifdef EXL3B_TC_DEBUG
void tc_set_debug_buffer(unsigned long long* d) { g_tc_dbg = d; }
#else
void tc_set_debug_buffer(unsigned long long*) { }
#endif

bool gemm_tc_supported(const GemmArgs& a)
{
    return a.k >= 128 && a.n >= 128 && a.k % 128 == 0 && a.n % 128 == 0 && a.m >= 1;
}

static int launch_had_tiled(cudaStream_t stream, const half* A, uint8_t* out, const half* suh, int m, int k, int NT,
                            const GateIn* gate)
{
    const dim3 grid((m * (k / 128) + 3) / 4);
    cudaError_t e;
    if (gate)
        e = suh ? launch_pdl<had_tiled_gated_kernel<true>>(stream, grid, 128, 0, *gate, out, suh, m, k, NT)
                : launch_pdl<had_tiled_gated_kernel<false>>(stream, grid, 128, 0, *gate, out, suh, m, k, NT);
    else
        e = suh ? launch_pdl<had_tiled_kernel<true>>(stream, grid, 128, 0, A, out, suh, m, k, NT)
                : launch_pdl<had_tiled_kernel<false>>(stream, grid, 128, 0, A, out, suh, m, k, NT);
    count_launch();
    EXL3B_CUDA(e);
    return 0;
}

// launch geometry of one pass (m <= F16_MAX_ROWS rows), also behind exl3b_gemm_plan
int plan_gemm_tc(int m, int k, int n, int K, int num_sms, int max_ctas, TcPlan* pl)
{
    EXL3B_CHECK(m >= 1 && m <= F16_MAX_ROWS, EXL3B_ERR_ARG, "plan_gemm_tc: one pass handles 1..%d rows", F16_MAX_ROWS);
    const int NT = (m + 15) / 16 * 16;
    // accumulators live in the consumer warpgroups' registers: no accumulator buffers to plan
    pl->d_bufs = 1;
    pl->b_load_bytes = m <= 8 ? 2048 : NT * 256;         // m <= 8: only the first row group is ever needed
    const int stages = f16_stages(K, NT);
    const TcSmemLayout L = f16_smem_layout(K, NT * 256, stages, NT);
    EXL3B_CHECK(L.total <= 220 * 1024, EXL3B_ERR_UNSUPPORTED, "exl3_gemm: shared-memory budget exceeded");
    const long long U = (long long) (k / 128) * (n / 128);
    int grid = num_sms;
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    if (grid > U) grid = (int) U;
    EXL3B_CHECK((size_t) 2 * grid * NT * 128 * 4 <= DevCtx::WS_BYTES_PER_SLOT, EXL3B_ERR_UNSUPPORTED,
                "exl3_gemm: split-K workspace too small");
    EXL3B_CHECK(n / 128 <= DevCtx::COUNTERS_PER_SLOT, EXL3B_ERR_UNSUPPORTED, "exl3_gemm: too many column strips");
    EXL3B_CHECK(partition_fits(U, grid), EXL3B_ERR_UNSUPPORTED, "exl3_gemm: too many units for the 32-bit stream-K partition");
    pl->rows = NT; pl->stages = stages; pl->b_bytes = L.b_bytes; pl->smem_total = L.total; pl->grid = grid; pl->units = U;
    return 0;
}

int launch_gemm_tc(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a, const GateIn* gate)
{
    EXL3B_CHECK(!gate || a.m <= F16_MAX_ROWS, EXL3B_ERR_UNSUPPORTED, "exl3_gemm_gated: gated input is one pass of rows");
    const size_t esz = a.c_fp32 ? 4 : 2;
    CUtensorMap tmap;
    { int r = get_weight_tmap(a.B, a.k, a.n, a.K, &tmap); if (r) return r; }
    for (int m0 = 0; m0 < a.m; m0 += F16_MAX_ROWS)
    {
        const int m = a.m - m0 < F16_MAX_ROWS ? a.m - m0 : F16_MAX_ROWS;
        TcPlan pl;
        { int r = plan_gemm_tc(m, a.k, a.n, a.K, ctx->num_sms, a.max_ctas, &pl); if (r) return r; }
        const int NT = pl.rows;
        const int slot = ctx->next_slot();
        { int r = ensure_xh_tiled(ctx, (size_t) (a.k / 128) * NT * 256); if (r) return r; }
        uint8_t* xh_tiled = ctx->xh_tiled + (size_t) (slot % DevCtx::XH_SLOTS) * ctx->xh_tiled_slot_bytes;
        { int r = launch_had_tiled(stream, a.A + (size_t) m0 * a.k, xh_tiled, a.suh, m, a.k, NT, gate); if (r) return r; }

        TcParams p{};
        p.xh_tiled = xh_tiled; p.B = a.B; p.C = (char*) a.C + (size_t) m0 * a.n * esz; p.svh = a.svh;
        p.m = m; p.k = a.k; p.n = a.n; p.NT = NT; p.c_fp32 = a.c_fp32; p.out_scale = a.out_scale;
        p.ws = ctx->ws_slot(slot); p.counters = ctx->counter_slot(slot);
        p.b_load_bytes = pl.b_load_bytes;
        p.stages = pl.stages;
        p.b_bytes = pl.b_bytes;
        p.dbg = g_tc_dbg;

        cudaError_t err = cudaSuccess;
        EXL3B_DISPATCH_K_CB(tc_launch_v, a.K, a.cb, stream, pl.grid, pl.smem_total, p, tmap, &err);
        count_launch();
        EXL3B_CUDA(err);
    }
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC;
}

}  // namespace exl3b
