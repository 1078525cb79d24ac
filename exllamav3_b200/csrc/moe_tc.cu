// Fused routed-expert MLP for sm_90a (exl3_moe, tag 230): for every routed position j of an expert e with 0 < c_e <= T tokens
//
//   g = gate_e(x_t), u = up_e(x_t)  (fp16, as exl3_gemm),  h = fp16(act(g) * u),  output_state[t] += w_j * down_e(h)  (fp32)
//
// Launches on the caller's stream, chained with programmatic dependent launch; each reads the work list the first one derives
// from expert_count on the device, so nothing is copied to the host.  Steps 2-7 run once per chunk of the work list: the passes
// are packed into chunks whose rows fit the fixed per-device work area (moe_chunk_rows), in position order.
//   1. route    one CTA: prefix sums of expert_count, the passes (<= 128 rows of one expert, padded to 16), the pass row of every
//               position, and per token the ascending list of its processed positions (the fixed order of the final sum)
//   2. gather   x[token] * suh -> 128-point Hadamard -> fp16 core-matrix tiles (the tag-200 input transform), for gate and up
//   3/4. GEMM   gate, then up: one persistent launch per matrix (K may differ), work items (pass, 128-column strip)
//   5. act      output Hadamard + svh already applied by the GEMM epilogue (fp16 g, u); act, clamp, * u -> fp16 h, * suh_down,
//               Hadamard -> down's tiles
//   6. GEMM     down, fp32 rows, one per position
//   7. reduce   output_state[t] += w_j * d_j over the token's positions of the chunk in ascending j.  Chunks cover ascending
//               position ranges, so every token's sum runs in ascending j whatever the chunking: deterministic, no atomics
//
// The GEMM is tag 200's unit (layout and helpers in f16_pipeline.cuh): decoded weights are the wgmma A fragments (m64n16k16,
// fp32 accumulation), activations the N = 16..128 operand.  Its own parts are the producer and the epilogue.  An item covers the
// whole k range of one strip, so there is no split-K exchange and the accumulators go straight to the output transform.
// Weights and activations arrive by plain 1-D bulk copies (eight 256K-byte trellis rows per 128 x 128 unit) from addresses
// read out of the device pointer tables: no tensor map has to be encoded on the host or patched per CTA and fenced when a
// CTA moves to another expert.
#include "f16_pipeline.cuh"
#include "act.cuh"
#include <mutex>
#include <vector>

namespace exl3b {

using namespace ptx;

constexpr int MOE_ROUTE_THREADS = 1024;

__host__ __device__ inline int moe_padded(int rows) { return (rows + 15) & ~15; }

// The work list of one call.  Experts in index order; an expert is processed when 0 < c_e <= T and its positions lie inside
// [end of the previous processed expert, num_positions), so processed ranges are disjoint and ascending even for malformed
// counts.  Each processed expert is cut into passes of <= F16_MAX_ROWS consecutive positions; passes are packed in order into
// chunks of at most chunk_rows padded rows.  The same function runs in the route kernel and behind exl3b_moe_plan.
struct MoePlanArrays
{
    MoePass* passes; int max_passes;
    int* chunk_first; int max_chunks;      // chunk c holds passes [chunk_first[c], chunk_first[c + 1]); max_chunks + 1 entries
    int* p_start; int* p_rows; int* p_pass0;   // per processed expert, in order: first position, rows, first pass
};
struct MoePlanCounts { int passes, chunks, experts, rows; };      // rows: most rows any chunk uses

__host__ __device__ inline bool moe_processed(long long c, long long s, long long lo, int T, int N)
{
    return c > 0 && c <= T && s >= lo && s + c <= N;
}
// returns false if the list does not fit max_passes / max_chunks (the host's bounds make that impossible)
__host__ __device__ inline bool moe_plan(const long long* count, int E, int T, int N, int chunk_rows, const MoePlanArrays& a,
                                         MoePlanCounts* out)
{
    long long s = 0, lo = 0;
    int P = 0, R = 0, C = 0, Rmax = 0, np = 0;
    if (a.max_chunks < 1) return false;
    a.chunk_first[0] = 0;
    for (int e = 0; e < E; ++e)
    {
        const long long c = count[e];
        if (moe_processed(c, s, lo, T, N))
        {
            a.p_start[np] = (int) s; a.p_rows[np] = (int) c; a.p_pass0[np] = P; ++np;
            for (int r0 = 0; r0 < (int) c; r0 += F16_MAX_ROWS)
            {
                const int rows = (int) c - r0 < F16_MAX_ROWS ? (int) c - r0 : F16_MAX_ROWS;
                const int pad = moe_padded(rows);
                if (R + pad > chunk_rows)
                {
                    if (++C >= a.max_chunks) return false;
                    a.chunk_first[C] = P;
                    R = 0;
                }
                if (P >= a.max_passes) return false;
                a.passes[P].expert = e; a.passes[P].pos0 = (int) s + r0; a.passes[P].rows = rows;
                a.passes[P].row0 = R; a.passes[P].chunk = C;
                R += pad;
                if (R > Rmax) Rmax = R;
                ++P;
            }
            lo = s + c;
        }
        s += c;
    }
    const int chunks = P > 0 ? C + 1 : 0;
    a.chunk_first[chunks] = P;
    out->passes = P; out->chunks = chunks; out->experts = np; out->rows = Rmax;
    return true;
}

// position j -> 128 * pass + row in the pass, -1 if j is not processed: the last processed expert starting at or before j,
// if its range holds j
__host__ __device__ inline int moe_pos_code(int j, int np, const int* p_start, const int* p_rows, const int* p_pass0)
{
    int lo = 0, hi = np;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (p_start[mid] <= j) lo = mid + 1; else hi = mid; }
    const int i = lo - 1;
    if (i < 0 || j >= p_start[i] + p_rows[i]) return -1;
    const int r = j - p_start[i];
    return (p_pass0[i] + r / F16_MAX_ROWS) * 128 + r % F16_MAX_ROWS;
}

// ---- fixed per-device work area ------------------------------------------------------------------------------------------
// Allocated once per device by the first exl3_moe call and never grown, freed or moved (captured graphs stay valid).  The
// work-list region bounds one call's positions and tokens; the row region holds one chunk's tiles and rows, so larger calls
// run in more chunks instead of needing more memory.
constexpr long long MOE_MAX_POSITIONS = 1 << 20;        // positions and tokens of one call
constexpr int MOE_MAX_PASSES = MOE_MAX_EXPERTS + (int) (MOE_MAX_POSITIONS / F16_MAX_ROWS);
constexpr int MOE_MAX_CHUNKS = 4096;
constexpr size_t MOE_ROW_BYTES = (size_t) 240 << 20;

// rows of one chunk: gate + up tiles (2 x fp16, later down's fp32 rows) 4 * hidden bytes, g / u / down tiles 6 * inter bytes
static int moe_chunk_rows(int hidden, int inter)
{
    const long long r = (long long) (MOE_ROW_BYTES / ((size_t) 4 * hidden + (size_t) 6 * inter)) & ~15ll;
    return r > (1 << 24) ? (1 << 24) : (int) r;
}

// Host bounds of one call, from sizes alone: at most min(N, E * T) positions are processed, each pass has >= 1 row, an expert
// with c rows has <= 1 + c / 128 passes, and every chunk but the last is filled beyond chunk_rows - 128 (rows are multiples
// of 16, so beyond chunk_rows - 112).
struct MoeBounds { long long passes, rows, chunks; };
static MoeBounds moe_bounds(long long N, long long E, long long T, int chunk_rows)
{
    MoeBounds b;
    const long long np = N < E * T ? N : E * T;
    b.passes = np < E + np / F16_MAX_ROWS ? np : E + np / F16_MAX_ROWS;
    b.rows = np + 15 * b.passes;
    b.chunks = b.rows == 0 ? 0 : 1 + b.rows / (chunk_rows - 112);
    return b;
}

// ---- 1. route ---------------------------------------------------------------------------------------------------------
struct MoeWork
{
    int* hdr;                  // [0] passes, [1] chunks
    MoePass* passes;
    int* chunk_first;          // [chunks + 1]
    int* pos_code;             // [N] 128 * pass + row in pass, -1 = not processed
    int* tok_cnt;              // [bsz] counts, then fill cursors
    int* tok_off;              // [bsz + 1]
    int* tok_list;             // [N] processed positions grouped by token, ascending within a token
};

__global__ void __launch_bounds__(MOE_ROUTE_THREADS)
moe_route_kernel(MoeWork w, const int64_t* __restrict__ expert_count, const int64_t* __restrict__ token_sorted,
                 int E, int T, int N, int bsz, int chunk_rows, int max_passes, int max_chunks)
{
    __shared__ long long s_count[MOE_MAX_EXPERTS];
    __shared__ int s_start[MOE_MAX_EXPERTS];        // processed experts in order: first position, rows, first pass
    __shared__ int s_rows[MOE_MAX_EXPERTS];
    __shared__ int s_pass0[MOE_MAX_EXPERTS];
    __shared__ int s_scan[MOE_ROUTE_THREADS];
    __shared__ int s_nproc;
    const int tid = threadIdx.x;
    pdl_launch_dependents();
    pdl_wait();                                      // the previous call's kernels read the work list

    for (int e = tid; e < E; e += MOE_ROUTE_THREADS) s_count[e] = expert_count[e];
    for (int t = tid; t < bsz; t += MOE_ROUTE_THREADS) w.tok_cnt[t] = 0;
    __syncthreads();
    if (tid == 0)
    {
        const MoePlanArrays arr{w.passes, max_passes, w.chunk_first, max_chunks, s_start, s_rows, s_pass0};
        MoePlanCounts pc{};
        const bool ok = moe_plan(s_count, E, T, N, chunk_rows, arr, &pc);     // always true: the host's bounds
        w.hdr[0] = ok ? pc.passes : 0; w.hdr[1] = ok ? pc.chunks : 0;
        s_nproc = ok ? pc.experts : 0;
    }
    __syncthreads();

    const int np = s_nproc;
    for (int j = tid; j < N; j += MOE_ROUTE_THREADS)
    {
        const int code = moe_pos_code(j, np, s_start, s_rows, s_pass0);
        w.pos_code[j] = code;
        const long long t = token_sorted[j];
        if (code >= 0 && t >= 0 && t < bsz) atomicAdd(&w.tok_cnt[t], 1);
    }
    __syncthreads();

    // exclusive scan of the token counts: each thread owns a contiguous chunk of tokens
    const int per = (bsz + MOE_ROUTE_THREADS - 1) / MOE_ROUTE_THREADS;
    const int t0 = tid * per, t1 = t0 + per < bsz ? t0 + per : bsz;
    int local = 0;
    for (int t = t0; t < t1; ++t) local += w.tok_cnt[t];
    s_scan[tid] = local;
    __syncthreads();
    for (int d = 1; d < MOE_ROUTE_THREADS; d <<= 1)
    {
        const int v = tid >= d ? s_scan[tid - d] : 0;
        __syncthreads();
        s_scan[tid] += v;
        __syncthreads();
    }
    int run = s_scan[tid] - local;
    for (int t = t0; t < t1; ++t) { w.tok_off[t] = run; run += w.tok_cnt[t]; w.tok_cnt[t] = 0; }
    if (tid == MOE_ROUTE_THREADS - 1) w.tok_off[bsz] = s_scan[tid];
    __syncthreads();

    for (int j = tid; j < N; j += MOE_ROUTE_THREADS)
    {
        const long long t = token_sorted[j];
        if (w.pos_code[j] >= 0 && t >= 0 && t < bsz) w.tok_list[w.tok_off[t] + atomicAdd(&w.tok_cnt[t], 1)] = j;
    }
    __syncthreads();
    for (int t = tid; t < bsz; t += MOE_ROUTE_THREADS)                 // the fill order above is arbitrary: sort each list
    {
        int* l = w.tok_list + w.tok_off[t];
        const int n = w.tok_off[t + 1] - w.tok_off[t];
        for (int a = 1; a < n; ++a)
        {
            const int v = l[a];
            int b = a - 1;
            while (b >= 0 && l[b] > v) { l[b + 1] = l[b]; --b; }
            l[b + 1] = v;
        }
    }
}

// ---- 2. gather + input transform --------------------------------------------------------------------------------------------
// One warp per (position, 128-k block): x[token] through the tag-200 input transform (xt_transform) into the pass's tile.
// Pass p's tiles start at row0 * k fp16; block kb of it is NT * 256 bytes.

__global__ void __launch_bounds__(128)
moe_gather_kernel(MoeWork w, const half* __restrict__ x, const int64_t* __restrict__ token_sorted,
                  const uint64_t* __restrict__ suh_g, const uint64_t* __restrict__ suh_u, uint8_t* xg, uint8_t* xu,
                  int N, int k, int bsz, int gated, int chunk)
{
    pdl_launch_dependents();
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int KB = k / 128;
    if (warp >= N * KB) return;
    const int j = warp / KB, kb = warp % KB;
    const int code = w.pos_code[j];
    if (code < 0) return;
    const MoePass ps = w.passes[code >> 7];
    if (ps.chunk != chunk) return;
    const int r = code & 127;
    const long long t = token_sorted[j];
    uint2 raw = make_uint2(0, 0);
    if (t >= 0 && t < bsz) raw = *reinterpret_cast<const uint2*>(x + (size_t) t * k + kb * 128 + lane * 4);
    const size_t off = (size_t) ps.row0 * k * 2 + (size_t) kb * moe_padded(ps.rows) * 256 + xt_tile_offset(r, lane);
    const int c0 = kb * 128 + lane * 4;
    if (gated) store_tile_pair(xg + off, xt_transform(raw, (const half*) suh_g[ps.expert] + c0, lane));
    store_tile_pair(xu + off, xt_transform(raw, (const half*) suh_u[ps.expert] + c0, lane));
}

// ---- 3, 4, 6. grouped decode-GEMM ---------------------------------------------------------------------------------------------
struct MoeGemmParams
{
    const int* hdr; const MoePass* passes; const int* chunk_first;
    int chunk;                         // items: (pass of this chunk, 128-column strip)
    const uint8_t* x;                  // tiles: pass p at x + row0 * k * 2
    const uint64_t* B_ptrs; const uint64_t* svh_ptrs;
    void* C; int c_fp32;               // [padded rows][n], row-major
    int k, n, stages;
};

template <int K, int cb>
__global__ void __launch_bounds__(F16_THREADS, 1)
moe_gemm_kernel(const MoeGemmParams p)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const TcSmemLayout L = f16_smem_layout(K, F16_MAX_ROWS * 256, p.stages, F16_MAX_ROWS);
    // values broadcast from lane 0 are warp-uniform to ptxas: without that, a loop bound or wgmma predicate loaded from memory
    // counts as divergent and ptxas serializes the wgmma (C7520)
    auto uni = [](int v) { return __shfl_sync(0xffffffffu, v, 0); };
    const int warp = uni(threadIdx.x >> 5), lane = threadIdx.x & 31;
    const int S = p.stages;
    const uint32_t bar0 = smem_u32(smem + L.off_bars);
    auto FULL = [&](int s) { return bar0 + 8u * s; };
    auto EMPTY = [&](int s) { return bar0 + 8u * (S + s); };

    pdl_launch_dependents();
    if (warp == 0)
    {
        for (int s = lane; s < S; s += 32) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), F16_CONS_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    pdl_wait();                                      // the work list and the tiles come from the previous kernels

    const int KB = p.k / 128, strips = p.n / 128;
    const bool live = p.chunk < uni(p.hdr[1]);
    const int pass0 = live ? uni(p.chunk_first[p.chunk]) : 0;
    const int items = live ? (uni(p.chunk_first[p.chunk + 1]) - pass0) * strips : 0;
    const int G = gridDim.x;

    if (warp == 0)
    {
        // =========================== producer ===========================
        const uint64_t pol_w = policy_evict_first(), pol_x = policy_evict_last();
        const uint32_t w_smem0 = smem_u32(smem), x_smem0 = smem_u32(smem + L.off_b);
        const size_t row_bytes = (size_t) strips * 256 * K;          // one trellis row: n / 16 tiles of 32 K bytes
        int s = 0, ph = 0;
        for (int it = blockIdx.x; it < items; it += G)
        {
            const int pi = it / strips, strip = it - pi * strips;
            const MoePass ps = p.passes[pass0 + pi];
            const int expert = uni(ps.expert), rows = uni(ps.rows), row0 = uni(ps.row0);
            const uint8_t* B = reinterpret_cast<const uint8_t*>(p.B_ptrs[expert]) + (size_t) strip * 256 * K;
            const uint32_t x_bytes = (uint32_t) moe_padded(rows) * 256;
            const uint8_t* xp = p.x + (size_t) row0 * p.k * 2;
            for (int kb = 0; kb < KB; ++kb)
            {
                mbar_wait<64>(EMPTY(s), ph ^ 1);
                if (elect_one())
                {
                    mbar_arrive_expect_tx(FULL(s), (uint32_t) L.w_bytes + x_bytes);
                    #pragma unroll
                    for (int r = 0; r < 8; ++r)
                        bulk_g2s(w_smem0 + s * L.w_bytes + r * 256 * K, B + (size_t) (kb * 8 + r) * row_bytes, 256 * K, FULL(s), pol_w);
                    bulk_g2s(x_smem0 + s * L.b_bytes, xp + (size_t) kb * x_bytes, x_bytes, FULL(s), pol_x);
                }
                __syncwarp();
                if (++s == S) { s = 0; ph ^= 1; }
            }
        }
    }
    else if (warp >= F16_CONS_WARP0)
    {
        // =========================== decode + MMA + epilogue (two warpgroups) ===========================
        const int ct = threadIdx.x - F16_CONS_WARP0 * 32;
        const int cw = ct >> 5;
        const int h = cw >> 2, wq = cw & 3;
        const int tl = 4 * h + wq;
        const int chunk = lane >> 2, c = lane & 3;
        float* tile = reinterpret_cast<float*>(smem + L.off_tile);
        auto cons_bar = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };
        const uint64_t desc0 = f16_tile_desc(smem + L.off_b);

        float acc[F16_MAX_ROWS / 16][8];
        int s = 0, sph = 0;
        for (int it = blockIdx.x; it < items; it += G)
        {
            const int pi = it / strips, strip = it - pi * strips;
            const MoePass ps = p.passes[pass0 + pi];
            const int expert = uni(ps.expert), rows = uni(ps.rows), row0 = uni(ps.row0);
            const int nchunks = moe_padded(rows) / 16;
            f16_zero(acc);

            for (int kb = 0; kb < KB; ++kb)
            {
                mbar_wait<32>(FULL(s), sph);
                uint32_t wr[2][K + 1];
                f16_load_unit<K>(reinterpret_cast<const uint32_t*>(smem + s * L.w_bytes), tl, chunk, c, wr);
                const uint64_t desc_s = desc0 + (uint64_t) ((s * L.b_bytes) >> 4);
                #pragma unroll
                for (int r = 0; r < 2; ++r)
                {
                    uint32_t o0[8], o1[8];
                    decode16<K, cb, 0>(wr[r], o0);
                    decode16<K, cb, 1>(wr[r], o1);
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
                if (lane == 0) mbar_arrive(EMPTY(s));
                if (++s == S) { s = 0; sph ^= 1; }
            }

            // accumulators -> tile -> output transform of the pass's rows
            cons_bar();                                              // the previous item's epilogue has read the tile
            f16_store_tile(tile, acc, tl, chunk, c, nchunks);
            cons_bar();
            const half* svh = reinterpret_cast<const half*>(p.svh_ptrs[expert]) + strip * 128;
            for (int j = cw; j < rows; j += F16_CONS_WARPS)
                output_row_128(tile + j * 128, (char*) p.C, (size_t) (row0 + j) * p.n + strip * 128, svh, 1.0f, p.c_fp32 != 0, lane);
        }
    }
    __syncthreads();
}

// ---- 5. activation into down's input ---------------------------------------------------------------------------------------
// g, u are fp16 exl3_gemm outputs (output Hadamard and svh applied).  h = fp16(act(g) * u) with the limit rule of act.cuh and
// exl3_moe's own SiLU / GELU expressions (act.cuh); then down's input transform.  ReLU^2 without a gate: act = max(u, 0), taken before the clamp.
__global__ void __launch_bounds__(128)
moe_act_kernel(MoeWork w, const half* __restrict__ g, const half* __restrict__ u, const uint64_t* __restrict__ suh_d,
               uint8_t* xd, int N, int k, int act, float limit, int chunk)
{
    pdl_launch_dependents();
    pdl_wait();
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    const int KB = k / 128;
    if (warp >= N * KB) return;
    const int j = warp / KB, kb = warp % KB;
    const int code = w.pos_code[j];
    if (code < 0) return;
    const MoePass ps = w.passes[code >> 7];
    if (ps.chunk != chunk) return;
    const int r = code & 127;
    const size_t e0 = (size_t) (ps.row0 + r) * k + kb * 128 + lane * 4;
    const uint2 ur = *reinterpret_cast<const uint2*>(u + e0);
    const uint2 gr = act == 2 ? ur : *reinterpret_cast<const uint2*>(g + e0);
    const half* uh = reinterpret_cast<const half*>(&ur);
    const half* gh = reinterpret_cast<const half*>(&gr);
    half hv[4];
    #pragma unroll
    for (int i = 0; i < 4; ++i)
    {
        const float uf = __half2float(uh[i]), gf = __half2float(gh[i]);
        hv[i] = act_limit_mul(act == ACT_SILU ? act_silu_moe(gf) : act == ACT_GELU ? act_gelu_moe(gf) : fmaxf(uf, 0.0f), uf, limit);
    }
    uint2 raw;
    raw.x = pack_half2(hv[0], hv[1]); raw.y = pack_half2(hv[2], hv[3]);
    const size_t off = (size_t) ps.row0 * k * 2 + (size_t) kb * moe_padded(ps.rows) * 256 + xt_tile_offset(r, lane);
    store_tile_pair(xd + off, xt_transform(raw, (const half*) suh_d[ps.expert] + kb * 128 + lane * 4, lane));
}

// ---- 7. fixed-order weighted sum into output_state ------------------------------------------------------------------------
__global__ void __launch_bounds__(128)
moe_reduce_kernel(MoeWork w, float* out, const half* __restrict__ weight_sorted, const float* __restrict__ d, int hidden, int chunk)
{
    pdl_launch_dependents();
    pdl_wait();
    const int t = blockIdx.x;
    const int col = (blockIdx.y * 128 + threadIdx.x) * 4;
    if (col >= hidden) return;
    const int b = w.tok_off[t], e = w.tok_off[t + 1];
    float4* o = reinterpret_cast<float4*>(out + (size_t) t * hidden + col);
    float4 acc;
    bool any = false;                                // no position in this chunk: the row keeps its bits
    for (int i = b; i < e; ++i)
    {
        const int j = w.tok_list[i];
        const int code = w.pos_code[j];
        const MoePass ps = w.passes[code >> 7];
        if (ps.chunk != chunk) continue;
        if (!any) { acc = *o; any = true; }
        const int row = ps.row0 + (code & 127);
        const float wt = __half2float(weight_sorted[j]);
        const float4 v = *reinterpret_cast<const float4*>(d + (size_t) row * hidden + col);
        acc.x = __fadd_rn(acc.x, __fmul_rn(wt, v.x));
        acc.y = __fadd_rn(acc.y, __fmul_rn(wt, v.y));
        acc.z = __fadd_rn(acc.z, __fmul_rn(wt, v.z));
        acc.w = __fadd_rn(acc.w, __fmul_rn(wt, v.w));
    }
    if (any) *o = acc;
}

// ---- host side -------------------------------------------------------------------------------------------------------------

// The per-device work area (see MOE_ROW_BYTES): work list [hdr | passes | chunk_first | pos_code | tok_cnt | tok_off | tok_list],
// then the row region.  One chunk's row region: gate + up tiles (later down's fp32 rows, aliasing them: both tiles are dead by
// then), g rows, u rows, down tiles.
static size_t align256(size_t b) { return (b + 255) & ~(size_t) 255; }
struct MoeLayout { size_t hdr, passes, chunk_first, pos_code, tok_cnt, tok_off, tok_list, rows, total; };
static MoeLayout moe_layout()
{
    MoeLayout L; size_t o = 0;
    L.hdr = o;         o += align256(16);
    L.passes = o;      o += align256((size_t) MOE_MAX_PASSES * sizeof(MoePass));
    L.chunk_first = o; o += align256((size_t) (MOE_MAX_CHUNKS + 1) * 4);
    L.pos_code = o;    o += align256((size_t) MOE_MAX_POSITIONS * 4);
    L.tok_cnt = o;     o += align256((size_t) MOE_MAX_POSITIONS * 4);
    L.tok_off = o;     o += align256((size_t) (MOE_MAX_POSITIONS + 1) * 4);
    L.tok_list = o;    o += align256((size_t) MOE_MAX_POSITIONS * 4);
    L.rows = o;        o += MOE_ROW_BYTES;
    L.total = o;
    return L;
}
static uint8_t* g_moe_area[32] = {};
static std::mutex g_moe_mu;

// the limits of one call (shared by the launcher and exl3b_moe_plan): positions and tokens within the work list, a chunk holds
// at least one full pass, and the host's bound on chunks fits the chunk table
static int moe_limits(long long N, int E, int T, long long bsz, int hidden, int inter, int* chunk_rows, MoeBounds* b)
{
    EXL3B_CHECK(N <= MOE_MAX_POSITIONS && bsz <= MOE_MAX_POSITIONS, EXL3B_ERR_UNSUPPORTED,
                "exl3_moe: at most %lld positions and tokens per call (got %lld, %lld)", MOE_MAX_POSITIONS, N, bsz);
    const long long kb = (hidden > inter ? hidden : inter) / 128;
    EXL3B_CHECK(N * kb * 32 <= 0x7fffffffll, EXL3B_ERR_UNSUPPORTED, "exl3_moe: positions x width too large for one call");
    *chunk_rows = moe_chunk_rows(hidden, inter);
    EXL3B_CHECK(*chunk_rows >= 2 * F16_MAX_ROWS, EXL3B_ERR_UNSUPPORTED, "exl3_moe: hidden %d / intermediate %d too large for the work area",
                hidden, inter);
    *b = moe_bounds(N, E, T, *chunk_rows);
    EXL3B_CHECK(b->passes <= MOE_MAX_PASSES && b->chunks <= MOE_MAX_CHUNKS, EXL3B_ERR_UNSUPPORTED, "exl3_moe: work list too long");
    return 0;
}

template <int K, int cb>
static void moe_gemm_launch(cudaStream_t stream, int grid, const MoeGemmParams& p, cudaError_t* err)
{
    *err = launch_pdl<moe_gemm_kernel<K, cb>>(stream, dim3(grid), F16_THREADS, f16_smem_layout(K, F16_MAX_ROWS * 256, p.stages, F16_MAX_ROWS).total, p);
}

static int moe_gemm(cudaStream_t stream, const MoeWork& w, int chunk, long long grid_passes, const uint8_t* x,
                    const uint64_t* B_ptrs, const uint64_t* svh_ptrs, void* C, int c_fp32, int k, int n, int K, int cb, int num_sms)
{
    MoeGemmParams p{};
    p.hdr = w.hdr; p.passes = w.passes; p.chunk_first = w.chunk_first; p.chunk = chunk;
    p.x = x; p.B_ptrs = B_ptrs; p.svh_ptrs = svh_ptrs; p.C = C; p.c_fp32 = c_fp32;
    p.k = k; p.n = n; p.stages = f16_stages(K, F16_MAX_ROWS);
    const long long items = grid_passes * (n / 128);
    const int grid = items < num_sms ? (int) items : num_sms;
    cudaError_t err = cudaSuccess;
    EXL3B_DISPATCH_K_CB(moe_gemm_launch, K, cb, stream, grid, p, &err);
    count_launch();
    EXL3B_CUDA(err);
    return 0;
}

int moe_plan_host(const int64_t* count, int E, int T, int N, int hidden, int inter, struct exl3b_moe_plan* out, int32_t* passes_out,
                  int32_t* pos_code_out)
{
    EXL3B_CHECK(count && out && E >= 1 && E <= MOE_MAX_EXPERTS && T >= 1 && N >= 0 && hidden >= 128 && hidden % 128 == 0
                && inter >= 128 && inter % 128 == 0, EXL3B_ERR_ARG, "exl3_moe_plan: bad argument");
    int chunk_rows; MoeBounds b;
    { int r = moe_limits(N, E, T, 1, hidden, inter, &chunk_rows, &b); if (r) return r; }
    std::vector<long long> c(count, count + E);
    std::vector<MoePass> ps((size_t) (b.passes > 0 ? b.passes : 1));
    std::vector<int> cf((size_t) b.chunks + 2), st(E), rw(E), p0(E);
    const MoePlanArrays arr{ps.data(), (int) b.passes, cf.data(), (int) b.chunks + 1, st.data(), rw.data(), p0.data()};
    MoePlanCounts pc{};
    EXL3B_CHECK(moe_plan(c.data(), E, T, N, chunk_rows, arr, &pc), EXL3B_ERR_UNSUPPORTED, "exl3_moe_plan: work list exceeds its bounds");
    out->passes = pc.passes; out->chunks = pc.chunks; out->rows = pc.rows; out->chunk_rows = chunk_rows;
    out->max_passes = (int32_t) b.passes; out->max_chunks = (int32_t) b.chunks;
    out->units_gate_up = (int64_t) pc.passes * (inter / 128); out->units_down = (int64_t) pc.passes * (hidden / 128);
    if (passes_out)
        for (int i = 0; i < pc.passes; ++i)
        {
            int32_t* q = passes_out + 5 * i;
            q[0] = ps[i].expert; q[1] = ps[i].pos0; q[2] = ps[i].rows; q[3] = ps[i].row0; q[4] = ps[i].chunk;
        }
    if (pos_code_out)
        for (int j = 0; j < N; ++j) pos_code_out[j] = moe_pos_code(j, pc.experts, st.data(), rw.data(), p0.data());
    return 0;
}

int launch_moe(cudaStream_t stream, DevCtx* ctx, const MoeArgs& a)
{
    const long long N = a.num_positions;
    int chunk_rows; MoeBounds b;
    { int r = moe_limits(N, a.num_experts, a.max_tokens, a.bsz, a.hidden, a.inter, &chunk_rows, &b); if (r) return r; }
    if (b.chunks == 0) return EXL3B_TAG_NOP;                 // no expert can be processed (E * T == 0 cannot happen: T >= 1)
    const MoeLayout L = moe_layout();
    uint8_t* base;
    {
        std::lock_guard<std::mutex> lock(g_moe_mu);
        uint8_t*& area = g_moe_area[ctx->device & 31];
        if (!area)
        {
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            EXL3B_CUDA(cudaStreamIsCapturing(stream, &cs));
            EXL3B_CHECK(cs == cudaStreamCaptureStatusNone, EXL3B_ERR_UNSUPPORTED,
                        "exl3_moe: the first call on a device allocates its work area; make it outside stream capture");
            EXL3B_CUDA(cudaMalloc(&area, L.total));
        }
        base = area;
    }
    MoeWork w;
    w.hdr = (int*) (base + L.hdr); w.passes = (MoePass*) (base + L.passes); w.chunk_first = (int*) (base + L.chunk_first);
    w.pos_code = (int*) (base + L.pos_code); w.tok_cnt = (int*) (base + L.tok_cnt); w.tok_off = (int*) (base + L.tok_off);
    w.tok_list = (int*) (base + L.tok_list);
    const size_t R = (size_t) chunk_rows;
    uint8_t* xg = base + L.rows;
    uint8_t* xu = xg + R * a.hidden * 2;
    float* d = (float*) xg;
    half* g = (half*) (xg + R * a.hidden * 4);
    half* u = g + R * a.inter;
    uint8_t* xd = (uint8_t*) (u + R * a.inter);
    const int gated = a.act != 2;
    const int KBh = a.hidden / 128, KBi = a.inter / 128;
    // persistent grids: a chunk has at most chunk_rows / 16 passes; num_active (processed experts, if the caller knows it)
    // narrows that further
    long long grid_passes = b.passes < chunk_rows / 16 ? b.passes : chunk_rows / 16;
    if (a.num_active > 0 && a.num_active + N / F16_MAX_ROWS < grid_passes) grid_passes = a.num_active + N / F16_MAX_ROWS;

    cudaError_t e = launch_pdl<moe_route_kernel>(stream, dim3(1), MOE_ROUTE_THREADS, 0, w, a.expert_count, a.token_sorted,
                                                 a.num_experts, a.max_tokens, a.num_positions, a.bsz, chunk_rows, (int) b.passes,
                                                 (int) b.chunks);
    count_launch(); EXL3B_CUDA(e);
    for (int c = 0; c < (int) b.chunks; ++c)
    {
        e = launch_pdl<moe_gather_kernel>(stream, dim3((unsigned) ((N * KBh + 3) / 4)), 128, 0, w, a.hidden_state, a.token_sorted,
                                          a.gate_suh, a.up_suh, xg, xu, a.num_positions, a.hidden, a.bsz, gated, c);
        count_launch(); EXL3B_CUDA(e);
        int r;
        if (gated)
        {
            r = moe_gemm(stream, w, c, grid_passes, xg, a.gate_trellis, a.gate_svh, g, 0, a.hidden, a.inter, a.K_gate, a.cb, ctx->num_sms);
            if (r) return r;
        }
        r = moe_gemm(stream, w, c, grid_passes, xu, a.up_trellis, a.up_svh, u, 0, a.hidden, a.inter, a.K_up, a.cb, ctx->num_sms);
        if (r) return r;
        e = launch_pdl<moe_act_kernel>(stream, dim3((unsigned) ((N * KBi + 3) / 4)), 128, 0, w, (const half*) g, (const half*) u,
                                       a.down_suh, xd, a.num_positions, a.inter, a.act, a.act_limit, c);
        count_launch(); EXL3B_CUDA(e);
        r = moe_gemm(stream, w, c, grid_passes, xd, a.down_trellis, a.down_svh, d, 1, a.inter, a.hidden, a.K_down, a.cb, ctx->num_sms);
        if (r) return r;
        e = launch_pdl<moe_reduce_kernel>(stream, dim3(a.bsz, (a.hidden + 511) / 512), 128, 0, w, a.output_state, a.weight_sorted,
                                          (const float*) d, a.hidden, c);
        count_launch(); EXL3B_CUDA(e);
    }
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC_MOE;
}

}  // namespace exl3b
