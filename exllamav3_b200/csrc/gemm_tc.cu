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
//                    starts BEFORE griddepcontrol.wait: PDL overlap with the previous kernel's tail)
//        warps 2-3   (optional, m <= 8) input transform fused in-kernel: A*suh -> 128-point Hadamard -> fp16 core-matrix tile
//                    written straight into the activation stage
//        warpgroups 1-2  decode + MMA + epilogue: warpgroup h owns output columns 64 h .. 64 h + 63 of the strip.  Lane
//                    (chunk, c) of warp w decodes tile column `chunk` (both halves) of tile 4 h + w for k-tiles c and 4 + c:
//                    the decoded fp16 pairs ARE the wgmma A fragments (rows chunk / chunk + 8, K pairs c / c + 4), so decoded
//                    weights never touch shared memory; the K order inside an instruction is permuted accordingly in the
//                    activation tile.  fp32 accumulators stay in registers over a k-segment, then go through shared memory
//                    into the split-K combine (global workspace, last arriver reduces in fixed order => deterministic),
//                    output Hadamard + svh, store.
//   * activations arrive pre-tiled in the no-swizzle K-major core-matrix layout wgmma reads, written by the input-transform
//     kernel (fused suh scale + 128-point Hadamard), so the B tile is one contiguous bulk copy.
//
// Reference behaviour being replaced: exllamav3_ext/quant/exl3_gemm_kernel.cuh:8-50, exl3_gemm_inner.cuh:22-733.
#include "common.cuh"
#include "decode.cuh"
#include "epilogue.cuh"
#include "tc_common.cuh"
#include <cstdlib>
#include <unordered_map>
#include <mutex>

namespace exl3b {

using namespace ptx;

// ---- input transform into the tiled activation layout ---------------------------------------------------------
// Tile of one unit: [NT / 8 row groups][16 K-chunks][8 rows][8 fp16], K-chunks 128 B apart, row groups 2048 B apart.  K order:
// k = 16 kt + 4 j + 2 h + e (kt = 4 r + c) sits in K-chunk 2 (4 r + j) + h at element 2 c + e, i.e. lane l's four values
// k = 4 l .. 4 l + 3 go to K-chunks 8 (l / 16) + 2 (l % 4) (+1 for the second pair), element pair (l / 4) % 4.
__device__ __forceinline__ int xt_tile_offset(int r, int lane)
{
    return (((r >> 3) * 16 + 8 * (lane >> 4) + 2 * (lane & 3)) * 8 + (r & 7)) * 16 + 4 * ((lane >> 2) & 3);
}
// the two 4-byte halves land 128 B apart (consecutive K-chunks)
__device__ __forceinline__ uint2 pack_tile_pair(half2 a, half2 b)
{
    uint2 o; o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
    return o;
}
__device__ __forceinline__ void store_tile_pair(uint8_t* p, uint2 o)
{
    *reinterpret_cast<uint32_t*>(p) = o.x;
    *reinterpret_cast<uint32_t*>(p + 128) = o.y;
}
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
    half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
    if constexpr (HAD)
    {
        uint2 scb = *reinterpret_cast<const uint2*>(suh + kb * 128 + lane * 4);
        a = __hmul2(a, *reinterpret_cast<half2*>(&scb.x));
        b = __hmul2(b, *reinterpret_cast<half2*>(&scb.y));
        float v0 = __low2float(a), v1 = __high2float(a), v2 = __low2float(b), v3 = __high2float(b);
        had128_warp(v0, v1, v2, v3, lane);
        a = __floats2half2_rn(v0 * R_SCALE, v1 * R_SCALE);
        b = __floats2half2_rn(v2 * R_SCALE, v3 * R_SCALE);
    }
    store_tile_pair(out + (size_t) kb * NT * 256 + xt_tile_offset(r, lane), pack_tile_pair(a, b));
}

// ---- the kernel -------------------------------------------------------------------------------------------------
constexpr int XT_THREADS = 384;
constexpr int XT_MAX_ROWS = 128;                 // activation rows per pass: NT / 16 accumulator chunks of 8 registers
constexpr int XT_CONS_WARP0 = 4, XT_CONS_WARPS = 8;

// smem: weight ring, activation ring, fp32 segment tile [NT][128], barriers
__host__ __device__ inline TcSmemLayout xt_smem_layout(int K, int b_bytes, int stages, int NT)
{
    TcSmemLayout L;
    L.w_bytes = 2048 * K;
    L.b_bytes = b_bytes;
    L.off_b = stages * L.w_bytes;
    L.off_tile = L.off_b + stages * L.b_bytes;
    L.off_bars = L.off_tile + NT * 128 * 4;
    L.total = L.off_bars + 1024;
    L.off_d = L.total;
    return L;
}

// D[64 x 16] (f32) += A[64 x 16] (f16, registers) * B[16 x 16] (f16, shared memory, K-major)
__device__ __forceinline__ void wgmma_f16_n16(float (&d)[8], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc)
{
    asm volatile("wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1, 1, 1, 0;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc) : "memory");
}

template <int K, int cb>
__global__ void __launch_bounds__(XT_THREADS, 1)
gemm_tc_kernel(const TcParams p, const __grid_constant__ CUtensorMap tmap_w)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const TcSmemLayout L = xt_smem_layout(K, p.b_bytes, p.stages, p.NT);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int S = p.stages;

    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    // barrier map: [0,S) w_full  [S,2S) w_empty  [2S,3S) x_full
    const uint32_t bar0 = smem_u32(bars);
    auto W_FULL = [&](int s) { return bar0 + 8u * s; };
    auto W_EMPTY = [&](int s) { return bar0 + 8u * (S + s); };
    auto X_FULL = [&](int s) { return bar0 + 8u * (2 * S + s); };
    int* s_flag = reinterpret_cast<int*>(smem + L.off_bars + 8 * (3 * TC_MAX_STAGES + 20));

    auto stamp = [&](int slot)
    {
#ifdef EXL3B_TC_DEBUG
        if (p.dbg) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); p.dbg[blockIdx.x * 64 + slot] = t; }
#else
        (void) slot;
#endif
    };
    if (threadIdx.x == 0) stamp(0);
    pdl_launch_dependents();

    if (warp == 0)
    {
        // W_EMPTY: the eight consumer warps, after their MMAs have read the stage
        for (int s = lane; s < S; s += 32) { mbar_init(W_FULL(s), 1); mbar_init(X_FULL(s), 1); mbar_init(W_EMPTY(s), XT_CONS_WARPS); }
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) stamp(1);

    // ---- this CTA's unit range ----
    const int KB = p.k / 128;
    const int strips = p.n / 128;
    const long long U = (long long) KB * strips;
    const int G = gridDim.x;
    const long long ubeg = unit_begin(U, G, blockIdx.x), uend = unit_begin(U, G, blockIdx.x + 1);
    const int n_units = (int) (uend - ubeg);

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
        const int strip0 = (int) (ubeg / KB), kb0 = (int) (ubeg % KB);
        int strip = strip0, kb = kb0;
        auto next_unit = [&] { if (++kb == KB) { kb = 0; ++strip; } };
        for (int u = 0; u < pre; ++u) { issue_w(u, strip, kb); next_unit(); }   // weights never depend on the previous kernel
        const bool fused_x = p.A_raw != nullptr;
        if (!fused_x)
        {
            pdl_wait();                                                          // activations do
            int kbx = kb0; for (int u = 0; u < pre; ++u) { issue_x(u, kbx); if (++kbx == KB) kbx = 0; }
        }
        if (lane == 0) stamp(2);
        int s = (pre == S) ? 0 : pre, ph = (pre == S) ? 1 : 0;                   // ring position of unit `pre`
        for (int u = pre; u < n_units; ++u)
        {
            mbar_wait<64>(W_EMPTY(s), ph ^ 1);
            issue_w(s, strip, kb);
            if (!fused_x) issue_x(s, kb);
            next_unit();
            if (++s == S) { s = 0; ph ^= 1; }
        }
        __syncwarp();
    }
    else if (warp >= TC_XF_WARP0 && warp < XT_CONS_WARP0)
    {
        // =========================== fused input transform (m <= 8) ===========================
        if (p.A_raw != nullptr)
        {
            pdl_wait();                                  // A is produced by the previous kernel
            const int xw = warp - TC_XF_WARP0;           // 0 / 1: units of alternating parity
            int kb = (int) ((ubeg + xw) % KB);
            int s = xw % S, ph = 0;
            if (xw >= S) { s = 0; ph = 1; }              // S >= 2 always
            const int kstep = 2 % KB;
            for (int u = xw; u < n_units; u += 2)
            {
                mbar_wait<64>(W_EMPTY(s), ph ^ 1);
                uint8_t* dst = smem + L.off_b + s * L.b_bytes;
                const uint2 scb = p.suh ? *reinterpret_cast<const uint2*>(p.suh + kb * 128 + lane * 4) : make_uint2(0, 0);
                for (int r = 0; r < p.m; ++r)
                {
                    uint2 raw = *reinterpret_cast<const uint2*>(p.A_raw + (size_t) r * p.k + kb * 128 + lane * 4);
                    half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
                    if (p.suh)
                    {
                        a = __hmul2(a, *reinterpret_cast<const half2*>(&scb.x));
                        b = __hmul2(b, *reinterpret_cast<const half2*>(&scb.y));
                        float v0 = __low2float(a), v1 = __high2float(a), v2 = __low2float(b), v3 = __high2float(b);
                        had128_warp(v0, v1, v2, v3, lane);
                        a = __floats2half2_rn(v0 * R_SCALE, v1 * R_SCALE);
                        b = __floats2half2_rn(v2 * R_SCALE, v3 * R_SCALE);
                    }
                    store_tile_pair(dst + xt_tile_offset(r, lane), pack_tile_pair(a, b));
                }
                fence_proxy_async_smem();                // generic-proxy writes -> visible to the tensor-core (async) proxy
                __syncwarp();
                if (lane == 0) mbar_arrive(X_FULL(s));
                kb += kstep; if (kb >= KB) kb -= KB;
                s += 2; if (s >= S) { s -= S; ph ^= 1; }
            }
        }
    }
    else if (warp >= XT_CONS_WARP0)
    {
        // =========================== decode + MMA + epilogue (two warpgroups) ===========================
        const int ct = threadIdx.x - XT_CONS_WARP0 * 32;             // 0..255
        const int cw = ct >> 5;                                      // consumer warp 0..7
        const int h = cw >> 2, wq = cw & 3;
        const int tl = 4 * h + wq;                                   // tile column of the strip owned by this warp
        const int chunk = lane >> 2, c = lane & 3;
        const int nchunks = p.NT / 16;
        float* tile = reinterpret_cast<float*>(smem + L.off_tile);   // [NT][128] fp32: one strip's k-segment sums
        auto cons_bar = [] { asm volatile("bar.sync 1, 256;" ::: "memory"); };
        const int part_stride = p.NT * 128;
        const uint64_t desc0 = smem_desc(smem_u32(smem + L.off_b), 128, 2048, 0);
        pdl_wait();                                                  // no global write before the previous grid has completed

        float acc[XT_MAX_ROWS / 16][8];
        #pragma unroll
        for (int i = 0; i < XT_MAX_ROWS / 16; ++i)
            #pragma unroll
            for (int e = 0; e < 8; ++e) acc[i][e] = 0.f;

        // all rows of one strip: tile (fp32 sums) -> output transform -> C
        auto emit_rows = [&](int strip)
        {
            cons_bar();
            for (int j = cw; j < p.m; j += XT_CONS_WARPS)
                output_row_128(tile + j * 128, (char*) p.C, (size_t) j * p.n + strip * 128,
                               p.svh ? p.svh + strip * 128 : nullptr, p.out_scale, p.c_fp32 != 0, lane);
            cons_bar();
        };

        int s = 0, sph = 0;
        int u = 0;
        while (u < n_units)
        {
            const long long g = ubeg + u;
            const int strip = (int) (g / KB), kb = (int) (g % KB);
            const int to_strip_end = KB - kb;
            const int seg = (n_units - u) < to_strip_end ? (n_units - u) : to_strip_end;
            const long long gs = (long long) strip * KB;
            const int c_a = cta_of_unit(U, G, gs), c_b = cta_of_unit(U, G, gs + KB - 1);
            const int n_contrib = c_b - c_a + 1;
            const bool full = n_contrib == 1;
            float* my_part = p.ws + (size_t) (2 * blockIdx.x + (ubeg >= gs ? 0 : 1)) * part_stride;

            for (int i = 0; i < seg; ++i)
            {
                mbar_wait<32>(W_FULL(s), sph);
                if (u + i == 0 && ct == 0) stamp(3);
                const uint32_t* wst = reinterpret_cast<const uint32_t*>(smem + s * L.w_bytes);
                uint32_t w[2][K + 1];
                #pragma unroll
                for (int r = 0; r < 2; ++r) load_chunk<K>(wst + ((4 * r + c) * 8 + tl) * (8 * K), chunk, w[r]);
                mbar_wait(X_FULL(s), sph);
                const uint64_t desc_s = desc0 + (uint64_t) ((s * L.b_bytes) >> 4);
                #pragma unroll
                for (int r = 0; r < 2; ++r)
                {
                    uint32_t o0[8], o1[8];
                    decode16<K, cb, 0>(w[r], o0);
                    decode16<K, cb, 1>(w[r], o1);
                    #pragma unroll
                    for (int ii = 0; ii < XT_MAX_ROWS / 16; ++ii)
                        #pragma unroll
                        for (int e = 0; e < 8; ++e) reg_fence(acc[ii][e]);
                    wgmma_fence();
                    #pragma unroll
                    for (int j = 0; j < 4; ++j)
                    {
                        // instruction 4 r + j: K-chunks 2 (4 r + j), +1;  N-chunk ii: row groups 2 ii, 2 ii + 1
                        #pragma unroll
                        for (int ii = 0; ii < XT_MAX_ROWS / 16; ++ii)
                            if (ii < nchunks)
                                wgmma_f16_n16(acc[ii], o0[2 * j], o1[2 * j], o0[2 * j + 1], o1[2 * j + 1],
                                              desc_s + (uint64_t) (16 * (4 * r + j) + 256 * ii));
                    }
                    wgmma_commit();
                    wgmma_wait<0>();
                    #pragma unroll
                    for (int e = 0; e < 8; ++e) { reg_fence(o0[e]); reg_fence(o1[e]); }
                    #pragma unroll
                    for (int ii = 0; ii < XT_MAX_ROWS / 16; ++ii)
                        #pragma unroll
                        for (int e = 0; e < 8; ++e) reg_fence(acc[ii][e]);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(W_EMPTY(s));
                if (++s == S) { s = 0; sph ^= 1; }
            }

            // accumulators -> tile[row][column]: fragment (row 16 ii + 2 c + e (+8), column 16 tl + chunk (+8))
            cons_bar();                                              // the previous segment's readers of the tile are done
            const int n0 = 16 * tl + chunk;
            #pragma unroll
            for (int ii = 0; ii < XT_MAX_ROWS / 16; ++ii)
            {
                if (ii < nchunks)
                {
                    const int r0 = 16 * ii + 2 * c;
                    tile[(r0 + 0) * 128 + n0] = acc[ii][0];
                    tile[(r0 + 1) * 128 + n0] = acc[ii][1];
                    tile[(r0 + 0) * 128 + n0 + 8] = acc[ii][2];
                    tile[(r0 + 1) * 128 + n0 + 8] = acc[ii][3];
                    tile[(r0 + 8) * 128 + n0] = acc[ii][4];
                    tile[(r0 + 9) * 128 + n0] = acc[ii][5];
                    tile[(r0 + 8) * 128 + n0 + 8] = acc[ii][6];
                    tile[(r0 + 9) * 128 + n0 + 8] = acc[ii][7];
                }
                #pragma unroll
                for (int e = 0; e < 8; ++e) acc[ii][e] = 0.f;
            }
            if (u + seg >= n_units && ct == 0) stamp(7);
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
        if (ct == 0) stamp(8);
    }

    // ---- teardown ----
    __syncthreads();
    if (threadIdx.x == 0) stamp(9);
}

// ---- host side -------------------------------------------------------------------------------------------------------

// ---- tensor map for the trellis: 2-D view [k/16 rows][n/16 * 32K bytes] in uint64 elements, box = 8 rows x 256K bytes ----
typedef CUresult (*PFN_encodeTiled)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                    const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

int get_weight_tmap(const void* B, int k, int n, int K, CUtensorMap* out)
{
#ifdef EXL3B_TC_DEBUG
    const bool flat = (g_tc_knob & 16) != 0;     // experiment: contiguous 8-row boxes (wrong data, same bytes)
#else
    constexpr bool flat = false;
#endif
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
    Key key{B, flat ? -k : k, n, K};
    auto it = cache.find(key);
    if (it == cache.end())
    {
        CUtensorMap tm;
        cuuint64_t row_bytes = (cuuint64_t) (n / 16) * 32 * K;
        cuuint64_t rows = (cuuint64_t) (k / 16);
        if (flat) { rows = rows * (n / 128); row_bytes = 256 * K; }
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
static cudaError_t tc_launch(cudaStream_t stream, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap)
{
    static bool attr_set[32] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (!attr_set[dev & 31])
    {
        cudaError_t e = cudaFuncSetAttribute(gemm_tc_kernel<K, cb>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 31] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(XT_THREADS); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, gemm_tc_kernel<K, cb>, p, tmap);
}

template <int K, int cb>
static void tc_launch_v(cudaStream_t stream, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap,
                        cudaError_t* err)
{
    *err = tc_launch<K, cb>(stream, grid, smem_bytes, p, tmap);
}

unsigned long long* g_tc_dbg = nullptr;
int g_tc_knob = 0;
// bring-up hooks: live only in the EXL3B_TC_DEBUG build (libexl3b200_dbg.so); the production library ignores them, so no
// exported call can change what its kernels compute
#ifdef EXL3B_TC_DEBUG
void tc_set_debug_buffer(unsigned long long* d) { g_tc_dbg = d; }
void tc_set_knob(int k) { g_tc_knob = k; }
#else
void tc_set_debug_buffer(unsigned long long*) { }
void tc_set_knob(int) { }
#endif

bool gemm_tc_supported(const GemmArgs& a)
{
    return a.k >= 128 && a.n >= 128 && a.k % 128 == 0 && a.n % 128 == 0 && a.m >= 1;
}

static int launch_had_tiled(cudaStream_t stream, const half* A, uint8_t* out, const half* suh, int m, int k, int NT)
{
    const int warps = m * (k / 128);
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((warps + 3) / 4); cfg.blockDim = dim3(128); cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    cudaError_t e = suh ? cudaLaunchKernelEx(&cfg, had_tiled_kernel<true>, A, out, suh, m, k, NT)
                        : cudaLaunchKernelEx(&cfg, had_tiled_kernel<false>, A, out, suh, m, k, NT);
    count_launch();
    EXL3B_CUDA(e);
    return 0;
}

// In-kernel input transform (two warps, per unit) or the separate had_tiled launch + tile loads?  The two transform warps do one
// 128-point Hadamard per row and unit and pace the kernel as rows grow, so the tiled path is the default for every row count;
// EXL3B_FUSED_X_ROWS=r (<= 8) brings the in-kernel transform back for up to r rows.
static bool tc_fused_x(int m, int k, int n, int num_sms)
{
    (void) k; (void) n; (void) num_sms;
    static int max_rows = -1;
    if (max_rows < 0)
    {
        const char* e = getenv("EXL3B_FUSED_X_ROWS");
        max_rows = e ? atoi(e) : 0;
        if (max_rows > 8) max_rows = 8;
    }
    return m <= max_rows;
}

// launch geometry of one pass (m <= XT_MAX_ROWS rows), also behind exl3b_gemm_plan
int plan_gemm_tc(int m, int k, int n, int K, int num_sms, int max_ctas, TcPlan* pl)
{
    EXL3B_CHECK(m >= 1 && m <= XT_MAX_ROWS, EXL3B_ERR_ARG, "plan_gemm_tc: one pass handles 1..%d rows", XT_MAX_ROWS);
    const int NT = (m + 15) / 16 * 16;
    const bool fused_x = tc_fused_x(m, k, n, num_sms);
    // accumulators live in the consumer warpgroups' registers: no operand stages or accumulator buffers to plan
    pl->tmem_cols = 0;
    pl->a_stages = 0;
    pl->d_bufs = 1;
    pl->b_load_bytes = m <= 8 ? 2048 : NT * 256;
    const int b_bytes = fused_x ? 2048 : NT * 256;       // m <= 8: only the first row group is ever written / needed
    const int stage_bytes = 2048 * K + b_bytes;
    const int budget = 200 * 1024 - NT * 128 * 4;
    int stages = budget / stage_bytes;
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages < 2) stages = 2;
    const TcSmemLayout L = xt_smem_layout(K, b_bytes, stages, NT);
    EXL3B_CHECK(L.total <= 220 * 1024, EXL3B_ERR_UNSUPPORTED, "exl3_gemm: shared-memory budget exceeded");
    const long long U = (long long) (k / 128) * (n / 128);
    int grid = num_sms;
    if (max_ctas > 0 && max_ctas < grid) grid = max_ctas;
    if (grid > U) grid = (int) U;
    EXL3B_CHECK((size_t) 2 * grid * NT * 128 * 4 <= DevCtx::WS_BYTES_PER_SLOT, EXL3B_ERR_UNSUPPORTED,
                "exl3_gemm: split-K workspace too small");
    EXL3B_CHECK(n / 128 <= DevCtx::COUNTERS_PER_SLOT, EXL3B_ERR_UNSUPPORTED, "exl3_gemm: too many column strips");
    pl->rows = NT; pl->stages = stages; pl->b_bytes = b_bytes; pl->smem_total = L.total; pl->grid = grid; pl->units = U;
    return 0;
}

int launch_gemm_tc(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a)
{
    const size_t esz = a.c_fp32 ? 4 : 2;
    CUtensorMap tmap;
    { int r = get_weight_tmap(a.B, a.k, a.n, a.K, &tmap); if (r) return r; }
    for (int m0 = 0; m0 < a.m; m0 += XT_MAX_ROWS)
    {
        const int m = a.m - m0 < XT_MAX_ROWS ? a.m - m0 : XT_MAX_ROWS;
        TcPlan pl;
        { int r = plan_gemm_tc(m, a.k, a.n, a.K, ctx->num_sms, a.max_ctas, &pl); if (r) return r; }
        const int NT = pl.rows;
        const int slot = ctx->next_slot();
        const bool fused_x = tc_fused_x(m, a.k, a.n, ctx->num_sms);
        uint8_t* xh_tiled = nullptr;
        if (!fused_x)
        {
            const size_t xh_bytes = (size_t) (a.k / 128) * NT * 256;
            int r = ensure_xh_tiled(ctx, xh_bytes); if (r) return r;
            xh_tiled = ctx->xh_tiled + (size_t) (slot % DevCtx::XH_SLOTS) * ctx->xh_tiled_slot_bytes;
            r = launch_had_tiled(stream, a.A + (size_t) m0 * a.k, xh_tiled, a.suh, m, a.k, NT); if (r) return r;
        }

        TcParams p{};
        p.xh_tiled = xh_tiled; p.B = a.B; p.C = (char*) a.C + (size_t) m0 * a.n * esz; p.svh = a.svh;
        p.m = m; p.k = a.k; p.n = a.n; p.NT = NT; p.c_fp32 = a.c_fp32; p.out_scale = a.out_scale;
        p.ws = ctx->ws_slot(slot); p.counters = ctx->counter_slot(slot);
        p.b_load_bytes = pl.b_load_bytes;
        p.stages = pl.stages;
        p.dbg = g_tc_dbg;
        p.knob_ = g_tc_knob;
        p.A_raw = fused_x ? a.A + (size_t) m0 * a.k : nullptr;
        p.suh = a.suh;
        p.b_bytes = pl.b_bytes;

        cudaError_t err = cudaSuccess;
        EXL3B_DISPATCH_K_CB(tc_launch_v, a.K, a.cb, stream, pl.grid, pl.smem_total, p, tmap, &err);
        count_launch();
        EXL3B_CUDA(err);
    }
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC;
}

}  // namespace exl3b
