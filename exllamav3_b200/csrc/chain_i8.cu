// Persistent multi-GEMM decode kernel for the mul1 codebook at <= 4 rows ("chain", tag 220): ONE launch runs a list of EXL3
// GEMMs -- a single exl3_gemm, the same-input projections of a block (q + k + v, gate + up), or a whole dependent block
// (gate + up -> silu * mul -> down: what the reference's BC_GatedMLP issues as three launches, libtorch/mlp.cpp:14-91; the
// projections of BC_Attention, libtorch/attention.cpp:286-365) -- with the weight stream never stopping at a GEMM boundary.
//
// Arithmetic per weight is that of gemm_tc_i8_body.cuh (the product word state * 0x83DCD12D as four u8 K-elements of a
// register A operand of wgmma, activations as balanced 16-bit integers in two int8 digits); what is new:
//
//   * ops and stages.  The list is cut into STAGES; the ops of a stage are independent (same or external inputs) and
//     their 128 x 128 units form one stream-K unit space over the persistent grid; a stage's inputs may be outputs of
//     earlier stages.  Between stages there is a grid-wide dependency: every finished 128-column output segment bumps
//     a global counter, and only the warps that PREPARE activations wait for it.  The TMA producer and the decode warps
//     run on into the next stage's weights (they depend on no activation), so HBM streams through the boundary and the
//     first operand stages of the next GEMM are decoded before its input exists.
//   * the unit pipeline itself is the one of gemm_tc_i8_body.cuh (two decode groups of two warpgroups, each warpgroup
//     decoding its weights straight into wgmma A fragments and accumulating in registers).
//   * activation scale without a Hadamard pass.  The quantisation scale only needs an upper bound of max |xh| over
//     the row; xh is a block-orthonormal transform of x * suh, so max_kb || (x * suh)_kb ||_2 is one -- a plain
//     reduction pass over the row by three warps (which also applies silu * mul for the gated-MLP input and caches
//     x * suh in shared memory) replaces the 18-warp Hadamard prologue every CTA of the single-GEMM kernel runs.
//     The 128-point Hadamard itself is done per unit by the digit warps from the cache, off the critical path.
//     (|q| <= 32512 still holds; the scale is up to ~3x larger than the exact maximum, i.e. activations carry ~14.5
//     instead of 16 bits: rel-RMS contribution 1e-4, tolerance tests in tests/test_chain.py.)
//
// Roles (768 threads): warp 0 TMA producer, warp 1 idle, warps 2-3 activation / digit warps, warps 4-19 decode + MMA (two
// groups of two warpgroups), warps 20-23 epilogue; accumulators reach the epilogue through two shared-memory buffers.
#include "tc_common.cuh"
#include "i8_math.cuh"
#include <mutex>
#include <vector>

namespace exl3b {

using namespace ptx;

constexpr int CH_THREADS = 768;
constexpr int CH_XF_WARP0 = 2, CH_XF_WARPS = 2;
constexpr int CH_DEC_WARP0 = 4, CH_DEC_WARPS = 16, CH_DEC_GROUPS = 2;
constexpr int CH_EPI_WARP0 = 20;
constexpr int CH_MR = 4;
constexpr int CH_B_BYTES = 4096, CH_B_STAGE = 4096 + 64;               // digit tile + per-row digit sums
constexpr int CH_SUB_UNITS = 96;                                       // int32 accumulator safety (see I8_SUB_UNITS)
constexpr int CH_MAX_STAGES = 16;
constexpr int CH_MAX_INLINE = 4;
constexpr int CH_SCALE_SLOTS = 32;
constexpr uint32_t CH_SENTINEL = 0xffffffffu;
constexpr int CH_CACHE_MAX = 64 * 1024;

struct ChainOp
{
    const void* A;            // in_mode 0: fp16 (m, k); 1: gate, fp32 (m, k); 2: gate, fp16 (m, k)
    const void* A2;           // in_mode 1 / 2: up, same dtype
    const half* suh; const half* svh;
    void* C;
    int m, k, n, K;
    int c_fp32, in_mode;
    int KB, strips;
    int stage;
    int cached;               // x * suh kept in shared memory (m * k * 2 <= cache bytes)
    int suh_cached;           // suh staged in shared memory by a bulk copy (k * 2 <= suh bytes)
    long long unit_off;       // first unit of this op in its stage's unit space
    float out_scale;
};

struct ChainStage { int op_begin, op_end; int strips_total; int pad_; long long U; };

struct ChainParams
{
    const ChainOp* ops; const ChainStage* stages; const CUtensorMap* tmaps;     // device tables (n_inline == 0)
    int n_ops, n_stages, n_inline;
    int S, w_bytes, cache_bytes, suh_bytes;
    unsigned int* ctr;        // [n_stages] finished output segments per stage, [n_stages] exit ticket; zero between launches
    float* parts;             // split-K exchange, [2][grid][MR * 128] words, sentinel between launches
    unsigned long long* dbg;
    ChainOp ops_inline[CH_MAX_INLINE];
    ChainStage stages_inline[CH_MAX_INLINE];
    CUtensorMap tmaps_inline[CH_MAX_INLINE];
};

// accumulator hand-off decode groups -> epilogue: [2 buffers][2 groups][128 columns][2 CH_MR] int32, then [2][2][8] digit sums
constexpr int CH_D_BYTES = 2 * 2 * 128 * 2 * CH_MR * 4 + 2 * 2 * 8 * 4;

struct ChainSmem { int off_b, off_tile, off_bars, off_d, off_cache, off_suh, total; };

__host__ __device__ inline ChainSmem chain_smem(int S, int w_bytes, int cache_bytes, int suh_bytes)
{
    ChainSmem L;
    L.off_b = S * w_bytes;
    L.off_tile = L.off_b + S * CH_B_STAGE;
    L.off_tile = (L.off_tile + 127) & ~127;
    L.off_bars = L.off_tile + CH_MR * 128 * 4;
    L.off_d = L.off_bars + 2048;
    L.off_cache = L.off_d + CH_D_BYTES;
    L.off_suh = L.off_cache + cache_bytes;
    L.total = L.off_suh + suh_bytes;
    return L;
}

// ---- the CTA's walk over its units: stage by stage, inside a stage op by op, strip by strip, k fastest ------------------
struct Cursor
{
    const ChainOp* ops; const ChainStage* stages;
    int n_stages, cta, G;
    int Gs;                   // CTAs that share the current stage: min(G, units of the stage), so that no CTA range is empty
    int stage, op, strip, kb, KB, strips;
    long long u, uend;
    int seq;                  // running index of the unit on this CTA over the whole chain: ring stage, quad, digit warp
    int run_begin, run_end;   // [seq range) of the CTA's units inside the current (op, strip)
    bool valid;

    __host__ __device__ __forceinline__ void start_run()
    {
        const long long left_cta = uend - u;
        const int left_strip = KB - kb;
        run_begin = seq;
        run_end = seq + (int) (left_cta < left_strip ? left_cta : left_strip);
    }
    __host__ __device__ __forceinline__ void enter_stage()
    {
        valid = false;
        while (++stage < n_stages)
        {
            const long long U = stages[stage].U;
            Gs = U < G ? (int) U : G;
            if (cta >= Gs) continue;
            const long long ub = unit_begin(U, Gs, cta), ue = unit_begin(U, Gs, cta + 1);
            u = ub; uend = ue;
            op = stages[stage].op_begin;
            while (u >= ops[op].unit_off + (long long) ops[op].KB * ops[op].strips) ++op;
            KB = ops[op].KB; strips = ops[op].strips;
            const long long rel = u - ops[op].unit_off;
            strip = (int) (rel / KB); kb = (int) (rel - (long long) strip * KB);
            start_run();
            valid = true;
            return;
        }
    }
    __host__ __device__ __forceinline__ void init(const ChainOp* o, const ChainStage* s, int ns, int cta_, int G_)
    {
        ops = o; stages = s; n_stages = ns; cta = cta_; G = G_;
        stage = -1; seq = 0;
        enter_stage();
    }
    __host__ __device__ __forceinline__ void next()
    {
        ++seq; ++u;
        if (u == uend) { enter_stage(); return; }
        if (++kb == KB)
        {
            kb = 0;
            if (++strip == strips) { strip = 0; ++op; KB = ops[op].KB; strips = ops[op].strips; }
            start_run();
        }
    }
    // bounds of the accumulation chunk (<= CH_SUB_UNITS units of the run) that holds the current unit
    __host__ __device__ __forceinline__ void sub_bounds(int& sb, int& se) const
    {
        sb = run_begin + (seq - run_begin) / CH_SUB_UNITS * CH_SUB_UNITS;
        se = sb + CH_SUB_UNITS < run_end ? sb + CH_SUB_UNITS : run_end;
    }
};

__device__ __forceinline__ float silu_f32(float x) { return x * __fdividef(1.0f, 1.0f + __expf(-x)); }

struct ChainCtx
{
    uint8_t* smem;
    uint32_t bar0;
    int S, w_bytes;
    ChainSmem L;
    unsigned long long* dbg;
    int trace_seq;            // bring-up: the unit (CTA-local index) whose steps are stamped
    __device__ __forceinline__ uint32_t W_FULL(int s) const { return bar0 + 8u * s; }
    __device__ __forceinline__ uint32_t W_EMPTY(int s) const { return bar0 + 8u * (CH_MAX_STAGES + s); }
    __device__ __forceinline__ uint32_t X_FULL(int s) const { return bar0 + 8u * (2 * CH_MAX_STAGES + s); }
    __device__ __forceinline__ uint32_t D_FULL(int b) const { return bar0 + 8u * (3 * CH_MAX_STAGES + 8 + b); }
    __device__ __forceinline__ uint32_t D_EMPTY(int b) const { return bar0 + 8u * (3 * CH_MAX_STAGES + 10 + b); }
    __device__ __forceinline__ uint32_t IN_BAR() const { return bar0 + 8u * (3 * CH_MAX_STAGES + 12); }
};
constexpr int CH_NUM_BARS = 3 * CH_MAX_STAGES + 13;                    // 61 barriers

#ifdef EXL3B_TC_DEBUG
#define CH_STAMP(cond, slot) do { if ((cond) && cx.dbg) { unsigned long long t__; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t__) :: "memory"); cx.dbg[blockIdx.x * 64 + (slot)] = t__; } } while (0)
#else
#define CH_STAMP(cond, slot) do { } while (0)
#endif

// One unit (128 k x 128 n weights) of a decode warpgroup: the pipeline of gemm_tc_i8_body.cuh -- weight words from the ring
// stage, the warp's tile column of k-tiles c and 4 + c decoded straight into wgmma A fragments, 16 MMAs into acc.
template <int K>
__device__ __forceinline__ void group_unit(const ChainCtx& cx, int tl, int lane, int s, int sph, int m, uint32_t (&acc)[CH_MR], int& tsum,
                                           [[maybe_unused]] bool trace)
{
    const int chunk = lane >> 2, c = lane & 3;
    [[maybe_unused]] const bool tr = trace && tl == 0 && lane == 0;
    CH_STAMP(tr, 0);
    mbar_wait<32>(cx.W_FULL(s), sph);
    CH_STAMP(tr, 1);
    const uint32_t* wst = reinterpret_cast<const uint32_t*>(cx.smem + s * cx.w_bytes);
    uint32_t w[2][K + 1];
    #pragma unroll
    for (int r = 0; r < 2; ++r) load_chunk<K>(wst + ((4 * r + c) * 8 + tl) * (8 * K), chunk, w[r]);
    mbar_wait(cx.X_FULL(s), sph);                                      // the unit's activation digits
    CH_STAMP(tr, 2);
    if (c < m) tsum += *reinterpret_cast<const int*>(cx.smem + cx.L.off_b + s * CH_B_STAGE + CH_B_BYTES + 4 * c);
    const uint64_t desc_s = smem_desc(smem_u32(cx.smem + cx.L.off_b + s * CH_B_STAGE), 128, 4096, 0);
    #pragma unroll
    for (int r = 0; r < 2; ++r)
    {
        uint32_t o0[16], o1[16];
        decode16_i8<K, 0>(w[r], o0);
        decode16_i8<K, 1>(w[r], o1);
        #pragma unroll
        for (int i = 0; i < CH_MR; ++i) reg_fence(acc[i]);
        wgmma_fence();
        #pragma unroll
        for (int j = 0; j < 8; ++j)
            wgmma_u8s8_n8(acc, o0[2 * j], o1[2 * j], o0[2 * j + 1], o1[2 * j + 1], desc_s + (uint64_t) (16 * (8 * r + j)));
        wgmma_commit();
        wgmma_wait<0>();
        #pragma unroll
        for (int i = 0; i < 16; ++i) { reg_fence(o0[i]); reg_fence(o1[i]); }
        #pragma unroll
        for (int i = 0; i < CH_MR; ++i) reg_fence(acc[i]);
    }
    CH_STAMP(tr, 3);
    __syncwarp();
    if (lane == 0) mbar_arrive(cx.W_EMPTY(s));
}

__device__ __forceinline__ void ch_watchdog(uint32_t& polls, unsigned long long& t0, const char* what, int a, int b)
{
    if ((++polls & 255u) == 0)
    {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (t0 == 0) t0 = t;
        else if (t - t0 > 4000000000ull) { printf("exl3b chain: %s timeout (block %d, %d, %d)\n", what, blockIdx.x, a, b); __trap(); }
    }
}

// KSEL = 0: ops of any bitrate (a switch per unit); KSEL = 1..8: every op of the chain has K = KSEL (smaller code: the
// instruction footprint of all concurrently running roles matters on a kernel this size)
template <int KSEL>
__global__ void __launch_bounds__(CH_THREADS, 1)
chain_i8_kernel(const __grid_constant__ ChainParams p)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const ChainOp* ops = p.n_inline ? p.ops_inline : p.ops;
    const ChainStage* stages = p.n_inline ? p.stages_inline : p.stages;
    const CUtensorMap* tmaps = p.n_inline ? p.tmaps_inline : p.tmaps;
    const int S = p.S;
    ChainCtx cx;
    cx.smem = smem; cx.S = S; cx.w_bytes = p.w_bytes; cx.L = chain_smem(S, p.w_bytes, p.cache_bytes, p.suh_bytes);
    cx.dbg = p.dbg; cx.trace_seq = 8;
    CH_STAMP(threadIdx.x == 0, 61);
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + cx.L.off_bars);
    cx.bar0 = smem_u32(bars);
    uint32_t* misc = reinterpret_cast<uint32_t*>(smem + cx.L.off_bars + 8 * CH_NUM_BARS);
    unsigned int* s_norm2 = reinterpret_cast<unsigned int*>(misc + 4);                                       // [MR] float bits
    float* s_scale = reinterpret_cast<float*>(misc + 8 + 8);                                                 // [CH_SCALE_SLOTS][MR]
    int32_t* s_d = reinterpret_cast<int32_t*>(smem + cx.L.off_d);                                            // [dbuf][group][128][2 MR]
    int* s_dt = reinterpret_cast<int*>(smem + cx.L.off_d + CH_D_BYTES - 2 * 2 * 8 * 4);                     // [dbuf][group][8]
    half* cache = reinterpret_cast<half*>(smem + cx.L.off_cache);
    half* suh_s = reinterpret_cast<half*>(smem + cx.L.off_suh);

    pdl_launch_dependents();
    if (warp == 0)
    {
        for (int i = lane; i < CH_NUM_BARS; i += 32)
        {
            int cnt = 1;
            if (i >= CH_MAX_STAGES && i < 2 * CH_MAX_STAGES) cnt = CH_DEC_WARPS / CH_DEC_GROUPS;         // W_EMPTY: the group's warps, after their MMAs
            else if (i >= 3 * CH_MAX_STAGES + 8 && i < 3 * CH_MAX_STAGES + 10) cnt = CH_DEC_WARPS;         // D_FULL: every decode warp
            else if (i >= 3 * CH_MAX_STAGES + 10 && i < 3 * CH_MAX_STAGES + 12) cnt = 4;                 // D_EMPTY: the 4 epilogue warps
            else if (i == 3 * CH_MAX_STAGES + 12) cnt = 2;                                               // IN_BAR: suh copy + input copy
            mbar_init(cx.bar0 + 8u * i, cnt);
        }
        fence_barrier_init();
    }
    __syncthreads();

    const int cta = blockIdx.x, G = gridDim.x;

    if (warp == 0)
    {
        // =========================== TMA producer: never waits for an activation ===========================
        Cursor c; c.init(ops, stages, p.n_stages, cta, G);
        const uint64_t pol_w = policy_evict_first();
        const uint32_t w_smem0 = smem_u32(smem);
        int s = 0, ph = 0, cur_op = -1, K = 0;
        const void* tm = nullptr;
        while (c.valid)
        {
            if (c.op != cur_op)
            {
                cur_op = c.op; K = ops[cur_op].K;
                tm = tmaps + cur_op;
                if (elect_one()) prefetch_tmap(tm);
            }
            mbar_wait<64>(cx.W_EMPTY(s), ph ^ 1);
            if (elect_one())
            {
                mbar_arrive_expect_tx(cx.W_FULL(s), (uint32_t) (2048 * K));
                tma_load_2d(w_smem0 + s * p.w_bytes, tm, c.strip * (32 * K), c.kb * 8, cx.W_FULL(s), pol_w);
            }
            if (++s == S) { s = 0; ph ^= 1; }
            c.next();
        }
        __syncwarp();
    }
    else if (warp >= CH_XF_WARP0 && warp < CH_DEC_WARP0)
    {
        // =========================== activation warps: scale pass per op, digits per unit ===========================
        const int xw = warp - CH_XF_WARP0;
        auto xf_bar = [] { asm volatile("bar.sync 2, %0;" :: "n"(CH_XF_WARPS * 32) : "memory"); };
        pdl_wait();                                                   // external inputs come from the previous kernel
        Cursor c; c.init(ops, stages, p.n_stages, cta, G);
        int s = 0, ph = 0, cur_op = -1, waited = 0, turn = 0, in_ph = 0;
        float inv_scale[CH_MR];
        #pragma unroll
        for (int r = 0; r < CH_MR; ++r) inv_scale[r] = 0.f;
        // the op's fields live in registers: `ops` is a generic pointer (kernel parameters or global memory), and every
        // shared-memory store in the loops below would otherwise force a reload of each field
        struct { const void* A; const void* A2; const half* suh; int m, k, KB, in_mode, cached, suh_cached, stage; } o{};
        while (c.valid)
        {
            if (c.op != cur_op)
            {
                cur_op = c.op;
                {
                    const ChainOp& g = ops[cur_op];
                    o.A = g.A; o.A2 = g.A2; o.suh = g.suh; o.m = g.m; o.k = g.k; o.KB = g.KB; o.in_mode = g.in_mode;
                    o.cached = g.cached; o.suh_cached = g.suh_cached; o.stage = g.stage;
                }
                CH_STAMP(warp == CH_XF_WARP0 && lane == 0 && c.seq == 0, 59);
                const bool bulk_x = o.in_mode == 0 && o.cached;       // input rows by one bulk copy straight into the cache
                const bool bulk_s = o.suh != nullptr && o.suh_cached;
                xf_bar();                                             // previous op's cache / suh no longer needed by any digit warp
                if (warp == CH_XF_WARP0)
                {
                    if (lane < CH_MR) s_norm2[lane] = 0u;
                    // suh does not depend on the previous stage: its copy is in flight while we wait for the stage
                    if (elect_one())
                    {
                        asm volatile("fence.proxy.async;" ::: "memory");
                        if (bulk_s)
                        {
                            mbar_arrive_expect_tx(cx.IN_BAR(), (uint32_t) (o.k * 2));
                            bulk_g2s(smem_u32(suh_s), o.suh, (uint32_t) (o.k * 2), cx.IN_BAR(), policy_evict_first());
                        }
                        else mbar_arrive(cx.IN_BAR());
                    }
                    __syncwarp();
                }
                // ---- stage dependency: every output segment of the previous stage has been written ----
                if (o.stage > waited)
                {
                    if (lane == 0)
                    {
                        const unsigned int want = (unsigned int) stages[o.stage - 1].strips_total;
                        uint32_t polls = 0; unsigned long long t0 = 0;
                        while (ld_acquire_gpu_u32(p.ctr + (o.stage - 1)) < want) { __nanosleep(32); ch_watchdog(polls, t0, "stage wait", o.stage, 0); }
                    }
                    __syncwarp();
                    waited = o.stage;
                }
                if (warp == CH_XF_WARP0)
                {
                    if (elect_one())
                    {
                        if (bulk_x)
                        {
                            asm volatile("fence.proxy.async;" ::: "memory");
                            const uint32_t bytes = (uint32_t) ((size_t) o.m * o.k * 2);
                            mbar_arrive_expect_tx(cx.IN_BAR(), bytes);
                            bulk_g2s(smem_u32(cache), o.A, bytes, cx.IN_BAR(), policy_evict_first());
                        }
                        else mbar_arrive(cx.IN_BAR());
                    }
                    __syncwarp();
                }
                mbar_wait(cx.IN_BAR(), in_ph);
                in_ph ^= 1;
                // ---- scale pass: t = input * suh (fp16, the reference's A_had input), cached; bound = max over 128-blocks of || t ||_2.
                //      Four blocks per step so that their loads and reductions overlap. ----
                const int KB = o.KB;
                for (int r = 0; r < o.m; ++r)
                {
                    float nmax = 0.f;
                    for (int kb0 = xw; kb0 < KB; kb0 += 4 * CH_XF_WARPS)
                    {
                        half2 a[4], b[4];
                        uint2 scb[4];
                        #pragma unroll
                        for (int j = 0; j < 4; ++j)
                        {
                            const int kb = kb0 + j * CH_XF_WARPS;
                            a[j] = __floats2half2_rn(0.f, 0.f); b[j] = a[j]; scb[j] = make_uint2(0, 0);
                            if (kb < KB)
                            {
                                const size_t e = (size_t) r * o.k + kb * 128 + lane * 4;
                                if (o.suh) scb[j] = bulk_s ? *reinterpret_cast<const uint2*>(suh_s + kb * 128 + lane * 4)
                                                           : *reinterpret_cast<const uint2*>(o.suh + kb * 128 + lane * 4);
                                if (bulk_x)
                                {
                                    const uint2 raw = *reinterpret_cast<const uint2*>(cache + e);
                                    a[j] = *reinterpret_cast<const half2*>(&raw.x); b[j] = *reinterpret_cast<const half2*>(&raw.y);
                                }
                                else if (o.in_mode == 0)
                                {
                                    const uint2 raw = __ldcg(reinterpret_cast<const uint2*>(reinterpret_cast<const half*>(o.A) + e));
                                    a[j] = *reinterpret_cast<const half2*>(&raw.x); b[j] = *reinterpret_cast<const half2*>(&raw.y);
                                }
                                else if (o.in_mode == 1)
                                {
                                    const float4 g = __ldcg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(o.A) + e));
                                    const float4 u = __ldcg(reinterpret_cast<const float4*>(reinterpret_cast<const float*>(o.A2) + e));
                                    a[j] = __floats2half2_rn(silu_f32(g.x) * u.x, silu_f32(g.y) * u.y);
                                    b[j] = __floats2half2_rn(silu_f32(g.z) * u.z, silu_f32(g.w) * u.w);
                                }
                                else
                                {
                                    const uint2 gr = __ldcg(reinterpret_cast<const uint2*>(reinterpret_cast<const half*>(o.A) + e));
                                    const uint2 ur = __ldcg(reinterpret_cast<const uint2*>(reinterpret_cast<const half*>(o.A2) + e));
                                    const float2 g0 = __half22float2(*reinterpret_cast<const half2*>(&gr.x)), g1 = __half22float2(*reinterpret_cast<const half2*>(&gr.y));
                                    const float2 u0 = __half22float2(*reinterpret_cast<const half2*>(&ur.x)), u1 = __half22float2(*reinterpret_cast<const half2*>(&ur.y));
                                    a[j] = __floats2half2_rn(silu_f32(g0.x) * u0.x, silu_f32(g0.y) * u0.y);
                                    b[j] = __floats2half2_rn(silu_f32(g1.x) * u1.x, silu_f32(g1.y) * u1.y);
                                }
                            }
                        }
                        float ss[4];
                        #pragma unroll
                        for (int j = 0; j < 4; ++j)
                        {
                            const int kb = kb0 + j * CH_XF_WARPS;
                            if (o.suh)
                            {
                                a[j] = __hmul2(a[j], *reinterpret_cast<const half2*>(&scb[j].x));
                                b[j] = __hmul2(b[j], *reinterpret_cast<const half2*>(&scb[j].y));
                            }
                            if (o.cached && kb < KB)
                            {
                                uint2 st; st.x = *reinterpret_cast<const uint32_t*>(&a[j]); st.y = *reinterpret_cast<const uint32_t*>(&b[j]);
                                *reinterpret_cast<uint2*>(cache + (size_t) r * o.k + kb * 128 + lane * 4) = st;
                            }
                            const float2 fa = __half22float2(a[j]), fb = __half22float2(b[j]);
                            ss[j] = fa.x * fa.x + fa.y * fa.y + fb.x * fb.x + fb.y * fb.y;
                        }
                        #pragma unroll
                        for (int d = 16; d > 0; d >>= 1)
                        {
                            #pragma unroll
                            for (int j = 0; j < 4; ++j) ss[j] += __shfl_xor_sync(0xffffffffu, ss[j], d);
                        }
                        nmax = fmaxf(fmaxf(nmax, fmaxf(ss[0], ss[1])), fmaxf(ss[2], ss[3]));
                    }
                    if (lane == 0) atomicMax(&s_norm2[r], __float_as_uint(nmax));
                }
                xf_bar();
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r)
                {
                    // bound on |xh|: block 2-norm, + margin for the fp32 reduction and the fp16 rounding of xh
                    const float bnd = sqrtf(__uint_as_float(s_norm2[r])) * 1.002f;
                    inv_scale[r] = bnd > 0.f ? (float) I8_QMAX / bnd : 0.f;
                    // every digit warp stores the (identical) value before its own first X_FULL arrive of this op: whichever
                    // arrive the MMA side observes, the scale the epilogue reads later is ordered before it
                    if (lane == r) s_scale[(cur_op % CH_SCALE_SLOTS) * CH_MR + r] = bnd / (float) I8_QMAX;
                }
                CH_STAMP(warp == CH_XF_WARP0 && lane == 0 && c.seq == 0, 60);
            }
            if (turn == xw)
            {
                // ---- digits of this unit: 128-point Hadamard of the cached block, quantise, two int8 digits x 4 bytes ----
                CH_STAMP(c.seq == cx.trace_seq && lane == 0, 56);
                mbar_wait<64>(cx.W_EMPTY(s), ph ^ 1);
                CH_STAMP(c.seq == cx.trace_seq && lane == 0, 57);
                uint8_t* dst = smem + cx.L.off_b + s * CH_B_STAGE;
                int qsum[CH_MR];
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r)
                {
                    qsum[r] = 0;
                    if (r < o.m)
                    {
                        half2 a, b;
                        if (o.cached)
                        {
                            const uint2 raw = *reinterpret_cast<const uint2*>(cache + (size_t) r * o.k + c.kb * 128 + lane * 4);
                            a = *reinterpret_cast<const half2*>(&raw.x); b = *reinterpret_cast<const half2*>(&raw.y);
                        }
                        else
                        {
                            // rows too long for the cache: recompute the block (plain fp16 input only, checked on the host)
                            const uint2 raw = __ldcg(reinterpret_cast<const uint2*>(reinterpret_cast<const half*>(o.A) + (size_t) r * o.k + c.kb * 128 + lane * 4));
                            a = *reinterpret_cast<const half2*>(&raw.x); b = *reinterpret_cast<const half2*>(&raw.y);
                            if (o.suh)
                            {
                                const uint2 scb = *reinterpret_cast<const uint2*>(o.suh + c.kb * 128 + lane * 4);
                                a = __hmul2(a, *reinterpret_cast<const half2*>(&scb.x));
                                b = __hmul2(b, *reinterpret_cast<const half2*>(&scb.y));
                            }
                        }
                        float v0 = __low2float(a), v1 = __high2float(a), v2 = __low2float(b), v3 = __high2float(b);
                        if (o.suh)
                        {
                            had128_warp(v0, v1, v2, v3, lane);
                            a = __floats2half2_rn(v0 * R_SCALE, v1 * R_SCALE);
                            b = __floats2half2_rn(v2 * R_SCALE, v3 * R_SCALE);
                            v0 = __low2float(a); v1 = __high2float(a); v2 = __low2float(b); v3 = __high2float(b);
                        }
                        uint32_t hi_w[4], lo_w[4];
                        int qs = 0;
                        i8_digits(v0, inv_scale[r], qs, hi_w[0], lo_w[0]);
                        i8_digits(v1, inv_scale[r], qs, hi_w[1], lo_w[1]);
                        i8_digits(v2, inv_scale[r], qs, hi_w[2], lo_w[2]);
                        i8_digits(v3, inv_scale[r], qs, hi_w[3], lo_w[3]);
                        // K order of the wgmma fragments (gemm_tc_i8_body.cuh): k = 4 lane + e -> K-chunk 16 (lane / 16) + 4 (lane % 4) + e,
                        // byte 4 ((lane / 4) % 4)
                        uint8_t* drow = dst + ((16 * (lane >> 4) + 4 * (lane & 3)) * 8 + 2 * r) * 16 + 4 * ((lane >> 2) & 3);
                        #pragma unroll
                        for (int e = 0; e < 4; ++e)
                        {
                            *reinterpret_cast<uint32_t*>(drow + e * 128) = hi_w[e];
                            *reinterpret_cast<uint32_t*>(drow + e * 128 + 16) = lo_w[e];
                        }
                        qsum[r] = qs;
                    }
                }
                #pragma unroll
                for (int d = 16; d > 0; d >>= 1)
                {
                    #pragma unroll
                    for (int r = 0; r < CH_MR; ++r) qsum[r] += __shfl_xor_sync(0xffffffffu, qsum[r], d);
                }
                if (lane < o.m)
                {
                    int mine = 0;
                    #pragma unroll
                    for (int r = 0; r < CH_MR; ++r) if (lane == r) mine = qsum[r];
                    *reinterpret_cast<int*>(dst + CH_B_BYTES + 4 * lane) = mine;
                }
                fence_proxy_async_smem();
                __syncwarp();
                if (lane == 0) mbar_arrive(cx.X_FULL(s));
                CH_STAMP(c.seq == cx.trace_seq && lane == 0, 58);
            }
            if (++turn == CH_XF_WARPS) turn = 0;
            if (++s == S) { s = 0; ph ^= 1; }
            c.next();
        }
    }
    else if (warp >= CH_DEC_WARP0 && warp < CH_EPI_WARP0)
    {
        // =========================== decode groups: four warpgroups ===========================
        // warpgroup (g, nh): units seq = g (mod 2), output columns 64 nh .. 64 nh + 63; both groups hand over (possibly zero)
        // accumulators at every accumulation-chunk boundary, the epilogue adds the two
        const int wq = warp & 3, wgi = (warp - CH_DEC_WARP0) >> 2;
        const int g = wgi & 1, nh = wgi >> 1, tl = 4 * nh + wq;
        const int chunk = lane >> 2, cq = lane & 3;
        Cursor c; c.init(ops, stages, p.n_stages, cta, G);
        int s = 0, ph = 0, dbuf = 0, dphase = 0;
        uint32_t acc[CH_MR] = {0u, 0u, 0u, 0u};
        int tsum = 0;
        while (c.valid)
        {
            int sb, se; c.sub_bounds(sb, se);
            const bool last = c.seq == se - 1;
            if ((c.seq & 1) == g)
            {
                const bool trace = c.seq == cx.trace_seq;
                const int m = ops[c.op].m;
                if constexpr (KSEL != 0) group_unit<KSEL>(cx, tl, lane, s, ph, m, acc, tsum, trace);
                else
                {
                    switch (ops[c.op].K)
                    {
                        case 1: group_unit<1>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        case 2: group_unit<2>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        case 3: group_unit<3>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        case 4: group_unit<4>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        case 5: group_unit<5>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        case 6: group_unit<6>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        case 7: group_unit<7>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                        default: group_unit<8>(cx, tl, lane, s, ph, m, acc, tsum, trace); break;
                    }
                }
            }
            if (last)
            {
                mbar_wait(cx.D_EMPTY(dbuf), dphase ^ 1);               // the epilogue has drained this buffer
                int32_t* dst = s_d + (size_t) ((dbuf * 2 + g) * 128 + 16 * tl + chunk) * (2 * CH_MR);
                *reinterpret_cast<int2*>(dst + 2 * cq) = make_int2((int) acc[0], (int) acc[1]);
                *reinterpret_cast<int2*>(dst + 8 * (2 * CH_MR) + 2 * cq) = make_int2((int) acc[2], (int) acc[3]);
                if (tl == 0 && lane < 4) s_dt[(dbuf * 2 + g) * 8 + cq] = tsum;
                acc[0] = acc[1] = acc[2] = acc[3] = 0u;
                tsum = 0;
                __syncwarp();
                if (lane == 0) mbar_arrive(cx.D_FULL(dbuf));
                dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
            }
            if (++s == S) { s = 0; ph ^= 1; }
            c.next();
        }
    }
    else if (warp >= CH_EPI_WARP0)
    {
        // =========================== epilogue ===========================
        pdl_wait();
        const int q = warp & 3;
        const int et = threadIdx.x - CH_EPI_WARP0 * 32;
        const int col = et;                                             // column of the strip this thread finishes
        float* tile = reinterpret_cast<float*>(smem + cx.L.off_tile);
        auto epi_bar = [] { asm volatile("bar.sync 1, 128;" ::: "memory"); };
        const int part_stride = CH_MR * 128;
        const float k_inv = __half2float(__ushort_as_half((unsigned short) 0x1eee));
        const float k_bias = __half2float(__ushort_as_half((unsigned short) 0xc931));
        const float c1 = 1534.0f * k_inv + k_bias;
        int dbuf = 0, dphase = 0, cur_op = -1;
        struct { void* C; const half* svh; long long unit_off; int m, n, KB, c_fp32; float out_scale; } o{};
        Cursor c; c.init(ops, stages, p.n_stages, cta, G);
        while (c.valid)
        {
            const int op = c.op, strip = c.strip, stage = c.stage;
            if (op != cur_op)
            {
                cur_op = op;
                const ChainOp& g = ops[op];
                o.C = g.C; o.svh = g.svh; o.m = g.m; o.n = g.n; o.KB = g.KB; o.c_fp32 = g.c_fp32; o.unit_off = g.unit_off; o.out_scale = g.out_scale;
            }
            const int run_begin = c.run_begin, run_end = c.run_end;
            const long long U = stages[stage].U;
            float* const parts = p.parts + (size_t) (stage & 1) * DevCtx::I8_PART_CTAS * part_stride;
            float facc[CH_MR];
            #pragma unroll
            for (int r = 0; r < CH_MR; ++r) facc[r] = 0.f;
            for (int sb = run_begin; sb < run_end; sb += CH_SUB_UNITS)
            {
                mbar_wait<32>(cx.D_FULL(dbuf), dphase);
                const int32_t* d0 = s_d + (size_t) ((dbuf * 2 + 0) * 128 + col) * (2 * CH_MR);
                const int32_t* d1 = s_d + (size_t) ((dbuf * 2 + 1) * 128 + col) * (2 * CH_MR);
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r)
                {
                    if (r < o.m)
                    {
                        const int T = s_dt[(dbuf * 2 + 0) * 8 + r] + s_dt[(dbuf * 2 + 1) * 8 + r];
                        const long long sp = i8_centred_sum(d0[2 * r] + d1[2 * r], d0[2 * r + 1] + d1[2 * r + 1], T);
                        facc[r] += i8_assemble(sp, T, s_scale[(op % CH_SCALE_SLOTS) * CH_MR + r], k_inv, c1);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(cx.D_EMPTY(dbuf));
                dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
            }

            // who else holds k-segments of this strip?
            const long long gs = o.unit_off + (long long) strip * o.KB;
            const int c_a = cta_of_unit(U, c.Gs, gs), c_b = cta_of_unit(U, c.Gs, gs + o.KB - 1);
            const bool full = c_a == c_b;
            bool emit = full;
            if (full)
            {
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r) if (r < o.m) tile[r * 128 + col] = facc[r];
            }
            else if (cta != c_a)
            {
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r)
                    if (r < o.m)
                    {
                        uint32_t bits = __float_as_uint(facc[r]);
                        if (bits == CH_SENTINEL) bits = 0x7fc00000u;
                        st_relaxed_gpu_u32(reinterpret_cast<uint32_t*>(parts + (size_t) cta * part_stride + r * 128 + col), bits);
                    }
            }
            else
            {
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r)
                {
                    if (r < o.m)
                    {
                        float a = facc[r];
                        int cc0 = c_a + 1;
                        while (cc0 <= c_b)
                        {
                            uint32_t v[8];
                            bool ok;
                            uint32_t polls = 0; unsigned long long t0 = 0;
                            do
                            {
                                ok = true;
                                #pragma unroll
                                for (int j = 0; j < 8; ++j)
                                {
                                    const int cc = cc0 + j;
                                    v[j] = 0u;
                                    if (cc <= c_b)
                                    {
                                        v[j] = ld_relaxed_gpu_u32(reinterpret_cast<const uint32_t*>(parts + (size_t) cc * part_stride + r * 128 + col));
                                        ok = ok && v[j] != CH_SENTINEL;
                                    }
                                }
                                if (!ok) ch_watchdog(polls, t0, "split-K exchange", stage, strip);
                            } while (!ok);
                            #pragma unroll
                            for (int j = 0; j < 8; ++j)
                            {
                                const int cc = cc0 + j;
                                if (cc <= c_b)
                                {
                                    a += __uint_as_float(v[j]);
                                    st_relaxed_gpu_u32(reinterpret_cast<uint32_t*>(parts + (size_t) cc * part_stride + r * 128 + col), CH_SENTINEL);
                                }
                            }
                            cc0 += 8;
                        }
                        tile[r * 128 + col] = a;
                    }
                }
                emit = true;
            }
            if (emit)
            {
                epi_bar();
                for (int r = q; r < o.m; r += 4)
                    output_row_128(tile + r * 128, (char*) o.C, (size_t) r * o.n + strip * 128,
                                   o.svh ? o.svh + strip * 128 : nullptr, o.out_scale, o.c_fp32 != 0, lane);
                epi_bar();
                if (et == 0)
                {
                    __threadfence();
                    atomicAdd(p.ctr + stage, 1u);
                }
            }
            // skip to the first unit after this run
            const int run_len = run_end - run_begin;
            for (int i = 0; i < run_len; ++i) c.next();
        }
    }

    __syncthreads();
    CH_STAMP(threadIdx.x == 0, 62);
    if (threadIdx.x == 0)
    {
        // last CTA out re-zeroes the counters for the next launch (which reads them only after griddepcontrol.wait)
        __threadfence();
        const unsigned int t = atomicAdd(p.ctr + p.n_stages, 1u);
        if (t == gridDim.x - 1)
        {
            for (int i = 0; i <= p.n_stages; ++i) p.ctr[i] = 0u;
            __threadfence();
        }
    }
}

// ---- host side ----------------------------------------------------------------------------------------------------------

struct Chain
{
    int device = -1;
    std::vector<ChainOp> ops;
    std::vector<ChainStage> stages;
    std::vector<CUtensorMap> tmaps;
    void* d_blob = nullptr;             // device copy: tmaps | ops | stages
    ChainParams p{};
    int smem_total = 0, grid = 0, ksel = 0;
};

const char* chain_op_unsupported(int m, int k, int n, int K, int cb, int in_mode)
{
    if (cb != 2) return "needs the mul1 codebook";
    if (m < 1 || m > CH_MR) return "needs 1 <= m <= 4";
    if (K < 1 || K > 8) return "K out of range";
    if (k < 128 || n < 128 || k % 128 || n % 128) return "k and n must be multiples of 128";
    if (in_mode < 0 || in_mode > 2) return "in_mode must be 0 (fp16 rows), 1 (silu(gate) * up, fp32) or 2 (same, fp16)";
    if (in_mode != 0 && (size_t) m * k * 2 > CH_CACHE_MAX) return "gated input needs m * k <= 32768";
    return nullptr;
}

// Fill ops / stages / launch geometry from the caller's list.  Pure host arithmetic (also behind exl3b_chain_plan).
static int chain_build(const exl3b_chain_op* in, int n_ops, int num_sms, Chain& ch)
{
    EXL3B_CHECK(in && n_ops >= 1, EXL3B_ERR_ARG, "exl3_chain: empty op list");
    EXL3B_CHECK(n_ops <= 4096, EXL3B_ERR_ARG, "exl3_chain: too many ops");
    ch.ops.resize(n_ops);
    ch.stages.clear();
    int Kmax = 1, Kmin = 9;
    size_t cache = 0, suhb = 0;
    long long Umax = 0;
    for (int i = 0; i < n_ops; ++i)
    {
        const exl3b_chain_op& a = in[i];
        const char* why = chain_op_unsupported(a.m, a.k, a.n, a.K, a.cb, a.in_mode);
        EXL3B_CHECK(!why, EXL3B_ERR_UNSUPPORTED, "exl3_chain: op %d: %s", i, why ? why : "");
        EXL3B_CHECK(a.A && a.B && a.C && (a.in_mode == 0 || a.A2), EXL3B_ERR_ARG, "exl3_chain: op %d: null tensor", i);
        if (i == 0 || a.new_stage)
        {
            ChainStage st{};
            st.op_begin = i; st.op_end = i; st.U = 0; st.strips_total = 0;
            ch.stages.push_back(st);
        }
        ChainStage& st = ch.stages.back();
        ChainOp& o = ch.ops[i];
        o = ChainOp{};
        o.A = a.A; o.A2 = a.A2; o.suh = (const half*) a.suh; o.svh = (const half*) a.svh; o.C = a.C;
        o.m = a.m; o.k = a.k; o.n = a.n; o.K = a.K; o.c_fp32 = a.c_fp32 != 0; o.in_mode = a.in_mode;
        o.KB = a.k / 128; o.strips = a.n / 128; o.stage = (int) ch.stages.size() - 1;
        o.unit_off = st.U; o.out_scale = 1.0f;
        const size_t cb_ = ((size_t) a.m * a.k * 2 + 127) / 128 * 128;
        o.cached = cb_ <= (size_t) CH_CACHE_MAX;
        if (o.cached && cb_ > cache) cache = cb_;
        o.suh_cached = a.suh != nullptr && (size_t) a.k * 2 <= (size_t) CH_CACHE_MAX && ((uintptr_t) a.suh & 15) == 0;
        if (o.suh_cached && (size_t) a.k * 2 > suhb) suhb = (size_t) a.k * 2;
        if (o.cached && o.in_mode == 0 && ((uintptr_t) a.A & 15) != 0) o.cached = 0;      // bulk copy needs 16-byte alignment
        if (a.K < Kmin) Kmin = a.K;
        st.U += (long long) o.KB * o.strips; st.strips_total += o.strips; st.op_end = i + 1;
        if (a.K > Kmax) Kmax = a.K;
    }
    EXL3B_CHECK(ch.stages.size() <= 255, EXL3B_ERR_UNSUPPORTED, "exl3_chain: more than 255 stages");
    for (const ChainStage& st : ch.stages) if (st.U > Umax) Umax = st.U;
    const int w_bytes = 2048 * Kmax;
    int S = (220 * 1024 - 128 - CH_MR * 128 * 4 - 2048 - CH_D_BYTES - (int) cache - (int) suhb) / (w_bytes + CH_B_STAGE);
    if (S > CH_MAX_STAGES) S = CH_MAX_STAGES;
    EXL3B_CHECK(S >= 2, EXL3B_ERR_UNSUPPORTED, "exl3_chain: shared-memory budget exceeded");
    const ChainSmem L = chain_smem(S, w_bytes, (int) cache, (int) suhb);
    EXL3B_CHECK(L.total <= 220 * 1024, EXL3B_ERR_UNSUPPORTED, "exl3_chain: shared-memory budget exceeded");
    int grid = num_sms;
    if (Umax < grid) grid = (int) Umax;
    EXL3B_CHECK(grid <= DevCtx::I8_PART_CTAS, EXL3B_ERR_UNSUPPORTED, "exl3_chain: grid exceeds the split-K exchange buffer");
    ch.p = ChainParams{};
    ch.p.n_ops = n_ops; ch.p.n_stages = (int) ch.stages.size();
    ch.p.S = S; ch.p.w_bytes = w_bytes; ch.p.cache_bytes = (int) cache; ch.p.suh_bytes = (int) suhb;
    ch.smem_total = L.total; ch.grid = grid; ch.ksel = Kmin == Kmax ? Kmax : 0;
    return 0;
}

template <int KSEL>
static cudaError_t chain_launch_k(cudaStream_t stream, int grid, int smem_bytes, const ChainParams& p)
{
    static bool attr_set[32] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (!attr_set[dev & 31])
    {
        cudaError_t e = cudaFuncSetAttribute(chain_i8_kernel<KSEL>, cudaFuncAttributeMaxDynamicSharedMemorySize, 220 * 1024);
        if (e != cudaSuccess) return e;
        attr_set[dev & 31] = true;
    }
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3(grid); cfg.blockDim = dim3(CH_THREADS); cfg.dynamicSmemBytes = smem_bytes; cfg.stream = stream;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    return cudaLaunchKernelEx(&cfg, chain_i8_kernel<KSEL>, p);
}

static cudaError_t chain_launch(cudaStream_t stream, int grid, int smem_bytes, const ChainParams& p, int ksel)
{
    switch (ksel)
    {
        case 1: return chain_launch_k<1>(stream, grid, smem_bytes, p);
        case 2: return chain_launch_k<2>(stream, grid, smem_bytes, p);
        case 3: return chain_launch_k<3>(stream, grid, smem_bytes, p);
        case 4: return chain_launch_k<4>(stream, grid, smem_bytes, p);
        case 5: return chain_launch_k<5>(stream, grid, smem_bytes, p);
        case 6: return chain_launch_k<6>(stream, grid, smem_bytes, p);
        case 7: return chain_launch_k<7>(stream, grid, smem_bytes, p);
        case 8: return chain_launch_k<8>(stream, grid, smem_bytes, p);
        default: return chain_launch_k<0>(stream, grid, smem_bytes, p);
    }
}

int chain_plan(const exl3b_chain_op* in, int n_ops, int num_sms, struct exl3b_chain_plan* out)
{
    Chain ch;
    int r = chain_build(in, n_ops, num_sms, ch); if (r) return r;
    out->stages = ch.p.n_stages; out->grid = ch.grid; out->ring_stages = ch.p.S; out->smem_bytes = ch.smem_total;
    out->cache_bytes = ch.p.cache_bytes; out->units = 0;
    for (const ChainStage& st : ch.stages) out->units += st.U;
    return 0;
}

// host-side replay of one CTA's walk with the kernel's own Cursor (tests: every unit visited exactly once, run bounds)
int chain_walk(const exl3b_chain_op* in, int n_ops, int num_sms, int cta, int32_t* out, int max_units)
{
    Chain ch;
    int r = chain_build(in, n_ops, num_sms, ch); if (r) return r;
    EXL3B_CHECK(cta >= 0 && cta < ch.grid && out && max_units >= 0, EXL3B_ERR_ARG, "exl3_chain_walk: bad argument");
    Cursor c; c.init(ch.ops.data(), ch.stages.data(), ch.p.n_stages, cta, ch.grid);
    int n = 0;
    while (c.valid)
    {
        if (n < max_units)
        {
            int sb, se; c.sub_bounds(sb, se);
            int32_t* o = out + (size_t) n * 8;
            o[0] = c.stage; o[1] = c.op; o[2] = c.strip; o[3] = c.kb; o[4] = c.seq; o[5] = c.run_begin; o[6] = c.run_end; o[7] = sb * 65536 + (se - sb);
        }
        ++n;
        c.next();
    }
    return n;
}

int chain_create(DevCtx* ctx, const exl3b_chain_op* in, int n_ops, void** out)
{
    EXL3B_CHECK(out, EXL3B_ERR_ARG, "exl3_chain_create: null output");
    Chain* ch = new Chain();
    int r = chain_build(in, n_ops, ctx->num_sms, *ch);
    if (r) { delete ch; return r; }
    ch->device = ctx->device;
    ch->tmaps.resize(n_ops);
    for (int i = 0; i < n_ops; ++i)
    {
        r = get_weight_tmap(in[i].B, in[i].k, in[i].n, in[i].K, &ch->tmaps[i]);
        if (r) { delete ch; return r; }
    }
    const size_t b_tm = sizeof(CUtensorMap) * n_ops, b_ops = sizeof(ChainOp) * n_ops, b_st = sizeof(ChainStage) * ch->stages.size();
    if (cudaMalloc(&ch->d_blob, b_tm + b_ops + b_st) != cudaSuccess) { delete ch; return fail(EXL3B_ERR_CUDA, "exl3_chain_create: cudaMalloc failed"); }
    uint8_t* d = (uint8_t*) ch->d_blob;
    cudaError_t e = cudaMemcpy(d, ch->tmaps.data(), b_tm, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d + b_tm, ch->ops.data(), b_ops, cudaMemcpyHostToDevice);
    if (e == cudaSuccess) e = cudaMemcpy(d + b_tm + b_ops, ch->stages.data(), b_st, cudaMemcpyHostToDevice);
    if (e != cudaSuccess) { cudaFree(ch->d_blob); delete ch; return fail(EXL3B_ERR_CUDA, "exl3_chain_create: %s", cudaGetErrorString(e)); }
    ch->p.tmaps = (const CUtensorMap*) d; ch->p.ops = (const ChainOp*) (d + b_tm); ch->p.stages = (const ChainStage*) (d + b_tm + b_ops);
    ch->p.n_inline = 0;
    ch->p.ctr = ctx->chain_ctr; ch->p.parts = ctx->chain_parts;
    *out = ch;
    return 0;
}

int chain_run(cudaStream_t stream, void* chain)
{
    Chain* ch = (Chain*) chain;
    EXL3B_CHECK(ch, EXL3B_ERR_ARG, "exl3_chain_run: null chain");
    int dev = -1; EXL3B_CUDA(cudaGetDevice(&dev));
    EXL3B_CHECK(dev == ch->device, EXL3B_ERR_ARG, "exl3_chain_run: chain was created on device %d, current device is %d", ch->device, dev);
    ch->p.dbg = g_tc_dbg;
    cudaError_t err = chain_launch(stream, ch->grid, ch->smem_total, ch->p, ch->ksel);
    count_launch();
    EXL3B_CUDA(err);
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC_I8_CHAIN;
}

int chain_destroy(void* chain)
{
    Chain* ch = (Chain*) chain;
    if (!ch) return 0;
    if (ch->d_blob) cudaFree(ch->d_blob);
    delete ch;
    return 0;
}

bool gemm_chain_supported(const GemmArgs& a)
{
    return chain_op_unsupported(a.m, a.k, a.n, a.K, a.cb, 0) == nullptr;
}

// a single exl3_gemm on the chain kernel: the op travels in the kernel parameters, nothing is allocated or copied
int launch_gemm_chain(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a)
{
    exl3b_chain_op in{};
    in.A = a.A; in.B = a.B; in.suh = a.suh; in.svh = a.svh; in.C = a.C;
    in.m = a.m; in.k = a.k; in.n = a.n; in.K = a.K; in.cb = a.cb; in.c_fp32 = a.c_fp32; in.in_mode = 0; in.new_stage = 0;
    Chain ch;
    { int r = chain_build(&in, 1, a.max_ctas > 0 && a.max_ctas < ctx->num_sms ? a.max_ctas : ctx->num_sms, ch); if (r) return r; }
    ch.ops[0].out_scale = a.out_scale;
    ChainParams& p = ch.p;
    { int r = get_weight_tmap(a.B, a.k, a.n, a.K, &p.tmaps_inline[0]); if (r) return r; }
    p.ops_inline[0] = ch.ops[0]; p.stages_inline[0] = ch.stages[0];
    p.n_inline = 1; p.ctr = ctx->chain_ctr; p.parts = ctx->chain_parts; p.dbg = g_tc_dbg;
    cudaError_t err = chain_launch(stream, ch.grid, ch.smem_total, p, ch.ksel);
    count_launch();
    EXL3B_CUDA(err);
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC_I8_CHAIN;
}

}  // namespace exl3b
