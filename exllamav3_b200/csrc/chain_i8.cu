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
//   * the unit pipeline itself is the one of gemm_tc_i8_body.cuh (i8_pipeline.cuh: two decode groups of two warpgroups,
//     each warpgroup decoding its weights straight into wgmma A fragments and accumulating in registers; the same ring
//     barriers, one W_FULL wait per unit for its weights and digits, the same row transform and split-K exchange).
//   * activation scale without a Hadamard pass.  The quantisation scale only needs an upper bound of max |xh| over
//     the row; xh is a block-orthonormal transform of x * suh, so max_kb || (x * suh)_kb ||_2 is one -- a plain
//     reduction pass over the row by three warps (which also applies silu * mul for the gated-MLP input and caches
//     x * suh in shared memory) replaces the 18-warp Hadamard prologue every CTA of the single-GEMM kernel runs.
//     The 128-point Hadamard itself is done per unit by the digit warps from the cache, off the critical path.
//     (|q| <= 32512 still holds; on Gaussian rows the bound is ~3.5x the exact maximum (medians 3.3x .. 3.8x for
//     k = 512 .. 14336, single rows 2.2x .. 4.7x), i.e. activations carry ~14 instead of 16 bits: rel-RMS
//     contribution 1e-4.  The rule is modelled bit for bit by oracle.exl3_gemm_i8_model(rule="blocknorm"):
//     tests/test_chain_host.py, tests/test_chain_exact.py.)
//
// Roles (768 threads): warp 0 TMA producer, warp 1 idle, warps 2-3 activation / digit warps, warps 4-19 decode + MMA (two
// groups of two warpgroups), warps 20-23 epilogue; accumulators reach the epilogue through two shared-memory buffers.
#include "i8_pipeline.cuh"
#include <mutex>
#include <vector>

namespace exl3b {

constexpr int CH_MR = 4;
constexpr int CH_XF_WARPS = TC_DEC_WARP0 - TC_XF_WARP0;
constexpr int CH_MAX_INLINE = 4;
constexpr int CH_SCALE_SLOTS = 32;

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
    ChainOp ops_inline[CH_MAX_INLINE];
    ChainStage stages_inline[CH_MAX_INLINE];
    CUtensorMap tmaps_inline[CH_MAX_INLINE];
};

struct ChainSmem { int off_b, off_tile, off_bars, off_d, off_cache, off_suh, total; };

__host__ __device__ inline ChainSmem chain_smem(int S, int w_bytes, int cache_bytes, int suh_bytes)
{
    ChainSmem L;
    L.off_b = S * w_bytes;
    L.off_tile = L.off_b + S * i8_b_stage(CH_MR);
    L.off_tile = (L.off_tile + 127) & ~127;
    L.off_bars = L.off_tile + CH_MR * 128 * 4;
    L.off_d = L.off_bars + 2048;
    L.off_cache = L.off_d + i8_d_bytes(CH_MR);
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
            const long long ub = unit_begin((int) U, Gs, cta), ue = unit_begin((int) U, Gs, cta + 1);
            u = ub; uend = ue;
            op = stages[stage].op_begin;
            while (u >= ops[op].unit_off + (long long) ops[op].KB * ops[op].strips) ++op;
            KB = ops[op].KB; strips = ops[op].strips;
            const int rel = (int) (u - ops[op].unit_off);
            strip = rel / KB; kb = rel - strip * KB;
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
    // bounds of the accumulation chunk (<= I8_SUB_UNITS units of the run) that holds the current unit
    __host__ __device__ __forceinline__ void sub_bounds(int& sb, int& se) const
    {
        sb = run_begin + (seq - run_begin) / I8_SUB_UNITS * I8_SUB_UNITS;
        se = sb + I8_SUB_UNITS < run_end ? sb + I8_SUB_UNITS : run_end;
    }
};

__device__ __forceinline__ float silu_f32(float x) { return x * __fdividef(1.0f, 1.0f + __expf(-x)); }

struct ChainCtx
{
    uint8_t* smem;
    I8Bars bars;
    int w_bytes;
    ChainSmem L;
    // after the ring's barriers: the op's suh copy and its input rows (bulk copies or plain arrivals)
    __device__ __forceinline__ uint32_t IN_BAR() const { return bars.end(); }
};
// the chain lays the ring's barrier block out for the deepest ring; IN_BAR follows it, then the misc words
constexpr int CH_NUM_BARS = I8Bars::words(TC_MAX_STAGES) + 1;

// One unit of a decode warp: wait for the ring stage's weights and digits (W_FULL), then i8_unit_mma.
template <int K>
__device__ __forceinline__ void group_unit(const ChainCtx& cx, int tl, int lane, int s, int sph, int m, uint32_t (&acc)[CH_MR], int& tsum)
{
    const int c = lane & 3;
    mbar_wait_ready<32>(cx.bars.W_FULL(s), sph);
    const uint8_t* b = cx.smem + cx.L.off_b + s * i8_b_stage(CH_MR);
    // the digit sum stays ahead of the MMAs here: read under k-half 0's batch, as the single-GEMM body does, it takes the
    // chain kernel past its spill budget
    if (c < m) tsum += *reinterpret_cast<const int*>(b + i8_b_bytes(CH_MR) + 4 * c);
    I8BatchClock clk{};
    i8_unit_mma<K, CH_MR>(reinterpret_cast<const uint32_t*>(cx.smem + s * cx.w_bytes), smem_desc(smem_u32(b), 128, 4096, 0), tl, lane, acc, clk,
                          [] {});
    __syncwarp();
    if (lane == 0) mbar_arrive(cx.bars.W_EMPTY(s));
}

// KSEL = 0: ops of any bitrate (a switch per unit); KSEL = 1..8: every op of the chain has K = KSEL (smaller code: the
// instruction footprint of all concurrently running roles matters on a kernel this size)
template <int KSEL>
__global__ void __launch_bounds__(TC_THREADS, 1)
chain_i8_kernel(const __grid_constant__ ChainParams p)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const ChainOp* ops = p.n_inline ? p.ops_inline : p.ops;
    const ChainStage* stages = p.n_inline ? p.stages_inline : p.stages;
    const CUtensorMap* tmaps = p.n_inline ? p.tmaps_inline : p.tmaps;
    const int S = p.S;
    ChainCtx cx;
    cx.smem = smem; cx.w_bytes = p.w_bytes; cx.L = chain_smem(S, p.w_bytes, p.cache_bytes, p.suh_bytes);
    cx.bars = I8Bars{smem_u32(smem + cx.L.off_bars), TC_MAX_STAGES};
    uint32_t* misc = reinterpret_cast<uint32_t*>(smem + cx.L.off_bars + 8 * CH_NUM_BARS);
    unsigned int* s_norm2 = reinterpret_cast<unsigned int*>(misc + 4);                                       // [MR] float bits
    float* s_scale = reinterpret_cast<float*>(misc + 8 + 8);                                                 // [CH_SCALE_SLOTS][MR]
    int32_t* s_d = reinterpret_cast<int32_t*>(smem + cx.L.off_d);                                            // [dbuf][group][128][2 MR]
    int* s_dt = reinterpret_cast<int*>(smem + cx.L.off_d + i8_d_bytes(CH_MR) - 2 * 2 * 8 * 4);              // [dbuf][group][8]
    half* cache = reinterpret_cast<half*>(smem + cx.L.off_cache);
    half* suh_s = reinterpret_cast<half*>(smem + cx.L.off_suh);

    pdl_launch_dependents();
    if (warp == 0)
    {
        for (int i = lane; i < CH_NUM_BARS; i += 32)
        {
            int cnt = 1;
            if (i < TC_MAX_STAGES) cnt = I8Bars::W_FULL_ARRIVALS;
            else if (i < 2 * TC_MAX_STAGES) cnt = I8Bars::W_EMPTY_ARRIVALS;
            else if (i >= 3 * TC_MAX_STAGES + 8 && i < 3 * TC_MAX_STAGES + 10) cnt = I8Bars::D_FULL_ARRIVALS;
            else if (i >= 3 * TC_MAX_STAGES + 10 && i < 3 * TC_MAX_STAGES + 12) cnt = I8Bars::D_EMPTY_ARRIVALS;
            else if (i == I8Bars::words(TC_MAX_STAGES)) cnt = 2;                                         // IN_BAR: suh copy + input copy
            mbar_init(cx.bars.bar0 + 8u * i, cnt);
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
            mbar_wait<64>(cx.bars.W_EMPTY(s), ph ^ 1);
            if (elect_one())
            {
                mbar_arrive_expect_tx(cx.bars.W_FULL(s), (uint32_t) (2048 * K));
                tma_load_2d(w_smem0 + s * p.w_bytes, tm, c.strip * (32 * K), c.kb * 8, cx.bars.W_FULL(s), pol_w);
            }
            if (++s == S) { s = 0; ph ^= 1; }
            c.next();
        }
        __syncwarp();
    }
    else if (warp >= TC_XF_WARP0 && warp < TC_DEC_WARP0)
    {
        // =========================== activation warps: scale pass per op, digits per unit ===========================
        const int xw = warp - TC_XF_WARP0;
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
                const bool bulk_x = o.in_mode == 0 && o.cached;       // input rows by one bulk copy straight into the cache
                const bool bulk_s = o.suh != nullptr && o.suh_cached;
                xf_bar();                                             // previous op's cache / suh no longer needed by any digit warp
                if (warp == TC_XF_WARP0)
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
                        while (ld_acquire_gpu_u32(p.ctr + (o.stage - 1)) < want) { __nanosleep(32); poll_watchdog<255u>(polls, t0, "chain stage wait", o.stage, 0); }
                    }
                    __syncwarp();
                    waited = o.stage;
                }
                if (warp == TC_XF_WARP0)
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
                    const float n2 = __uint_as_float(s_norm2[r]);
                    const float bnd = (n2 > 0.f ? i8_sqrt_rn(n2) : 0.f) * 1.002f;   // n2: 0 or in [2^-48, 2^40]
                    inv_scale[r] = bnd > 0.f ? i8_qmax_over(bnd) : 0.f;
                    // every digit warp stores the (identical) value before its own first W_FULL arrival of this op: whichever
                    // arrival the MMA side observes, the scale the epilogue reads later is ordered before it
                    if (lane == r) s_scale[(cur_op % CH_SCALE_SLOTS) * CH_MR + r] = i8_over_qmax(bnd);
                }
            }
            if (turn == xw)
            {
                // ---- digits of this unit: 128-point Hadamard of the cached block, quantise, two int8 digits x 4 bytes ----
                mbar_wait<64>(cx.bars.W_EMPTY(s), ph ^ 1);
                i8_write_digit_tile<CH_MR>(smem + cx.L.off_b + s * i8_b_stage(CH_MR), inv_scale, o.m, lane, cx.bars.W_FULL(s),
                                           [&](int r, float (&v)[4])
                {
                    uint2 raw;
                    if (o.cached) raw = *reinterpret_cast<const uint2*>(cache + (size_t) r * o.k + c.kb * 128 + lane * 4);
                    else
                    {
                        // rows too long for the cache: recompute x * suh (plain fp16 input only, checked on the host)
                        raw = __ldcg(reinterpret_cast<const uint2*>(reinterpret_cast<const half*>(o.A) + (size_t) r * o.k + c.kb * 128 + lane * 4));
                        if (o.suh)
                        {
                            const uint2 scb = *reinterpret_cast<const uint2*>(o.suh + c.kb * 128 + lane * 4);
                            half2* h = reinterpret_cast<half2*>(&raw);
                            h[0] = __hmul2(h[0], *reinterpret_cast<const half2*>(&scb.x));
                            h[1] = __hmul2(h[1], *reinterpret_cast<const half2*>(&scb.y));
                        }
                    }
                    // one Hadamard for both: x * suh is already applied (the cache holds it)
                    if (o.suh) raw = had128_fp16(raw, nullptr, lane);
                    const half2 a = *reinterpret_cast<const half2*>(&raw.x), b = *reinterpret_cast<const half2*>(&raw.y);
                    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
                });
            }
            if (++turn == CH_XF_WARPS) turn = 0;
            if (++s == S) { s = 0; ph ^= 1; }
            c.next();
        }
    }
    else if (warp >= TC_DEC_WARP0 && warp < TC_EPI_WARP0)
    {
        // =========================== decode groups: four warpgroups ===========================
        // warpgroup (g, nh): units seq = g (mod 2), output columns 64 nh .. 64 nh + 63; both groups hand over (possibly zero)
        // accumulators at every accumulation-chunk boundary, the epilogue adds the two
        const int wq = warp & 3, wgi = (warp - TC_DEC_WARP0) >> 2;
        const int g = wgi & 1, nh = wgi >> 1, tl = 4 * nh + wq;
        Cursor c; c.init(ops, stages, p.n_stages, cta, G);
        int s = 0, ph = 0, dbuf = 0, dphase = 0;
        uint32_t acc[CH_MR] = {0u, 0u, 0u, 0u};
        int tsum = 0, t_hi = 0;                                          // t_hi: rows 4..7, none at MR = 4
        while (c.valid)
        {
            int sb, se; c.sub_bounds(sb, se);
            const bool last = c.seq == se - 1;
            if ((c.seq & 1) == g)
            {
                const int m = ops[c.op].m;
                if constexpr (KSEL != 0) group_unit<KSEL>(cx, tl, lane, s, ph, m, acc, tsum);
                else EXL3B_DISPATCH_K(ops[c.op].K, group_unit<KK>(cx, tl, lane, s, ph, m, acc, tsum));
            }
            if (last)
            {
                mbar_wait(cx.bars.D_EMPTY(dbuf), dphase ^ 1);          // the epilogue has drained this buffer
                i8_hand_off<CH_MR>(s_d, s_dt, dbuf, g, nh, wq, lane, acc, tsum, t_hi);
                __syncwarp();
                if (lane == 0) mbar_arrive(cx.bars.D_FULL(dbuf));
                dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
            }
            if (++s == S) { s = 0; ph ^= 1; }
            c.next();
        }
    }
    else if (warp >= TC_EPI_WARP0)
    {
        // =========================== epilogue ===========================
        pdl_wait();
        const int q = warp & 3;
        const int et = threadIdx.x - TC_EPI_WARP0 * 32;
        const int col = et;                                             // column of the strip this thread finishes
        float* tile = reinterpret_cast<float*>(smem + cx.L.off_tile);
        auto epi_bar = [] { asm volatile("bar.sync 1, 128;" ::: "memory"); };
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
            // consecutive stages alternate between two exchange buffers
            float* const parts = p.parts + (size_t) (stage & 1) * DevCtx::I8_PART_CTAS * (CH_MR * 128);
            float facc[CH_MR];
            #pragma unroll
            for (int r = 0; r < CH_MR; ++r) facc[r] = 0.f;
            for (int sb = run_begin; sb < run_end; sb += I8_SUB_UNITS)
            {
                mbar_wait<32>(cx.bars.D_FULL(dbuf), dphase);
                i8_drain<CH_MR>(s_d, s_dt, dbuf, col, o.m, [&](int r) { return s_scale[(op % CH_SCALE_SLOTS) * CH_MR + r]; }, facc);
                __syncwarp();
                if (lane == 0) mbar_arrive(cx.bars.D_EMPTY(dbuf));
                dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
            }

            // who else holds k-segments of this strip?
            const long long gs = o.unit_off + (long long) strip * o.KB;
            const int c_a = cta_of_unit((int) U, c.Gs, (int) gs), c_b = cta_of_unit((int) U, c.Gs, (int) (gs + o.KB - 1));
            const bool full = c_a == c_b;
            if (full)
            {
                #pragma unroll
                for (int r = 0; r < CH_MR; ++r) if (r < o.m) tile[r * 128 + col] = facc[r];
            }
            else if (cta != c_a) i8_splitk_publish<CH_MR>(parts, cta, facc, o.m, col);
            else i8_splitk_reduce<CH_MR>(parts, 0, c_a, c_b, facc, o.m, col, tile);
            if (full || cta == c_a)
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
    static_assert(CH_MR == 4, "the chain takes the int8 rule's 1..4 rows");
    if (const char* why = i8_shape_unsupported(m, k, n, K, cb, false)) return why;
    if (in_mode < 0 || in_mode > 2) return "in_mode must be 0 (fp16 rows), 1 (silu(gate) * up, fp32) or 2 (same, fp16)";
    if (in_mode != 0 && (size_t) m * k * 2 > I8_CACHE_MAX_BYTES) return "gated input needs m * k <= 32768";
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
        // the kernel's vector accesses: fp32 gate / up by float4, fp16 rows / suh / svh by uint2, C by float4 (fp32) or uint2
        // (fp16); k and n are multiples of 128, so an aligned base keeps every row aligned
        {
            const int a_align = a.in_mode == 1 ? 16 : 8, c_align = a.c_fp32 ? 16 : 8;
            const char* bad = nullptr; int need = 0;
            if ((uintptr_t) a.A % a_align) { bad = a.in_mode ? "gate (A)" : "A"; need = a_align; }
            else if (a.in_mode != 0 && (uintptr_t) a.A2 % a_align) { bad = "up (A2)"; need = a_align; }
            else if ((uintptr_t) a.suh % 8) { bad = "suh"; need = 8; }
            else if ((uintptr_t) a.svh % 8) { bad = "svh"; need = 8; }
            else if ((uintptr_t) a.C % c_align) { bad = "C"; need = c_align; }
            EXL3B_CHECK(!bad, EXL3B_ERR_ARG, "exl3_chain: op %d: %s must be %d-byte aligned", i, bad ? bad : "", need);
        }
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
        o.cached = cb_ <= (size_t) I8_CACHE_MAX_BYTES;
        if (o.cached && cb_ > cache) cache = cb_;
        o.suh_cached = a.suh != nullptr && (size_t) a.k * 2 <= (size_t) I8_CACHE_MAX_BYTES && ((uintptr_t) a.suh & 15) == 0;
        if (o.suh_cached && (size_t) a.k * 2 > suhb) suhb = (size_t) a.k * 2;
        if (o.cached && o.in_mode == 0 && ((uintptr_t) a.A & 15) != 0) o.cached = 0;      // bulk copy needs 16-byte alignment
        if (a.K < Kmin) Kmin = a.K;
        st.U += (long long) o.KB * o.strips; st.strips_total += o.strips; st.op_end = i + 1;
        if (a.K > Kmax) Kmax = a.K;
    }
    EXL3B_CHECK(ch.stages.size() <= 255, EXL3B_ERR_UNSUPPORTED, "exl3_chain: more than 255 stages");
    for (const ChainStage& st : ch.stages) if (st.U > Umax) Umax = st.U;
    const int w_bytes = 2048 * Kmax;
    int S = (220 * 1024 - 128 - CH_MR * 128 * 4 - 2048 - i8_d_bytes(CH_MR) - (int) cache - (int) suhb) / (w_bytes + i8_b_stage(CH_MR));
    if (S > TC_MAX_STAGES) S = TC_MAX_STAGES;
    EXL3B_CHECK(S >= 2, EXL3B_ERR_UNSUPPORTED, "exl3_chain: shared-memory budget exceeded");
    const ChainSmem L = chain_smem(S, w_bytes, (int) cache, (int) suhb);
    EXL3B_CHECK(L.total <= 220 * 1024, EXL3B_ERR_UNSUPPORTED, "exl3_chain: shared-memory budget exceeded");
    int grid = num_sms;
    if (Umax < grid) grid = (int) Umax;
    EXL3B_CHECK(grid <= DevCtx::I8_PART_CTAS, EXL3B_ERR_UNSUPPORTED, "exl3_chain: grid exceeds the split-K exchange buffer");
    EXL3B_CHECK(partition_fits(Umax, grid), EXL3B_ERR_UNSUPPORTED, "exl3_chain: too many units for the 32-bit stream-K partition");
    ch.p = ChainParams{};
    ch.p.n_ops = n_ops; ch.p.n_stages = (int) ch.stages.size();
    ch.p.S = S; ch.p.w_bytes = w_bytes; ch.p.cache_bytes = (int) cache; ch.p.suh_bytes = (int) suhb;
    ch.smem_total = L.total; ch.grid = grid; ch.ksel = Kmin == Kmax ? Kmax : 0;
    return 0;
}

static cudaError_t chain_launch(cudaStream_t stream, int grid, int smem_bytes, const ChainParams& p, int ksel)
{
    cudaError_t err = cudaSuccess;
    if (ksel == 0) err = launch_pdl<chain_i8_kernel<0>>(stream, dim3(grid), TC_THREADS, smem_bytes, p);
    else EXL3B_DISPATCH_K(ksel, err = launch_pdl<chain_i8_kernel<KK>>(stream, dim3(grid), TC_THREADS, smem_bytes, p));
    return err;
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
    p.n_inline = 1; p.ctr = ctx->chain_ctr; p.parts = ctx->chain_parts;
    cudaError_t err = chain_launch(stream, ch.grid, ch.smem_total, p, ch.ksel);
    count_launch();
    EXL3B_CUDA(err);
    EXL3B_CUDA(cudaPeekAtLastError());
    return EXL3B_TAG_TC_I8_CHAIN;
}

}  // namespace exl3b
