// The unit pipeline of the int8 codebook path (mul1, m <= 8): the data formats and protocols that the single-GEMM body
// (gemm_tc_i8_body.cuh: plain, row-parallel AR and routed kernels) and the persistent chain kernel (chain_i8.cu) share --
// the ring's barrier block, the digit tile and its K order, one unit's decode + wgmma, the accumulator hand-off to the
// epilogue, the mul1 reassembly and the sentinel split-K exchange.
#pragma once
#include "tc_common.cuh"
#include "i8_math.cuh"

namespace exl3b {

using namespace ptx;

constexpr int I8_MAX_M = 8;                                    // rows per launch: kernel instantiated for MR = 4 and MR = 8 rows
constexpr int I8_DEC_GROUPS = 2;
constexpr int I8_NT = 16;                                      // N: rows 2r = hi digit, 2r+1 = lo digit of row r
// digit tile of a unit: 32 K-chunks x (8 N-rows x 16 B) per row group; N-rows 2r / 2r+1 = hi / lo digit of activation row r, so
// MR = 4 rows fill one row group (4096 B) and MR = 8 rows two (SBO = 4096 B); + 64 B of per-row digit sums behind the tile.
// K order: the value of unit k-index 16 kt + 2 j + b (kt = 4 r + c) sits in K-chunk 2 (8 r + j) + b at byte 4 c -- the slot the
// decode lane holding that weight feeds to wgmma (8 r + j).
__host__ __device__ constexpr int i8_b_bytes(int MR) { return MR <= 4 ? 4096 : 8192; }
__host__ __device__ constexpr int i8_b_stage(int MR) { return i8_b_bytes(MR) + 64; }
constexpr int I8_SUB_UNITS = 96;                               // int32 accumulator safety: <= 12288 k per accumulation
constexpr uint32_t I8_SENTINEL = 0xffffffffu;                  // "no partial sum here yet" in the split-K exchange buffer

// optional shared-memory cache of the whole transformed activation (m x k fp16) and of the per-block digit sums, filled by
// the CTA prologue: the per-unit transform then is an 8-byte LDS + quantise instead of a global load + Hadamard
// (without it the two transform warps do a global load and a Hadamard per row and unit, on the per-unit critical path)
constexpr int I8_CACHE_MAX_BYTES = 64 * 1024;

// accumulator hand-off to the epilogue: [2 buffers][2 decode groups][128 columns][2 MR] int32, then [2][2][8] digit sums
__host__ __device__ constexpr int i8_d_bytes(int MR) { return 2 * 2 * 128 * 2 * MR * 4 + 2 * 2 * 8 * 4; }

#ifdef __CUDACC__

// Barrier block of the unit ring (S = the launch's ring depth), mbarriers at `bar0`:
//   W_FULL(s)   word s          the stage's weights (the producer's expect_tx) and its digit tile (the digit warp's arrival):
//                               a decode warp takes one barrier per unit
//   W_EMPTY(s)  word S + s      the eight decode warps of the unit's group, after their MMAs have read weights and digits;
//                               the producer and the digit warp wait for it before they refill the stage
//   D_FULL(b)   word 3 S + 8 + b   accumulator hand-off buffer b written, by every decode warp
//   D_EMPTY(b)  word 3 S + 10 + b  buffer b drained, by the four epilogue warps
// end() is the first word after the block, words(S) its size.
struct I8Bars
{
    static constexpr int W_FULL_ARRIVALS = 2, W_EMPTY_ARRIVALS = TC_DEC_WARPS / I8_DEC_GROUPS;
    static constexpr int D_FULL_ARRIVALS = TC_DEC_WARPS, D_EMPTY_ARRIVALS = 4;
    __host__ __device__ static constexpr int words(int S) { return 3 * S + 12; }
    uint32_t bar0;
    int S;
    __device__ __forceinline__ uint32_t W_FULL(int s) const { return bar0 + 8u * s; }
    __device__ __forceinline__ uint32_t W_EMPTY(int s) const { return bar0 + 8u * (S + s); }
    __device__ __forceinline__ uint32_t D_FULL(int b) const { return bar0 + 8u * (3 * S + 8 + b); }
    __device__ __forceinline__ uint32_t D_EMPTY(int b) const { return bar0 + 8u * (3 * S + 10 + b); }
    __device__ __forceinline__ uint32_t end() const { return bar0 + 8u * words(S); }
    // by the 32 lanes of one warp, one barrier per lane and round; other() runs on the lanes >= 2 (the caller's own
    // initialisation), then the warp fences the barriers' initialisation
    template <typename Other>
    __device__ __forceinline__ void init(int lane, Other&& other) const
    {
        for (int s = lane; s < S; s += 32) { mbar_init(W_FULL(s), W_FULL_ARRIVALS); mbar_init(W_EMPTY(s), W_EMPTY_ARRIVALS); }
        if (lane < 2) { mbar_init(D_FULL(lane), D_FULL_ARRIVALS); mbar_init(D_EMPTY(lane), D_EMPTY_ARRIVALS); }
        else other();
        fence_barrier_init();
    }
};

// Digit tile of one unit, written by one activation warp into the stage's tile at `dst` after the stage's W_EMPTY:
// row_values(r, v) gives lane's four transformed values k = 4 lane .. 4 lane + 3 of row r < m.  Each value becomes two digits
// replicated over the 4 product bytes, stored in the wgmma K order; the per-row digit sums go behind the tile.  Then the tile is
// made visible to the async proxy and the warp arrives on the stage's `w_full`.
template <int MR, typename RowValues>
__device__ __forceinline__ void i8_write_digit_tile(uint8_t* dst, const float (&inv_scale)[MR], int m, int lane, uint32_t w_full,
                                                    RowValues&& row_values)
{
    int qsum[MR];
    #pragma unroll
    for (int r = 0; r < MR; ++r)
    {
        qsum[r] = 0;
        if (r < m)
        {
            float v[4];
            row_values(r, v);
            uint32_t hi_w[4], lo_w[4];
            int qs = 0;
            #pragma unroll
            for (int e = 0; e < 4; ++e)
            {
                i8_digits(v[e], inv_scale[r], qs, hi_w[e], lo_w[e]);     // digits replicated over the 4 product bytes
            }
            // k = 4 lane + e: K-chunk 16 (lane / 16) + 4 (lane % 4) + e, byte 4 ((lane / 4) % 4); N-rows 2r (hi) and
            // 2r+1 (lo): row group r / 4, local rows 2 (r % 4), +1
            uint8_t* drow = dst + (r >> 2) * 4096 + ((16 * (lane >> 4) + 4 * (lane & 3)) * 8 + 2 * (r & 3)) * 16 + 4 * ((lane >> 2) & 3);
            #pragma unroll
            for (int e = 0; e < 4; ++e)
            {
                *reinterpret_cast<uint32_t*>(drow + e * 128) = hi_w[e];
                *reinterpret_cast<uint32_t*>(drow + e * 128 + 16) = lo_w[e];
            }
            qsum[r] = qs;
        }
    }
    // digit sums of all rows: the butterfly steps of different rows are independent, issued side by side
    #pragma unroll
    for (int o = 16; o > 0; o >>= 1)
    {
        #pragma unroll
        for (int r = 0; r < MR; ++r) qsum[r] += __shfl_xor_sync(0xffffffffu, qsum[r], o);
    }
    if (lane < m)
    {
        int mine = 0;
        #pragma unroll
        for (int r = 0; r < MR; ++r) if (lane == r) mine = qsum[r];
        *reinterpret_cast<int*>(dst + i8_b_bytes(MR) + 4 * lane) = mine;
    }
    fence_proxy_async_smem();
    __syncwarp();
    if (lane == 0) mbar_arrive(w_full);
}

#ifdef EXL3B_TC_DEBUG
__device__ __forceinline__ uint32_t sm_clock()
{
    uint32_t t; asm volatile("mov.u32 %0, %%clock;" : "=r"(t) :: "memory"); return t;
}
// The SM clock once `v` is available: both predicated reads wait for the compare, so for a register loaded from shared memory
// the stamp includes the load's latency (an unconditional read of %clock would issue right behind the load).
__device__ __forceinline__ uint32_t sm_clock_after(uint32_t v)
{
    uint32_t t;
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.u32 p, %1, 0x9e3779b9;\n\t@p mov.u32 %0, %%clock;\n\t@!p mov.u32 %0, %%clock;\n\t}"
                 : "=r"(t) : "r"(v) : "memory");
    return t;
}
#endif

// Timeline of a decode warp's k-half wgmma batches in the EXL3B_TC_DEBUG build (tools/i8_phase_profile.py): the SM clock at
// the issue and at the retirement of each batch, and for the unit-gap split the clock once k-half 0's weight words are in
// registers, after its first wgmma, and after the register fences that end the unit.  The other builds keep no state and
// emit nothing.
struct I8BatchClock
{
#ifdef EXL3B_TC_DEBUG
    unsigned long long* dbg;                 // slots of the CTA's timeline row (16 batches), null: no stamps
    int i;                                   // next batch
    uint32_t t_issue;
    uint32_t t_loaded0, t_issue0, t_mma0;    // k-half 0: weight words loaded, fence reached (decoded), first wgmma issued
    uint32_t t_retired1, t_end;              // k-half 1: batch retired, register fences passed
    __device__ __forceinline__ void loaded(int r, uint32_t w) { if (r == 0) t_loaded0 = sm_clock_after(w); }
    __device__ __forceinline__ void issue(int r) { t_issue = sm_clock(); if (r == 0) t_issue0 = t_issue; }
    __device__ __forceinline__ void first_mma(int r) { if (r == 0) t_mma0 = sm_clock(); }
    __device__ __forceinline__ void retired(int r)
    {
        const uint32_t t = sm_clock();
        if (dbg && i < 16) dbg[i] = ((unsigned long long) t << 32) | t_issue;          // retirement (high word), issue (low)
        ++i;
        if (r == 1) t_retired1 = t;
    }
    __device__ __forceinline__ void end() { t_end = sm_clock(); }
#else
    __device__ __forceinline__ void loaded(int, uint32_t) {}
    __device__ __forceinline__ void issue(int) {}
    __device__ __forceinline__ void first_mma(int) {}
    __device__ __forceinline__ void retired(int) {}
    __device__ __forceinline__ void end() {}
#endif
};

// One unit (128 k x 128 n weights) of a decode warp: lane (chunk, c) decodes tile column `tl`, both halves, of k-tile 4 r + c
// (r = 0, 1) from the weight stage `wst` straight into wgmma A fragments, 8 wgmma.m64nNk32 per r against the digit tile at
// `desc_s`, into acc.  The caller has waited for the stage's W_FULL.  `in_flight()` runs while k-half 0's batch
// is in flight (the caller's per-unit bookkeeping; it must not touch acc).  `clk` takes the batches' issue and retirement
// times (debug timeline).
template <int K, int MR, typename InFlight>
__device__ __forceinline__ void i8_unit_mma(const uint32_t* wst, uint64_t desc_s, int tl, int lane, uint32_t (&acc)[MR], I8BatchClock& clk,
                                            InFlight&& in_flight)
{
    const int chunk = lane >> 2, c = lane & 3;
    // k-half 0's weight words are loaded here, k-half 1's while k-half 0's batch is in flight: its decode then starts on
    // words already in registers (K + 1 registers next to the fragments the batch reads)
    uint32_t w[K + 1];
    load_chunk<K>(wst + (c * 8 + tl) * (8 * K), chunk, w);
    #pragma unroll
    for (int r = 0; r < 2; ++r)
    {
        uint32_t o0[16], o1[16];
        clk.loaded(r, w[K]);
        decode16_i8<K, 0>(w, o0);
        decode16_i8<K, 1>(w, o1);
        #pragma unroll
        for (int i = 0; i < MR; ++i) reg_fence(acc[i]);
        clk.issue(r);
        wgmma_fence();
        #pragma unroll
        for (int j = 0; j < 8; ++j)
        {
            wgmma_u8s8<MR>(acc, o0[2 * j], o1[2 * j], o0[2 * j + 1], o1[2 * j + 1], desc_s + (uint64_t) (16 * (8 * r + j)));
            if (j == 0) clk.first_mma(r);
        }
        wgmma_commit();
        if (r == 0)
        {
            in_flight();
            load_chunk<K>(wst + ((4 + c) * 8 + tl) * (8 * K), chunk, w);
        }
        wgmma_wait<0>();
        clk.retired(r);
        #pragma unroll
        for (int i = 0; i < 16; ++i) { reg_fence(o0[i]); reg_fence(o1[i]); }
        #pragma unroll
        for (int i = 0; i < MR; ++i) reg_fence(acc[i]);
    }
    clk.end();
}

// Hand a sub-segment's accumulators of decode group g to the epilogue: the registers into s_d [dbuf][g][128][2 MR], the digit
// sums of rows c and c + 4 (one warp of the group stores them) into s_dt [dbuf][g][8]; then both start again from zero.
// The caller waits for D_EMPTY before and arrives on D_FULL after.
template <int MR>
__device__ __forceinline__ void i8_hand_off(int32_t* s_d, int* s_dt, int dbuf, int g, int nh, int wq, int lane, uint32_t (&acc)[MR],
                                            int& t_lo, int& t_hi)
{
    const int chunk = lane >> 2, c = lane & 3;
    int32_t* dst = s_d + (size_t) ((dbuf * 2 + g) * 128 + 64 * nh + 16 * wq + chunk) * (2 * MR);
    #pragma unroll
    for (int i = 0; i < MR / 4; ++i)
    {
        *reinterpret_cast<int2*>(dst + 8 * i + 2 * c) = make_int2((int) acc[4 * i], (int) acc[4 * i + 1]);
        *reinterpret_cast<int2*>(dst + 8 * (2 * MR) + 8 * i + 2 * c) = make_int2((int) acc[4 * i + 2], (int) acc[4 * i + 3]);
    }
    if (nh == 0 && wq == 0 && lane < 4)
    {
        s_dt[(dbuf * 2 + g) * 8 + c] = t_lo;
        s_dt[(dbuf * 2 + g) * 8 + c + 4] = t_hi;
    }
    #pragma unroll
    for (int i = 0; i < MR; ++i) acc[i] = 0u;
    t_lo = 0; t_hi = 0;
}

// Epilogue side of the hand-off: one sub-segment of both decode groups, column `col`, into facc[r] for the rows r < m;
// scale(r) is row r's activation scale (max / I8_QMAX).  The mul1 reassembly: w = k_inv * (1024 + bytesum) + k_bias.
template <int MR, typename RowScale>
__device__ __forceinline__ void i8_drain(const int32_t* s_d, const int* s_dt, int dbuf, int col, int m, RowScale&& scale,
                                         float (&facc)[MR])
{
    const float k_inv = __half2float(__ushort_as_half((unsigned short) 0x1eee));
    const float k_bias = __half2float(__ushort_as_half((unsigned short) 0xc931));
    const float c1 = 1534.0f * k_inv + k_bias;        // (1024 + 510) k_inv + k_bias: residue of the fp16-rounded bias
    const int32_t* d0 = s_d + (size_t) ((dbuf * 2 + 0) * 128 + col) * (2 * MR);
    const int32_t* d1 = s_d + (size_t) ((dbuf * 2 + 1) * 128 + col) * (2 * MR);
    #pragma unroll
    for (int r = 0; r < MR; ++r)
    {
        if (r < m)
        {
            const int T = s_dt[(dbuf * 2 + 0) * 8 + r] + s_dt[(dbuf * 2 + 1) * 8 + r];
            // sum_k q_k (bytesum_kn - 510), exact in 64-bit (the two groups' int32 partials add without loss)
            const long long sp = i8_centred_sum(d0[2 * r] + d1[2 * r], d0[2 * r + 1] + d1[2 * r + 1], T);
            facc[r] += i8_assemble(sp, T, scale(r), k_inv, c1);
        }
    }
}

// ---- split-K exchange --------------------------------------------------------------------------------------------------
// A strip whose k-segments several CTAs hold is summed through a buffer with one slot of MR x 128 floats per CTA: parts +
// (cta_off + c) * MR * 128 for the c-th CTA of the unit space.  Contributors publish their partial sums and move on.  The data
// is its own flag: the exchange buffer holds the sentinel everywhere outside a launch, a 32-bit store is single-copy atomic,
// so no fence, counter or ticket.
template <int MR>
__device__ __forceinline__ void i8_splitk_publish(float* parts, int cta, const float (&facc)[MR], int m, int col)
{
    #pragma unroll
    for (int r = 0; r < MR; ++r)
        if (r < m)
        {
            uint32_t bits = __float_as_uint(facc[r]);
            if (bits == I8_SENTINEL) bits = 0x7fc00000u;                 // a NaN stays a NaN
            st_relaxed_gpu_u32(reinterpret_cast<uint32_t*>(parts + (size_t) cta * (MR * 128) + r * 128 + col), bits);
        }
}

// The CTA c_a that owns the strip's FIRST k-segment works on it LAST (segments are processed in unit order), so it is the
// natural reducer: own sums from registers, then those of CTAs c_a + 1 .. c_b in fixed CTA order (bit-reproducible), each slot
// re-armed with the sentinel once read.  One global round trip in the common case.  Result: tile[r * 128 + col].
template <int MR>
__device__ __forceinline__ void i8_splitk_reduce(float* parts, int cta_off, int c_a, int c_b, const float (&facc)[MR], int m, int col,
                                                 float* tile)
{
    #pragma unroll
    for (int r = 0; r < MR; ++r)
    {
        if (r < m)
        {
            float a = 0.f;
            a += facc[r];
            int c = c_a + 1;
            while (c <= c_b)
            {
                uint32_t v[8];
                bool ok;
                uint32_t polls = 0;
                unsigned long long t0 = 0;
                do
                {
                    ok = true;
                    #pragma unroll
                    for (int j = 0; j < 8; ++j)
                    {
                        const int cc = c + j;
                        v[j] = 0u;
                        if (cc <= c_b)
                        {
                            v[j] = ld_relaxed_gpu_u32(reinterpret_cast<const uint32_t*>(parts + (size_t) (cta_off + cc) * (MR * 128) + r * 128 + col));
                            ok = ok && v[j] != I8_SENTINEL;
                        }
                    }
                    if (!ok) poll_watchdog<255>(polls, t0, "split-K exchange", c_a, c_b);
                } while (!ok);
                #pragma unroll
                for (int j = 0; j < 8; ++j)
                {
                    const int cc = c + j;
                    if (cc <= c_b)
                    {
                        a += __uint_as_float(v[j]);
                        // re-arm the slot for the launch that uses this exchange buffer next
                        st_relaxed_gpu_u32(reinterpret_cast<uint32_t*>(parts + (size_t) (cta_off + cc) * (MR * 128) + r * 128 + col), I8_SENTINEL);
                    }
                }
                c += 8;
            }
            tile[r * 128 + col] = a;
        }
    }
}

#endif  // __CUDACC__

}  // namespace exl3b
