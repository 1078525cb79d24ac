// wgmma u8 x s8 EXL3 decode-GEMM for the mul1 codebook, m <= 4 (instantiated for up to 8 rows, see api.cu) ("TC-i8 path", tag 210).
//
// Why: the bit-exact mul1 decode needs IMAD + IDP.4A per weight on the same issue pipe plus pack + HFMA2.
// The mul1 value is AFFINE in the byte sum of x = state * 0x83DCD12D:
//        w = k_inv * (1024 + b0 + b1 + b2 + b3) + k_bias              (codebook.cuh:77-89, before its fp16 rounding)
// so   sum_k a_k w_kn = k_inv * sum_k a_k (b0+b1+b2+b3)_kn + (1024 k_inv + k_bias) * sum_k a_k.
// The first sum is an integer GEMM whose K-elements are the four product BYTES: the decode thread stores the raw
// 32-bit product into a register A operand of wgmma (4 u8 along K) and the tensor core sums the bytes while contracting
// with the activation, which is quantised per row to a balanced pair of signed 8-bit digits (q = 256 hi + lo,
// |q| <= 32512, i.e. 16-bit activations; hi and lo are two N-columns, each digit replicated over the 4 bytes).
// Per weight that leaves window extraction + ONE IMAD.
//
// Numerics: integer accumulation is exact; what differs from the reference's fp16 kernel is (a) the per-weight fp16
// rounding of the codebook value is skipped (rel-RMS ~3e-4 of the output, unbiased) and (b) activations carry
// 16-bit instead of fp16 quantisation noise (smaller).  The reference's own default decode path for mul1 at m <= 2 is
// its int8-activation GEMV with ~0.9 % output RMS deviation (exl3_gemv_int8.cu:19-20); this path is ~30x closer to
// the fp16 kernel than that.  Tolerances are asserted in tests/test_gpu_parity.py::test_gemm_i8_*.
//
// Structure: stream-K units of 128x128 weights, a TMA ring of weight stages, warp roles:
//   * four decode warpgroups (warps 4..19): warpgroup (g, nh) takes the units u = g (mod 2) and their 64 output columns
//     nh*64 .. nh*64+63.  A warp owns one 16x16-tile column of the strip; lane (chunk, c) decodes tile column `chunk`, both
//     halves, of k-tile 4r + c (r = 0, 1).  Its 2 x 16 products ARE the wgmma A fragments (rows chunk / chunk + 8, K slots
//     c / c + 4) of 8 wgmma.m64nNk32 per r; the K order inside each instruction is permuted accordingly in the digit tile.
//     int32 accumulators stay in registers for a sub-segment and are then handed to the epilogue through shared memory
//   * a CTA prologue (warps 1..23, redundantly per CTA) transforms the rows once into a shared-memory cache and finds the
//     per-row |xh| maximum; the two transform warps then write per-unit activation digits + digit sums
//   * split-K partial sums travel through a sentinel-armed exchange buffer: contributors store and leave, the CTA owning the
//     strip's first k-segment (it processes it last) adds them to its registers in fixed CTA order and re-arms the slots --
//     no fence, no ticket, one global round trip, bit-reproducible
//   * multi-matrix launches (dense exl3_mgemm: the model's k+v and gate+up calls): the grid is cut into one CTA group per
//     matrix; the pointer tables stay in device memory, each CTA patches the weight tensor map's address on the device
//   * instantiated for MR = 4 and MR = 8 activation rows (digit tile with one / two row groups); api.cu auto-selects m <= 4
#pragma once
#include "i8_pipeline.cuh"
#include "act.cuh"
#include <type_traits>

namespace exl3b {

// (row, k-block) input loads a prologue warp keeps in flight per round trip: 2 registers each, plus 2 per block for suh.
// 5 covers k = 23 * 5 * 128 = 14720 (Llama's down projection) at m = 1 in one round trip; more blocks per round trip made
// ptxas spill in the routed kernel, whose spill-free register allocation is kept (ptxas -v).
constexpr int I8_PRO_SLOTS = 5;

__host__ __device__ inline TcSmemLayout i8_smem_layout(int K, int MR, int stages, int cache_bytes)
{
    TcSmemLayout L = tc_smem_layout(K, i8_b_stage(MR), stages);
    L.off_d = L.total;                 // accumulator hand-off after the barrier block
    L.total += i8_d_bytes(MR);
    L.total += cache_bytes;            // cache after that
    return L;
}

// The kernel body, shared by the plain kernel (gemm_tc_i8.cu) and the row-parallel variant whose epilogue sums the
// tensor-parallel partial outputs over NVLink peer memory (gemm_tc_i8_ar.cu, AR = true).
// ROUTED = true (gemm_tc_i8_routed.cu): multi-matrix launch whose CTA groups are the ACTIVE SLOTS of an exl3_mgemm call with
// indices / weights / expert-range filter (MoE decode); slot -> matrix and the slot's output weight come from the table the
// resolve kernel wrote just before this launch.
// GATED = true (gemm_tc_i8.cu, exl3b_gemm_gated): the rows are fp16(act(G) * U) (act.cuh), formed where the plain kernel loads
// A_raw; everything from the input transform on is the plain kernel's.
template <int K, int MR, bool AR, bool ROUTED = false, bool GATED = false>
__device__ __forceinline__ void gemm_tc_i8_body(const TcParams& p, const CUtensorMap* tmap_w, const ArArgs* ar,
                                                const RouteArgs* route = nullptr, const GateIn* gate = nullptr)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int I8_B_BYTES = i8_b_bytes(MR);
    const TcSmemLayout L = i8_smem_layout(K, MR, p.stages, 0);          // offsets only; the cache starts at L.total
    int32_t* const s_d = reinterpret_cast<int32_t*>(smem + L.off_d);     // accumulator hand-off, [dbuf][group][128][2 MR]
    int* const s_dt = reinterpret_cast<int*>(smem + L.off_d + i8_d_bytes(MR) - 2 * 2 * 8 * 4);   // digit sums, [dbuf][group][8]
    const bool cached = p.b_load_bytes > 0;                            // host: cache_bytes (0 = recompute per unit)
    half* xh_cache = reinterpret_cast<half*>(smem + L.total);
    // warp index broadcast from lane 0: ptxas then knows it is warp-uniform, so the role branches and everything derived from
    // the warp index (decode group, stage, wgmma descriptors) stay in uniform registers; a descriptor in per-thread registers
    // costs a 64-bit add and two R2UR in front of every wgmma (tests/test_i8_issue_sass_host.py)
    const int warp = __shfl_sync(0xffffffffu, (int) (threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const int S = p.stages;

    // multi-matrix launch (exl3_mgemm): group `mat` of g_per_mat CTAs works on matrix `mat` exactly like a single-matrix
    // launch of g_per_mat CTAs; `cta` is the index inside the group
    int cta = blockIdx.x, G = gridDim.x, mat = 0;
    const half* suh = p.suh; const half* svh = p.svh; const half* A_raw = p.A_raw;
    char* Cout = (char*) p.C;
    const bool multi = p.num_mats > 0;
    float* const parts = p.parts;                    // split-K exchange buffer, one slot of MR x 128 floats per CTA of the grid
    int cta0 = 0;                                    // first CTA of this matrix's group
    int n_loc = p.n;                                 // output width of this CTA's matrix
    [[maybe_unused]] float routed_scale = 1.f;
    if (multi)
    {
        if (p.rag)
        {
            // fan-out: CTA groups proportional to the matrices' unit counts (host-computed boundaries)
            #pragma unroll
            for (int j = 1; j < TC_RAG_MAX_MATS; ++j) if (j < p.num_mats && (int) blockIdx.x >= p.rag_cta0[j]) mat = j;
            #pragma unroll
            for (int j = 0; j < TC_RAG_MAX_MATS; ++j) if (j == mat) { cta0 = p.rag_cta0[j]; G = p.rag_cta0[j + 1] - cta0; n_loc = p.rag_n[j]; }
            cta = blockIdx.x - cta0;
        }
        else { G = p.g_per_mat; mat = blockIdx.x / G; cta = blockIdx.x - mat * G; cta0 = mat * G; }
        const int slot = mat;                        // inputs / outputs are per slot, the pointer tables per matrix
        if constexpr (ROUTED)
        {
            // the slot table is written by the resolve kernel that precedes this launch: nothing can start before it is
            // complete (the weight prefetch of the plain kernel is given up here).  Slots beyond the active ones, and
            // skipped slots (negative index), have no work: the whole CTA group leaves before it allocates anything.
            pdl_wait();
            if (slot >= route->tab->n_active) return;
            mat = route->tab->mat[slot];
            if (mat < 0) return;
            if (route->has_weights) routed_scale = __half2float(route->tab->weight[slot]);
        }
        suh = reinterpret_cast<const half*>(p.suh_ptrs[mat]); svh = reinterpret_cast<const half*>(p.svh_ptrs[mat]);
        A_raw += (size_t) slot * p.a_mat_stride;
        if (p.rag) Cout = reinterpret_cast<char*>(p.c_ptrs[mat]); else Cout += (size_t) slot * p.c_mat_stride;
    }

    if (multi && warp == 0)
    {
        // per-CTA tensor map: the template (dims / strides / box of this shape) with matrix `mat`'s address -- and, in a fan-out
        // launch, its own width (innermost extent in 8-byte elements, row pitch in bytes).  Patched here, where `mat` is at
        // hand, so that it is not kept live until the producer's loop (it was spilled there).
        const size_t w_pitch = (size_t) (n_loc / 16) * 32 * K;           // bytes per 16-row tile row of the packed tensor
        uint8_t* stm = smem + ((L.off_bars + 640 + 127) & ~127);
        reinterpret_cast<uint32_t*>(stm)[lane] = reinterpret_cast<const uint32_t*>(tmap_w)[lane];
        __syncwarp();
        void* gtm = p.tmap_slots + (size_t) blockIdx.x * 128;
        if (p.rag) tmap_patch_address_width(smem_u32(stm), gtm, p.B_ptrs[mat], (uint32_t) (w_pitch / 8), (uint64_t) w_pitch, lane);
        else tmap_patch_address(smem_u32(stm), gtm, p.B_ptrs[mat], lane);
    }

    const I8Bars bars{smem_u32(smem + L.off_bars), S};
    uint32_t* misc = reinterpret_cast<uint32_t*>(smem + L.off_bars + 8 * (3 * TC_MAX_STAGES + 16));
    unsigned int* s_absmax = reinterpret_cast<unsigned int*>(misc + 4);           // [MR] float bits, >= 0
    [[maybe_unused]] volatile unsigned int* s_ar = reinterpret_cast<volatile unsigned int*>(misc + 28);   // AR: epoch of this launch

#ifdef EXL3B_TC_DEBUG
    // how often did a role find its barrier not yet complete (= it had to wait)?  slots 56.. of the CTA's debug row
    int wf_a = 0, wf_b = 0, wf_c = 0;
#define I8_WAITCNT(cnt, bar, par) do { if (!mbar_test_wait((bar), (par))) ++(cnt); } while (0)
#else
#define I8_WAITCNT(cnt, bar, par) do { } while (0)
#endif
    if (threadIdx.x == 0) tc_stamp(p.dbg, 0);
    pdl_launch_dependents();

    if (warp == 0) bars.init(lane, [&] { if (lane < 2 + MR) s_absmax[lane - 2] = 0u; });
    __syncthreads();
    if (threadIdx.x == 0) tc_stamp(p.dbg, 1);

    const int KB = p.k / 128;
    const int strips = n_loc / 128;
    const int U = KB * strips;
    const int ubeg = unit_begin(U, G, cta), uend = unit_begin(U, G, cta + 1);
    const int n_units = uend - ubeg;

    // the raw fp16 inputs k = kb * 128 + 4 lane .. + 3 of row r
    auto raw_block = [&](int r, int kb) -> uint2
    {
        const size_t e = (size_t) r * p.k + kb * 128 + lane * 4;
        if constexpr (GATED) return gated_load4(*gate, e);
        else return *reinterpret_cast<const uint2*>(A_raw + e);
    };

    // fp16 transformed activation of (row r, k-block kb), 4 values per lane, exactly as the reference's A_had
    auto xh_finish = [&](uint2 raw, uint2 scb, float (&v)[4])
    {
        if (suh) raw = had128_fp16(raw, &scb, lane);
        const half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
        v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
    };
    auto xh_block = [&](int r, int kb, float (&v)[4])
    {
        const uint2 raw = raw_block(r, kb);
        uint2 scb = make_uint2(0, 0);
        if (suh) scb = *reinterpret_cast<const uint2*>(suh + kb * 128 + lane * 4);
        xh_finish(raw, scb, v);
    };
    // one transformed block: into the cache, its |max| into the row maximum
    auto xh_publish = [&](int r, int kb, const float (&v)[4])
    {
        if (cached)
        {
            const half2 a = __floats2half2_rn(v[0], v[1]), b = __floats2half2_rn(v[2], v[3]);     // exact: values are fp16
            uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&b);
            *reinterpret_cast<uint2*>(xh_cache + (size_t) r * p.k + kb * 128 + lane * 4) = o;
        }
        float mx = fmaxf(fmaxf(fabsf(v[0]), fabsf(v[1])), fmaxf(fabsf(v[2]), fabsf(v[3])));
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        if (lane == 0) atomicMax(&s_absmax[r], __float_as_uint(mx));
    };

    // ---- prologue: per-row max |xh| over the whole row (every warp but the producer), overlapped with the first weight loads ----
    // The decode warps can start only after it, so it is on every launch's critical path, and its cost is the number of
    // dependent memory round trips.  Warp w (1..23) takes the k-blocks w - 1, w - 1 + 23, ... with all rows of each block and
    // issues the loads of up to I8_PRO_SLOTS (row, block) pairs before its first Hadamard: at m = 1 that is one round trip up
    // to k = 23 * I8_PRO_SLOTS * 128.  suh is a weight (it does not depend on the previous kernel) and usually comes from DRAM: the first
    // round's blocks are fetched BEFORE griddepcontrol.wait, the activations only after it.  The epilogue warps take part too;
    // their pdl_wait here comes before their first use of A.
    if (warp != 0)
    {
        constexpr int nw = TC_THREADS / 32 - 1;
        const int w0 = warp - 1;
        auto transform = [&](auto rows)
        {
            constexpr int M = decltype(rows)::value;     // rows loaded per block: the register arrays are sized for M
            constexpr int NB = I8_PRO_SLOTS / M > 0 ? I8_PRO_SLOTS / M : 1;
            uint2 sc[NB];
            auto load_suh = [&](int kb0)
            {
                #pragma unroll
                for (int j = 0; j < NB; ++j)
                {
                    const int kb = kb0 + j * nw;
                    sc[j] = make_uint2(0, 0);
                    if (suh && kb < KB) sc[j] = *reinterpret_cast<const uint2*>(suh + kb * 128 + lane * 4);
                }
            };
            load_suh(w0);
            if constexpr (!ROUTED) pdl_wait();            // A is produced by the previous kernel (ROUTED waited at the top)
            for (int kb0 = w0; kb0 < KB; kb0 += NB * nw)
            {
                if (kb0 != w0) load_suh(kb0);
                uint2 raw[NB][M];
                #pragma unroll
                for (int j = 0; j < NB; ++j)
                {
                    #pragma unroll
                    for (int r = 0; r < M; ++r)
                    {
                        raw[j][r] = make_uint2(0, 0);
                        if (kb0 + j * nw < KB && r < p.m) raw[j][r] = raw_block(r, kb0 + j * nw);
                    }
                }
                #pragma unroll
                for (int j = 0; j < NB; ++j)
                {
                    #pragma unroll
                    for (int r = 0; r < M; ++r)
                    {
                        if (kb0 + j * nw < KB && r < p.m)
                        {
                            float v[4];
                            xh_finish(raw[j][r], sc[j], v);
                            xh_publish(r, kb0 + j * nw, v);
                        }
                    }
                }
            }
        };
        // batch 1 (the decode token) gets the widest round trip; otherwise the arrays are sized for MR rows
        if (p.m == 1) transform(std::integral_constant<int, 1>());
        else transform(std::integral_constant<int, MR>());
        asm volatile("bar.sync 2, %0;" :: "n"(TC_THREADS - 32) : "memory");
        if (warp == TC_DEC_WARP0 && lane == 0) tc_stamp(p.dbg, 2);
    }

    if (warp == 0)
    {
        // =========================== producer ===========================
        // multi-matrix launch: this CTA's tensor map was patched at the top of the kernel
        const void* tm = multi ? static_cast<const void*>(p.tmap_slots + (size_t) blockIdx.x * 128) : static_cast<const void*>(tmap_w);
        if (!multi && elect_one()) prefetch_tmap(tmap_w);
        const uint64_t pol_w = policy_evict_first();
        const uint32_t w_smem0 = smem_u32(smem);
        int strip = ubeg / KB, kb = ubeg % KB;
        int s = 0, ph = 0;
        for (int u = 0; u < n_units; ++u)
        {
            if (u >= S) { I8_WAITCNT(wf_a, bars.W_EMPTY(s), ph ^ 1); mbar_wait<64>(bars.W_EMPTY(s), ph ^ 1); }
            if (elect_one())
            {
                mbar_arrive_expect_tx(bars.W_FULL(s), (uint32_t) L.w_bytes);
                tma_load_2d(w_smem0 + s * L.w_bytes, tm, strip * (32 * K), kb * 8, bars.W_FULL(s), pol_w);
            }
            if (++kb == KB) { kb = 0; ++strip; }
            if (++s == S) { s = 0; ph ^= 1; }
        }
        __syncwarp();
#ifdef EXL3B_TC_DEBUG
        if (lane == 0 && p.dbg) p.dbg[blockIdx.x * 64 + 56] = wf_a;
#endif
    }
    else if (warp >= TC_XF_WARP0 && warp < TC_DEC_WARP0)
    {
        // =========================== activation digits (per unit) ===========================
        const int xw = warp - TC_XF_WARP0;
        float inv_scale[MR];
        #pragma unroll
        for (int r = 0; r < MR; ++r)
        {
            const float mx = __uint_as_float(s_absmax[r]);
            inv_scale[r] = mx > 0.f ? i8_qmax_over(mx) : 0.f;
        }
        int kb = (ubeg + xw) % KB;
        int s = xw % S, ph = 0;
        const int kstep = 2 % KB;
        for (int u = xw; u < n_units; u += 2)
        {
            I8_WAITCNT(wf_a, bars.W_EMPTY(s), ph ^ 1);
            mbar_wait<64>(bars.W_EMPTY(s), ph ^ 1);
            i8_write_digit_tile<MR>(smem + L.off_b + s * L.b_bytes, inv_scale, p.m, lane, bars.W_FULL(s), [&](int r, float (&v)[4])
            {
                if (cached)
                {
                    const uint2 raw = *reinterpret_cast<const uint2*>(xh_cache + (size_t) r * p.k + kb * 128 + lane * 4);
                    const half2 a = *reinterpret_cast<const half2*>(&raw.x), b = *reinterpret_cast<const half2*>(&raw.y);
                    v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
                }
                else xh_block(r, kb, v);
            });
            kb += kstep; if (kb >= KB) kb -= KB;
            s += 2; if (s >= S) { s -= S; ph ^= 1; }
        }
#ifdef EXL3B_TC_DEBUG
        if (xw == 0 && lane == 0 && p.dbg) p.dbg[blockIdx.x * 64 + 61] = wf_a;
#endif
    }
    else if (warp >= TC_DEC_WARP0 && warp < TC_EPI_WARP0)
    {
        // =========================== decode + MMA ===========================
        // Warpgroup (g, nh): units u = g (mod 2), output columns 64 nh .. 64 nh + 63 of the strip.  A group steps through its
        // own units only, but hands over (possibly zero) accumulators at every sub-segment boundary; the epilogue adds the two.
        const int wq = warp & 3, wgi = (warp - TC_DEC_WARP0) >> 2;
        const int g = wgi & 1, nh = wgi >> 1;
        const int tl = 4 * nh + wq;                      // tile column of the strip owned by this warp
        const int c = lane & 3;
        const uint64_t desc0 = smem_desc(smem_u32(smem + L.off_b), 128, 4096, 0);
        uint32_t acc[MR];
        #pragma unroll
        for (int i = 0; i < MR; ++i) acc[i] = 0u;
        int t_lo = 0, t_hi = 0;                          // digit sums of activation rows c and c + 4 over the group's units
        // debug timeline: lane 0 of the group's first warp stamps its first 16 batches into slots 16 + 16 g ..
        I8BatchClock clk{};
#ifdef EXL3B_TC_DEBUG
        unsigned long long* const dbg_row = p.dbg && nh == 0 && wq == 0 && lane == 0 ? p.dbg + blockIdx.x * 64 : nullptr;
        clk.dbg = dbg_row ? dbg_row + 16 + 16 * g : nullptr;
        // unit-gap split: row gridDim.x + blockIdx.x, seen as 128 words; words 8 + 12 (4 g + j) .. + 11 follow the group's
        // step from its unit j < 4 to unit j + 1 (tools/i8_phase_profile.py, "unit_gap_split")
        uint32_t* const att = dbg_row ? reinterpret_cast<uint32_t*>(p.dbg + (gridDim.x + blockIdx.x) * 64) + 8 + 48 * g : nullptr;
        uint32_t t_ho = 0;                               // clocks in hand-offs since the group's last W_EMPTY arrival
        int du = 0;                                      // the group's unit count
#endif
        int dbuf = 0, dphase = 0;
        auto hand_off = [&]
        {
#ifdef EXL3B_TC_DEBUG
            const uint32_t t0 = sm_clock();
#endif
            // hand the sub-segment's accumulators to the epilogue
            mbar_wait(bars.D_EMPTY(dbuf), dphase ^ 1);
            i8_hand_off<MR>(s_d, s_dt, dbuf, g, nh, wq, lane, acc, t_lo, t_hi);
            __syncwarp();
            if (lane == 0) mbar_arrive(bars.D_FULL(dbuf));
            dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
#ifdef EXL3B_TC_DEBUG
            t_ho += sm_clock() - t0;
#endif
        };
        auto unit = [&](int u, int s, int sph)
        {
#ifdef EXL3B_TC_DEBUG
            const uint32_t t_in = sm_clock();
            uint32_t wait_info = 0;                      // bit 31: the first probe failed; bits 0..30: ns slept after it
            if (att)
            {
                // the release wait below, taken apart: mbar_wait_ready<32>
                if (!mbar_test_wait(bars.W_FULL(s), sph))
                {
                    wait_info = 1u << 31;
                    uint32_t ns = 32, polls = 0;
                    unsigned long long t0 = 0;
                    while (!mbar_try_wait(bars.W_FULL(s), sph))
                    {
                        __nanosleep(ns); wait_info += ns; if (ns < 512u) ns <<= 1;
                        poll_watchdog<1023u>(polls, t0, "mbarrier", (int) bars.W_FULL(s), sph);
                    }
                }
            }
            else
#endif
            mbar_wait_ready<32>(bars.W_FULL(s), sph);                             // the unit's weights and activation digits
#ifdef EXL3B_TC_DEBUG
            const uint32_t t_out = sm_clock();
#endif
            if (u == 0 && warp == TC_DEC_WARP0 && lane == 0) { tc_stamp(p.dbg, 3); tc_stamp(p.dbg, 4); }
            const uint32_t* wst = reinterpret_cast<const uint32_t*>(smem + s * L.w_bytes);
#ifdef EXL3B_TC_DEBUG
            // slots 48 + 4 g + j: SM clock before (low word) and after (high word) the wait of the group's unit j < 4
            if (dbg_row && du < 4) dbg_row[48 + 4 * g + du] = ((unsigned long long) t_out << 32) | t_in;
#endif
            // the unit's digit sums are read and added while k-half 0's batch is in flight
            const int* dsum = reinterpret_cast<const int*>(smem + L.off_b + s * L.b_bytes + I8_B_BYTES);
            auto digit_sums = [&]
            {
                if (c < p.m) t_lo += dsum[c];
                if (MR > 4 && c + 4 < p.m) t_hi += dsum[c + 4];
            };
#ifdef EXL3B_TC_DEBUG
            const uint32_t t_dsum = sm_clock_after((uint32_t) (t_lo + t_hi));
            if (att && du >= 1 && du <= 4)
            {
                uint32_t* a = att + 12 * (du - 1);
                a[4] = t_in; a[5] = t_out; a[6] = wait_info; a[7] = t_dsum;
            }
#endif
            i8_unit_mma<K, MR>(wst, desc0 + (uint64_t) ((s * L.b_bytes) >> 4), tl, lane, acc, clk, digit_sums);
            __syncwarp();
            if (lane == 0) mbar_arrive(bars.W_EMPTY(s));
            if (u == n_units - 1 && wq == 0 && lane == 0) tc_stamp(p.dbg, 10);
#ifdef EXL3B_TC_DEBUG
            if (att && du >= 1 && du <= 4)
            {
                uint32_t* a = att + 12 * (du - 1);
                a[8] = clk.t_loaded0; a[9] = clk.t_issue0; a[10] = clk.t_mma0; a[11] = 1u;
            }
            if (att && du < 4)
            {
                uint32_t* a = att + 12 * du;
                a[0] = clk.t_retired1; a[1] = clk.t_end; a[2] = sm_clock();
            }
            t_ho = 0;
            ++du;
#endif
        };
        // the group walks its own units only; `b` is the last unit of the current sub-segment (the epilogue's sub-segments:
        // strip ends and every I8_SUB_UNITS units), and every boundary before the group's next unit is handed off first
        auto sub_end = [&](int u0)
        {
            const int to_strip_end = KB - (ubeg + u0) % KB;
            const int seg_end = u0 + ((n_units - u0) < to_strip_end ? (n_units - u0) : to_strip_end) - 1;
            return seg_end < u0 + I8_SUB_UNITS - 1 ? seg_end : u0 + I8_SUB_UNITS - 1;
        };
        int b = sub_end(0);
        int s = g < S ? g : g - S, sph = 0;
        for (int u = g; ; u += 2)
        {
            while (b < u && b < n_units)
            {
                hand_off();
                b = b + 1 < n_units ? sub_end(b + 1) : n_units;
            }
#ifdef EXL3B_TC_DEBUG
            if (att && du >= 1 && du <= 4) att[12 * (du - 1) + 3] = t_ho;
#endif
            if (u >= n_units) break;
            unit(u, s, sph);
            s += 2; if (s >= S) { s -= S; sph ^= 1; }
        }
    }
    else if (warp >= TC_EPI_WARP0)
    {
        // =========================== epilogue ===========================
        pdl_wait();
        const int q = warp & 3;
        const int et = threadIdx.x - TC_EPI_WARP0 * 32;
        const int col = et;                              // column of the strip this thread finishes
        float* tile = reinterpret_cast<float*>(smem + L.off_tile);
        auto epi_bar = [] { asm volatile("bar.sync 1, 128;" ::: "memory"); };

        // ---- AR: which exchange slot does this launch use?  ----------------------------------------------------------------
        // The slot must alternate between consecutive row-parallel launches of the rank (a peer may run one launch ahead, see
        // emit_rows), also across replays of a CUDA graph, so it cannot be a host-chosen kernel argument: it is the parity of
        // a device-resident epoch.  Every CTA reads the epoch (stable: the previous launch has completed, pdl_wait above),
        // then takes a ticket; the CTA that takes the last ticket -- every CTA has read by then -- advances the epoch.
        [[maybe_unused]] long long ar_base = 0;           // word offset of (slot, source rank 0) inside a receive buffer
        if constexpr (AR)
        {
            if (et == 0)
            {
                // ordering: the epoch load must be performed before this CTA's ticket is visible (otherwise the last ticket
                // holder could already have advanced the epoch and this CTA would pick the other slot than its peers): acquire
                // load, acq_rel ticket; the advance is a release store after the ticket reset
                const unsigned int e = ld_acquire_gpu_u32(ar->state);
                const unsigned int ticket = atom_add_acq_rel_gpu_u32(ar->state + 1, 1u);
                if (ticket == gridDim.x - 1)
                {
                    st_relaxed_gpu_u32(ar->state + 1, 0u);
                    st_release_gpu_u32(ar->state, e + 1u);
                }
                *s_ar = e;
            }
            epi_bar();
            ar_base = (long long) (*s_ar % AR_SLOTS) * ar->world * ar->slot_elems;
        }

        auto emit_rows = [&](int strip)
        {
            epi_bar();
            if constexpr (!AR)
            {
                for (int r = q; r < p.m; r += 4)
                    output_row_128(tile + r * 128, Cout, (size_t) r * n_loc + strip * 128,
                                   svh ? svh + strip * 128 : nullptr, ROUTED ? routed_scale : p.out_scale, p.c_fp32 != 0, lane);
            }
            else
            {
                // Row-parallel output: y = sum over ranks of this rank's finished partial (own output Hadamard and svh applied,
                // fp32).  One warp per row and 128-column segment, four values per lane.  The exchange is the split-K protocol
                // stretched over NVLink: the receive buffers hold the sentinel outside a launch, each 32-bit word is its own
                // flag.  (1) store the partial into slot [rank] of every peer's buffer, (2) read slots [j] of the own buffer
                // until they are all there, (3) add in RANK order -- every rank computes bit-identical sums -- and (4) put the
                // sentinel back.  No fence, no flag, no second kernel; segments finish independently, so the transfer of one
                // overlaps the contraction of the others.
                // Why two alternating slots are enough: a peer can write launch L+2's data only after it completed launch
                // L+1, which needed this rank's launch-L+1 partials, which this rank sends only after pdl_wait in launch L+1,
                // i.e. after launch L (and its step 4) has completed.
                const int rank = ar->rank, world = ar->world;
                for (int r = q; r < p.m; r += 4)
                {
                    float v[4];
                    finish_row_128_f32(tile + r * 128, svh ? svh + strip * 128 : nullptr, ROUTED ? routed_scale : p.out_scale, lane, v);
                    const long long e0 = (long long) r * n_loc + strip * 128 + lane * 4;
                    uint4 mine = make_uint4(__float_as_uint(v[0]), __float_as_uint(v[1]), __float_as_uint(v[2]), __float_as_uint(v[3]));
                    if (mine.x == I8_SENTINEL) mine.x = 0x7fc00000u;            // a NaN stays a NaN
                    if (mine.y == I8_SENTINEL) mine.y = 0x7fc00000u;
                    if (mine.z == I8_SENTINEL) mine.z = 0x7fc00000u;
                    if (mine.w == I8_SENTINEL) mine.w = 0x7fc00000u;
                    for (int j = 1; j < world; ++j)
                    {
                        int pj = rank + j; if (pj >= world) pj -= world;           // staggered: not every rank hits rank 0 first
                        st_relaxed_sys_v4(ar->recv[pj] + ar_base + (long long) rank * ar->slot_elems + e0, mine);
                    }
                    uint4 x[AR_MAX_WORLD];
                    uint32_t have = 1u << rank;
                    const uint32_t all = (1u << world) - 1u;
                    uint32_t polls = 0;
                    unsigned long long t0 = 0;
                    const uint32_t* mybuf = ar->recv[rank] + ar_base + e0;
                    while (true)
                    {
                        #pragma unroll
                        for (int j = 0; j < AR_MAX_WORLD; ++j)
                        {
                            if (j < world && !((have >> j) & 1u))
                            {
                                x[j] = ld_relaxed_sys_v4(mybuf + (long long) j * ar->slot_elems);
                                if (x[j].x != I8_SENTINEL && x[j].y != I8_SENTINEL && x[j].z != I8_SENTINEL && x[j].w != I8_SENTINEL)
                                    have |= 1u << j;
                            }
                        }
                        if (__all_sync(0xffffffffu, have == all)) break;
                        poll_watchdog<255u, 20000000000ull>(polls, t0, "tensor-parallel exchange", strip, (int) have);
                    }
                    float s0 = 0.f, s1 = 0.f, s2 = 0.f, s3 = 0.f;
                    #pragma unroll
                    for (int j = 0; j < AR_MAX_WORLD; ++j)
                    {
                        if (j < world)
                        {
                            const uint4 xv = j == rank ? mine : x[j];
                            s0 += __uint_as_float(xv.x); s1 += __uint_as_float(xv.y); s2 += __uint_as_float(xv.z); s3 += __uint_as_float(xv.w);
                            if (j != rank)
                                st_relaxed_sys_v4(const_cast<uint32_t*>(mybuf) + (long long) j * ar->slot_elems,
                                                  make_uint4(I8_SENTINEL, I8_SENTINEL, I8_SENTINEL, I8_SENTINEL));
                        }
                    }
                    if (p.c_fp32)
                        *reinterpret_cast<float4*>((float*) Cout + e0) = make_float4(s0, s1, s2, s3);
                    else
                    {
                        const half2 a = __floats2half2_rn(s0, s1), b = __floats2half2_rn(s2, s3);
                        uint2 o; o.x = *reinterpret_cast<const uint32_t*>(&a); o.y = *reinterpret_cast<const uint32_t*>(&b);
                        *reinterpret_cast<uint2*>((half*) Cout + e0) = o;
                    }
                }
            }
            epi_bar();
        };

        int dbuf = 0, dphase = 0;
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

            float facc[MR];
            #pragma unroll
            for (int r = 0; r < MR; ++r) facc[r] = 0.f;
            for (int done = 0; done < seg; )
            {
                const int sub = (seg - done) < I8_SUB_UNITS ? (seg - done) : I8_SUB_UNITS;
                mbar_wait<32>(bars.D_FULL(dbuf), dphase);
                if (et == 0 && u + seg >= n_units) tc_stamp(p.dbg, 7);
                // the prologue result is needed here too: the first D_FULL orders it (the MMA warps only get operands after the
                // transform warps passed the prologue barrier)
                i8_drain<MR>(s_d, s_dt, dbuf, col, p.m, [&](int r) { return i8_over_qmax(__uint_as_float(s_absmax[r])); }, facc);
                __syncwarp();
                if (lane == 0) mbar_arrive(bars.D_EMPTY(dbuf));
                dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
                done += sub;
            }

            if (full)
            {
                #pragma unroll
                for (int r = 0; r < MR; ++r) if (r < p.m) tile[r * 128 + col] = facc[r];
                emit_rows(strip);
            }
            else if (cta != c_a)
            {
                // contributor: the exchange slots of this matrix's CTA group start at cta0
                i8_splitk_publish<MR>(parts, cta0 + cta, facc, p.m, col);
                if (et == 0 && u + seg >= n_units) tc_stamp(p.dbg, 11);
            }
            else
            {
                // reducer; its slots are re-armed for the launch that uses this exchange buffer next (8 launches from now)
                i8_splitk_reduce<MR>(parts, cta0, c_a, c_b, facc, p.m, col, tile);
                if (et == 0 && u + seg >= n_units) tc_stamp(p.dbg, 13);
                emit_rows(strip);
            }
            u += seg;
        }
        if (et == 0) tc_stamp(p.dbg, 8);
    }
}

}  // namespace exl3b
