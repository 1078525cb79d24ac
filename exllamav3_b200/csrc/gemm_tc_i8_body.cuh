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
//   * a CTA prologue (warps 2..19, redundantly per CTA) transforms the rows once into a shared-memory cache and finds the
//     per-row |xh| maximum; the two transform warps then write per-unit activation digits + digit sums
//   * split-K partial sums travel through a sentinel-armed exchange buffer: contributors store and leave, the CTA owning the
//     strip's first k-segment (it processes it last) adds them to its registers in fixed CTA order and re-arms the slots --
//     no fence, no ticket, one global round trip, bit-reproducible
//   * multi-matrix launches (dense exl3_mgemm: the model's k+v and gate+up calls): the grid is cut into one CTA group per
//     matrix; the pointer tables stay in device memory, each CTA patches the weight tensor map's address on the device
//   * instantiated for MR = 4 and MR = 8 activation rows (digit tile with one / two row groups); api.cu auto-selects m <= 4
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
template <int K, int MR, bool AR, bool ROUTED = false>
__device__ __forceinline__ void gemm_tc_i8_body(const TcParams& p, const CUtensorMap* tmap_w, const ArArgs* ar,
                                                const RouteArgs* route = nullptr)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    constexpr int I8_B_BYTES = i8_b_bytes(MR);
    const TcSmemLayout L = i8_smem_layout(K, MR, p.stages, 0);          // offsets only; the cache starts at L.total
    int32_t* const s_d = reinterpret_cast<int32_t*>(smem + L.off_d);     // accumulator hand-off, [dbuf][group][128][2 MR]
    int* const s_dt = reinterpret_cast<int*>(smem + L.off_d + i8_d_bytes(MR) - 2 * 2 * 8 * 4);   // digit sums, [dbuf][group][8]
    const bool cached = p.b_load_bytes > 0;                            // host: cache_bytes (0 = recompute per unit)
    half* xh_cache = reinterpret_cast<half*>(smem + L.total);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
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

    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + L.off_bars);
    const uint32_t bar0 = smem_u32(bars);
    auto W_FULL = [&](int s) { return bar0 + 8u * s; };
    auto W_EMPTY = [&](int s) { return bar0 + 8u * (S + s); };
    auto X_FULL = [&](int s) { return bar0 + 8u * (2 * S + s); };
    auto D_FULL = [&](int s) { return bar0 + 8u * (3 * S + 8 + s); };
    auto D_EMPTY = [&](int s) { return bar0 + 8u * (3 * S + 10 + s); };
    uint32_t* misc = reinterpret_cast<uint32_t*>(smem + L.off_bars + 8 * (3 * TC_MAX_STAGES + 16));
    unsigned int* s_absmax = reinterpret_cast<unsigned int*>(misc + 4);           // [MR] float bits, >= 0
    [[maybe_unused]] volatile unsigned int* s_ar = reinterpret_cast<volatile unsigned int*>(misc + 28);   // AR: epoch of this launch

#ifdef EXL3B_TC_DEBUG
    const int KNOB = p.knob_;
#else
    constexpr int KNOB = 0;
#endif
    auto stamp = [&](int slot)
    {
#ifdef EXL3B_TC_DEBUG
        if (p.dbg) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory"); p.dbg[blockIdx.x * 64 + slot] = t; }
#else
        (void) slot;
#endif
    };
#ifdef EXL3B_TC_DEBUG
    // how often did a role find its barrier not yet complete (= it had to wait)?  slots 56.. of the CTA's debug row
    int wf_a = 0, wf_b = 0, wf_c = 0;
#define I8_WAITCNT(cnt, bar, par) do { if (!mbar_test_wait((bar), (par))) ++(cnt); } while (0)
#else
#define I8_WAITCNT(cnt, bar, par) do { } while (0)
#endif
    if (threadIdx.x == 0) stamp(0);
    pdl_launch_dependents();

    if (warp == 0)
    {
        // one barrier per lane and round instead of ~60 serial initialisations by one thread
        // W_EMPTY: the eight decode warps of the unit's group, after their MMAs have read the weights' digit tile
        for (int s = lane; s < S; s += 32) { mbar_init(W_FULL(s), 1); mbar_init(X_FULL(s), 1); mbar_init(W_EMPTY(s), TC_DEC_WARPS / I8_DEC_GROUPS); }
        if (lane < 2) { mbar_init(D_FULL(lane), TC_DEC_WARPS); mbar_init(D_EMPTY(lane), 4); }
        else if (lane < 2 + MR) s_absmax[lane - 2] = 0u;
        fence_barrier_init();
    }
    __syncthreads();
    if (threadIdx.x == 0) stamp(1);

    const int KB = p.k / 128;
    const int strips = n_loc / 128;
    const long long U = (long long) KB * strips;
    const long long ubeg = unit_begin(U, G, cta), uend = unit_begin(U, G, cta + 1);
    const int n_units = (int) (uend - ubeg);

    // fp16 transformed activation of (row r, k-block kb), 4 values per lane, exactly as the reference's A_had
    auto xh_finish = [&](uint2 raw, uint2 scb, float (&v)[4])
    {
        half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
        if (suh)
        {
            a = __hmul2(a, *reinterpret_cast<const half2*>(&scb.x));
            b = __hmul2(b, *reinterpret_cast<const half2*>(&scb.y));
            float v0 = __low2float(a), v1 = __high2float(a), v2 = __low2float(b), v3 = __high2float(b);
            had128_warp(v0, v1, v2, v3, lane);
            a = __floats2half2_rn(v0 * R_SCALE, v1 * R_SCALE);
            b = __floats2half2_rn(v2 * R_SCALE, v3 * R_SCALE);
        }
        v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
    };
    auto xh_block = [&](int r, int kb, float (&v)[4])
    {
        const uint2 raw = *reinterpret_cast<const uint2*>(A_raw + (size_t) r * p.k + kb * 128 + lane * 4);
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

    // ---- prologue: per-row max |xh| over the whole row (warps 2..19), overlapped with the first weight loads ----
    if (warp == 0)
    {
        // producer starts streaming weights immediately (below); it does not take part in the prologue
    }
    if (warp >= TC_XF_WARP0 && warp < TC_EPI_WARP0)
    {
        const int nw = TC_EPI_WARP0 - TC_XF_WARP0;       // 18 warps
        if constexpr (MR <= 4)
        {
            // Two tasks (row, k-block) per step with both loads in flight together, and the suh blocks of the first step fetched
            // BEFORE griddepcontrol.wait: suh is a weight (it does not depend on the previous kernel) and usually comes from
            // DRAM, the activations come from L2 -- one DRAM latency and one L2 latency less on every launch's critical path.
            const int T = p.m * KB, w0 = warp - TC_XF_WARP0;
            uint2 sc0 = make_uint2(0, 0), sc1 = make_uint2(0, 0);
            if (suh)
            {
                if (w0 < T) sc0 = *reinterpret_cast<const uint2*>(suh + (w0 % KB) * 128 + lane * 4);
                if (w0 + nw < T) sc1 = *reinterpret_cast<const uint2*>(suh + ((w0 + nw) % KB) * 128 + lane * 4);
            }
            if constexpr (!ROUTED) pdl_wait();            // A is produced by the previous kernel (ROUTED waited at the top)
            for (int task = w0; task < T; task += 2 * nw)
            {
                const int ta = task, tb = task + nw;
                const int ra = ta / KB, ka = ta % KB, rb = tb / KB, kb_ = tb % KB;
                if (task != w0 && suh)
                {
                    sc0 = *reinterpret_cast<const uint2*>(suh + ka * 128 + lane * 4);
                    if (tb < T) sc1 = *reinterpret_cast<const uint2*>(suh + kb_ * 128 + lane * 4);
                }
                const uint2 raw0 = *reinterpret_cast<const uint2*>(A_raw + (size_t) ra * p.k + ka * 128 + lane * 4);
                uint2 raw1 = make_uint2(0, 0);
                if (tb < T) raw1 = *reinterpret_cast<const uint2*>(A_raw + (size_t) rb * p.k + kb_ * 128 + lane * 4);
                float v[4];
                xh_finish(raw0, sc0, v);
                xh_publish(ra, ka, v);
                if (tb < T)
                {
                    xh_finish(raw1, sc1, v);
                    xh_publish(rb, kb_, v);
                }
            }
        }
        else
        {
            pdl_wait();                                   // A is produced by the previous kernel
            // up to 8 rows: one k-block of ALL rows per step, the rows' loads in flight together (one L2 round trip per step
            // instead of one per row)
            for (int kb = warp - TC_XF_WARP0; kb < KB; kb += nw)
            {
                uint2 scb = make_uint2(0, 0), raw[MR];
                if (suh) scb = *reinterpret_cast<const uint2*>(suh + kb * 128 + lane * 4);
                #pragma unroll
                for (int r = 0; r < MR; ++r)
                {
                    raw[r] = make_uint2(0, 0);
                    if (r < p.m) raw[r] = *reinterpret_cast<const uint2*>(A_raw + (size_t) r * p.k + kb * 128 + lane * 4);
                }
                #pragma unroll
                for (int r = 0; r < MR; ++r)
                {
                    if (r < p.m)
                    {
                        float v[4];
                        xh_finish(raw[r], scb, v);
                        xh_publish(r, kb, v);
                    }
                }
            }
        }
        asm volatile("bar.sync 2, %0;" :: "n"((TC_EPI_WARP0 - TC_XF_WARP0) * 32) : "memory");
        if (warp == TC_DEC_WARP0 && lane == 0) stamp(2);
    }

    if (warp == 0)
    {
        // =========================== producer ===========================
        const void* tm = tmap_w;
        const size_t w_pitch = (size_t) (n_loc / 16) * 32 * K;               // bytes per 16-row tile row of the packed tensor
        if (multi)
        {
            // per-CTA tensor map: the template (dims / strides / box of this shape) with matrix `mat`'s address -- and, in a fan-out
            // launch, its own width (innermost extent in 8-byte elements, row pitch in bytes)
            uint8_t* stm = smem + ((L.off_bars + 640 + 127) & ~127);
            reinterpret_cast<uint32_t*>(stm)[lane] = reinterpret_cast<const uint32_t*>(tmap_w)[lane];
            __syncwarp();
            void* gtm = p.tmap_slots + (size_t) blockIdx.x * 128;
            if (p.rag) tmap_patch_address_width(smem_u32(stm), gtm, p.B_ptrs[mat], (uint32_t) (w_pitch / 8), (uint64_t) w_pitch, lane);
            else tmap_patch_address(smem_u32(stm), gtm, p.B_ptrs[mat], lane);
            tm = gtm;
        }
        else if (elect_one()) prefetch_tmap(tmap_w);
        const uint64_t pol_w = policy_evict_first();
        const uint32_t w_smem0 = smem_u32(smem);
        int strip = (int) (ubeg / KB), kb = (int) (ubeg % KB);
        int s = 0, ph = 0;
        for (int u = 0; u < n_units; ++u)
        {
            if (u >= S) { I8_WAITCNT(wf_a, W_EMPTY(s), ph ^ 1); mbar_wait<64>(W_EMPTY(s), ph ^ 1); }
            if (elect_one())
            {
                mbar_arrive_expect_tx(W_FULL(s), (uint32_t) L.w_bytes);
                tma_load_2d(w_smem0 + s * L.w_bytes, tm, strip * (32 * K), kb * 8, W_FULL(s), pol_w);
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
            inv_scale[r] = mx > 0.f ? (float) I8_QMAX / mx : 0.f;
        }
        int kb = (int) ((ubeg + xw) % KB);
        int s = xw % S, ph = 0;
        const int kstep = 2 % KB;
        for (int u = xw; u < n_units; u += 2)
        {
            I8_WAITCNT(wf_a, W_EMPTY(s), ph ^ 1);
            mbar_wait<64>(W_EMPTY(s), ph ^ 1);
            uint8_t* dst = smem + L.off_b + s * L.b_bytes;
            int qsum[MR];
            #pragma unroll
            for (int r = 0; r < MR; ++r)
            {
                qsum[r] = 0;
                if (r < p.m && !(KNOB & 8))
                {
                    float v[4];
                    if (cached)
                    {
                        const uint2 raw = *reinterpret_cast<const uint2*>(xh_cache + (size_t) r * p.k + kb * 128 + lane * 4);
                        const half2 a = *reinterpret_cast<const half2*>(&raw.x), b = *reinterpret_cast<const half2*>(&raw.y);
                        v[0] = __low2float(a); v[1] = __high2float(a); v[2] = __low2float(b); v[3] = __high2float(b);
                    }
                    else xh_block(r, kb, v);
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
            if (lane < p.m)
            {
                int mine = 0;
                #pragma unroll
                for (int r = 0; r < MR; ++r) if (lane == r) mine = qsum[r];
                *reinterpret_cast<int*>(dst + I8_B_BYTES + 4 * lane) = mine;
            }
            fence_proxy_async_smem();
            __syncwarp();
            if (lane == 0) mbar_arrive(X_FULL(s));
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
        // Warpgroup (g, nh): units u = g (mod 2), output columns 64 nh .. 64 nh + 63 of the strip.  Both groups walk the same
        // sub-segment boundaries and hand over (possibly zero) accumulators at every boundary; the epilogue adds the two.
        const int wq = warp & 3, wgi = (warp - TC_DEC_WARP0) >> 2;
        const int g = wgi & 1, nh = wgi >> 1;
        const int tl = 4 * nh + wq;                      // tile column of the strip owned by this warp
        const int chunk = lane >> 2, c = lane & 3;
        const uint64_t desc0 = smem_desc(smem_u32(smem + L.off_b), 128, 4096, 0);
        uint32_t acc[MR];
        #pragma unroll
        for (int i = 0; i < MR; ++i) acc[i] = 0u;
        int t_lo = 0, t_hi = 0;                          // digit sums of activation rows c and c + 4 over the group's units
        int s = 0, sph = 0, dbuf = 0, dphase = 0, seg_left = 0, sub_left = 0;
        int kb = (int) (ubeg % KB);
        for (int u = 0; u < n_units; ++u)
        {
            if (seg_left == 0)
            {
                const int to_strip_end = KB - kb;
                seg_left = (n_units - u) < to_strip_end ? (n_units - u) : to_strip_end;
            }
            if (sub_left == 0) sub_left = seg_left < I8_SUB_UNITS ? seg_left : I8_SUB_UNITS;
            if ((u & 1) == g)
            {
                mbar_wait<32>(W_FULL(s), sph);
                if (u == 0 && warp == TC_DEC_WARP0 && lane == 0) stamp(3);
                const uint32_t* wst = reinterpret_cast<const uint32_t*>(smem + s * L.w_bytes);
                uint32_t w[2][K + 1];
                #pragma unroll
                for (int r = 0; r < 2; ++r) load_chunk<K>(wst + ((4 * r + c) * 8 + tl) * (8 * K), chunk, w[r]);
                mbar_wait(X_FULL(s), sph);                                   // the unit's activation digits
                const int* dsum = reinterpret_cast<const int*>(smem + L.off_b + s * L.b_bytes + I8_B_BYTES);
                if (c < p.m) t_lo += dsum[c];
                if (MR > 4 && c + 4 < p.m) t_hi += dsum[c + 4];
                const uint64_t desc_s = desc0 + (uint64_t) ((s * L.b_bytes) >> 4);
                #pragma unroll
                for (int r = 0; r < 2; ++r)
                {
                    uint32_t o0[16], o1[16];
                    decode16_i8<K, 0>(w[r], o0);
                    decode16_i8<K, 1>(w[r], o1);
                    #pragma unroll
                    for (int i = 0; i < MR; ++i) reg_fence(acc[i]);
                    wgmma_fence();
                    #pragma unroll
                    for (int j = 0; j < 8; ++j)
                        wgmma_u8s8<MR>(acc, o0[2 * j], o1[2 * j], o0[2 * j + 1], o1[2 * j + 1], desc_s + (uint64_t) (16 * (8 * r + j)));
                    wgmma_commit();
                    wgmma_wait<0>();
                    #pragma unroll
                    for (int i = 0; i < 16; ++i) { reg_fence(o0[i]); reg_fence(o1[i]); }
                    #pragma unroll
                    for (int i = 0; i < MR; ++i) reg_fence(acc[i]);
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(W_EMPTY(s));
                if (u == n_units - 1 && wq == 0 && lane == 0) stamp(10);
            }
            --seg_left; --sub_left;
            if (sub_left == 0)
            {
                // hand the sub-segment's accumulators to the epilogue
                mbar_wait(D_EMPTY(dbuf), dphase ^ 1);
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
                __syncwarp();
                if (lane == 0) mbar_arrive(D_FULL(dbuf));
                dbuf ^= 1; if (dbuf == 0) dphase ^= 1;
            }
            if (++kb == KB) kb = 0;
            if (++s == S) { s = 0; sph ^= 1; }
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
        const int part_stride = MR * 128;

        // the prologue result is needed here too: wait for it through the first D_FULL (the MMA warp only gets
        // operands after the transform warps passed the prologue barrier), then read the maxima
        const float k_inv = __half2float(__ushort_as_half((unsigned short) 0x1eee));
        const float k_bias = __half2float(__ushort_as_half((unsigned short) 0xc931));
        const float c1 = 1534.0f * k_inv + k_bias;        // (1024 + 510) k_inv + k_bias: residue of the fp16-rounded bias

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
                        if ((++polls & 255u) == 0)
                        {
                            unsigned long long t;
                            asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                            if (t0 == 0) t0 = t;
                            else if (t - t0 > 20000000000ull)
                            {
                                if (lane == 0) printf("exl3b: tensor-parallel exchange timeout (rank %d block %d strip %d have %x)\n", rank, blockIdx.x, strip, have);
                                __trap();
                            }
                        }
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
            const long long g = ubeg + u;
            const int strip = (int) (g / KB), kb = (int) (g % KB);
            const int to_strip_end = KB - kb;
            const int seg = (n_units - u) < to_strip_end ? (n_units - u) : to_strip_end;
            const long long gs = (long long) strip * KB;
            const int c_a = cta_of_unit(U, G, gs), c_b = cta_of_unit(U, G, gs + KB - 1);
            const int n_contrib = c_b - c_a + 1;
            const bool full = n_contrib == 1;

            float facc[MR];
            #pragma unroll
            for (int r = 0; r < MR; ++r) facc[r] = 0.f;
            for (int done = 0; done < seg; )
            {
                const int sub = (seg - done) < I8_SUB_UNITS ? (seg - done) : I8_SUB_UNITS;
                mbar_wait<32>(D_FULL(dbuf), dphase);
                if (et == 0 && u + seg >= n_units) stamp(7);
                const int32_t* d0 = s_d + (size_t) ((dbuf * 2 + 0) * 128 + col) * (2 * MR);
                const int32_t* d1 = s_d + (size_t) ((dbuf * 2 + 1) * 128 + col) * (2 * MR);
                #pragma unroll
                for (int r = 0; r < MR; ++r)
                {
                    if (r < p.m)
                    {
                        const int T = s_dt[(dbuf * 2 + 0) * 8 + r] + s_dt[(dbuf * 2 + 1) * 8 + r];
                        // sum_k q_k (bytesum_kn - 510), exact in 64-bit (the two groups' int32 partials add without loss)
                        const long long sp = i8_centred_sum(d0[2 * r] + d1[2 * r], d0[2 * r + 1] + d1[2 * r + 1], T);
                        const float mx = __uint_as_float(s_absmax[r]);
                        const float scale = mx / (float) I8_QMAX;
                        facc[r] += i8_assemble(sp, T, scale, k_inv, c1);
                    }
                }
                __syncwarp();
                if (lane == 0) mbar_arrive(D_EMPTY(dbuf));
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
                // Contributor: publish the partial sums and move on.  The data is its own flag: the exchange buffer holds the
                // sentinel everywhere outside a launch, a 32-bit store is single-copy atomic, so no fence, counter or ticket.
                #pragma unroll
                for (int r = 0; r < MR; ++r)
                    if (r < p.m)
                    {
                        uint32_t bits = __float_as_uint(facc[r]);
                        if (bits == I8_SENTINEL) bits = 0x7fc00000u;                 // a NaN stays a NaN
                        st_relaxed_gpu_u32(reinterpret_cast<uint32_t*>(parts + (size_t) (cta0 + cta) * part_stride + r * 128 + col), bits);
                    }
                if (et == 0 && u + seg >= n_units) stamp(11);
            }
            else
            {
                // The CTA that owns the strip's FIRST k-segment works on it LAST (segments are processed in unit order), so it is the
                // natural reducer: own sums from registers, then the others' in fixed CTA order (bit-reproducible).  One global
                // round trip in the common case -- the old protocol needed three (fence + ticket, then the loads).
                #pragma unroll
                for (int r = 0; r < MR; ++r)
                {
                    if (r < p.m)
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
                                        v[j] = ld_relaxed_gpu_u32(reinterpret_cast<const uint32_t*>(parts + (size_t) (cta0 + cc) * part_stride + r * 128 + col));
                                        ok = ok && v[j] != I8_SENTINEL;
                                    }
                                }
                                if (!ok && (++polls & 255u) == 0)
                                {
                                    unsigned long long t;
                                    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
                                    if (t0 == 0) t0 = t;
                                    else if (t - t0 > 4000000000ull) { printf("exl3b: split-K exchange timeout (block %d strip %d)\n", blockIdx.x, strip); __trap(); }
                                }
                            } while (!ok);
                            #pragma unroll
                            for (int j = 0; j < 8; ++j)
                            {
                                const int cc = c + j;
                                if (cc <= c_b)
                                {
                                    a += __uint_as_float(v[j]);
                                    // re-arm the slot for the launch that uses this exchange buffer next (8 launches from now)
                                    st_relaxed_gpu_u32(reinterpret_cast<uint32_t*>(parts + (size_t) (cta0 + cc) * part_stride + r * 128 + col), I8_SENTINEL);
                                }
                            }
                            c += 8;
                        }
                        tile[r * 128 + col] = a;
                    }
                }
                if (et == 0 && u + seg >= n_units) stamp(13);
                emit_rows(strip);
            }
            u += seg;
        }
        if (et == 0) stamp(8);
    }
}

}  // namespace exl3b
