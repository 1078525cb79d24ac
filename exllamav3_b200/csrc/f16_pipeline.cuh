// The unit pipeline of the exact fp16 path: the data layout and the per-unit work that the tag-200 decode-GEMM (gemm_tc.cu)
// and the exl3_moe grouped GEMM (moe_tc.cu) share -- the shared-memory ring and its stage count, the wgmma descriptor of the
// activation tile, one unit's weight words and the accumulators' scatter into the fp32 tile.  The kernels keep their own
// producers, barrier waits and epilogues, and each writes one unit's decode + wgmma itself: the lane (chunk, c) decodes its
// weight words (f16_load_unit) straight into wgmma A fragments (rows chunk / chunk + 8, K pairs c / c + 4) and issues
// 4 x nchunks wgmma.m64n16k16 per k-half against the activation tile, whose K order (xt_tile_offset) is permuted to match.
// That block stays in the kernels because ptxas orders tag 200's 3inst / mcg decode differently when it comes through a
// function; a build with it shared ran those kernels 4-8 % slower on an H100 (80 GB HBM3, 700 W).
#pragma once
#include "tc_common.cuh"

namespace exl3b {

using namespace ptx;

constexpr int F16_MAX_ROWS = 128;                  // activation rows per pass: F16_MAX_ROWS / 16 accumulator chunks of 8 registers
constexpr int F16_THREADS = 384;                   // warp 0 producer, warps 4-11 decode + MMA + epilogue (two warpgroups)
constexpr int F16_CONS_WARP0 = 4, F16_CONS_WARPS = 8;

// smem: weight ring (2048 K bytes per unit), activation ring (b_bytes = NT * 256 per unit: NT / 8 row groups of 2048 bytes),
// fp32 tile [NT][128], barriers
__host__ __device__ inline TcSmemLayout f16_smem_layout(int K, int b_bytes, int stages, int NT)
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

// ring depth: as many stages as fit 200 KiB beside the tile, 2..TC_MAX_STAGES
__host__ __device__ inline int f16_stages(int K, int NT)
{
    const int budget = 200 * 1024 - NT * 128 * 4;
    int stages = budget / (2048 * K + NT * 256);
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    return stages < 2 ? 2 : stages;
}

#ifdef __CUDACC__

// wgmma descriptor of an activation tile in the xt_tile_offset layout (tc_common.cuh): K-chunks 128 B, row groups 2048 B apart
__device__ __forceinline__ uint64_t f16_tile_desc(const uint8_t* tile) { return smem_desc(smem_u32(tile), 128, 2048, 0); }

// Weight words of one unit (128 k x 128 n) for lane (chunk, c) = (lane / 4, lane % 4) of the warp that owns tile column `tl`
// of the strip: k-tiles c (w[0]) and 4 + c (w[1]) of the weight stage `wst`.
template <int K>
__device__ __forceinline__ void f16_load_unit(const uint32_t* wst, int tl, int chunk, int c, uint32_t (&w)[2][K + 1])
{
    #pragma unroll
    for (int r = 0; r < 2; ++r) load_chunk<K>(wst + ((4 * r + c) * 8 + tl) * (8 * K), chunk, w[r]);
}

__device__ __forceinline__ void f16_zero(float (&acc)[F16_MAX_ROWS / 16][8])
{
    #pragma unroll
    for (int ii = 0; ii < F16_MAX_ROWS / 16; ++ii)
        #pragma unroll
        for (int e = 0; e < 8; ++e) acc[ii][e] = 0.f;
}

// accumulators -> tile[row][column] (fp32, [NT][128]) for the first 16 nchunks rows: fragment (row 16 ii + 2 c + e (+8),
// column 16 tl + chunk (+8))
__device__ __forceinline__ void f16_store_tile(float* tile, const float (&acc)[F16_MAX_ROWS / 16][8], int tl, int chunk, int c,
                                               int nchunks)
{
    const int n0 = 16 * tl + chunk;
    #pragma unroll
    for (int ii = 0; ii < F16_MAX_ROWS / 16; ++ii)
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
    }
}

#endif  // __CUDACC__

}  // namespace exl3b
