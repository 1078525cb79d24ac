// had_r_128, reconstruct, reconstruct_had -- the memory-bound helpers of the EXL3 path.
//
// Reference behaviour restated (not copied): exllamav3_ext/quant/hadamard.cu:88-173 + hadamard_inner.cuh:93-277,
// exllamav3_ext/quant/reconstruct.cu:11-144 (plain), :159-373 (fused both-side Hadamard).
#include "common.cuh"
#include "decode.cuh"

namespace exl3b {

// ==================================================================================================================
// had_r_128: one warp per (row, 128-column block); 4 warps per CTA.
// ==================================================================================================================

template <bool FP32, int SCALE_MODE /*0 none, 1 pre, 2 post*/>
__global__ void __launch_bounds__(128)
had_r_128_kernel(const void* __restrict__ in, void* __restrict__ out, const half* __restrict__ scale,
                 float r_scale, int rows, int blocks_per_row)
{
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    int lane = threadIdx.x & 31;
    int total = rows * blocks_per_row;
    if (warp >= total) return;
    int blk = warp % blocks_per_row;
    size_t off = (size_t) warp * 128 + lane * 4;

    float sc0 = 1.f, sc1 = 1.f, sc2 = 1.f, sc3 = 1.f;
    uint2 scb = make_uint2(0, 0);
    if constexpr (SCALE_MODE != 0)
    {
        scb = *reinterpret_cast<const uint2*>(scale + blk * 128 + lane * 4);
        const half2 a = *reinterpret_cast<const half2*>(&scb.x), b = *reinterpret_cast<const half2*>(&scb.y);
        sc0 = __low2float(a); sc1 = __high2float(a); sc2 = __low2float(b); sc3 = __high2float(b);
    }

    float v0, v1, v2, v3;
    bool pre_done = false;
    if constexpr (FP32)
    {
        float4 v = *reinterpret_cast<const float4*>((const float*) in + off);
        v0 = v.x; v1 = v.y; v2 = v.z; v3 = v.w;
        if constexpr (SCALE_MODE == 1)
        {
            // Explicitly the contraction the reference binary performs for this (cold) variant, so results are
            // bit-identical to it and independent of compiler mood: t = x1*a1; s = fma(x0,a0,t); d = fma(x0,a0,-t).
            float t1 = __fmul_rn(v1, sc1), t3 = __fmul_rn(v3, sc3);
            float s0 = __fmaf_rn(v0, sc0, t1), d0 = __fmaf_rn(v0, sc0, -t1);
            float s1 = __fmaf_rn(v2, sc2, t3), d1 = __fmaf_rn(v2, sc2, -t3);
            v0 = __fadd_rn(s0, s1); v1 = __fadd_rn(d0, d1); v2 = __fsub_rn(s0, s1); v3 = __fsub_rn(d0, d1);
            had128_warp_tail(v0, v1, v2, v3, lane);
            pre_done = true;
        }
    }
    else
    {
        uint2 raw = *reinterpret_cast<const uint2*>((const half*) in + off);
        half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
        if constexpr (SCALE_MODE == 1)
        {
            a = __hmul2(a, *reinterpret_cast<const half2*>(&scb.x));     // fp16 product, as the reference
            b = __hmul2(b, *reinterpret_cast<const half2*>(&scb.y));
        }
        v0 = __low2float(a); v1 = __high2float(a); v2 = __low2float(b); v3 = __high2float(b);
    }

    if (!pre_done) had128_warp(v0, v1, v2, v3, lane);
    v0 *= r_scale; v1 *= r_scale; v2 *= r_scale; v3 *= r_scale;

    if constexpr (FP32)
    {
        if constexpr (SCALE_MODE == 2) { v0 *= sc0; v1 *= sc1; v2 *= sc2; v3 *= sc3; }
        *reinterpret_cast<float4*>((float*) out + off) = make_float4(v0, v1, v2, v3);
    }
    else
    {
        half2 a = __floats2half2_rn(v0, v1), b = __floats2half2_rn(v2, v3);
        if constexpr (SCALE_MODE == 2)
        {
            a = __hmul2(a, *reinterpret_cast<const half2*>(&scb.x));
            b = __hmul2(b, *reinterpret_cast<const half2*>(&scb.y));
        }
        uint2 o;
        o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
        *reinterpret_cast<uint2*>((half*) out + off) = o;
    }
}

int launch_had_r_128(cudaStream_t stream, const void* in, void* out, const half* pre, const half* post,
                     float scale, int rows, int cols, bool fp32)
{
    int blocks_per_row = cols / 128;
    long total_warps = (long) rows * blocks_per_row;
    if (total_warps == 0) return 0;
    int grid = (int) ((total_warps + 3) / 4);
    float r_scale = scale * R_SCALE;
    int mode = pre ? 1 : (post ? 2 : 0);
    const half* sc = pre ? pre : post;
#define L(FP, MD) had_r_128_kernel<FP, MD><<<grid, 128, 0, stream>>>(in, out, sc, r_scale, rows, blocks_per_row)
    if (fp32) { if (mode == 0) L(true, 0); else if (mode == 1) L(true, 1); else L(true, 2); }
    else      { if (mode == 0) L(false, 0); else if (mode == 1) L(false, 1); else L(false, 2); }
#undef L
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

// ==================================================================================================================
// reconstruct: CTA = 128 threads = one 16(k) x 128(n) strip.  Thread decodes one column (16 k-values), the strip is
// transposed through shared memory and written as 16 rows of 256 contiguous bytes.
// ==================================================================================================================

template <int K, int cb>
__global__ void __launch_bounds__(128)
reconstruct_kernel(half* __restrict__ out, const uint32_t* __restrict__ packed, int n_out, int packed_tiles_n,
                   int tile_n_offset)
{
    __shared__ __align__(16) half tile[16][128 + 8];
    const int q = threadIdx.x >> 5, i = threadIdx.x & 31;
    const int kt = blockIdx.y, strip = blockIdx.x;
    const int tl = strip_tile(q, i);
    const uint32_t* tp = packed + ((size_t) kt * packed_tiles_n + tile_n_offset + strip * 8 + tl) * (8 * K);

    uint32_t w[K + 1], o[8];
    load_chunk<K>(tp, i & 7, w);
    if (q & 1) decode16<K, cb, 1>(w, o); else decode16<K, cb, 0>(w, o);

    const int col = strip_col(q, i);
    #pragma unroll
    for (int j = 0; j < 8; ++j)
    {
        tile[2 * j][col]     = __ushort_as_half((unsigned short) (o[j] & 0xffff));
        tile[2 * j + 1][col] = __ushort_as_half((unsigned short) (o[j] >> 16));
    }
    __syncthreads();
    // 16 rows x 256 B: thread t writes 16 B chunks (t, t+128)
    #pragma unroll
    for (int r = 0; r < 2; ++r)
    {
        int idx = threadIdx.x + r * 128;
        int row = idx >> 4, ch = idx & 15;
        uint4 v = *reinterpret_cast<const uint4*>(&tile[row][ch * 8]);
        *reinterpret_cast<uint4*>(out + ((size_t) kt * 16 + row) * n_out + strip * 128 + ch * 8) = v;
    }
}

template <int K, int cb>
static void reconstruct_launch(cudaStream_t stream, half* out, const uint16_t* packed, int k, int n_out,
                               int packed_tiles_n, int tile_n_offset)
{
    dim3 grid(n_out / 128, k / 16);
    reconstruct_kernel<K, cb><<<grid, 128, 0, stream>>>(out, (const uint32_t*) packed, n_out, packed_tiles_n,
                                                        tile_n_offset);
}


int launch_reconstruct(cudaStream_t stream, half* unpacked, const uint16_t* packed, int k, int n_out,
                       int packed_tiles_n, int K, int cb, int64_t n_offset)
{
    if (k == 0 || n_out == 0) return 0;
    EXL3B_DISPATCH_K_CB(reconstruct_launch, K, cb, stream, unpacked, packed, k, n_out, packed_tiles_n,
                        (int) (n_offset / 16));
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

// ==================================================================================================================
// reconstruct_had: CTA = 128 threads = one 128 x 128 block.  Each thread decodes ALL 128 k-values of its column into
// registers, runs the k-side (left) 128-point Hadamard entirely in registers (fp32), applies suh, and parks the
// column in shared memory (fp16, like the reference's intermediate tile).  The n-side (right) Hadamard then runs one
// row per warp with shuffles, fused with svh and the coalesced 256-byte row store.
// ==================================================================================================================

template <int N>
__device__ __forceinline__ void fwht_regs(float (&v)[N])
{
    #pragma unroll
    for (int w = 1; w < N; w <<= 1)
    {
        #pragma unroll
        for (int b = 0; b < N; b += 2 * w)
        {
            #pragma unroll
            for (int j = 0; j < w; ++j)
            {
                float a = v[b + j], c = v[b + w + j];
                v[b + j] = a + c;
                v[b + w + j] = a - c;
            }
        }
    }
}

template <int K, int cb>
__global__ void __launch_bounds__(128)
reconstruct_had_kernel(half* __restrict__ out, const uint32_t* __restrict__ packed, const half* __restrict__ suh,
                       const half* __restrict__ svh, int n_out, int packed_tiles_n, int tile_n_offset)
{
    __shared__ __align__(16) half tile[128][128 + 8];
    const int q = threadIdx.x >> 5, i = threadIdx.x & 31;
    const int kb = blockIdx.y, nb = blockIdx.x;
    const int tl = strip_tile(q, i);
    const int col = strip_col(q, i);

    float v[128];
    #pragma unroll
    for (int t = 0; t < 8; ++t)
    {
        const uint32_t* tp = packed + ((size_t) (kb * 8 + t) * packed_tiles_n + tile_n_offset + nb * 8 + tl) * (8 * K);
        uint32_t w[K + 1], o[8];
        load_chunk<K>(tp, i & 7, w);
        if (q & 1) decode16<K, cb, 1>(w, o); else decode16<K, cb, 0>(w, o);
        #pragma unroll
        for (int j = 0; j < 8; ++j)
        {
            half2 h = *reinterpret_cast<half2*>(&o[j]);
            v[t * 16 + 2 * j] = __low2float(h);
            v[t * 16 + 2 * j + 1] = __high2float(h);
        }
    }
    fwht_regs<128>(v);
    #pragma unroll
    for (int r = 0; r < 128; ++r)
    {
        // left transform scaled and rounded to fp16 (the reference keeps an fp16 tile between the passes)
        tile[r][col] = __float2half_rn(v[r] * R_SCALE);
    }
    __syncthreads();

    const uint2 svb = *reinterpret_cast<const uint2*>(svh + nb * 128 + i * 4);
    for (int r = q; r < 128; r += 4)
    {
        uint2 raw = *reinterpret_cast<const uint2*>(&tile[r][i * 4]);
        half2 a = *reinterpret_cast<half2*>(&raw.x), b = *reinterpret_cast<half2*>(&raw.y);
        float v0 = __low2float(a), v1 = __high2float(a), v2 = __low2float(b), v3 = __high2float(b);
        had128_warp(v0, v1, v2, v3, i);
        // scale order as the reference's fused kernel (reconstruct.cu:300-304): (h * suh[row]) * svh[col], fp16
        const half2 su2 = __half2half2(suh[kb * 128 + r]);
        a = __hmul2(__hmul2(__floats2half2_rn(v0 * R_SCALE, v1 * R_SCALE), su2), *reinterpret_cast<const half2*>(&svb.x));
        b = __hmul2(__hmul2(__floats2half2_rn(v2 * R_SCALE, v3 * R_SCALE), su2), *reinterpret_cast<const half2*>(&svb.y));
        uint2 o2;
        o2.x = *reinterpret_cast<uint32_t*>(&a); o2.y = *reinterpret_cast<uint32_t*>(&b);
        *reinterpret_cast<uint2*>(out + ((size_t) kb * 128 + r) * n_out + nb * 128 + i * 4) = o2;
    }
}

template <int K, int cb>
static void reconstruct_had_launch(cudaStream_t stream, half* out, const uint16_t* packed, const half* suh,
                                   const half* svh, int k, int n_out, int packed_tiles_n, int tile_n_offset)
{
    dim3 grid(n_out / 128, k / 128);
    reconstruct_had_kernel<K, cb><<<grid, 128, 0, stream>>>(out, (const uint32_t*) packed, suh, svh, n_out,
                                                            packed_tiles_n, tile_n_offset);
}

int launch_reconstruct_had(cudaStream_t stream, half* unpacked, const uint16_t* packed, const half* suh,
                           const half* svh, int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset)
{
    if (k == 0 || n_out == 0) return 0;
    EXL3B_DISPATCH_K_CB(reconstruct_had_launch, K, cb, stream, unpacked, packed, suh, svh, k, n_out,
                        packed_tiles_n, (int) (n_offset / 16));
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

}  // namespace exl3b
