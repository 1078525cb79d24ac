// reconstruct_had on the tensor cores:  W = diag(suh) . H128 . W_hat . H128 . diag(svh)  per 128 x 128 block, both 128-point
// Hadamards as wgmma GEMMs against the +-1 matrix H128 (exact in fp16, fp32 accumulation) instead of 2 x 7 butterfly
// stages on the CUDA cores (kernels_basic.cu).  Replaces the reference's reconstruct_had_kernel
// (exllamav3_ext/quant/reconstruct.cu:159-306).
//
// Per block (one CTA of two warpgroups, persistent over the blocks; the next block's packed words are fetched one block ahead):
//   1. thread pair = one column n: decode its 128 k-values (4 tiles each, decode16) and store them as the B operand W_hat^T [n][k]
//      (K-major core-matrix layout) in shared memory
//   2. GEMM 1 (warpgroup h: rows 64 h .. 64 h + 63):  D[k'][n] = sum_k H[k'][k] W_hat[k][n]        (A = H from shared memory)
//   3. the accumulator fragment, * 1/sqrt(128) and rounded to fp16 (the reference keeps an fp16 tile between the passes), IS
//      the register A fragment of the second GEMM
//   4. GEMM 2:  D[k'][n'] = sum_n T[k'][n] H[n][n']                                                   (B = the same H)
//   5. * 1/sqrt(128) -> fp16, * suh[row] * svh[col] in fp16 (the rounding order of reconstruct.cu:300-304), stored from the fragment
// H128 is written to shared memory once per CTA.
#include "tc_common.cuh"
#include <cstdlib>

namespace exl3b {

using namespace ptx;

constexpr int RT_THREADS = 256;
constexpr int RT_H_BYTES = 128 * 256;                  // H128 fp16, K-major core-matrix layout
constexpr int RT_B_BYTES = 128 * 256;                  // W_hat^T block
constexpr int RT_SMEM = RT_H_BYTES + RT_B_BYTES + 256;

// (row, k) of a 128 x 128 fp16 operand in the K-major no-swizzle core-matrix layout: 8 rows x 16 B core matrices,
// K-adjacent ones 128 B apart (LBO), 8-row groups 2048 B apart (SBO)
__device__ __forceinline__ uint32_t rt_off(int row, int k) { return (row >> 3) * 2048 + (k >> 3) * 128 + (row & 7) * 16 + (k & 7) * 2; }

// D[64 x 128] (f32) = / += A[64 x 16] (f16, shared memory) * B[16 x 128] (f16, shared memory, K-major)
__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t a_desc, uint64_t b_desc, int accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a_desc), "l"(b_desc), "r"(accumulate) : "memory");
}
// D[64 x 128] (f32) = / += A[64 x 16] (f16, registers) * B[16 x 128] (f16, shared memory, K-major)
__device__ __forceinline__ void wgmma_rs_n128(float (&d)[64], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc,
                                              int accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %69, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "{%64, %65, %66, %67}, %68, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]),
                   "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]),
                   "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]),
                   "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]),
                   "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]),
                   "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]),
                   "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]),
                   "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc), "r"(accumulate) : "memory");
}

__device__ __forceinline__ uint32_t pack_scaled(float a, float b)
{
    const half2 h = __floats2half2_rn(a * R_SCALE, b * R_SCALE);
    return *reinterpret_cast<const uint32_t*>(&h);
}

template <int K, int cb>
__global__ void __launch_bounds__(RT_THREADS, 1)
reconstruct_had_tc_kernel(half* __restrict__ out, const uint32_t* __restrict__ packed, const half* __restrict__ suh,
                          const half* __restrict__ svh, int n_out, int packed_tiles_n, int tile_n_offset, int blocks_n, int n_blocks)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    uint8_t* sH = smem;
    uint8_t* sB = smem + RT_H_BYTES;
    half* s_svh = reinterpret_cast<half*>(smem + RT_H_BYTES + RT_B_BYTES);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int q = warp & 3, part = warp >> 2;                 // lane quarter, half of the column's tiles / warpgroup
    const int row = q * 32 + lane;                            // the thread's column in phase 1

    // H128[row][c] = (-1)^popcount(row & c): 16 x 16 bytes per row, shared by the row's two threads
    #pragma unroll
    for (int kc = part; kc < 16; kc += 2)
    {
        uint32_t wv[4];
        #pragma unroll
        for (int j = 0; j < 4; ++j)
        {
            const int c0 = kc * 8 + 2 * j;
            const uint32_t lo = (__popc(row & c0) & 1) ? 0xbc00u : 0x3c00u;
            const uint32_t hi = (__popc(row & (c0 + 1)) & 1) ? 0xbc00u : 0x3c00u;
            wv[j] = lo | (hi << 16);
        }
        *reinterpret_cast<uint4*>(sH + rt_off(row, kc * 8)) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
    }
    const uint32_t h_addr = smem_u32(sH), b_addr = smem_u32(sB);
    const uint64_t desc_a1 = smem_desc(h_addr + part * 64 * 256, 128, 2048, 0);   // this warpgroup's 64 rows of H
    const uint64_t desc_h = smem_desc(h_addr, 128, 2048, 0);
    const uint64_t desc_b = smem_desc(b_addr, 128, 2048, 0);
    // fragment coordinates of the accumulators: rows r0, r0 + 8 of the block, columns 8 j + 2 c, +1
    const int r0 = 64 * part + 16 * q + (lane >> 2), c2 = 2 * (lane & 3);

    const int tl = strip_tile(q, lane), col = strip_col(q, lane);
    // the packed words, suh and svh of a block are fetched one block AHEAD (registers), right after the previous block's decode:
    // the DRAM latency then runs under the two GEMMs and the read-outs instead of opening the block's serial chain
    uint32_t w[4][K + 1];
    half nx_suh0, nx_suh1, nx_svh = __float2half(0.f);
    auto fetch = [&](int blk)
    {
        const int kb = blk / blocks_n, nb = blk - kb * blocks_n;
        #pragma unroll
        for (int i = 0; i < 4; ++i)
        {
            const int t = part + i * 2;
            load_chunk<K>(packed + ((size_t) (kb * 8 + t) * packed_tiles_n + tile_n_offset + nb * 8 + tl) * (8 * K), lane & 7, w[i]);
        }
        nx_suh0 = suh[kb * 128 + r0];
        nx_suh1 = suh[kb * 128 + r0 + 8];
        if (threadIdx.x < 128) nx_svh = svh[nb * 128 + threadIdx.x];
    };
    if ((int) blockIdx.x < n_blocks) fetch(blockIdx.x);
    for (int blk = blockIdx.x; blk < n_blocks; blk += gridDim.x)
    {
        const int kb = blk / blocks_n, nb = blk - kb * blocks_n;
        // ---- 1. decode this thread's share of its column into the B operand ----
        #pragma unroll
        for (int i = 0; i < 4; ++i)
        {
            const int t = part + i * 2;
            uint32_t o[8];
            if (q & 1) decode16<K, cb, 1>(w[i], o); else decode16<K, cb, 0>(w[i], o);
            *reinterpret_cast<uint4*>(sB + rt_off(col, 16 * t)) = make_uint4(o[0], o[1], o[2], o[3]);
            *reinterpret_cast<uint4*>(sB + rt_off(col, 16 * t + 8)) = make_uint4(o[4], o[5], o[6], o[7]);
        }
        if (threadIdx.x < 128) s_svh[threadIdx.x] = nx_svh;
        const half su0 = nx_suh0, su1 = nx_suh1;
        if (blk + (int) gridDim.x < n_blocks) fetch(blk + gridDim.x);
        fence_proxy_async_smem();
        __syncthreads();                                       // B complete (generic writes visible to the async proxy)
        // ---- 2. left Hadamard: D = H x W_hat ----
        float d[64];
        #pragma unroll
        for (int i = 0; i < 64; ++i) d[i] = 0.f;
        wgmma_fence();
        #pragma unroll
        for (int j = 0; j < 8; ++j) wgmma_ss_n128(d, desc_a1 + (uint64_t) (16 * j), desc_b + (uint64_t) (16 * j), j > 0);
        wgmma_commit();
        wgmma_wait<0>();
        #pragma unroll
        for (int i = 0; i < 64; ++i) reg_fence(d[i]);
        // ---- 3. * 1/sqrt(128) -> fp16: the A fragments of the right Hadamard (K = n, 16 columns per instruction) ----
        uint32_t t[32];
        #pragma unroll
        for (int j = 0; j < 8; ++j)
        {
            t[4 * j + 0] = pack_scaled(d[8 * j + 0], d[8 * j + 1]);        // row r0,     n = 16 j + 2c, +1
            t[4 * j + 1] = pack_scaled(d[8 * j + 2], d[8 * j + 3]);        // row r0 + 8
            t[4 * j + 2] = pack_scaled(d[8 * j + 4], d[8 * j + 5]);        // row r0,     n = 16 j + 8 + 2c, +1
            t[4 * j + 3] = pack_scaled(d[8 * j + 6], d[8 * j + 7]);        // row r0 + 8
        }
        // ---- 4. right Hadamard: D = T x H (A from registers) ----
        #pragma unroll
        for (int i = 0; i < 64; ++i) reg_fence(d[i]);
        wgmma_fence();
        #pragma unroll
        for (int j = 0; j < 8; ++j) wgmma_rs_n128(d, t[4 * j], t[4 * j + 1], t[4 * j + 2], t[4 * j + 3], desc_h + (uint64_t) (16 * j), j > 0);
        wgmma_commit();
        wgmma_wait<0>();
        #pragma unroll
        for (int i = 0; i < 32; ++i) reg_fence(t[i]);
        #pragma unroll
        for (int i = 0; i < 64; ++i) reg_fence(d[i]);
        // ---- 5. scale and store: (fp16(h / sqrt(128)) * suh[row]) * svh[col], fp16 multiplies ----
        half* orow0 = out + ((size_t) kb * 128 + r0) * n_out + nb * 128;
        half* orow1 = orow0 + (size_t) 8 * n_out;
        const half2 sa = __half2half2(su0), sb = __half2half2(su1);
        #pragma unroll
        for (int j = 0; j < 16; ++j)
        {
            const int cc = 8 * j + c2;
            const half2 sv = *reinterpret_cast<const half2*>(s_svh + cc);
            uint32_t v0 = pack_scaled(d[4 * j + 0], d[4 * j + 1]), v1 = pack_scaled(d[4 * j + 2], d[4 * j + 3]);
            half2 h0 = __hmul2(__hmul2(*reinterpret_cast<half2*>(&v0), sa), sv);
            half2 h1 = __hmul2(__hmul2(*reinterpret_cast<half2*>(&v1), sb), sv);
            *reinterpret_cast<half2*>(orow0 + cc) = h0;
            *reinterpret_cast<half2*>(orow1 + cc) = h1;
        }
        // sB and s_svh are rewritten by the next block: every thread must be through with them
        __syncthreads();
    }
}

template <int K, int cb>
static void reconstruct_had_tc_launch(cudaStream_t stream, half* out, const uint16_t* packed, const half* suh, const half* svh,
                                      int k, int n_out, int packed_tiles_n, int tile_n_offset, int num_sms, cudaError_t* err)
{
    static bool attr_set[32] = {};
    int dev = 0; cudaGetDevice(&dev);
    if (!attr_set[dev & 31])
    {
        *err = cudaFuncSetAttribute(reconstruct_had_tc_kernel<K, cb>, cudaFuncAttributeMaxDynamicSharedMemorySize, RT_SMEM);
        if (*err != cudaSuccess) return;
        attr_set[dev & 31] = true;
    }
    const int blocks_n = n_out / 128, n_blocks = blocks_n * (k / 128);
    int grid = 2 * num_sms; if (grid > n_blocks) grid = n_blocks;
    reconstruct_had_tc_kernel<K, cb><<<grid, RT_THREADS, RT_SMEM, stream>>>(out, (const uint32_t*) packed, suh, svh, n_out,
                                                                            packed_tiles_n, tile_n_offset, blocks_n, n_blocks);
    *err = cudaSuccess;
}

// EXL3B_RECONSTRUCT_HAD=simt keeps the CUDA-core kernel (kernels_basic.cu), the twin the tests compare against;
// reconstruct_had_set_mode (test hook): 0 = environment / default, 1 = CUDA cores, 2 = tensor cores
static int g_rt_mode = 0;
void reconstruct_had_set_mode(int mode)
{
    g_rt_mode = mode;
}
bool reconstruct_had_tc_enabled()
{
    if (g_rt_mode) return g_rt_mode == 2;
    static int on = -1;
    if (on < 0) { const char* e = getenv("EXL3B_RECONSTRUCT_HAD"); on = (e && e[0] == 's') ? 0 : 1; }
    return on != 0;
}

int launch_reconstruct_had_tc(cudaStream_t stream, half* unpacked, const uint16_t* packed, const half* suh, const half* svh,
                              int k, int n_out, int packed_tiles_n, int K, int cb, int64_t n_offset, int num_sms)
{
    if (k == 0 || n_out == 0) return 0;
    cudaError_t err = cudaSuccess;
    EXL3B_DISPATCH_K_CB(reconstruct_had_tc_launch, K, cb, stream, unpacked, packed, suh, svh, k, n_out, packed_tiles_n,
                        (int) (n_offset / 16), num_sms, &err);
    count_launch();
    EXL3B_CUDA(err);
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

}  // namespace exl3b
