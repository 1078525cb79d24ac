// Dense fp16 GEMM on wgmma for the reconstruct -> hgemm prefill path:  C[m,n] = A[m,k] @ B[k,n], fp32 accumulate.
// Replaces the reference's cuBLAS call (exllamav3_ext/hgemm.cu:19-102); no library GEMM is used.
//
//   * persistent CTAs, one 128(m) x 128(n) output tile at a time, K in steps of 64
//   * warp 0: TMA producer (A box 128 x 64 K-major, B as two 64(k) x 64(n) boxes, both 128-byte swizzled) into a 4-stage
//     mbarrier ring;  warpgroups 1-2: wgmma.m64n128k16 (A K-major / B MN-major straight from the row-major operands, no
//     transposes), 64 rows each, accumulators in registers, then convert -> masked stores from the fragments
//   * ragged m / n / k: TMA zero-fills out-of-bounds operand elements, stores are masked
#include "tc_common.cuh"
#include <unordered_map>
#include <mutex>

namespace exl3b {

using namespace ptx;

constexpr int HG_BM = 128, HG_BN = 128, HG_BK = 64, HG_STAGES = 4;
constexpr int HG_A_BYTES = HG_BM * HG_BK * 2;          // 16 KB
constexpr int HG_B_BYTES = HG_BK * HG_BN * 2;          // 16 KB
constexpr int HG_THREADS = 384;

struct HgParams
{
    void* C;
    int m, k, n;
    int c_fp32;
    long long c_stride;
    int tiles_m, tiles_n, k_iters;
};

// D[64 x 128] (f32) (+)= A[64 x 16] (f16, K-major, shared memory) * B[16 x 128] (f16, MN-major, shared memory)
__device__ __forceinline__ void wgmma_hg(float (&d)[64], uint64_t a_desc, uint64_t b_desc, int accumulate)
{
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, "
                 "%16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, "
                 "%32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, "
                 "%48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, "
                 "%64, %65, p, 1, 1, 0, 1;\n\t}"
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

__global__ void __launch_bounds__(HG_THREADS, 1)
hgemm_tc_kernel(const HgParams p, const __grid_constant__ CUtensorMap tmA, const __grid_constant__ CUtensorMap tmB)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* sA = smem;                                   // HG_STAGES x 16 KB
    uint8_t* sB = smem + HG_STAGES * HG_A_BYTES;          // HG_STAGES x 16 KB
    uint64_t* bars = reinterpret_cast<uint64_t*>(smem + HG_STAGES * (HG_A_BYTES + HG_B_BYTES));
    const uint32_t bar0 = smem_u32(bars);
    auto FULL = [&](int s) { return bar0 + 8u * s; };
    auto EMPTY = [&](int s) { return bar0 + 8u * (HG_STAGES + s); };

    if (threadIdx.x == 0)
    {
        for (int s = 0; s < HG_STAGES; ++s) { mbar_init(FULL(s), 1); mbar_init(EMPTY(s), 8); }     // EMPTY: the 8 consumer warps
        fence_barrier_init();
    }
    __syncthreads();
    const int tiles = p.tiles_m * p.tiles_n;

    if (warp == 0)
    {
        // =========================== TMA producer ===========================
        if (elect_one()) { prefetch_tmap(&tmA); prefetch_tmap(&tmB); }
        const uint64_t pol = policy_evict_last();
        int s = 0, ph = 0, it = 0;
        for (int t = blockIdx.x; t < tiles; t += gridDim.x)
        {
            const int tm = t / p.tiles_n, tn = t - tm * p.tiles_n;
            for (int ki = 0; ki < p.k_iters; ++ki, ++it)
            {
                if (it >= HG_STAGES) mbar_wait<64>(EMPTY(s), ph ^ 1);
                if (elect_one())
                {
                    mbar_arrive_expect_tx(FULL(s), HG_A_BYTES + HG_B_BYTES);
                    tma_load_2d(smem_u32(sA + s * HG_A_BYTES), &tmA, ki * HG_BK, tm * HG_BM, FULL(s), pol);
                    #pragma unroll
                    for (int j = 0; j < HG_BN / 64; ++j)
                        tma_load_2d(smem_u32(sB + s * HG_B_BYTES + j * 8192), &tmB, tn * HG_BN + 64 * j, ki * HG_BK, FULL(s), pol);
                }
                __syncwarp();
                if (++s == HG_STAGES) { s = 0; ph ^= 1; }
            }
        }
    }
    else if (warp >= 4)
    {
        // =========================== consumers: warpgroup h = rows 64 h .. 64 h + 63 of the tile ===========================
        const int h = (warp - 4) >> 2, wq = warp & 3;
        // A: K-major, 128-byte swizzle (8-row atoms 1024 B apart); B: MN-major, 128-byte swizzle (8-k atoms 1024 B apart,
        // 64-column boxes 8192 B apart)
        const uint64_t descA0 = smem_desc(smem_u32(sA) + h * 64 * 128, 16, 1024, 1);
        const uint64_t descB0 = smem_desc(smem_u32(sB), 8192, 1024, 1);
        const int r_in = 64 * h + 16 * wq + (lane >> 2), c2 = 2 * (lane & 3);
        int s = 0, ph = 0;
        for (int t = blockIdx.x; t < tiles; t += gridDim.x)
        {
            const int tm = t / p.tiles_n, tn = t - tm * p.tiles_n;
            float d[64];
            #pragma unroll
            for (int i = 0; i < 64; ++i) d[i] = 0.f;
            for (int ki = 0; ki < p.k_iters; ++ki)
            {
                mbar_wait<32>(FULL(s), ph);
                #pragma unroll
                for (int i = 0; i < 64; ++i) reg_fence(d[i]);
                wgmma_fence();
                #pragma unroll
                for (int j = 0; j < HG_BK / 16; ++j)
                    wgmma_hg(d, descA0 + (uint64_t) ((s * HG_A_BYTES + 32 * j) >> 4), descB0 + (uint64_t) ((s * HG_B_BYTES + 2048 * j) >> 4), 1);
                wgmma_commit();
                wgmma_wait<0>();
                #pragma unroll
                for (int i = 0; i < 64; ++i) reg_fence(d[i]);
                __syncwarp();
                if (lane == 0) mbar_arrive(EMPTY(s));
                if (++s == HG_STAGES) { s = 0; ph ^= 1; }
            }
            // ---- epilogue from the fragments: rows r, r + 8, columns 8 j + 2c, +1 ----
            #pragma unroll
            for (int hr = 0; hr < 2; ++hr)
            {
                const int row = tm * HG_BM + r_in + 8 * hr;
                if (row >= p.m) continue;
                #pragma unroll
                for (int j = 0; j < 16; ++j)
                {
                    const int col = tn * HG_BN + 8 * j + c2;
                    if (col >= p.n) continue;                  // n % 8 == 0: a column pair is in or out as a whole
                    const float v0 = d[4 * j + 2 * hr], v1 = d[4 * j + 2 * hr + 1];
                    if (p.c_fp32)
                        *reinterpret_cast<float2*>((float*) p.C + (size_t) row * p.c_stride + col) = make_float2(v0, v1);
                    else
                        *reinterpret_cast<half2*>((half*) p.C + (size_t) row * p.c_stride + col) = __floats2half2_rn(v0, v1);
                }
            }
        }
    }
}

// ---- host -------------------------------------------------------------------------------------------------------------

typedef CUresult (*PFN_encodeTiled2)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                     const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                     CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static int make_tmap_fp16_2d(const void* base, uint64_t inner, uint64_t outer, uint64_t row_stride_bytes, uint32_t box_inner,
                             uint32_t box_outer, CUtensorMap* out)
{
    static PFN_encodeTiled2 encode = nullptr;
    static std::mutex mu;
    std::lock_guard<std::mutex> lock(mu);
    if (!encode)
    {
        void* fn = nullptr;
        cudaDriverEntryPointQueryResult qres;
        EXL3B_CUDA(cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &fn, cudaEnableDefault, &qres));
        EXL3B_CHECK(fn && qres == cudaDriverEntryPointSuccess, EXL3B_ERR_CUDA, "cuTensorMapEncodeTiled not available from the driver");
        encode = (PFN_encodeTiled2) fn;
    }
    cuuint64_t gdim[2] = { inner, outer };
    cuuint64_t gstride[1] = { row_stride_bytes };
    cuuint32_t box[2] = { box_inner, box_outer };
    cuuint32_t estr[2] = { 1, 1 };
    CUresult r = encode(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2, const_cast<void*>(base), gdim, gstride, box, estr,
                        CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                        CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    EXL3B_CHECK(r == CUDA_SUCCESS, EXL3B_ERR_CUDA, "cuTensorMapEncodeTiled failed (%d) for hgemm operand", (int) r);
    return 0;
}

bool hgemm_tc_supported(const void* a, const void* b, const void* c, int m, int k, int n, int64_t c_stride)
{
    // TMA needs 16-byte aligned bases and row pitches.  Anything else (e.g. an unaligned view) takes the CUDA-core kernel
    // instead of an error.
    const bool aligned = (((uintptr_t) a | (uintptr_t) b | (uintptr_t) c) & 15) == 0;
    return aligned && m >= 1 && k >= 8 && n >= 8 && k % 8 == 0 && n % 8 == 0 && c_stride % 8 == 0;
}

int launch_hgemm_tc(cudaStream_t stream, const half* a, const half* b, void* c, int m, int k, int n, bool c_fp32,
                    int64_t c_stride)
{
    EXL3B_CHECK(((uintptr_t) a & 15) == 0 && ((uintptr_t) b & 15) == 0 && ((uintptr_t) c & 15) == 0, EXL3B_ERR_ARG,
                "hgemm: operands must be 16-byte aligned");
    CUtensorMap tmA, tmB;
    int r = make_tmap_fp16_2d(a, (uint64_t) k, (uint64_t) m, (uint64_t) k * 2, HG_BK, HG_BM, &tmA); if (r) return r;
    r = make_tmap_fp16_2d(b, (uint64_t) n, (uint64_t) k, (uint64_t) n * 2, 64, HG_BK, &tmB); if (r) return r;
    HgParams p{};
    p.C = c; p.m = m; p.k = k; p.n = n; p.c_fp32 = c_fp32; p.c_stride = c_stride;
    p.tiles_m = (m + HG_BM - 1) / HG_BM; p.tiles_n = (n + HG_BN - 1) / HG_BN; p.k_iters = (k + HG_BK - 1) / HG_BK;
    static bool attr_set[32] = {};
    int dev = 0; cudaGetDevice(&dev);
    const int smem_bytes = HG_STAGES * (HG_A_BYTES + HG_B_BYTES) + 256;
    if (!attr_set[dev & 31])
    {
        EXL3B_CUDA(cudaFuncSetAttribute(hgemm_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem_bytes));
        attr_set[dev & 31] = true;
    }
    int sms = 0; cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    int grid = p.tiles_m * p.tiles_n; if (grid > sms) grid = sms;
    hgemm_tc_kernel<<<grid, HG_THREADS, smem_bytes, stream>>>(p, tmA, tmB);
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

}  // namespace exl3b
