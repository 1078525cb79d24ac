// Dense fp16 GEMM  c = a @ b  (row-major, fp32 accumulate) -- replaces the reference's cuBLAS call
// (exllamav3_ext/hgemm.cu:19-102) on the reconstruct -> hgemm prefill path.
//
// Dispatch: the wgmma kernel (hgemm_tc.cu) for 16-byte-aligned operands; this shared-memory tiled CUDA-core kernel
// only for shapes TMA cannot address (k, n or the C row pitch not a multiple of 8).
#include "common.cuh"

namespace exl3b {

template <bool C_FP32>
__global__ void __launch_bounds__(256)
hgemm_simt_kernel(const half* __restrict__ a, const half* __restrict__ b, void* __restrict__ c,
                  int m, int k, int n, int64_t c_stride)
{
    constexpr int BM = 64, BN = 64, BK = 16;
    __shared__ float as[BK][BM + 1];
    __shared__ float bs[BK][BN + 1];
    const int tx = threadIdx.x % 16, ty = threadIdx.x / 16;
    const int m0 = blockIdx.y * BM, n0 = blockIdx.x * BN;
    float acc[4][4] = {};
    for (int k0 = 0; k0 < k; k0 += BK)
    {
        for (int e = threadIdx.x; e < BM * BK; e += 256)
        {
            int r = e / BK, kk = e % BK;
            as[kk][r] = (m0 + r < m && k0 + kk < k) ? __half2float(a[(size_t) (m0 + r) * k + k0 + kk]) : 0.f;
        }
        for (int e = threadIdx.x; e < BK * BN; e += 256)
        {
            int kk = e / BN, cc = e % BN;
            bs[kk][cc] = (n0 + cc < n && k0 + kk < k) ? __half2float(b[(size_t) (k0 + kk) * n + n0 + cc]) : 0.f;
        }
        __syncthreads();
        #pragma unroll
        for (int kk = 0; kk < BK; ++kk)
        {
            float av[4], bv[4];
            #pragma unroll
            for (int i = 0; i < 4; ++i) { av[i] = as[kk][ty * 4 + i]; bv[i] = bs[kk][tx * 4 + i]; }
            #pragma unroll
            for (int i = 0; i < 4; ++i)
                #pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }
    #pragma unroll
    for (int i = 0; i < 4; ++i)
        #pragma unroll
        for (int j = 0; j < 4; ++j)
        {
            int r = m0 + ty * 4 + i, cc = n0 + tx * 4 + j;
            if (r < m && cc < n)
            {
                if constexpr (C_FP32) ((float*) c)[(size_t) r * c_stride + cc] = acc[i][j];
                else ((half*) c)[(size_t) r * c_stride + cc] = __float2half_rn(acc[i][j]);
            }
        }
}

int launch_hgemm_tc(cudaStream_t stream, const half* a, const half* b, void* c, int m, int k, int n, bool c_fp32,
                    int64_t c_stride);
bool hgemm_tc_supported(const void* a, const void* b, const void* c, int m, int k, int n, int64_t c_stride);

int launch_hgemm(cudaStream_t stream, const half* a, const half* b, void* c, int m, int k, int n, bool c_fp32,
                 int64_t c_stride)
{
    if (hgemm_tc_supported(a, b, c, m, k, n, c_stride))
        return launch_hgemm_tc(stream, a, b, c, m, k, n, c_fp32, c_stride);
    dim3 grid((n + 63) / 64, (m + 63) / 64);
    if (c_fp32) hgemm_simt_kernel<true><<<grid, 256, 0, stream>>>(a, b, c, m, k, n, c_stride);
    else        hgemm_simt_kernel<false><<<grid, 256, 0, stream>>>(a, b, c, m, k, n, c_stride);
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

}  // namespace exl3b
