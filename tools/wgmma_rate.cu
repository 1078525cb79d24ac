// Sustained throughput of back-to-back wgmma.m64nNk32.s32.u8.s8 (A from registers, B from shared memory) on one SM, the
// instruction the int8 decode-GEMM (gemm_tc_i8_body.cuh) issues.  Built and run by tools/wgmma_rate.py.
//
// Every CTA (one per SM) runs `iters` batches of 8 wgmma per warpgroup, each batch one commit group, in the kernel's form:
//   chain  all 8 accumulate into the same registers (the decode-GEMM's form), or 8 independent accumulators
//   wait   wait_group 0 after every batch (the batch drains before the next is issued), or wait_group 1 (one batch stays in
//          flight while the next is issued)
// and prints one JSON line per configuration: SM clocks per wgmma per SM, and the SM clock rate during the run.
#include <cstdio>
#include <cstdint>
#include <cstdlib>
#include <vector>
#include <algorithm>
#include <cuda_runtime.h>
#include "../exllamav3_b200/csrc/ptx.cuh"

using namespace exl3b::ptx;

#define CK(x) do { cudaError_t e_ = (x); if (e_ != cudaSuccess) { fprintf(stderr, "%s: %s\n", #x, cudaGetErrorString(e_)); exit(1); } } while (0)

template <int N, bool INDEP, int WAIT>
__global__ void __launch_bounds__(512, 1) wgmma_rate_kernel(int iters, unsigned long long* out)
{
    extern __shared__ __align__(1024) uint8_t smem[];
    // B: the decode-GEMM's digit-tile layout (K-chunks of 8 N-rows x 16 B, second 8-row group 4096 B further)
    for (int i = threadIdx.x; i < 8192 / 4; i += blockDim.x) reinterpret_cast<uint32_t*>(smem)[i] = 0x01010101u * (i & 7);
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
    __syncthreads();
    const uint64_t desc0 = smem_desc(smem_u32(smem), 128, 4096, 0);
    constexpr int NA = INDEP ? 8 : 1;
    uint32_t acc[NA][N / 2];
    #pragma unroll
    for (int c = 0; c < NA; ++c)
        #pragma unroll
        for (int i = 0; i < N / 2; ++i) acc[c][i] = 0u;
    uint32_t a[4][4];                                    // A fragments (their values do not matter), shared by the 8 MMAs of a batch
    #pragma unroll
    for (int j = 0; j < 4; ++j)
        #pragma unroll
        for (int i = 0; i < 4; ++i) a[j][i] = (threadIdx.x * 0x9E3779B9u) ^ (0x01000193u * (4 * j + i));
    unsigned long long t0 = 0, c0 = 0;
    __syncthreads();
    if (threadIdx.x == 0) { asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t0)); c0 = clock64(); }
    for (int it = 0; it < iters; ++it)
    {
        // (with a batch in flight, any other access of its accumulators makes ptxas wait for the MMAs: no fences then)
        if constexpr (WAIT == 0)
        {
            #pragma unroll
            for (int c = 0; c < NA; ++c)
                #pragma unroll
                for (int i = 0; i < N / 2; ++i) reg_fence(acc[c][i]);
        }
        wgmma_fence();
        #pragma unroll
        for (int j = 0; j < 8; ++j)
        {
            const uint64_t d = desc0 + (uint64_t) (16 * (j + 8 * (it & 1)));
            if constexpr (N == 8) wgmma_u8s8_n8(acc[INDEP ? j : 0], a[j & 3][0], a[j & 3][1], a[j & 3][2], a[j & 3][3], d);
            else wgmma_u8s8_n16(acc[INDEP ? j : 0], a[j & 3][0], a[j & 3][1], a[j & 3][2], a[j & 3][3], d);
        }
        wgmma_commit();
        wgmma_wait<WAIT>();
        if constexpr (WAIT == 0)
        {
            #pragma unroll
            for (int c = 0; c < NA; ++c)
                #pragma unroll
                for (int i = 0; i < N / 2; ++i) reg_fence(acc[c][i]);
        }
    }
    wgmma_wait<0>();
    __syncthreads();
    if (threadIdx.x == 0)
    {
        unsigned long long t1;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t1));
        out[2 * blockIdx.x] = clock64() - c0;
        out[2 * blockIdx.x + 1] = t1 - t0;
    }
    // keep the accumulators alive
    uint32_t x = 0;
    #pragma unroll
    for (int c = 0; c < NA; ++c)
        #pragma unroll
        for (int i = 0; i < N / 2; ++i) x ^= acc[c][i];
    if (x == 0x12345678u && iters < 0) out[0] = x;
}

template <int N, bool INDEP, int WAIT>
static void run(int num_sms, int wgs, int iters)
{
    auto k = wgmma_rate_kernel<N, INDEP, WAIT>;
    const int smem = 120 * 1024;                         // one CTA per SM
    CK(cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    unsigned long long* d_out;
    CK(cudaMalloc(&d_out, 2 * num_sms * sizeof(unsigned long long)));
    k<<<num_sms, 128 * wgs, smem>>>(iters / 10, d_out);  // warm-up
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    k<<<num_sms, 128 * wgs, smem>>>(iters, d_out);
    CK(cudaGetLastError());
    CK(cudaDeviceSynchronize());
    std::vector<unsigned long long> h(2 * num_sms);
    CK(cudaMemcpy(h.data(), d_out, h.size() * sizeof(unsigned long long), cudaMemcpyDeviceToHost));
    CK(cudaFree(d_out));
    std::vector<double> cpi, mhz;
    for (int b = 0; b < num_sms; ++b)
    {
        cpi.push_back((double) h[2 * b] / ((double) iters * 8 * wgs));
        mhz.push_back((double) h[2 * b] / (double) h[2 * b + 1] * 1e3);
    }
    std::sort(cpi.begin(), cpi.end());
    std::sort(mhz.begin(), mhz.end());
    printf("{\"shape\": \"m64n%dk32\", \"warpgroups\": %d, \"chain\": \"%s\", \"wait_group\": %d, \"iters\": %d, "
           "\"clocks_per_wgmma_per_sm\": {\"median\": %.2f, \"min\": %.2f, \"max\": %.2f}, \"sm_mhz_median\": %.0f}\n",
           N, wgs, INDEP ? "independent" : "same_accumulator", WAIT, iters,
           cpi[cpi.size() / 2], cpi.front(), cpi.back(), mhz[mhz.size() / 2]);
    fflush(stdout);
}

template <int N>
static void run_all(int num_sms, int iters)
{
    for (int wgs : {1, 4})
    {
        run<N, false, 0>(num_sms, wgs, iters);
        run<N, true, 0>(num_sms, wgs, iters);
        run<N, false, 1>(num_sms, wgs, iters);
        run<N, true, 1>(num_sms, wgs, iters);
    }
}

int main(int argc, char** argv)
{
    const int iters = argc > 1 ? atoi(argv[1]) : 20000;
    int dev = 0, num_sms = 0;
    CK(cudaGetDevice(&dev));
    CK(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    run_all<8>(num_sms, iters);
    run_all<16>(num_sms, iters);
    return 0;
}
