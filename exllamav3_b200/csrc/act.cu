// Standalone gated activation, a = fp16(act(g) * u) elementwise (exl3b_act_mul: the reference's silu_mul / gelu_mul / relu2_mul,
// exllamav3_ext/activation.cu).  The arithmetic is act.cuh's, shared with the gated input stage of exl3b_gemm_gated.
// `a` may alias `g` or `u`: every element is read and written by the same thread, reads first.
#include "act.cuh"
#include "ptx.cuh"

namespace exl3b {

using namespace ptx;

constexpr int ACT_THREADS = 256;

// thread t handles elements 4 t .. 4 t + 3: one vector load per input and one 8-byte store when the block is whole and aligned
template <bool F32>
__global__ void __launch_bounds__(ACT_THREADS)
act_mul_kernel(const void* g, const void* u, half* a, long long numel, int act, float limit, int vec)
{
    pdl_launch_dependents();
    pdl_wait();
    const long long e = ((long long) blockIdx.x * ACT_THREADS + threadIdx.x) * 4;
    if (e >= numel) return;
    if (vec && e + 4 <= numel)
    {
        const uint2 o = gated_load4(GateIn{g, u, F32, act, limit}, (size_t) e);
        *reinterpret_cast<uint2*>(a + e) = o;
        return;
    }
    for (long long i = e; i < numel && i < e + 4; ++i)
    {
        const float gf = F32 ? static_cast<const float*>(g)[i] : __half2float(static_cast<const half*>(g)[i]);
        const float uf = F32 ? static_cast<const float*>(u)[i] : __half2float(static_cast<const half*>(u)[i]);
        a[i] = act_mul(gf, uf, act, limit);
    }
}

int launch_act_mul(cudaStream_t stream, const void* g, const void* u, half* a, long long numel, bool in_fp32, int act, float limit)
{
    const size_t in_align = in_fp32 ? 16 : 8;
    const int vec = (uintptr_t) g % in_align == 0 && (uintptr_t) u % in_align == 0 && (uintptr_t) a % 8 == 0;
    const long long blocks = (numel + 4LL * ACT_THREADS - 1) / (4LL * ACT_THREADS);
    EXL3B_CHECK(blocks <= 0x7fffffffLL, EXL3B_ERR_SHAPE, "act_mul: %lld elements are too many", numel);
    const dim3 grid((unsigned) blocks);
    const cudaError_t e = in_fp32 ? launch_pdl<act_mul_kernel<true>>(stream, grid, ACT_THREADS, 0, g, u, a, numel, act, limit, vec)
                                  : launch_pdl<act_mul_kernel<false>>(stream, grid, ACT_THREADS, 0, g, u, a, numel, act, limit, vec);
    count_launch();
    EXL3B_CUDA(e);
    return 0;
}

}  // namespace exl3b
