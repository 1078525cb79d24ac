// The gated activations of the MLP blocks, one definition for every kernel that applies them: the standalone operators
// (act.cu: silu_mul / gelu_mul / relu2_mul), the gated input stage of the down projection (exl3b_gemm_gated: gemm_tc_i8_body.cuh,
// gemm_tc.cu) and the fused MoE block (moe_tc.cu: the limit rule and rounding; it keeps its own SiLU / GELU expressions and ungated ReLU^2).  The down projection is bit-identical to act_mul + exl3_gemm only because
// both run these functions on the same fp32 values.
//
//   a = fp16( act(g) * u )      in fp32, rounded once; act = silu g / (1 + exp(-g)), gelu (tanh form) or relu2 max(g, 0)^2
//                               act_limit L != 0: u clamped to [-L, L], act(g) clamped from above at L (the reference's limit
//                               rule, exllamav3_ext/activation_kernels.cuh)
#pragma once
#include "common.cuh"

namespace exl3b {

// activation kinds of exl3b_act_mul / exl3b_gemm_gated (include/exl3b200.h); exl3_moe's act_function uses 0 and 1 the same way
constexpr int ACT_SILU = 0, ACT_GELU = 1, ACT_RELU2 = 2;

// Gated input of a GEMM: the rows it reads are fp16(act(G) * U), G and U (m, k) fp16 or fp32, contiguous
struct GateIn
{
    const void* g;
    const void* u;
    int fp32;                // G and U are fp32 (else fp16)
    int act;                 // ACT_*
    float limit;             // act_limit, 0 = none
};

#ifdef __CUDACC__
// The divisions are __fdividef (2 ulp, no subroutine): the IEEE division's slow path is a CALL, and a wgmma kernel that contains
// one has every wgmma serialized by ptxas (tests/test_wgmma_sass_host.py).  A divisor overflowing to inf gives +-0, the limit
// of both functions there.
__device__ __forceinline__ float act_silu(float g) { return __fdividef(g, 1.0f + expf(-g)); }
// gelu, tanh form: 0.5 g (1 + tanh(t)), t = 0.797884560803 (g + 0.044715 g^3), evaluated as g / (1 + exp(-2 t)) -- the same function
// without the cancellation of 1 + tanh(t) in fp32 for negative g, which costs several fp16 steps of the result there
__device__ __forceinline__ float act_gelu(float g)
{
    return __fdividef(g, 1.0f + expf(-2.0f * (0.797884560803f * (g + 0.044715f * g * g * g))));
}
// exl3_moe's own expressions (IEEE division, the literal tanh form), kept so that the fused MoE operator computes the bits it
// always has; it contains no wgmma
__device__ __forceinline__ float act_silu_moe(float g) { return g / (1.0f + expf(-g)); }
__device__ __forceinline__ float act_gelu_moe(float g) { return 0.5f * g * (1.0f + tanhf(0.797884560803f * (g + 0.044715f * g * g * g))); }
__device__ __forceinline__ float act_relu2(float g) { const float r = fmaxf(g, 0.0f); return r * r; }

__device__ __forceinline__ float act_gate(float g, int act)
{
    if (act == ACT_SILU) return act_silu(g);
    if (act == ACT_GELU) return act_gelu(g);
    return act_relu2(g);
}

// fp16(a * u) after the limit rule; `a` is the activation already applied
__device__ __forceinline__ half act_limit_mul(float a, float u, float limit)
{
    if (limit != 0.0f) { u = fminf(fmaxf(u, -limit), limit); a = fminf(a, limit); }
    return __float2half_rn(a * u);
}

__device__ __forceinline__ half act_mul(float g, float u, int act, float limit)
{
    return act_limit_mul(act_gate(g, act), u, limit);
}

// the four gated inputs of elements e .. e + 3 (e % 4 == 0) as fp16, packed like four raw fp16 inputs
__device__ __forceinline__ uint2 gated_load4(const GateIn& gi, size_t e)
{
    float g[4], u[4];
    if (gi.fp32)
    {
        const float4 a = *reinterpret_cast<const float4*>(static_cast<const float*>(gi.g) + e);
        const float4 b = *reinterpret_cast<const float4*>(static_cast<const float*>(gi.u) + e);
        g[0] = a.x; g[1] = a.y; g[2] = a.z; g[3] = a.w;
        u[0] = b.x; u[1] = b.y; u[2] = b.z; u[3] = b.w;
    }
    else
    {
        const uint2 a = *reinterpret_cast<const uint2*>(static_cast<const half*>(gi.g) + e);
        const uint2 b = *reinterpret_cast<const uint2*>(static_cast<const half*>(gi.u) + e);
        const half2 a0 = *reinterpret_cast<const half2*>(&a.x), a1 = *reinterpret_cast<const half2*>(&a.y);
        const half2 b0 = *reinterpret_cast<const half2*>(&b.x), b1 = *reinterpret_cast<const half2*>(&b.y);
        g[0] = __low2float(a0); g[1] = __high2float(a0); g[2] = __low2float(a1); g[3] = __high2float(a1);
        u[0] = __low2float(b0); u[1] = __high2float(b0); u[2] = __low2float(b1); u[3] = __high2float(b1);
    }
    half h[4];
    #pragma unroll
    for (int i = 0; i < 4; ++i) h[i] = act_mul(g[i], u[i], gi.act, gi.limit);
    uint2 o;
    o.x = pack_half2(h[0], h[1]); o.y = pack_half2(h[2], h[3]);
    return o;
}
#endif

}  // namespace exl3b
