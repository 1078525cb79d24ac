// Scalar arithmetic of the int8 tensor-core codebook path (gemm_tc_i8_body.cuh), host + device: the activation -> digit
// decomposition its transform warps apply per value, and the reassembly its epilogue applies per accumulator pair.  Kept in
// one place so that the CPU tests can run exactly this code against the oracle's model of the path
// (tests/emu/decode_emu.cpp, tests/test_decode_emu.py); the kernels inline it (SASS unchanged by the extraction).
#pragma once
#include <stdint.h>
#include <string.h>
#ifdef __CUDACC__
#define EXL3B_HD __host__ __device__ __forceinline__
#else
#include <math.h>
#define EXL3B_HD inline
#endif

namespace exl3b {

constexpr int I8_QMAX = 32512;                                 // |q| <= 127 * 256 + 0  -> hi in [-127, 127]

EXL3B_HD int i8_rint(float x)
{
#ifdef __CUDA_ARCH__
    return __float2int_rn(x);
#else
    return (int) lrintf(x);                                    // round to nearest even (default rounding mode)
#endif
}

EXL3B_HD float i8_bits_to_f32(uint32_t u) { float f; memcpy(&f, &u, 4); return f; }
EXL3B_HD uint32_t i8_f32_to_bits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }
EXL3B_HD float i8_mul_rn(float a, float b)
{
#ifdef __CUDA_ARCH__
    return __fmul_rn(a, b);                                    // never contracted into an FMA
#else
    return a * b;
#endif
}

// The two scale divisions of the path, I8_QMAX / mx (digit warps) and mx / I8_QMAX (epilogue), rounded exactly like IEEE
// division (div.rn), from multiplies and FMAs only.  The compiler's fp32 division branches to a slow-path subroutine, and a
// call inside a kernel that issues wgmma makes ptxas serialize every wgmma of it.  Exact for every x in [2^-24, 2^20): the
// positive fp16 magnitudes (the row maxima of the decode-GEMM) and the chain's block-norm bounds; tests/test_i8_div_host.py
// checks every float of that range against IEEE division.  Outside it the results are not those of division: +inf gives NaN
// instead of 0 (only an fp16 overflow of the activations reaches that, where the output is meaningless either way).
EXL3B_HD float i8_qmax_over(float x)
{
    float y = i8_bits_to_f32(0x7ef311c3u - i8_f32_to_bits(x));   // 1 / x within 13 %
    y = fmaf(y, fmaf(-x, y, 1.f), y);                          // Newton steps: 13 % -> 1.6 % -> 3e-4 -> 7e-8 -> < 1 ulp
    y = fmaf(y, fmaf(-x, y, 1.f), y);
    y = fmaf(y, fmaf(-x, y, 1.f), y);
    y = fmaf(y, fmaf(-x, y, 1.f), y);
    const float q = i8_mul_rn((float) I8_QMAX, y);
    return fmaf(fmaf(-x, q, (float) I8_QMAX), y, q);           // one correction with the exact residual
}
EXL3B_HD float i8_over_qmax(float x)
{
    constexpr float r = 1.f / (float) I8_QMAX;
    const float q = i8_mul_rn(x, r);
    return fmaf(fmaf(-(float) I8_QMAX, q, x), r, q);
}

// sqrtf (round to nearest even) from multiplies and FMAs only, for the chain kernel's block norms: the compiler's sqrtf
// branches to a slow-path subroutine, with the same effect on wgmma as the division's.  Exact for every x in [2^-48, 2^40]
// (the nonzero sums of squares of fp16 values the chain can produce); tests/test_i8_div_host.py checks every float of that
// range against IEEE sqrt.  Not for 0 or non-finite x.
EXL3B_HD float i8_sqrt_rn(float x)
{
    float y = i8_bits_to_f32(0x5f3759dfu - (i8_f32_to_bits(x) >> 1));   // 1 / sqrt(x) within 3.5 %
    #pragma unroll
    for (int i = 0; i < 4; ++i)                                // Newton steps: 3.5 % -> 2e-3 -> 5e-6 -> 4e-11 -> < 1 ulp
        y = fmaf(0.5f * y, fmaf(-i8_mul_rn(x, y), y, 1.f), y);
    const float s = i8_mul_rn(x, y);
    return fmaf(fmaf(-s, s, x), 0.5f * y, s);                  // one correction with the exact residual
}

// One transformed activation value -> q = round(v * inv_scale) = 256 * hi + lo with BALANCED signed 8-bit digits
// (hi in [-127, 127], lo in [-128, 127]); each digit is replicated over the four product bytes of a weight, which is how
// the tensor core ends up summing them: sum_k digit_k * (b0 + b1 + b2 + b3)_k.
EXL3B_HD void i8_digits(float v, float inv_scale, int& q_sum, uint32_t& hi_w, uint32_t& lo_w)
{
    const int q = i8_rint(v * inv_scale);
    const int hi = (q + 128) >> 8;
    const int lo = q - (hi << 8);
    q_sum += q;                                                // the row's digit sum T = sum q_k goes into the epilogue
    hi_w = (uint32_t) (hi & 0xff) * 0x01010101u;
    lo_w = (uint32_t) (lo & 0xff) * 0x01010101u;
}

// One row's s32 accumulators of a column (d_hi = sum hi_k * bytesum_k, d_lo = sum lo_k * bytesum_k) and the row's digit sum
// T = sum q_k  ->  scale * sum_k q_k * w_k  with  w = k_inv * (1024 + bytesum) + k_bias, in two steps:
//     i8_centred_sum   sp = sum_k q_k (bytesum_k - 510), exact in 64-bit (the byte sum is centred to keep the fp32 part small)
//     i8_assemble      scale * (k_inv * sp + c1 * T),  c1 = (1024 + 510) * k_inv + k_bias
EXL3B_HD long long i8_centred_sum(int d_hi, int d_lo, int T)
{
    return 256ll * d_hi + (long long) d_lo - 510ll * T;
}
EXL3B_HD float i8_assemble(long long sp, int T, float scale, float k_inv, float c1)
{
    return scale * (k_inv * (float) sp + c1 * (float) T);
}

}  // namespace exl3b
