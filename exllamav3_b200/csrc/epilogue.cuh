// Output transform shared by the SIMT and tensor-core GEMM paths.
#pragma once
#include "common.cuh"

namespace exl3b {

#ifdef __CUDACC__
// One warp finishes one 128-column segment of one output row: fp32 sums (shared memory) -> 128-point Hadamard (fp32)
// -> * scale/sqrt(128) -> * svh -> C dtype.  Rounding points follow the reference's had_ff_r_128_inner /
// had_fh_r_128_inner (hadamard_inner.cuh:151-277): fp32 C multiplies by float(svh); fp16 C rounds to fp16 first and
// then multiplies in fp16.  svh == nullptr: no output transform, plain conversion.
__device__ __forceinline__ void output_row_128(const float* row, char* C, size_t elem_off, const half* svh,
                                               float out_scale, bool c_fp32, int lane)
{
    float4 v = *reinterpret_cast<const float4*>(row + lane * 4);
    float v0 = v.x, v1 = v.y, v2 = v.z, v3 = v.w;
    uint2 scb = make_uint2(0, 0);
    if (svh)
    {
        scb = *reinterpret_cast<const uint2*>(svh + lane * 4);
        had128_warp(v0, v1, v2, v3, lane);
        const float r = R_SCALE * out_scale;
        v0 *= r; v1 *= r; v2 *= r; v3 *= r;
    }
    if (c_fp32)
    {
        if (svh)
        {
            const half2 a = *reinterpret_cast<const half2*>(&scb.x), b = *reinterpret_cast<const half2*>(&scb.y);
            v0 *= __low2float(a); v1 *= __high2float(a); v2 *= __low2float(b); v3 *= __high2float(b);
        }
        *reinterpret_cast<float4*>((float*) C + elem_off + lane * 4) = make_float4(v0, v1, v2, v3);
    }
    else
    {
        half2 a = __floats2half2_rn(v0, v1), b = __floats2half2_rn(v2, v3);
        if (svh)
        {
            a = __hmul2(a, *reinterpret_cast<const half2*>(&scb.x));
            b = __hmul2(b, *reinterpret_cast<const half2*>(&scb.y));
        }
        uint2 o; o.x = *reinterpret_cast<uint32_t*>(&a); o.y = *reinterpret_cast<uint32_t*>(&b);
        *reinterpret_cast<uint2*>((half*) C + elem_off + lane * 4) = o;
    }
}

// The same transform without the store: the fp32 values of one 128-column segment after Hadamard, scale and float(svh)
// (the fp32-C arithmetic of output_row_128).  Used where the segment is summed over the tensor-parallel ranks first.
__device__ __forceinline__ void finish_row_128_f32(const float* row, const half* svh, float out_scale, int lane, float (&o)[4])
{
    float4 v = *reinterpret_cast<const float4*>(row + lane * 4);
    float v0 = v.x, v1 = v.y, v2 = v.z, v3 = v.w;
    if (svh)
    {
        const uint2 scb = *reinterpret_cast<const uint2*>(svh + lane * 4);
        had128_warp(v0, v1, v2, v3, lane);
        const float r = R_SCALE * out_scale;
        v0 *= r; v1 *= r; v2 *= r; v3 *= r;
        const half2 a = *reinterpret_cast<const half2*>(&scb.x), b = *reinterpret_cast<const half2*>(&scb.y);
        v0 *= __low2float(a); v1 *= __high2float(a); v2 *= __low2float(b); v3 *= __high2float(b);
    }
    o[0] = v0; o[1] = v1; o[2] = v2; o[3] = v3;
}
#endif

}  // namespace exl3b
