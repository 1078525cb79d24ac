// Host build of the int8 path's inline scale divisions and square root (exllamav3_b200/csrc/i8_math.cuh: i8_qmax_over,
// i8_over_qmax, i8_sqrt_rn) for tests/test_i8_div_host.py: every float of a range is compared bit for bit with IEEE division
// or sqrt.  The helpers use only fmaf, single multiplies and bit casts, which round the same way on the host as on the GPU.
// Test infrastructure only.
#include <stdint.h>
#include <string.h>
#include <math.h>

#include "../../exllamav3_b200/csrc/i8_math.cuh"

using namespace exl3b;

extern "C" {

// Checks every float with bit pattern in [lo, hi), stepping by `step`.  Returns the number of mismatches; the first one's
// bit pattern goes to *first (0 when there is none).
long long emu_check_divisions(uint32_t lo, uint32_t hi, uint32_t step, uint32_t* first)
{
    volatile float qmax = (float) I8_QMAX;                     // volatile: the reference is a run-time IEEE division
    long long bad = 0;
    *first = 0;
    for (uint64_t b = lo; b < hi; b += step)
    {
        const float x = i8_bits_to_f32((uint32_t) b);
        const bool ok = i8_f32_to_bits(i8_qmax_over(x)) == i8_f32_to_bits(qmax / x)
                     && i8_f32_to_bits(i8_over_qmax(x)) == i8_f32_to_bits(x / qmax);
        if (!ok && bad++ == 0) *first = (uint32_t) b;
    }
    return bad;
}

// The same for i8_sqrt_rn against IEEE sqrtf.
long long emu_check_sqrt(uint32_t lo, uint32_t hi, uint32_t step, uint32_t* first)
{
    long long bad = 0;
    *first = 0;
    for (uint64_t b = lo; b < hi; b += step)
    {
        volatile float x = i8_bits_to_f32((uint32_t) b);
        if (i8_f32_to_bits(i8_sqrt_rn(x)) != i8_f32_to_bits(sqrtf(x)) && bad++ == 0) *first = (uint32_t) b;
    }
    return bad;
}

}
