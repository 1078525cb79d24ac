// EXL3 trellis decode primitives.
//
// Format facts (reference: exllamav3_ext/quant/exl3_dq.cuh:15-31, codebook.cuh:56-90, pack.cu:9-57,
// modules/quant/exl3_lib/quantize.py:22-44):
//   * a 16x16 tile is 256*K bits = 8K little-endian uint32 words; word w holds stream bits [32w, 32w+32) MSB first
//   * the 16-bit state of position t is the window ending at stream bit (t+1)*K, wrapping modulo 256*K
//   * position t = 8*l + i  (l = 0..31, i = 0..7) sits at  k = 2*(l%4) + (i&1) + 8*((i>>1)&1),  n = l/4 + 8*(i>>2)
//
// Work decomposition used by every kernel in this library (different from the reference's mma.sync fragment order):
//   a tile is cut into 8 "chunks" c = 0..7 of 32 positions (K words).  Chunk c holds tile columns n = c (positions
//   with i < 4, "half 0") and n = c + 8 (i >= 4, "half 1"), all 16 k-rows each.  One thread decodes one
//   (chunk, half) = ONE tile column x 16 k-values from K+1 words (the chunk plus the preceding word), with every
//   bit offset a compile-time constant.  `half` is warp-uniform in all kernels, so there is no divergence.
//
//   Output order matches what a K-major operand row wants: out[j] = packed fp16 pair (k = 2j, 2j+1).
#pragma once
#include <stdint.h>
#ifndef EXL3B_HOST_EMU
#include <cuda_fp16.h>
#endif

namespace exl3b {

#ifndef EXL3B_HOST_EMU
__device__ __forceinline__ uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel)
{
    uint32_t r;
    asm("prmt.b32 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(sel));
    return r;
}

__device__ __forceinline__ uint32_t lop3_and_xor(uint32_t x, uint32_t b, uint32_t c)
{
    uint32_t r;
    asm("lop3.b32 %0, %1, %2, %3, 0x6a;" : "=r"(r) : "r"(x), "r"(b), "r"(c));   // (x & b) ^ c
    return r;
}

__device__ __forceinline__ uint32_t hadd2_u32(uint32_t a, uint32_t b)
{
    uint32_t r;
    asm("add.rn.f16x2 %0, %1, %2;" : "=r"(r) : "r"(a), "r"(b));
    return r;
}

__device__ __forceinline__ uint32_t hfma2_u32(uint32_t a, uint32_t b, uint32_t c)
{
    uint32_t r;
    asm("fma.rn.f16x2 %0, %1, %2, %3;" : "=r"(r) : "r"(a), "r"(b), "r"(c));
    return r;
}
#else
// Host restatement of the four PTX instructions above (and of __funnelshift_r / __dp4a, provided by the including file) so
// that the SAME decode templates below compile with g++ and can be checked against the oracle without a GPU
// (tests/emu/decode_emu.cpp, tests/test_decode_emu.py).  Never part of the library.
inline uint32_t prmt(uint32_t a, uint32_t b, uint32_t sel)
{
    const uint64_t src = ((uint64_t) b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; ++i)
    {
        const uint32_t s = (sel >> (4 * i)) & 0xf;
        uint32_t byte = (uint32_t) (src >> (8 * (s & 7))) & 0xff;
        if (s & 8) byte = (byte & 0x80) ? 0xff : 0x00;            // sign-replicate mode of prmt.b32
        r |= byte << (8 * i);
    }
    return r;
}
inline uint32_t lop3_and_xor(uint32_t x, uint32_t b, uint32_t c) { return (x & b) ^ c; }
inline uint32_t hadd2_u32(uint32_t a, uint32_t b) { return exl3b_emu_f16x2_fma(a, 0x3c003c00u, b); }            // a * 1 + b, one rounding
inline uint32_t hfma2_u32(uint32_t a, uint32_t b, uint32_t c) { return exl3b_emu_f16x2_fma(a, b, c); }
#endif

// Two 16-bit states -> packed fp16x2 (lo = value(s0), hi = value(s1)), bit-exact with the reference's
// decode_3inst_2<cb> (codebook.cuh:92-123).
template <int cb>
__device__ __forceinline__ uint32_t decode_pair(uint32_t s0, uint32_t s1)
{
    if constexpr (cb == 0)
    {
        uint32_t x0 = s0 * 89226354u + 64248484u;
        uint32_t x1 = s1 * 89226354u + 64248484u;
        x0 = lop3_and_xor(x0, 0x8fff8fffu, 0x3b603b60u);
        x1 = lop3_and_xor(x1, 0x8fff8fffu, 0x3b603b60u);
        return hadd2_u32(prmt(x0, x1, 0x5410), prmt(x0, x1, 0x7632));
    }
    else if constexpr (cb == 1)
    {
        uint32_t x0 = s0 * 0xCBAC1FEDu;
        uint32_t x1 = s1 * 0xCBAC1FEDu;
        x0 = lop3_and_xor(x0, 0x8fff8fffu, 0x3b603b60u);
        x1 = lop3_and_xor(x1, 0x8fff8fffu, 0x3b603b60u);
        return hadd2_u32(prmt(x0, x1, 0x5410), prmt(x0, x1, 0x7632));
    }
    else
    {
        uint32_t x0 = s0 * 0x83DCD12Du;
        uint32_t x1 = s1 * 0x83DCD12Du;
        uint32_t h0 = __dp4a(x0, 0x01010101u, 0x6400u);          // fp16 bits of (1024 + bytesum), exact
        uint32_t h1 = __dp4a(x1, 0x01010101u, 0x6400u);
        return hfma2_u32(prmt(h0, h1, 0x5410), 0x1eee1eeeu, 0xc931c931u);
    }
}

// state of the position whose window ends at chunk-relative stream bit E (K <= E <= 32K); w[0] = word preceding
// the chunk, w[1..K] = chunk words.  All indices/shifts are compile-time.
template <int K, int E>
__device__ __forceinline__ uint32_t window16(const uint32_t (&w)[K + 1])
{
    constexpr int wi = (E - 1) / 32;            // chunk word holding the last bit
    constexpr int sh = (wi + 1) * 32 - E;       // 0..31
    uint32_t v;
    if constexpr (sh == 0)       v = w[1 + wi];
    else if constexpr (sh <= 16) v = w[1 + wi] >> sh;            // window entirely inside one word
    else                         v = __funnelshift_r(w[1 + wi], w[wi], sh);
    return v & 0xffffu;
}

template <int K, int cb, int HALF, int J>
__device__ __forceinline__ void decode4(const uint32_t (&w)[K + 1], uint32_t& lo_pair, uint32_t& hi_pair)
{
    // positions 8*J + 4*HALF + {0,1,2,3} of the chunk -> k = 2J, 2J+1 (lo_pair) and 2J+8, 2J+9 (hi_pair)
    constexpr int P = 8 * J + 4 * HALF;
    uint32_t s0 = window16<K, (P + 1) * K>(w);
    uint32_t s1 = window16<K, (P + 2) * K>(w);
    uint32_t s2 = window16<K, (P + 3) * K>(w);
    uint32_t s3 = window16<K, (P + 4) * K>(w);
    lo_pair = decode_pair<cb>(s0, s1);
    hi_pair = decode_pair<cb>(s2, s3);
}

// One tile column (16 k-values) from K+1 words.  out[j] = fp16x2 (k = 2j, 2j+1), j = 0..7.
template <int K, int cb, int HALF>
__device__ __forceinline__ void decode16(const uint32_t (&w)[K + 1], uint32_t (&out)[8])
{
    decode4<K, cb, HALF, 0>(w, out[0], out[4]);
    decode4<K, cb, HALF, 1>(w, out[1], out[5]);
    decode4<K, cb, HALF, 2>(w, out[2], out[6]);
    decode4<K, cb, HALF, 3>(w, out[3], out[7]);
}

// ---- int8 tensor-core codebook path (mul1 only) -----------------------------------------------------------------
// The mul1 value is k_inv * (1024 + bytesum(state * 0x83DCD12D)) + k_bias (codebook.cuh:77-89).  Instead of summing the
// four product bytes on the IMAD pipe (IDP.4A shares it) the product word itself
// becomes four unsigned 8-bit K-elements of a wgmma u8 operand and the tensor core does the byte sum while
// contracting with the (4x replicated) int8 activation digits.  Cost per weight: window extraction + ONE IMAD.
// out[k] = state(k) * 0x83DCD12D for the 16 k-rows of the thread's tile column, in k order.
template <int K, int HALF, int J>
__device__ __forceinline__ void products4(const uint32_t (&w)[K + 1], uint32_t& x0, uint32_t& x1, uint32_t& x2, uint32_t& x3)
{
    constexpr int P = 8 * J + 4 * HALF;
    uint32_t s0, s1, s2, s3;
    if constexpr (K == 4)
    {
        // the four windows live in one 32-bit span ending at chunk bit 32J + 16 (HALF 0) or 32J + 32 (HALF 1)
        const uint32_t v = HALF == 0 ? __funnelshift_r(w[1 + J], w[J], 16) : w[1 + J];
        const uint32_t t = v >> 4;
        s3 = prmt(v, 0u, 0x4410);          // v & 0xffff
        s1 = prmt(v, 0u, 0x4421);          // (v >> 8) & 0xffff
        s2 = prmt(t, 0u, 0x4410);          // (v >> 4) & 0xffff
        s0 = prmt(t, 0u, 0x4421);          // (v >> 12) & 0xffff
    }
    else if constexpr (K == 8)
    {
        // byte-aligned windows: positions end at chunk bytes P+1 .. P+4
        s0 = window16<K, (P + 1) * K>(w); s1 = window16<K, (P + 2) * K>(w);
        s2 = window16<K, (P + 3) * K>(w); s3 = window16<K, (P + 4) * K>(w);
    }
    else
    {
        s0 = window16<K, (P + 1) * K>(w); s1 = window16<K, (P + 2) * K>(w);
        s2 = window16<K, (P + 3) * K>(w); s3 = window16<K, (P + 4) * K>(w);
    }
    x0 = s0 * 0x83DCD12Du; x1 = s1 * 0x83DCD12Du; x2 = s2 * 0x83DCD12Du; x3 = s3 * 0x83DCD12Du;
}

template <int K, int HALF>
__device__ __forceinline__ void decode16_i8(const uint32_t (&w)[K + 1], uint32_t (&out)[16])
{
    // positions 8J + 4*HALF + {0,1,2,3} -> k = 2J, 2J+1, 2J+8, 2J+9
    products4<K, HALF, 0>(w, out[0], out[1], out[8], out[9]);
    products4<K, HALF, 1>(w, out[2], out[3], out[10], out[11]);
    products4<K, HALF, 2>(w, out[4], out[5], out[12], out[13]);
    products4<K, HALF, 3>(w, out[6], out[7], out[14], out[15]);
}

// K = 4 with the half as a RUN-TIME (warp-uniform) value: span_shift = 16 (half 0) or 0 (half 1) selects the 32-bit span
// holding the group's four windows with one funnel shift, so both halves run the same instruction stream and the
// per-tile branch of the kernels' decode loop disappears (experiment switch EXL3B_I8_K4_BRANCHFREE in gemm_tc_i8_body.cuh;
// checked against the oracle on the host by tests/test_decode_emu.py).
__device__ __forceinline__ void decode16_i8_k4_rt(const uint32_t (&w)[5], uint32_t span_shift, uint32_t (&out)[16])
{
    #pragma unroll
    for (int J = 0; J < 4; ++J)
    {
        const uint32_t v = __funnelshift_r(w[1 + J], w[J], span_shift);       // (w[J] : w[1+J]) >> 16, or w[1+J] itself
        const uint32_t t = v >> 4;
        const uint32_t s3 = prmt(v, 0u, 0x4410), s1 = prmt(v, 0u, 0x4421), s2 = prmt(t, 0u, 0x4410), s0 = prmt(t, 0u, 0x4421);
        out[2 * J] = s0 * 0x83DCD12Du; out[2 * J + 1] = s1 * 0x83DCD12Du;
        out[2 * J + 8] = s2 * 0x83DCD12Du; out[2 * J + 9] = s3 * 0x83DCD12Du;
    }
}

// Thread -> column mapping inside a 128-column strip (8 tiles).  q = lane quarter (warp index % 4), i = lane.
//   tile-in-strip = 4*(q>>1) + (i>>3), chunk = i&7, half = q&1   =>   n_local = 16*tile + 8*half + chunk
__device__ __forceinline__ int strip_tile(int q, int i)  { return 4 * (q >> 1) + (i >> 3); }
__device__ __forceinline__ int strip_col(int q, int i)   { return 16 * strip_tile(q, i) + 8 * (q & 1) + (i & 7); }

// Load the K+1 words of (tile, chunk) from a tile base pointer (global or shared), 8K words per tile.
template <int K>
__device__ __forceinline__ void load_chunk(const uint32_t* tile, int chunk, uint32_t (&w)[K + 1])
{
    const uint32_t* p = tile + chunk * K;
    w[0] = tile[chunk == 0 ? 8 * K - 1 : chunk * K - 1];
    #pragma unroll
    for (int j = 0; j < K; ++j) w[1 + j] = p[j];
}

}  // namespace exl3b
