// EXL3 trellis encoder: tail-biting Viterbi over the 16-bit codebook trellis (quantize_tiles) and the K-bit packer
// (pack_trellis).  Replaces the reference's quant/quantize_tiles_kernel.cuh and quant/pack.cu:9-57.
//
// Trellis: s[t] = ((s[t-1] << K) | q_t) & 0xffff, so s[t] >> K == s[t-1] & (2^(16-K) - 1).  A path cost is kept per "edge",
// the 16-K low bits a state passes on; the 2^K states ending in edge e are (k << (16-K)) | e, k = 0 .. 2^K-1, and state s
// continues the path that ended in edge s >> K.  Per position, every edge takes the cheapest of its 2^K candidates.
//
// Differences from the reference kernel:
//   * path costs and the input are fp32 (the reference rounds both to fp16, whose spacing at a typical path cost is the size
//     of the per-step differences Viterbi compares), and the value of a state is the GEMMs' own decode_pair<cb>.
//   * a backpointer is the K-bit choice k, stored as K bit planes of 32 edges (one warp ballot per bit) in a fixed per-device
//     scratch region: 256 * K * 2^(16-K) bits per tile instead of the reference's 16 bits per edge in the caller's buffer.
//   * one CTA walks many tiles (persistent grid), so any number of tiles runs in the fixed scratch.
// Anchor rule (the reference's): pass 1 starts at position 128 unconstrained; the overlap e = s[0] >> K of its best path is
// the anchor; pass 2 starts at position 0 with only states whose predecessor edge is e, and backtracks from edge e at
// position 255, so the result is the exact (fp32) minimum-error tail-biting path with that overlap.
#include "common.cuh"
#include "decode.cuh"
#include <mutex>

namespace exl3b {

namespace {

constexpr size_t ENC_SCRATCH_PER_SM = (size_t) 2 << 20;     // backpointer scratch: 2 MB per SM, allocated once per device

template <int K>
struct EncGeom
{
    static constexpr int Kr = 16 - K;
    static constexpr int E = 1 << Kr;                        // path-cost entries (edges)
    static constexpr int NP = E / 2;                         // a thread relaxes edge pairs (2j, 2j+1): one decode_pair
    // K = 1 keeps ONE fp32 cost buffer (128 KB, two do not fit) and stages each thread's inputs in registers
    static constexpr int NT = K == 1 ? 1024 : (NP < 512 ? NP : 512);
    static constexpr int PPT = NP / NT;                      // pairs per thread and step
    static constexpr int NC = NP / 32;                       // 32-pair warp chunks per step
    static constexpr int BP_WORDS = 256 * NC * 2 * K;        // backpointer words per tile: K bit planes x 2 parities per chunk
    static constexpr int COST_BUFS = K == 1 ? 1 : 2;
    static constexpr size_t SMEM = 256 * 4 + (size_t) COST_BUFS * E * 4 + 256 * 2 + 32 * 8;
};

__device__ __forceinline__ float value_f32(uint32_t pair, int hi)
{
    return __half2float(__ushort_as_half((unsigned short) (hi ? pair >> 16 : pair & 0xffff)));
}

// One trellis position: relax every edge pair from cin into cout and, if RECORD, store the choices of the position.
template <int K, int cb, bool RECORD>
__device__ __forceinline__ void viterbi_step(const float* cin, float* cout, uint32_t* bp_pos, float x, int tid)
{
    using G = EncGeom<K>;
    const int lane = tid & 31;
    float staged[K == 1 ? G::PPT : 1][2];
    if constexpr (K == 1)
    {
        // the pair (2j, 2j+1) continues edges j and j + NP; read all of them before anyone overwrites the single buffer
        #pragma unroll
        for (int i = 0; i < G::PPT; ++i)
        {
            const int j = tid + i * G::NT;
            staged[i][0] = cin[j];
            staged[i][1] = cin[j + G::NP];
        }
        __syncthreads();
    }
    #pragma unroll (K == 1 ? G::PPT : 1)
    for (int i = 0; i < G::PPT; ++i)
    {
        const int pair = tid + i * G::NT;
        const uint32_t e0 = 2u * pair;
        float best0 = __int_as_float(0x7f800000), best1 = best0;
        int arg0 = 0, arg1 = 0;
        #pragma unroll 16
        for (int k = 0; k < (1 << K); ++k)
        {
            const uint32_t s0 = ((uint32_t) k << G::Kr) | e0;          // s0 and s0 + 1 continue the same edge s0 >> K
            float c;
            if constexpr (K == 1) c = staged[i][k];
            else                  c = cin[s0 >> K];
            const uint32_t v = decode_pair<cb>(s0, s0 + 1);
            const float d0 = value_f32(v, 0) - x, d1 = value_f32(v, 1) - x;
            const float c0 = fmaf(d0, d0, c), c1 = fmaf(d1, d1, c);
            if constexpr (RECORD)
            {
                if (c0 < best0) { best0 = c0; arg0 = k; }
                if (c1 < best1) { best1 = c1; arg1 = k; }
            }
            else
            {
                best0 = fminf(best0, c0);
                best1 = fminf(best1, c1);
            }
        }
        *reinterpret_cast<float2*>(cout + e0) = make_float2(best0, best1);
        if constexpr (RECORD)
        {
            uint32_t word = 0;
            #pragma unroll
            for (int b = 0; b < K; ++b)
            {
                const uint32_t w0 = __ballot_sync(0xffffffffu, (arg0 >> b) & 1);
                const uint32_t w1 = __ballot_sync(0xffffffffu, (arg1 >> b) & 1);
                if (lane == 2 * b) word = w0;
                if (lane == 2 * b + 1) word = w1;
            }
            if (lane < 2 * K) bp_pos[(pair >> 5) * 2 * K + lane] = word;
        }
    }
    __syncthreads();
}

// choice k recorded for edge e at position p
template <int K>
__device__ __forceinline__ uint32_t bp_choice(const uint32_t* bp, int p, uint32_t e)
{
    using G = EncGeom<K>;
    const uint32_t pair = e >> 1, bit = pair & 31;
    const uint32_t* w = bp + ((size_t) p * G::NC + (pair >> 5)) * 2 * K + (e & 1);
    uint32_t k = 0;
    #pragma unroll
    for (int b = 0; b < K; ++b) k |= ((w[2 * b] >> bit) & 1u) << b;
    return k;
}

template <int K, int cb>
__global__ void __launch_bounds__(EncGeom<K>::NT)
quantize_tiles_kernel(const float* __restrict__ in, float* __restrict__ out_values, uint16_t* __restrict__ out_states,
                      uint32_t* __restrict__ bp_all, int64_t num_tiles)
{
    using G = EncGeom<K>;
    extern __shared__ float4 smem4[];
    float* xs = reinterpret_cast<float*>(smem4);
    float* cost = xs + 256;
    uint16_t* path = reinterpret_cast<uint16_t*>(cost + G::COST_BUFS * G::E);
    float* red_c = reinterpret_cast<float*>(path + 256);
    int* red_i = reinterpret_cast<int*>(red_c + 32);
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    uint32_t* bp = bp_all + (size_t) blockIdx.x * G::BP_WORDS;
    const float inf = __int_as_float(0x7f800000);

    for (int64_t tile = blockIdx.x; tile < num_tiles; tile += gridDim.x)
    {
        __syncthreads();                                               // previous tile's readers of xs / path are done
        for (int i = tid; i < 256; i += G::NT) xs[i] = in[tile * 256 + i];
        for (int i = tid; i < G::E; i += G::NT) cost[i] = 0.0f;
        __syncthreads();

        // pass 1: positions 128 .. 255, 0 .. 127 from a free start; only the choices of 0 .. 127 are ever read back
        int cur = 0;
        for (int i = 0; i < 256; ++i)
        {
            const int p = (128 + i) & 255;
            float* cin = cost + cur * G::E;
            float* cout = cost + (G::COST_BUFS - 1 - cur) * G::E;
            if (i < 128) viterbi_step<K, cb, false>(cin, cout, nullptr, xs[p], tid);
            else         viterbi_step<K, cb, true>(cin, cout, bp + (size_t) p * G::NC * 2 * K, xs[p], tid);
            cur = G::COST_BUFS - 1 - cur;
        }

        // cheapest final edge, lowest index on ties
        const float* fin = cost + cur * G::E;
        float bc = inf; int bi = G::E;
        for (int e = tid; e < G::E; e += G::NT)
            if (fin[e] < bc) { bc = fin[e]; bi = e; }
        #pragma unroll
        for (int o = 16; o > 0; o >>= 1)
        {
            const float oc = __shfl_xor_sync(0xffffffffu, bc, o);
            const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
            if (oc < bc || (oc == bc && oi < bi)) { bc = oc; bi = oi; }
        }
        if (lane == 0) { red_c[warp] = bc; red_i[warp] = bi; }
        __syncthreads();
        if (warp == 0)
        {
            bc = lane < G::NT / 32 ? red_c[lane] : inf;
            bi = lane < G::NT / 32 ? red_i[lane] : G::E;
            #pragma unroll
            for (int o = 16; o > 0; o >>= 1)
            {
                const float oc = __shfl_xor_sync(0xffffffffu, bc, o);
                const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
                if (oc < bc || (oc == bc && oi < bi)) { bc = oc; bi = oi; }
            }
            if (lane == 0)
            {
                // back from position 127 to 0: the edge left before position 0 is the anchor
                uint32_t e = (uint32_t) bi;
                for (int p = 127; p >= 0; --p) e = ((bp_choice<K>(bp, p, e) << G::Kr) | e) >> K;
                red_i[0] = (int) e;
            }
        }
        __syncthreads();
        const int anchor = red_i[0];

        // pass 2: positions 0 .. 255, starting from the anchor edge only
        for (int i = tid; i < G::E; i += G::NT) cost[cur * G::E + i] = i == anchor ? 0.0f : inf;
        __syncthreads();
        for (int p = 0; p < 256; ++p)
        {
            float* cin = cost + cur * G::E;
            float* cout = cost + (G::COST_BUFS - 1 - cur) * G::E;
            viterbi_step<K, cb, true>(cin, cout, bp + (size_t) p * G::NC * 2 * K, xs[p], tid);
            cur = G::COST_BUFS - 1 - cur;
        }
        if (tid == 0)
        {
            uint32_t e = (uint32_t) anchor;                            // s[255] must pass on the anchor edge
            for (int p = 255; p >= 0; --p)
            {
                const uint32_t s = (bp_choice<K>(bp, p, e) << G::Kr) | e;
                path[p] = (uint16_t) s;
                e = s >> K;
            }
        }
        __syncthreads();
        for (int p = tid; p < 256; p += G::NT)
        {
            const uint32_t s = path[p];
            out_states[tile * 256 + p] = (uint16_t) s;
            out_values[tile * 256 + p] = value_f32(decode_pair<cb>(s, s), 0);
        }
    }
}

template <int K, int cb>
int launch_quantize_kc(cudaStream_t stream, const float* in, float* out_values, uint16_t* out_states, int64_t num_tiles,
                       uint32_t* scratch, int num_sms, int* grid_out)
{
    using G = EncGeom<K>;
    auto kern = quantize_tiles_kernel<K, cb>;
    EXL3B_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int) G::SMEM));
    int per_sm = 0;
    EXL3B_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, kern, G::NT, G::SMEM));
    EXL3B_CHECK(per_sm >= 1, EXL3B_ERR_CUDA, "quantize_tiles: kernel K=%d does not fit on an SM", K);
    int64_t grid = (int64_t) per_sm * num_sms;
    const int64_t fit = (int64_t) (ENC_SCRATCH_PER_SM * num_sms / ((size_t) G::BP_WORDS * 4));
    if (grid > fit) grid = fit;
    if (grid > num_tiles) grid = num_tiles;
    kern<<<(int) grid, G::NT, G::SMEM, stream>>>(in, out_values, out_states, scratch, num_tiles);
    EXL3B_CUDA(cudaPeekAtLastError());
    count_launch();
    *grid_out = (int) grid;
    return 0;
}

// The packed stream: the low K bits of every state, MSB first, as big-endian 16-bit words, pairwise swapped per 32-bit word.
template <int K>
__global__ void __launch_bounds__(256)
pack_trellis_kernel(uint16_t* __restrict__ packed, const uint16_t* __restrict__ unpacked, int64_t num_words)
{
    const int64_t g = (int64_t) blockIdx.x * 256 + threadIdx.x;
    if (g >= num_words) return;
    const int64_t tile = g / (16 * K);
    const int w = (int) (g - tile * 16 * K);
    const uint16_t* s = unpacked + tile * 256;
    uint32_t v = 0;
    #pragma unroll
    for (int i = 0; i < 16; ++i)
    {
        const int b = 16 * w + i, t = b / K;
        v = (v << 1) | ((s[t] >> (K - 1 - (b - t * K))) & 1u);
    }
    packed[tile * 16 * K + (w ^ 1)] = (uint16_t) v;
}

template <int K>
int launch_pack_k(cudaStream_t stream, uint16_t* packed, const uint16_t* unpacked, int64_t num_tiles)
{
    const int64_t words = num_tiles * 16 * K;
    const int64_t blocks = (words + 255) / 256;
    EXL3B_CHECK(blocks <= 0x7fffffff, EXL3B_ERR_SHAPE, "pack_trellis: too many tiles (%lld)", (long long) num_tiles);
    pack_trellis_kernel<K><<<(unsigned) blocks, 256, 0, stream>>>(packed, unpacked, words);
    EXL3B_CUDA(cudaPeekAtLastError());
    count_launch();
    return 0;
}

template <int K, int cb>
void quantize_dispatch(int* r, cudaStream_t stream, const float* in, float* out_values, uint16_t* out_states, int64_t num_tiles,
                       uint32_t* scratch, int num_sms, int* grid_out)
{
    *r = launch_quantize_kc<K, cb>(stream, in, out_values, out_states, num_tiles, scratch, num_sms, grid_out);
}

std::mutex g_enc_mu;
uint32_t* g_enc_scratch[32];

}  // namespace

int launch_quantize_tiles(cudaStream_t stream, DevCtx* ctx, const float* in, float* out_values, uint16_t* out_states,
                          int64_t num_tiles, int K, int cb)
{
    uint32_t* scratch;
    {
        std::lock_guard<std::mutex> lock(g_enc_mu);
        uint32_t*& s = g_enc_scratch[ctx->device & 31];
        if (!s)
        {
            cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
            EXL3B_CUDA(cudaStreamIsCapturing(stream, &cs));
            EXL3B_CHECK(cs == cudaStreamCaptureStatusNone, EXL3B_ERR_UNSUPPORTED,
                        "quantize_tiles: the first call on a device allocates its scratch; make it outside stream capture");
            EXL3B_CUDA(cudaMalloc(&s, ENC_SCRATCH_PER_SM * ctx->num_sms));
        }
        scratch = s;
    }
    int grid = 0, r = 0;
    EXL3B_DISPATCH_K_CB(quantize_dispatch, K, cb, &r, stream, in, out_values, out_states, num_tiles, scratch, ctx->num_sms, &grid);
    return r;
}

int launch_pack_trellis(cudaStream_t stream, uint16_t* packed, const uint16_t* unpacked, int64_t num_tiles, int K)
{
    switch (K)
    {
        case 1: return launch_pack_k<1>(stream, packed, unpacked, num_tiles);
        case 2: return launch_pack_k<2>(stream, packed, unpacked, num_tiles);
        case 3: return launch_pack_k<3>(stream, packed, unpacked, num_tiles);
        case 4: return launch_pack_k<4>(stream, packed, unpacked, num_tiles);
        case 5: return launch_pack_k<5>(stream, packed, unpacked, num_tiles);
        case 6: return launch_pack_k<6>(stream, packed, unpacked, num_tiles);
        case 7: return launch_pack_k<7>(stream, packed, unpacked, num_tiles);
        default: return launch_pack_k<8>(stream, packed, unpacked, num_tiles);
    }
}

}  // namespace exl3b
