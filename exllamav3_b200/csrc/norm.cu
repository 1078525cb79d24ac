// RMSNorm operators (exl3b_rms_norm, exl3b_gated_rms_norm): the reference's rms_norm / rms_norm_res_in / gated_rms_norm
// (exllamav3_ext/norm.cu), computed in fp32.
//
//   rms_norm        v = (x * w) * rmf,  rmf = rsqrt(sum(x^2) / dim + eps) * constant_scale,  w = w + constant_bias (or 1)
//                   RES_NONE  y = v                 RES_POST  y = y + v (fp32, rounded once)
//                   RES_IN    r = round_r(x + r), then v is taken of that r instead of x; y fp16
//                   fp16 x is clamped to +-65504 where it is read; r and the old y are not.
//   gated_rms_norm  bf16 x, s = silu(g):  gate_first  y = norm(x * s) * w,  else  y = (norm(x) * w) * s;  w row i % w_groups
//
// One HBM read of every input: a row is loaded once, with 16-byte vectors where the row allows it (E = 8 elements per load
// unit, else 4), and kept in registers from the load to the store.  A row is owned by `tpr` threads (a power of two, about
// two load units each; up to 512), so short rows (head norms) share a CTA of 256 threads and long rows have a CTA of their
// own.  Every load of the row, of w and of the old y is issued before the reduction, so a decode call costs one memory round
// trip for the inputs instead of one for x and one for w.  The sum of squares is reduced in a fixed order (per thread, then
// xor-shuffles, then the warp sums in warp order), so the result of a row depends on its values, dim and the unit width only:
// not on the row count, the row's position in the call or earlier calls.
#include "act.cuh"
#include "ptx.cuh"
#include <cuda_bf16.h>
#include <type_traits>

namespace exl3b {

using namespace ptx;
using bf16 = __nv_bfloat16;

constexpr int NORM_CTA = 256;          // threads of a CTA that holds several rows
constexpr int NORM_MAX_TPR = 512;      // threads of one row, at most
constexpr int NORM_UNITS = 4;          // load units per thread the registers are sized for (E = 8; 8 units of E = 4)
static_assert(NORM_MAX_TPR * NORM_UNITS * 8 == NORM_MAX_DIM, "a row of NORM_MAX_DIM elements fills the registers of its threads");

// E consecutive elements of one tensor, as loaded: E * sizeof(T) bytes in 8-, 16- or 32-byte vectors
template <typename T, int E>
struct Pack
{
    static constexpr int WORDS = E * (int) sizeof(T) / 4;
    uint32_t w[WORDS];

    __device__ __forceinline__ void load(const T* p)
    {
        if constexpr (WORDS == 2)
        {
            const uint2 a = *reinterpret_cast<const uint2*>(p);
            w[0] = a.x; w[1] = a.y;
        }
        else
        {
            #pragma unroll
            for (int i = 0; i < WORDS / 4; ++i)
            {
                const uint4 a = reinterpret_cast<const uint4*>(p)[i];
                w[4 * i] = a.x; w[4 * i + 1] = a.y; w[4 * i + 2] = a.z; w[4 * i + 3] = a.w;
            }
        }
    }

    __device__ __forceinline__ float get(int e) const
    {
        if constexpr (std::is_same_v<T, float>) return __uint_as_float(w[e]);
        else if constexpr (std::is_same_v<T, half>)
        {
            const half2 h = *reinterpret_cast<const half2*>(&w[e / 2]);
            return e & 1 ? __high2float(h) : __low2float(h);
        }
        else
        {
            const __nv_bfloat162 h = *reinterpret_cast<const __nv_bfloat162*>(&w[e / 2]);
            return e & 1 ? __high2float(h) : __low2float(h);
        }
    }

    // f rounded to T (round to nearest even); T is fp16 or fp32
    __device__ __forceinline__ void set(const float (&f)[E])
    {
        #pragma unroll
        for (int e = 0; e < E; ++e)
        {
            if constexpr (std::is_same_v<T, float>) w[e] = __float_as_uint(f[e]);
            else if (e % 2 == 0) w[e / 2] = pack_half2(__float2half_rn(f[e]), __float2half_rn(f[e + 1]));
        }
    }

    __device__ __forceinline__ void store(T* p) const
    {
        if constexpr (WORDS == 2) *reinterpret_cast<uint2*>(p) = make_uint2(w[0], w[1]);
        else
        {
            #pragma unroll
            for (int i = 0; i < WORDS / 4; ++i)
                reinterpret_cast<uint4*>(p)[i] = make_uint4(w[4 * i], w[4 * i + 1], w[4 * i + 2], w[4 * i + 3]);
        }
    }
};

// Sum over the `tpr` threads of a row (aligned groups of tpr consecutive threads), in a fixed order: xor-shuffles inside the
// warp, then, for rows wider than a warp, the warp sums of the row reduced the same way.  Every thread of the CTA calls it.
__device__ __forceinline__ float row_sum(float s, int tpr)
{
    __shared__ float warp_sums[NORM_MAX_TPR / 32];
    const int width = tpr < 32 ? tpr : 32;
    for (int o = width / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (tpr <= 32) return s;
    const int lane = threadIdx.x % 32, warp = threadIdx.x / 32, nw = tpr / 32;
    if (lane == 0) warp_sums[warp] = s;
    __syncthreads();
    // every aligned group of nw lanes holds the row's warp sums in warp order, so every lane ends with the same sum
    s = warp_sums[warp / nw * nw + lane % nw];
    for (int o = nw / 2; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    return s;
}

template <int MODE, typename XT, typename WT, typename YT, typename RT, int E>
__global__ void __launch_bounds__(NORM_MAX_TPR)
rms_norm_kernel(const XT* x, const WT* w, YT* y, RT* r, long long rows, int dim, int tpr, float eps, float bias, float scale)
{
    constexpr int V = NORM_UNITS * 8 / E;
    pdl_launch_dependents();
    const int t = threadIdx.x % tpr;
    const long long row = (long long) blockIdx.x * (blockDim.x / tpr) + threadIdx.x / tpr;
    const bool live = row < rows;
    const int units = dim / E;
    const size_t base = (size_t) row * dim;

    Pack<XT, E> xp[V];
    Pack<RT, E> rp[V];
    Pack<WT, E> wp[V];
    Pack<YT, E> yp[V];
    pdl_wait();                                     // x, r and the old y may be the previous kernel's output
    if (live)
    {
        #pragma unroll
        for (int i = 0; i < V; ++i)
        {
            const int u = t + i * tpr;
            if (u >= units) break;
            xp[i].load(x + base + (size_t) u * E);
            if constexpr (MODE == EXL3B_RES_IN) rp[i].load(r + base + (size_t) u * E);
            if (w) wp[i].load(w + (size_t) u * E);
            if constexpr (MODE == EXL3B_RES_POST) yp[i].load(y + base + (size_t) u * E);
        }
    }

    float v[V][E];
    float s = 0.0f;
    #pragma unroll
    for (int i = 0; i < V; ++i)
    {
        const int u = t + i * tpr;
        if (!live || u >= units) break;
        #pragma unroll
        for (int e = 0; e < E; ++e)
        {
            v[i][e] = xp[i].get(e);
            if constexpr (std::is_same_v<XT, half>) v[i][e] = fminf(fmaxf(v[i][e], -65504.0f), 65504.0f);
        }
        if constexpr (MODE == EXL3B_RES_IN)
        {
            float sum[E];
            #pragma unroll
            for (int e = 0; e < E; ++e) sum[e] = v[i][e] + rp[i].get(e);
            rp[i].set(sum);
            rp[i].store(r + base + (size_t) u * E);
            #pragma unroll
            for (int e = 0; e < E; ++e) v[i][e] = rp[i].get(e);
        }
        #pragma unroll
        for (int e = 0; e < E; ++e) s = fmaf(v[i][e], v[i][e], s);
    }
    s = row_sum(s, tpr);
    const float rmf = rsqrtf(s / (float) dim + eps) * scale;
    if (!live) return;

    #pragma unroll
    for (int i = 0; i < V; ++i)
    {
        const int u = t + i * tpr;
        if (u >= units) break;
        float o[E];
        #pragma unroll
        for (int e = 0; e < E; ++e)
        {
            // products kept apart from the POST add (no fma contraction): POST is exactly the old y plus NONE's value
            o[e] = w ? __fmul_rn(__fmul_rn(v[i][e], bias != 0.0f ? wp[i].get(e) + bias : wp[i].get(e)), rmf)
                     : __fmul_rn(v[i][e], rmf);
            if constexpr (MODE == EXL3B_RES_POST) o[e] = o[e] + yp[i].get(e);
        }
        Pack<YT, E> out;
        out.set(o);
        out.store(y + base + (size_t) u * E);
    }
}

template <typename WT, typename YT, typename GT, int E>
__global__ void __launch_bounds__(NORM_MAX_TPR)
gated_rms_norm_kernel(const bf16* x, const WT* w, YT* y, const GT* g, long long rows, int dim, int tpr, float eps, float bias,
                      int w_groups, int gate_first)
{
    constexpr int V = NORM_UNITS * 8 / E;
    pdl_launch_dependents();
    const int t = threadIdx.x % tpr;
    const long long row = (long long) blockIdx.x * (blockDim.x / tpr) + threadIdx.x / tpr;
    const bool live = row < rows;
    const int units = dim / E;
    const size_t base = (size_t) row * dim;
    const WT* w_row = w + (size_t) (live ? row % w_groups : 0) * dim;

    Pack<bf16, E> xp[V];
    Pack<GT, E> gp[V];
    Pack<WT, E> wp[V];
    pdl_wait();
    if (live)
    {
        #pragma unroll
        for (int i = 0; i < V; ++i)
        {
            const int u = t + i * tpr;
            if (u >= units) break;
            xp[i].load(x + base + (size_t) u * E);
            gp[i].load(g + base + (size_t) u * E);
            wp[i].load(w_row + (size_t) u * E);
        }
    }

    float v[V][E], sg[V][E];
    float s = 0.0f;
    #pragma unroll
    for (int i = 0; i < V; ++i)
    {
        const int u = t + i * tpr;
        if (!live || u >= units) break;
        #pragma unroll
        for (int e = 0; e < E; ++e)
        {
            sg[i][e] = act_silu(gp[i].get(e));
            v[i][e] = gate_first ? xp[i].get(e) * sg[i][e] : xp[i].get(e);
            s = fmaf(v[i][e], v[i][e], s);
        }
    }
    s = row_sum(s, tpr);
    const float rmf = rsqrtf(s / (float) dim + eps);
    if (!live) return;

    #pragma unroll
    for (int i = 0; i < V; ++i)
    {
        const int u = t + i * tpr;
        if (u >= units) break;
        float o[E];
        #pragma unroll
        for (int e = 0; e < E; ++e)
        {
            const float we = bias != 0.0f ? wp[i].get(e) + bias : wp[i].get(e);
            o[e] = __fmul_rn(__fmul_rn(v[i][e], we), rmf);
            if (!gate_first) o[e] = __fmul_rn(o[e], sg[i][e]);
        }
        Pack<YT, E> out;
        out.set(o);
        out.store(y + base + (size_t) u * E);
    }
}

// ---- host ---------------------------------------------------------------------------------------------------------------

// threads per row: a power of two giving each thread about two load units, within [1, NORM_MAX_TPR]
int norm_threads_per_row(int dim, int e)
{
    const int units = dim / e;
    int tpr = 1;
    while (tpr < NORM_MAX_TPR && 2 * tpr < units) tpr *= 2;
    return tpr;
}

// grid and CTA for `rows` rows of `tpr` threads: one row per CTA from 256 threads up, else 256 / tpr rows per CTA
static void norm_geometry(long long rows, int tpr, dim3* grid, int* threads)
{
    *threads = tpr >= NORM_CTA ? tpr : NORM_CTA;
    const long long per_cta = *threads / tpr;
    *grid = dim3((unsigned) ((rows + per_cta - 1) / per_cta));
}

template <typename F>
static int with_dtype(int dt, F&& f)
{
    if (dt == EXL3B_DTYPE_FP16) return f(half{});
    if (dt == EXL3B_DTYPE_FP32) return f(float{});
    return f(bf16{});
}

template <int MODE>
static int launch_rms_norm_mode(cudaStream_t stream, const NormArgs& a, dim3 grid, int threads, int tpr)
{
    // the reference's 24 combinations (exl3b_rms_norm checked them): w fp16 when absent, r of the x dtype unless RES_IN
    const int w_dt = a.w ? a.w_dtype : EXL3B_DTYPE_FP16;
    const int r_dt = MODE == EXL3B_RES_IN ? a.r_dtype : a.x_dtype;
    return with_dtype(a.x_dtype, [&](auto xt) { return with_dtype(w_dt, [&](auto wt) {
           return with_dtype(a.y_dtype, [&](auto yt) { return with_dtype(r_dt, [&](auto rt) {
        using XT = decltype(xt); using WT = decltype(wt); using YT = decltype(yt); using RT = decltype(rt);
        constexpr bool ok = !std::is_same_v<XT, bf16> && !std::is_same_v<WT, float> && !std::is_same_v<YT, bf16>
                            && !std::is_same_v<RT, bf16> && (MODE == EXL3B_RES_IN ? std::is_same_v<YT, half> : std::is_same_v<RT, XT>);
        if constexpr (!ok) return fail(EXL3B_ERR_ARG, "rms_norm: Invalid datatypes for input/output");
        else
        {
            const cudaError_t e = a.e == 8
                ? launch_pdl<rms_norm_kernel<MODE, XT, WT, YT, RT, 8>>(stream, grid, threads, 0, (const XT*) a.x, (const WT*) a.w,
                      (YT*) a.y, (RT*) a.r, a.rows, a.dim, tpr, a.eps, a.bias, a.scale)
                : launch_pdl<rms_norm_kernel<MODE, XT, WT, YT, RT, 4>>(stream, grid, threads, 0, (const XT*) a.x, (const WT*) a.w,
                      (YT*) a.y, (RT*) a.r, a.rows, a.dim, tpr, a.eps, a.bias, a.scale);
            count_launch();
            EXL3B_CUDA(e);
            return 0;
        }
    }); }); }); });
}

int launch_rms_norm(cudaStream_t stream, const NormArgs& a)
{
    const int tpr = norm_threads_per_row(a.dim, a.e);
    dim3 grid; int threads;
    norm_geometry(a.rows, tpr, &grid, &threads);
    if (a.res_mode == EXL3B_RES_IN) return launch_rms_norm_mode<EXL3B_RES_IN>(stream, a, grid, threads, tpr);
    if (a.res_mode == EXL3B_RES_POST) return launch_rms_norm_mode<EXL3B_RES_POST>(stream, a, grid, threads, tpr);
    return launch_rms_norm_mode<EXL3B_RES_NONE>(stream, a, grid, threads, tpr);
}

int launch_gated_rms_norm(cudaStream_t stream, const NormArgs& a)
{
    const int tpr = norm_threads_per_row(a.dim, a.e);
    dim3 grid; int threads;
    norm_geometry(a.rows, tpr, &grid, &threads);
    return with_dtype(a.w_dtype, [&](auto wt) { return with_dtype(a.y_dtype, [&](auto yt) { return with_dtype(a.g_dtype, [&](auto gt) {
        using WT = decltype(wt); using YT = decltype(yt); using GT = decltype(gt);
        constexpr bool ok = !std::is_same_v<WT, half> && !std::is_same_v<YT, bf16> && !std::is_same_v<GT, half>;
        if constexpr (!ok) return fail(EXL3B_ERR_ARG, "gated_rms_norm: Invalid datatypes for input/output");
        else
        {
            const cudaError_t e = a.e == 8
                ? launch_pdl<gated_rms_norm_kernel<WT, YT, GT, 8>>(stream, grid, threads, 0, (const bf16*) a.x, (const WT*) a.w,
                      (YT*) a.y, (const GT*) a.g, a.rows, a.dim, tpr, a.eps, a.bias, a.w_groups, a.gate_first)
                : launch_pdl<gated_rms_norm_kernel<WT, YT, GT, 4>>(stream, grid, threads, 0, (const bf16*) a.x, (const WT*) a.w,
                      (YT*) a.y, (const GT*) a.g, a.rows, a.dim, tpr, a.eps, a.bias, a.w_groups, a.gate_first);
            count_launch();
            EXL3B_CUDA(e);
            return 0;
        }
    }); }); });
}

}  // namespace exl3b
