// Shared declarations of the tensor-core kernels (exact fp16 path: gemm_tc.cu, moe_tc.cu; int8 codebook path: gemm_tc_i8.cu).
#pragma once
#include "common.cuh"
#include "decode.cuh"
#include "epilogue.cuh"
#include "ptx.cuh"
#include <cuda.h>

namespace exl3b {

constexpr int TC_THREADS = 768;
constexpr int TC_XF_WARP0 = 2;               // warps 2,3: in-kernel input transform (small m)
constexpr int TC_DEC_WARP0 = 4;
constexpr int TC_DEC_WARPS = 16;             // four decode warpgroups
constexpr int TC_EPI_WARP0 = TC_DEC_WARP0 + TC_DEC_WARPS;
constexpr int TC_MAX_STAGES = 16;
constexpr int TC_RAG_MAX_MATS = 8;          // matrices of a fan-out launch (per-matrix widths)

struct TcParams
{
    const uint8_t* xh_tiled;     // [k/128][NT/8][16][8][8] fp16 (core-matrix tiles)
    const uint32_t* B;
    void* C;
    const half* svh;
    int m, k, n, NT;
    int c_fp32;
    float out_scale;
    float* ws;
    int* counters;
    int stages;                  // smem ring depth
    int b_bytes;                 // bytes reserved per activation stage
    int b_load_bytes;            // bytes of the activation tile copied per unit
    const half* A_raw;           // int8 kernels: raw activations (m, k), transformed in-kernel with suh
    const half* suh;
    // multi-matrix launch (exl3_mgemm, dense case): the grid is num_mats groups of g_per_mat CTAs, group j works on
    // matrix j exactly like a single-matrix launch with g_per_mat CTAs.  num_mats == 0: single matrix, fields unused.
    int num_mats, g_per_mat;
    const uint64_t* B_ptrs; const uint64_t* suh_ptrs; const uint64_t* svh_ptrs;
    long long a_mat_stride;      // elements between the inputs of consecutive matrices (0 = shared input)
    long long c_mat_stride;      // bytes between the outputs of consecutive matrices
    // fan-out (exl3_mgemm with per-matrix output widths, size_n_list / c_ptrs): matrix j is rag_n[j] columns wide, writes to
    // c_ptrs[j] (device table) with row stride rag_n[j], and owns the CTAs rag_cta0[j] .. rag_cta0[j + 1] - 1 (proportional
    // to its number of units).  rag == 0: uniform widths, fields unused.
    int rag;
    int rag_n[TC_RAG_MAX_MATS];
    int rag_cta0[TC_RAG_MAX_MATS + 1];
    const uint64_t* c_ptrs;
    float* parts;                // i8 path: sentinel-managed split-K exchange buffer (one 4 x 128 fp32 slot per CTA)
    uint8_t* tmap_slots;         // one 128-byte tensor-map slot per CTA (global memory)
    unsigned long long* dbg;     // optional per-CTA timeline (16 x u64 per CTA), bring-up only
};

// Tensor-parallel group of this device for the row-parallel GEMM whose epilogue sums the ranks' partial outputs over
// NVLink peer memory (gemm_tc_i8_ar.cu).  recv[j] = rank j's receive buffer as mapped into THIS process (recv[rank] is
// local memory); every buffer is [AR_SLOTS][world][slot_elems] 32-bit words holding the sentinel outside a launch.
constexpr int AR_MAX_WORLD = 8;
constexpr int AR_SLOTS = 2;
struct ArArgs
{
    uint32_t* recv[AR_MAX_WORLD];
    unsigned int* state;         // local device memory: [0] epoch (AR launches completed), [1] CTA arrival ticket
    long long slot_elems;        // words per (slot, source rank)
    int rank, world;
};

// Routed multi-matrix launch (exl3_mgemm with indices / weights / expert-range filter): the active-slot table of the call
struct RouteArgs
{
    const MSlotTable* tab;       // written by mgemm_resolve_kernel earlier on the same stream
    int has_weights;             // multiply each slot's output by tab->weight[slot]
};

struct TcSmemLayout
{
    int w_bytes, b_bytes, off_b, off_tile, off_bars, off_d, total;
};

__host__ __device__ inline TcSmemLayout tc_smem_layout(int K, int b_bytes, int stages)
{
    TcSmemLayout L;
    L.w_bytes = 2048 * K;
    L.b_bytes = b_bytes;
    L.off_b = stages * L.w_bytes;
    L.off_tile = L.off_b + stages * L.b_bytes;
    L.off_bars = L.off_tile + 16 * 128 * 4;
    L.total = L.off_bars + 1024;
    L.off_d = L.total;
    return L;
}

// ---- work partition helpers -------------------------------------------------------------------------------------
// (host + device: the CPU tests walk the same partition the kernels use, exl3b_plan_* in api.cu)
// 32-bit arithmetic: a 64-bit division is a subroutine call in SASS, and a call inside a kernel that issues wgmma makes
// ptxas serialize every wgmma of it.  The planners only launch grids for which partition_fits(U, G) holds, so U * c and
// (g + 1) * G - 1 (c <= G, g < U) never exceed 32 unsigned bits.
__host__ __device__ __forceinline__ bool partition_fits(long long U, long long G)
{
    return U >= 1 && G >= 1 && U <= 0x7fffffffll && U * G <= 0xffffffffll;
}
__host__ __device__ __forceinline__ int unit_begin(int U, int G, int c) { return (int) ((uint32_t) U * (uint32_t) c / (uint32_t) G); }
__host__ __device__ __forceinline__ int cta_of_unit(int U, int G, int g)
{
    return (int) ((((uint32_t) g + 1u) * (uint32_t) G - 1u) / (uint32_t) U);
}


#ifdef __CUDACC__
// ---- input transform into the tiled activation layout ---------------------------------------------------------
// Tile of one unit: [NT / 8 row groups][16 K-chunks][8 rows][8 fp16], K-chunks 128 B apart, row groups 2048 B apart.  K order:
// k = 16 kt + 4 j + 2 h + e (kt = 4 r + c) sits in K-chunk 2 (4 r + j) + h at element 2 c + e, i.e. lane l's four values
// k = 4 l .. 4 l + 3 go to K-chunks 8 (l / 16) + 2 (l % 4) (+1 for the second pair), element pair (l / 4) % 4.
__device__ __forceinline__ int xt_tile_offset(int r, int lane)
{
    return (((r >> 3) * 16 + 8 * (lane >> 4) + 2 * (lane & 3)) * 8 + (r & 7)) * 16 + 4 * ((lane >> 2) & 3);
}
// the two 4-byte halves land 128 B apart (consecutive K-chunks)
__device__ __forceinline__ void store_tile_pair(uint8_t* p, uint2 o)
{
    *reinterpret_cast<uint32_t*>(p) = o.x;
    *reinterpret_cast<uint32_t*>(p + 128) = o.y;
}
// The input transform (had128_fp16) of lane's four values of one row, `suh` pointing at lane's four scales, as a tile pair
__device__ __forceinline__ uint2 xt_transform(uint2 raw, const half* suh, int lane)
{
    const uint2 scb = *reinterpret_cast<const uint2*>(suh);
    return had128_fp16(raw, &scb, lane);
}

// Bring-up timeline of the tensor-core kernels (EXL3B_TC_DEBUG builds, tools/i8_phase_profile.py): the %globaltimer into slot
// `slot` of this CTA's row of `dbg` (64 u64 per CTA; null: no stamp).  Compiles to nothing in the other builds.
__device__ __forceinline__ void tc_stamp([[maybe_unused]] unsigned long long* dbg, [[maybe_unused]] int slot)
{
#ifdef EXL3B_TC_DEBUG
    if (dbg) { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t) :: "memory"); dbg[blockIdx.x * 64 + slot] = t; }
#endif
}
#endif

int get_weight_tmap(const void* B, int k, int n, int K, CUtensorMap* out);
extern unsigned long long* g_tc_dbg;

// ---- int8 decode-GEMM launches (gemm_tc_i8.cu) ----------------------------------------------------------------------
// The TcParams every int8 launch shares, on launch slot `slot` with plan `pl`: one matrix (a), or the pointer tables of `mats`
// matrices (multi-matrix launches; g_per_mat and the fan-out fields are the caller's).
TcParams i8_params(DevCtx* ctx, int slot, const TcPlan& pl, const GemmArgs& a);
TcParams i8_params(DevCtx* ctx, int slot, const TcPlan& pl, const MGemmArgs& a, int mats);
// One launch of the kernel entry the extra arguments select: plain rows, or gated rows (gate), the row-parallel sum (ar) or
// routed slots (route).  Counted; 0 or the launch error.
int i8_launch(cudaStream_t stream, int K, int grid, int smem_bytes, const TcParams& p, const CUtensorMap& tmap,
              const GateIn* gate = nullptr, const ArArgs* ar = nullptr, const RouteArgs* route = nullptr);

}  // namespace exl3b
