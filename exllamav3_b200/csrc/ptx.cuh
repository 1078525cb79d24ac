// Thin inline-PTX wrappers for the sm_90a features this library uses: mbarrier, bulk async copy (TMA engine,
// SASS UBLKCP), wgmma (warpgroup MMA), programmatic dependent launch.
#pragma once
#include <stdint.h>
#include <cuda_runtime.h>

namespace exl3b { namespace ptx {

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t) __cvta_generic_to_shared(p); }

// One elected lane of a fully converged warp.  Keeping the surrounding control flow warp-uniform lets ptxas keep TMA
// operands in uniform registers instead of a per-lane R2UR loop.
__device__ __forceinline__ bool elect_one()
{
    uint32_t pred;
    asm volatile("{\n\t.reg .pred p;\n\telect.sync _|p, 0xffffffff;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(pred));
    return pred != 0;
}

// ---- mbarrier -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count)
{
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void fence_barrier_init()
{
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
__device__ __forceinline__ void fence_proxy_async_smem()
{
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar)
{
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_arrive_expect_tx(uint32_t bar, uint32_t bytes)
{
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
// try_wait with a suspend-time hint: the warp sleeps in hardware until the phase completes (or the hint expires)
// instead of polling, so waiting warps do not take issue slots from the decode warps.
__device__ __forceinline__ bool mbar_try_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity), "r"(0x989680u) : "memory");
    return ok != 0;
}
// non-blocking probe
__device__ __forceinline__ bool mbar_test_wait(uint32_t bar, uint32_t parity)
{
    uint32_t ok;
    asm volatile("{\n\t.reg .pred p;\n\t"
                 "mbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
                 "selp.u32 %0, 1, 0, p;\n\t}"
                 : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    return ok != 0;
}
// Watchdog of a bounded poll loop, called after every failed poll (polls and t0 start at 0): a protocol bug traps (reported
// as a CUDA error) instead of hanging the GPU.  The bound is wall-clock (%globaltimer, read every MASK + 1 polls), not an
// iteration count: an mbarrier try_wait returns early whenever ANY barrier activity wakes the warp, and a global-memory poll
// takes as long as the memory system makes it, so iteration counts say nothing about elapsed time.
// The timeout message is printed only in the bring-up build with messages (EXL3B_TC_DEBUG=2): printf is a function call, and any
// call in a kernel that issues wgmma makes ptxas wait for every wgmma on its own (C7510), so the timeline build
// (EXL3B_TC_DEBUG=1) leaves it out to time the production MMA schedule; the trap alone still ends the launch with an error.
template <uint32_t MASK, unsigned long long LIMIT_NS = 4000000000ull>
__device__ __forceinline__ void poll_watchdog(uint32_t& polls, unsigned long long& t0, const char* what, int a, int b)
{
    if ((++polls & MASK) == 0)
    {
        unsigned long long t;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
        if (t0 == 0) t0 = t;
        else if (t - t0 > LIMIT_NS)
        {
#if EXL3B_TC_DEBUG >= 2
            printf("exl3b: %s timeout (block %d thread %d: %d %d)\n", what, blockIdx.x, threadIdx.x, a, b);
#else
            (void) what; (void) a; (void) b;
#endif
            __trap();
        }
    }
}

// Bounded mbarrier wait (poll_watchdog, every 1024 polls).
// BACKOFF_NS > 0: exponential back-off (BACKOFF_NS, 2x, ... capped at 16x) between polls for roles whose waits can be
// long: polling warps otherwise burn issue slots the decode warps need.
template <int BACKOFF_NS = 0>
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity)
{
    if (mbar_try_wait(bar, parity)) return;
    uint32_t polls = 0;
    unsigned long long t0 = 0;
    [[maybe_unused]] uint32_t ns = BACKOFF_NS;
    while (!mbar_try_wait(bar, parity))
    {
        if constexpr (BACKOFF_NS > 0) { __nanosleep(ns); if (ns < 16u * BACKOFF_NS) ns <<= 1; }
        poll_watchdog<1023u>(polls, t0, "mbarrier", (int) bar, (int) parity);
    }
}

// mbar_wait for a phase that has usually completed already: one non-blocking test_wait first.
template <int BACKOFF_NS = 0>
__device__ __forceinline__ void mbar_wait_ready(uint32_t bar, uint32_t parity)
{
    if (mbar_test_wait(bar, parity)) return;
    mbar_wait<BACKOFF_NS>(bar, parity);
}

// ---- bulk async copy global -> shared (1-D), completion on an mbarrier ----------------------------------------
__device__ __forceinline__ uint64_t policy_evict_first()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ uint64_t policy_evict_last()
{
    uint64_t p;
    asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p));
    return p;
}
__device__ __forceinline__ void bulk_g2s(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t policy)
{
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(policy) : "memory");
}

// 2-D tiled TMA copy (SASS UTMALDG): box at element coordinates (c0 = innermost, c1 = row) of a CUtensorMap
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const void* tmap, int c0, int c1, uint32_t bar, uint64_t policy)
{
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes.L2::cache_hint"
                 " [%0], [%1, {%2, %3}], [%4], %5;"
                 :: "r"(dst), "l"(tmap), "r"(c0), "r"(c1), "r"(bar), "l"(policy) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const void* tmap)
{
    asm volatile("prefetch.tensormap [%0];" :: "l"(tmap) : "memory");
}

// ---- device-side tensor-map patching (multi-matrix launches: one template, per-CTA global address) ----------------
// smem_tmap: 128-byte aligned shared-memory copy of the template; gmem_tmap: this CTA's 128-byte slot in global memory.
// Warp-collective (cp_fenceproxy is .sync.aligned).  After this the slot can be used by cp.async.bulk.tensor.
__device__ __forceinline__ void tmap_patch_address(uint32_t smem_tmap, void* gmem_tmap, uint64_t new_addr, int lane)
{
    if (lane == 0)
        asm volatile("tensormap.replace.tile.global_address.shared::cta.b1024.b64 [%0], %1;" :: "r"(smem_tmap), "l"(new_addr) : "memory");
    __syncwarp();
    asm volatile("tensormap.cp_fenceproxy.global.shared::cta.tensormap::generic.release.gpu.sync.aligned [%0], [%1], 128;"
                 :: "l"(gmem_tmap), "r"(smem_tmap) : "memory");
    asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" :: "l"(gmem_tmap) : "memory");
}

// The same for a matrix whose WIDTH differs from the template's: innermost extent (elements) and row pitch (bytes) too.
// (global_stride takes the byte value as of CUDA 12.5; older assemblers wanted it >> 4.)
__device__ __forceinline__ void tmap_patch_address_width(uint32_t smem_tmap, void* gmem_tmap, uint64_t new_addr, uint32_t dim0_elems,
                                                         uint64_t pitch_bytes, int lane)
{
    if (lane == 0)
    {
        asm volatile("tensormap.replace.tile.global_address.shared::cta.b1024.b64 [%0], %1;" :: "r"(smem_tmap), "l"(new_addr) : "memory");
        asm volatile("tensormap.replace.tile.global_dim.shared::cta.b1024.b32 [%0], 0, %1;" :: "r"(smem_tmap), "r"(dim0_elems) : "memory");
        asm volatile("tensormap.replace.tile.global_stride.shared::cta.b1024.b64 [%0], 0, %1;" :: "r"(smem_tmap), "l"(pitch_bytes) : "memory");
    }
    __syncwarp();
    asm volatile("tensormap.cp_fenceproxy.global.shared::cta.tensormap::generic.release.gpu.sync.aligned [%0], [%1], 128;"
                 :: "l"(gmem_tmap), "r"(smem_tmap) : "memory");
    asm volatile("fence.proxy.tensormap::generic.acquire.gpu [%0], 128;" :: "l"(gmem_tmap) : "memory");
}

// ---- relaxed gpu-scope accesses (flag-in-data exchange through L2) ------------------------------------------------------
__device__ __forceinline__ uint32_t ld_relaxed_gpu_u32(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.relaxed.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_gpu_u32(uint32_t* p, uint32_t v)
{
    asm volatile("st.relaxed.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t ld_acquire_gpu_u32(const uint32_t* p)
{
    uint32_t v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_release_gpu_u32(uint32_t* p, uint32_t v)
{
    asm volatile("st.release.gpu.global.u32 [%0], %1;" :: "l"(p), "r"(v) : "memory");
}
__device__ __forceinline__ uint32_t atom_add_acq_rel_gpu_u32(uint32_t* p, uint32_t v)
{
    uint32_t old;
    asm volatile("atom.acq_rel.gpu.global.add.u32 %0, [%1], %2;" : "=r"(old) : "l"(p), "r"(v) : "memory");
    return old;
}

// ---- relaxed system-scope vector accesses (flag-in-data exchange between GPUs over NVLink peer memory) -------------------
// A vector access is a set of 32-bit accesses, each of them single-copy atomic: every word is its own flag.
__device__ __forceinline__ uint4 ld_relaxed_sys_v4(const uint32_t* p)
{
    uint4 v;
    asm volatile("ld.relaxed.sys.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void st_relaxed_sys_v4(uint32_t* p, uint4 v)
{
    asm volatile("st.relaxed.sys.global.v4.u32 [%0], {%1, %2, %3, %4};" :: "l"(p), "r"(v.x), "r"(v.y), "r"(v.z), "r"(v.w) : "memory");
}

// ---- programmatic dependent launch ------------------------------------------------------------------------------
__device__ __forceinline__ void pdl_wait() { asm volatile("griddepcontrol.wait;" ::: "memory"); }
__device__ __forceinline__ void pdl_launch_dependents() { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); }

// ---- wgmma (sm_90a warpgroup MMA) -------------------------------------------------------------------------------
// All four warps of a warpgroup (warps 4w .. 4w+3) execute these together.  The A operand comes from registers (the decode
// threads' own decoded weights), B from shared memory through a descriptor, D lives in registers.
// The .aligned instructions need every lane of the warp converged: lanes that left an mbarrier poll loop at different
// iterations are joined first.
__device__ __forceinline__ void wgmma_fence()  { __syncwarp(); asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait()   { asm volatile("wgmma.wait_group.sync.aligned %0;" :: "n"(N) : "memory"); }
// keeps the compiler from moving accesses of a register across the asynchronous MMA (or reusing it while the MMA reads it)
__device__ __forceinline__ void reg_fence(uint32_t& r) { asm volatile("" : "+r"(r) :: "memory"); }
__device__ __forceinline__ void reg_fence(float& r)    { asm volatile("" : "+f"(r) :: "memory"); }

// Shared-memory matrix descriptor of wgmma: start address, leading-dimension byte offset (K-adjacent core matrices for a
// K-major operand without swizzle, the unused 1 for a swizzled K-major one) and stride-dimension byte offset (8-row groups),
// all in 16-byte units; layout type in bits 62..63 (0 = no swizzle / 8 x 16 B core matrices, 1 = 128-byte swizzle).
__device__ __forceinline__ uint64_t smem_desc(uint32_t saddr, uint32_t lbo_bytes, uint32_t sbo_bytes, uint32_t layout_type)
{
    uint64_t d = 0;
    d |= (uint64_t) ((saddr >> 4) & 0x3fff);
    d |= (uint64_t) ((lbo_bytes >> 4) & 0x3fff) << 16;
    d |= (uint64_t) ((sbo_bytes >> 4) & 0x3fff) << 32;
    d |= (uint64_t) (layout_type & 3) << 62;
    return d;
}

// D[64 x 16] (f32) += A[64 x 16] (f16, registers) * B[16 x 16] (f16, shared memory, K-major)
__device__ __forceinline__ void wgmma_f16_n16(float (&d)[8], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc)
{
    asm volatile("wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1, 1, 1, 0;"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc) : "memory");
}

// D[64 x 8] (s32) += A[64 x 32] (u8, registers) * B[32 x 8] (s8, shared memory, K-major)
__device__ __forceinline__ void wgmma_u8s8_n8(uint32_t (&d)[4], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc)
{
    asm volatile("wgmma.mma_async.sync.aligned.m64n8k32.s32.u8.s8 {%0, %1, %2, %3}, {%4, %5, %6, %7}, %8, 1;"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc) : "memory");
}
// D[64 x 16] (s32) += A[64 x 32] (u8, registers) * B[32 x 16] (s8, shared memory, K-major)
__device__ __forceinline__ void wgmma_u8s8_n16(uint32_t (&d)[8], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc)
{
    asm volatile("wgmma.mma_async.sync.aligned.m64n16k32.s32.u8.s8 {%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, 1;"
                 : "+r"(d[0]), "+r"(d[1]), "+r"(d[2]), "+r"(d[3]), "+r"(d[4]), "+r"(d[5]), "+r"(d[6]), "+r"(d[7])
                 : "r"(a0), "r"(a1), "r"(a2), "r"(a3), "l"(b_desc) : "memory");
}
template <int MR>
__device__ __forceinline__ void wgmma_u8s8(uint32_t (&d)[MR], uint32_t a0, uint32_t a1, uint32_t a2, uint32_t a3, uint64_t b_desc)
{
    if constexpr (MR == 4) wgmma_u8s8_n8(d, a0, a1, a2, a3, b_desc);
    else wgmma_u8s8_n16(d, a0, a1, a2, a3, b_desc);
}

}}  // namespace exl3b::ptx
