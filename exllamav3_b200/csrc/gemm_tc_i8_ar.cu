// Row-parallel EXL3 decode-GEMM with the tensor-parallel sum fused into its epilogue (tag 211):
//
//      C = sum over ranks r of  had128( xh_r @ W_r ) * svh          (o_proj / down_proj of a tensor-parallel model)
//
// Replaces, for the row-parallel linears of the reference's TP mode, the pair  exl3_gemm  +  all_reduce  that its callers
// issue (modules/mlp.py:769-770, modules/attn.py:546-547 -> model/model_tp_backend.py:119-126, one NCCL launch per
// output): the kernel is gemm_tc_i8_body<K, 4, AR = true> (entry in gemm_tc_i8.cu) -- the same decode-GEMM, whose epilogue exchanges each finished
// 128-column segment with the peer GPUs through NVLink peer memory (flag-in-data, see emit_rows in gemm_tc_i8_body.cuh).
//
// Setup (one process per GPU): every rank allocates a receive buffer (tp_alloc), the ranks exchange the 64-byte CUDA IPC
// handles over their existing torch.distributed group, and map each other's buffers (tp_attach).  A loop-back mode maps
// "peer" buffers to local allocations so that the protocol can be exercised on one GPU (tests, bring-up).
//
// STATUS: world-1 equality with the plain kernel and the loop-back protocol (scatter, rank-ordered sum, re-arming, slot
// alternation) tested on one GPU; multi-GPU runs: tests/test_tp_fused.py -m multigpu, bench.py --gpus N.
#include "i8_pipeline.cuh"
#include <mutex>

namespace exl3b {

// bring-up: place a "peer" partial into the own receive buffer, in the slot the NEXT row-parallel launch will read
__global__ void tp_inject_kernel(const unsigned int* state, uint32_t* local, long long slot_elems, int world, int src,
                                 const uint32_t* data, long long count)
{
    const long long base = ((long long) (state[0] % AR_SLOTS) * world + src) * slot_elems;
    for (long long i = blockIdx.x * (long long) blockDim.x + threadIdx.x; i < count; i += (long long) gridDim.x * blockDim.x)
    {
        uint32_t v = data[i];
        if (v == I8_SENTINEL) v = 0x7fc00000u;
        local[base + i] = v;
    }
}

// ---- host side -------------------------------------------------------------------------------------------------------

struct TpGroup
{
    int rank = -1, world = 0;
    long long slot_elems = 0;
    uint32_t* local = nullptr;                    // own receive buffer [AR_SLOTS][world][slot_elems]
    unsigned int* state = nullptr;                // [0] epoch, [1] ticket
    uint32_t* recv[AR_MAX_WORLD] = {};            // recv[j] as mapped here
    bool peer_is_ipc[AR_MAX_WORLD] = {};
    bool attached = false;
};
static TpGroup g_tp[32];
static std::mutex g_tp_mutex;

static size_t tp_buffer_bytes(const TpGroup& g) { return (size_t) AR_SLOTS * g.world * g.slot_elems * sizeof(uint32_t); }

static int tp_current(TpGroup** out)
{
    int dev = -1;
    EXL3B_CUDA(cudaGetDevice(&dev));
    EXL3B_CHECK(dev >= 0 && dev < 32, EXL3B_ERR_CUDA, "device index %d out of range", dev);
    *out = &g_tp[dev];
    return 0;
}

int tp_free()
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    std::lock_guard<std::mutex> lock(g_tp_mutex);
    if (g->rank < 0) return 0;
    EXL3B_CUDA(cudaDeviceSynchronize());
    for (int j = 0; j < g->world; ++j)
    {
        if (j == g->rank || !g->recv[j]) continue;
        if (g->peer_is_ipc[j]) cudaIpcCloseMemHandle(g->recv[j]); else cudaFree(g->recv[j]);
    }
    if (g->local) cudaFree(g->local);
    if (g->state) cudaFree(g->state);
    *g = TpGroup();
    return 0;
}

int tp_alloc(int rank, int world, long long max_elems, void* handle_out)
{
    EXL3B_CHECK(world >= 1 && world <= AR_MAX_WORLD, EXL3B_ERR_ARG, "tp_alloc: world size %d not in 1..%d", world, AR_MAX_WORLD);
    EXL3B_CHECK(rank >= 0 && rank < world, EXL3B_ERR_ARG, "tp_alloc: rank %d not in 0..%d", rank, world - 1);
    EXL3B_CHECK(max_elems >= 128 && max_elems % 128 == 0 && max_elems <= (1ll << 26), EXL3B_ERR_ARG,
                "tp_alloc: max_elems (%lld) must be a multiple of 128 in [128, 2^26]", max_elems);
    { int r = tp_free(); if (r) return r; }
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    DevCtx* ctx; r = get_ctx(&ctx); if (r) return r;                 // also rejects devices other than sm_90
    std::lock_guard<std::mutex> lock(g_tp_mutex);
    g->rank = rank; g->world = world; g->slot_elems = max_elems;
    EXL3B_CUDA(cudaMalloc(&g->local, tp_buffer_bytes(*g)));
    EXL3B_CUDA(cudaMemset(g->local, 0xff, tp_buffer_bytes(*g)));    // sentinel everywhere
    EXL3B_CUDA(cudaMalloc(&g->state, 2 * sizeof(unsigned int)));
    EXL3B_CUDA(cudaMemset(g->state, 0, 2 * sizeof(unsigned int)));
    EXL3B_CUDA(cudaDeviceSynchronize());
    g->recv[rank] = g->local;
    if (handle_out)
    {
        cudaIpcMemHandle_t h;
        EXL3B_CUDA(cudaIpcGetMemHandle(&h, g->local));
        static_assert(sizeof(h) == EXL3B_TP_HANDLE_BYTES, "CUDA IPC handle size");
        memcpy(handle_out, &h, sizeof(h));
    }
    return 0;
}

int tp_attach(const void* handles, int world)
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    std::lock_guard<std::mutex> lock(g_tp_mutex);
    EXL3B_CHECK(g->rank >= 0, EXL3B_ERR_ARG, "tp_attach: call tp_alloc first");
    EXL3B_CHECK(world == g->world, EXL3B_ERR_ARG, "tp_attach: %d handles for a group of %d", world, g->world);
    EXL3B_CHECK(!g->attached, EXL3B_ERR_ARG, "tp_attach: already attached");
    EXL3B_CHECK(handles || world == 1, EXL3B_ERR_ARG, "tp_attach: null handle table");
    for (int j = 0; j < world; ++j)
    {
        if (j == g->rank) continue;
        cudaIpcMemHandle_t h;
        memcpy(&h, (const char*) handles + (size_t) j * EXL3B_TP_HANDLE_BYTES, sizeof(h));
        void* ptr = nullptr;
        EXL3B_CUDA(cudaIpcOpenMemHandle(&ptr, h, cudaIpcMemLazyEnablePeerAccess));
        g->recv[j] = (uint32_t*) ptr;
        g->peer_is_ipc[j] = true;
    }
    g->attached = true;
    return 0;
}

int tp_attach_loopback()
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    std::lock_guard<std::mutex> lock(g_tp_mutex);
    EXL3B_CHECK(g->rank >= 0, EXL3B_ERR_ARG, "tp_attach_loopback: call tp_alloc first");
    EXL3B_CHECK(!g->attached, EXL3B_ERR_ARG, "tp_attach_loopback: already attached");
    for (int j = 0; j < g->world; ++j)
    {
        if (j == g->rank) continue;
        EXL3B_CUDA(cudaMalloc(&g->recv[j], tp_buffer_bytes(*g)));
        EXL3B_CUDA(cudaMemset(g->recv[j], 0xff, tp_buffer_bytes(*g)));
        g->peer_is_ipc[j] = false;
    }
    EXL3B_CUDA(cudaDeviceSynchronize());
    g->attached = true;
    return 0;
}

int tp_info(int* rank, int* world, long long* max_elems, int* attached)
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    if (rank) *rank = g->rank;
    if (world) *world = g->world;
    if (max_elems) *max_elems = g->slot_elems;
    if (attached) *attached = g->attached ? 1 : 0;
    return 0;
}

int tp_debug_inject(cudaStream_t stream, int src_rank, const void* partial, long long count)
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    EXL3B_CHECK(g->attached, EXL3B_ERR_ARG, "tp_debug_inject: no tensor-parallel group attached");
    EXL3B_CHECK(src_rank >= 0 && src_rank < g->world && src_rank != g->rank, EXL3B_ERR_ARG, "tp_debug_inject: bad source rank %d", src_rank);
    EXL3B_CHECK(count >= 0 && count <= g->slot_elems, EXL3B_ERR_SHAPE, "tp_debug_inject: %lld words exceed the slot (%lld)", count, g->slot_elems);
    if (count == 0) return 0;
    tp_inject_kernel<<<64, 256, 0, stream>>>(g->state, g->local, g->slot_elems, g->world, src_rank, (const uint32_t*) partial, count);
    count_launch();
    EXL3B_CUDA(cudaPeekAtLastError());
    return 0;
}

int tp_debug_peek(int buffer_rank, int slot, int src_rank, void* host_out, long long count)
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    EXL3B_CHECK(g->attached, EXL3B_ERR_ARG, "tp_debug_peek: no tensor-parallel group attached");
    EXL3B_CHECK(buffer_rank >= 0 && buffer_rank < g->world && src_rank >= 0 && src_rank < g->world && slot >= 0 && slot < AR_SLOTS,
                EXL3B_ERR_ARG, "tp_debug_peek: index out of range");
    EXL3B_CHECK(count >= 0 && count <= g->slot_elems, EXL3B_ERR_SHAPE, "tp_debug_peek: count exceeds the slot");
    EXL3B_CUDA(cudaDeviceSynchronize());
    const uint32_t* src = g->recv[buffer_rank] + ((long long) slot * g->world + src_rank) * g->slot_elems;
    EXL3B_CUDA(cudaMemcpy(host_out, src, (size_t) count * 4, cudaMemcpyDeviceToHost));
    return 0;
}

long long tp_debug_epoch()
{
    TpGroup* g; int r = tp_current(&g); if (r) return r;
    EXL3B_CHECK(g->rank >= 0, EXL3B_ERR_ARG, "tp_debug_epoch: no tensor-parallel group");
    unsigned int st[2];
    EXL3B_CUDA(cudaDeviceSynchronize());
    EXL3B_CUDA(cudaMemcpy(st, g->state, sizeof(st), cudaMemcpyDeviceToHost));
    EXL3B_CHECK(st[1] == 0, EXL3B_ERR_CUDA, "tp_debug_epoch: arrival ticket not reset (%u)", st[1]);
    return (long long) st[0];
}

// why a call cannot take the fused path (nullptr = it can); checked without touching the device
const char* gemm_tc_i8_ar_unsupported(int m, int k, int n, int K, int cb, int world, long long slot_elems)
{
    if (const char* why = i8_shape_unsupported(m, k, n, K, cb, false)) return why;
    if (world < 1 || world > AR_MAX_WORLD) return "world size out of range";
    if ((long long) m * n > slot_elems) return "m * n exceeds the exchange slot (tp_alloc max_elems)";
    return nullptr;
}

// Same launch geometry as launch_gemm_tc_i8 (plan_gemm_tc_i8, gemm_tc_i8.cu); every rank must issue the same sequence of
// row-parallel calls (the requirement any collective has).
int launch_gemm_tc_i8_ar(cudaStream_t stream, DevCtx* ctx, const GemmArgs& a)
{
    TpGroup* g; { int r = tp_current(&g); if (r) return r; }
    EXL3B_CHECK(g->attached, EXL3B_ERR_UNSUPPORTED, "exl3_gemm_allreduce: no tensor-parallel group attached on this device (tp_alloc / tp_attach)");
    const char* why = gemm_tc_i8_ar_unsupported(a.m, a.k, a.n, a.K, a.cb, g->world, g->slot_elems);
    EXL3B_CHECK(!why, EXL3B_ERR_UNSUPPORTED, "exl3_gemm_allreduce: %s", why ? why : "");
    CUtensorMap tmap;
    { int r = get_weight_tmap(a.B, a.k, a.n, a.K, &tmap); if (r) return r; }
    const int slot = ctx->next_slot();
    TcPlan pl;
    { int r = plan_gemm_tc_i8(a.m, a.k, a.n, a.K, ctx->num_sms, a.max_ctas, &pl); if (r) return r; }      // m <= 4: the MR = 4 variant
    ArArgs ar{};
    for (int j = 0; j < g->world; ++j) ar.recv[j] = g->recv[j];
    ar.state = g->state; ar.slot_elems = g->slot_elems; ar.rank = g->rank; ar.world = g->world;
    { int r = i8_launch(stream, a.K, pl.grid, pl.smem_total, i8_params(ctx, slot, pl, a), tmap, nullptr, &ar); if (r) return r; }
    return EXL3B_TAG_TC_I8_AR;
}

}  // namespace exl3b
