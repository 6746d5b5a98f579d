// vq_group.cu — the device group of vqcuda_group.h: peer access, flag arrays, rank orders and signals of a multi-GPU world in
// one process, and the band plans (the row splits that vqengine_b200/distributed.py's equal_tiles, even_tiles and
// InterleavedSpecularPlan compute for the torch path). Two kernels: the arrival of a rank whose signalled call was refused, and the
// barrier of a rank with no pass.
#include "vq_common.cuh"
#include "../../include/vqcuda_group.h"

#include <new>

struct VqGroup {
    int n = 0;
    int device[8] = {};
    VqContext* ctx[8] = {};           // rank r's context: its rendezvous policy (vqcuda_rendezvous.h)
    uint32_t* flags[8] = {};
    bool owned = false;              // the flag arrays are the group's (cudaMalloc on each rank's device)
};

// one thread: the store a signalled call's last CTA makes after its own stores (peer_rendezvous, vq_common.cuh)
__global__ void group_arrive_kernel(PeerSync y) {
    __threadfence_system();
    for (int k = 1; k < y.n; ++k)
        asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(y.flags[k] + y.myIndex), "r"(y.epoch) : "memory");
}

// one thread: a signalled call's rendezvous without its pass (the epoch into the peers' arrays, then the wait under the rank's policy)
__global__ void group_barrier_kernel(const PeerSync y) {
    __threadfence_system();
    vq::peer_rendezvous(y);
}

// rank r's PeerSync at `epoch` (vq_group_signal's flag arrays and the rank's policy)
static int group_peer_sync(const VqGroup* g, int rank, uint32_t epoch, PeerSync* y) {
    VqPeerSignal sig;
    vq_group_signal(g, rank, epoch, &sig);
    return vq_fill_peer_sync(g->ctx[rank], &sig, y);
}

static void vq_group_free_flags(VqGroup* g) {
    if (!g->owned) return;
    for (int r = 0; r < g->n; ++r)
        if (g->flags[r]) { cudaSetDevice(g->device[r]); cudaFree(g->flags[r]); g->flags[r] = nullptr; }
}

extern "C" {

int vq_group_create(VqContext* const* ctxs, int n_ranks, uint32_t* const* flag_arrays, VqGroup** out) {
    VQ_REQUIRE(out, "out is null");
    *out = nullptr;
    VQ_REQUIRE(ctxs, "ctxs is null");
    VQ_REQUIRE(n_ranks >= 1 && n_ranks <= 8, "n_ranks must be 1..8");
    for (int r = 0; r < n_ranks; ++r) {
        VQ_REQUIRE(ctxs[r], "null context");
        for (int q = 0; q < r; ++q) VQ_REQUIRE(ctxs[q] != ctxs[r], "a context appears twice (each rank needs its own)");
        if (flag_arrays) VQ_REQUIRE(flag_arrays[r], "null flag array");
    }
    int dev[8];
    for (int r = 0; r < n_ranks; ++r) dev[r] = ctxs[r]->device;
    // every pair first, so that a refusal changes nothing
    for (int a = 0; a < n_ranks; ++a)
        for (int b = 0; b < n_ranks; ++b) {
            if (dev[a] == dev[b]) continue;
            int can = 0;
            VQ_CUDA_OK(cudaDeviceCanAccessPeer(&can, dev[a], dev[b]));
            if (!can) { vq_set_error("device %d cannot access device %d (cudaDeviceCanAccessPeer)", dev[a], dev[b]); return VQ_ERR_UNSUPPORTED; }
        }
    for (int a = 0; a < n_ranks; ++a)
        for (int b = 0; b < n_ranks; ++b) {
            if (dev[a] == dev[b]) continue;
            VQ_CUDA_OK(cudaSetDevice(dev[a]));
            const cudaError_t e = cudaDeviceEnablePeerAccess(dev[b], 0);
            if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); continue; }
            VQ_CUDA_OK(e);
        }
    // load the arrival and barrier kernels on every rank's device now: a first launch loads its module, and a module load waits for
    // the kernels already running, which include the signalled calls the arrival would release
    for (int r = 0; r < n_ranks; ++r) {
        cudaFuncAttributes attr;
        VQ_CUDA_OK(cudaSetDevice(dev[r]));
        VQ_CUDA_OK(cudaFuncGetAttributes(&attr, group_arrive_kernel));
        VQ_CUDA_OK(cudaFuncGetAttributes(&attr, group_barrier_kernel));
    }
    VqGroup* g = new (std::nothrow) VqGroup();
    if (!g) { vq_set_error("out of host memory"); return VQ_ERR_OUT_OF_MEMORY; }
    g->n = n_ranks;
    for (int r = 0; r < n_ranks; ++r) { g->device[r] = dev[r]; g->ctx[r] = ctxs[r]; }
    if (flag_arrays) {
        for (int r = 0; r < n_ranks; ++r) g->flags[r] = flag_arrays[r];
    } else {
        g->owned = true;
        for (int r = 0; r < n_ranks; ++r) {
            cudaError_t e = cudaSetDevice(dev[r]);
            if (e == cudaSuccess) e = cudaMalloc(&g->flags[r], (size_t)n_ranks * sizeof(uint32_t));
            if (e == cudaSuccess) e = cudaMemset(g->flags[r], 0, (size_t)n_ranks * sizeof(uint32_t));
            if (e != cudaSuccess) {
                cudaGetLastError();
                vq_set_error("flag array of rank %d: %s", r, cudaGetErrorString(e));
                vq_group_free_flags(g);
                delete g;
                return e == cudaErrorMemoryAllocation ? VQ_ERR_OUT_OF_MEMORY : VQ_ERR_CUDA;
            }
        }
        for (int r = 0; r < n_ranks; ++r) {     // the zeroes land before any rank's first signalled call, on any stream, reads them
            VQ_CUDA_OK(cudaSetDevice(dev[r]));
            VQ_CUDA_OK(cudaDeviceSynchronize());
        }
    }
    *out = g;
    return VQ_OK;
}

int vq_group_destroy(VqGroup* g) {
    if (!g) return VQ_OK;
    vq_group_free_flags(g);
    delete g;
    return VQ_OK;
}

int vq_group_rank_order(const VqGroup* g, int rank, int order[8]) {
    VQ_REQUIRE(g && order, "null group or order");
    VQ_REQUIRE(rank >= 0 && rank < g->n, "rank out of range");
    for (int k = 0; k < 8; ++k) order[k] = k < g->n ? (rank + k) % g->n : -1;
    return VQ_OK;
}

int vq_group_signal(const VqGroup* g, int rank, uint32_t epoch, VqPeerSignal* out) {
    VQ_REQUIRE(g && out, "null group or signal");
    VQ_REQUIRE(rank >= 0 && rank < g->n, "rank out of range");
    memset(out, 0, sizeof(*out));
    for (int k = 0; k < g->n; ++k) out->flags[k] = g->flags[(rank + k) % g->n];
    out->n_ranks = g->n;
    out->my_index = rank;
    out->epoch = epoch;
    return VQ_OK;
}

int vq_group_arrive(const VqGroup* g, int rank, uint32_t epoch, void* stream) {
    VQ_REQUIRE(g, "null group");
    VQ_REQUIRE(rank >= 0 && rank < g->n, "rank out of range");
    if (g->n == 1) return VQ_OK;
    PeerSync y;
    memset(&y, 0, sizeof(y));
    for (int k = 0; k < g->n; ++k) y.flags[k] = g->flags[(rank + k) % g->n];
    y.n = g->n; y.myIndex = rank; y.epoch = epoch;
    VQ_CUDA_OK(cudaSetDevice(g->device[rank]));
    group_arrive_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(y);
    return vq_check_launch("group_arrive");
}

int vq_group_set_rendezvous_deadline(const VqGroup* g, uint64_t ns) {
    VQ_REQUIRE(g, "null group");
    VQ_REQUIRE(ns >= 1 && ns <= VQ_RENDEZVOUS_MAX_DEADLINE_NS, "the deadline must be 1 ns..20 s");
    for (int r = 0; r < g->n; ++r) { const int rc = vq_ctx_set_rendezvous_deadline(g->ctx[r], ns); if (rc) return rc; }
    return VQ_OK;
}

int vq_group_cancel(const VqGroup* g) {
    VQ_REQUIRE(g, "null group");
    // every rank checked before any is cancelled: a refusal cancels nothing
    for (int r = 0; r < g->n; ++r)
        VQ_REQUIRE(g->ctx[r]->rv_deadline_ns.load(std::memory_order_acquire) != 0, "a rank's context has no rendezvous deadline registered");
    for (int r = 0; r < g->n; ++r) { const int rc = vq_ctx_cancel_rendezvous(g->ctx[r]); if (rc) return rc; }
    return VQ_OK;
}

int vq_group_barrier(const VqGroup* g, int rank, uint32_t epoch, void* stream) {
    VQ_REQUIRE(g, "null group");
    VQ_REQUIRE(rank >= 0 && rank < g->n, "rank out of range");
    if (g->n == 1) return VQ_OK;
    PeerSync y;
    int rc = group_peer_sync(g, rank, epoch, &y); if (rc) return rc;
    VQ_CUDA_OK(cudaSetDevice(g->device[rank]));
    group_barrier_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(y);
    return vq_check_launch("group_barrier");
}

int vq_band_rows(int n_rows, int n_ranks, int rank, int even, int* row_begin, int* row_end) {
    VQ_REQUIRE(row_begin && row_end, "null output");
    VQ_REQUIRE(n_rows >= 0, "n_rows must not be negative");
    VQ_REQUIRE(n_ranks >= 1 && n_ranks <= 8, "n_ranks must be 1..8");
    VQ_REQUIRE(rank >= 0 && rank < n_ranks, "rank out of range");
    VQ_REQUIRE(even == 0 || even == 1, "even must be 0 or 1");
    const int64_t n = n_rows, w = n_ranks;
    if (!even) {
        *row_begin = (int)(n * rank / w);
        *row_end = (int)(n * (rank + 1) / w);
    } else {
        // even_tiles: cut r = 2 * ceil(pairs * r / world), the last cut at n_rows
        const int64_t pairs = n / 2;
        *row_begin = (int)(2 * ((pairs * rank + w - 1) / w));
        *row_end = rank + 1 == n_ranks ? n_rows : (int)(2 * ((pairs * (rank + 1) + w - 1) / w));
    }
    return VQ_OK;
}

int vq_specular_rank_ranges(int res, int mips, int n_ranks, int rank, int* ranges, int capacity, int* n_ranges) {
    VQ_REQUIRE(n_ranges, "n_ranges is null");
    *n_ranges = 0;
    VQ_REQUIRE(res >= 1, "res must be at least 1");
    VQ_REQUIRE(mips >= 1 && mips <= vq_mip_level_count((uint64_t)res, (uint64_t)res), "mips must be 1..vq_mip_level_count(res, res)");
    VQ_REQUIRE(n_ranks >= 1 && n_ranks <= 8, "n_ranks must be 1..8");
    VQ_REQUIRE(rank >= 0 && rank < n_ranks, "rank out of range");
    VQ_REQUIRE(capacity >= 0 && (ranges || capacity == 0), "null ranges with a capacity");
    // mips are laid out in increasing row order, one range per mip: the list is increasing and disjoint as it is built
    int count = 0, row0 = 0;
    for (int m = 0; m < mips; ++m) {
        const int rows = 6 * (res >> m);
        int a = row0, b = row0 + rows;
        if (n_ranks > 1 && rows % n_ranks == 0) { const int k = rows / n_ranks; a = row0 + rank * k; b = a + k; }
        if (b > a) {
            if (count < capacity) { ranges[2 * count] = a; ranges[2 * count + 1] = b; }
            ++count;
        }
        row0 += rows;
    }
    *n_ranges = count;
    VQ_REQUIRE(count <= capacity, "capacity is smaller than the number of ranges (*n_ranges)");
    return VQ_OK;
}

}  // extern "C"
