// vq_context.cu — context lifetime, error plumbing, packed-layout helpers and the host-side
// FidelityFX constant setup (== the A_CPU functions the engine calls, PostProcess.cpp:39-99).
#include "vq_common.cuh"
#include <stdlib.h>
#include <stdarg.h>
#include <string.h>
#include <math.h>
#include <new>

std::atomic<uint64_t> g_vq_launches{0};
static thread_local char t_err[512] = "";

void vq_set_error(const char* fmt, ...) {
    va_list ap; va_start(ap, fmt);
    vsnprintf(t_err, sizeof(t_err), fmt, ap);
    va_end(ap);
}

int vq_enter(VqContext* ctx) {
    if (!ctx) { vq_set_error("null context"); return VQ_ERR_INVALID_ARG; }
    VQ_CUDA_OK(cudaSetDevice(ctx->device));
    return VQ_OK;
}
int vq_check_launch(const char* what) {
    cudaError_t e = cudaGetLastError();
    if (e != cudaSuccess) { vq_set_error("%s launch failed: %s", what, cudaGetErrorString(e)); return VQ_ERR_CUDA; }
    vq_count_launch();
    return VQ_OK;
}

// The one place context scratch grows. A launch enqueued by an earlier call, on any stream, may still be reading the old
// buffer (e.g. K1 on another stream reading the sampling copies), so the whole device is drained before it is released.
// The contents do not survive a regrow. Once a renderer's sizes are fixed no call regrows, so steady frames never wait here.
int vq_scratch_reserve(VqScratch& s, size_t need, const char* what) {
    if (s.bytes >= need) return VQ_OK;
    if (s.p) {
        VQ_CUDA_OK(cudaDeviceSynchronize());
        cudaFree(s.p);
        s.p = nullptr; s.bytes = 0;
    }
    if (cudaMalloc(&s.p, need) != cudaSuccess) {
        cudaGetLastError(); s.p = nullptr;
        vq_set_error("cudaMalloc(%zu) failed (%s)", need, what);
        return VQ_ERR_OUT_OF_MEMORY;
    }
    s.bytes = need;
    return VQ_OK;
}

int vq_fill_peer_sync(const VqContext* ctx, const VqPeerSignal* sig, PeerSync* out) {
    memset(out, 0, sizeof(*out));
    if (!sig || sig->n_ranks <= 1) return VQ_OK;
    VQ_REQUIRE(sig->n_ranks <= 8 && sig->my_index >= 0 && sig->my_index < sig->n_ranks, "bad peer signal descriptor");
    for (int k = 0; k < sig->n_ranks; ++k) { VQ_REQUIRE(sig->flags[k], "null flag array in the peer signal"); out->flags[k] = sig->flags[k]; }
    out->n = sig->n_ranks; out->myIndex = sig->my_index; out->epoch = sig->epoch;
    const uint64_t deadline = ctx ? ctx->rv_deadline_ns.load(std::memory_order_acquire) : 0;
    if (deadline) { out->deadlineNs = deadline; out->cancel = ctx->rv_cancel_dev; out->status = ctx->rv_status; }
    return VQ_OK;
}

// ---- the band contract (every *_multi_signal call) ----------------------------------------------------------------------------
int vq_band_list(const void* outs, int n_outs) {
    VQ_REQUIRE(outs, "null destination list");
    VQ_REQUIRE(n_outs >= 1 && n_outs <= 8, "1..8 destinations");
    return VQ_OK;
}

int vq_band_check(const VqContext* ctx, int n_outs, int dst_row_offset, int H, int row_begin, int row_end, const VqPeerSignal* sig,
                  PeerSync& sync) {
    VQ_REQUIRE(dst_row_offset >= 0, "negative destination row offset");
    VQ_REQUIRE(row_begin >= 0 && row_end <= H && row_begin <= row_end, "row range out of bounds");
    VQ_REQUIRE(row_begin < row_end || !(sig && sig->n_ranks > 1), "a rendezvous needs a non-empty row range (the kernel runs it)");
    const int rc = vq_fill_peer_sync(ctx, sig, &sync); if (rc) return rc;
    VQ_REQUIRE(sync.n == 0 || n_outs > 1, "a rendezvous only makes sense with peer destinations");
    return VQ_OK;
}

uint32_t* vq_band_ticket(VqContext* ctx, const PeerSync& sync) { return sync.n > 1 ? vq_ticket_pair(ctx) : nullptr; }

// vq_ctx_rendezvous_clear: the record and the cancel word zeroed in stream order (loaded when the first deadline is registered)
__global__ void rendezvous_clear_kernel(VqRendezvousStatus* status, uint32_t* cancel) {
    *status = VqRendezvousStatus{};
    asm volatile("st.relaxed.sys.global.u32 [%0], %1;" :: "l"(cancel), "r"(0u) : "memory");
}

extern "C" {

const char* vq_last_error(void) { return t_err; }
const char* vq_version(void) { return "vqcuda 0.1 (sm_90a)"; }
uint64_t vq_launch_count(void) { return g_vq_launches.load(); }

int vq_ctx_create(int device, VqContext** out_ctx) {
    if (!out_ctx) { vq_set_error("out_ctx is null"); return VQ_ERR_INVALID_ARG; }
    *out_ctx = nullptr;
    int n = 0;
    cudaError_t e = cudaGetDeviceCount(&n);
    if (e != cudaSuccess || n == 0) {
        // no CPU fallback by design: fail loudly
        vq_set_error("no CUDA device available (%s): this backend has no CPU path", e == cudaSuccess ? "count=0" : cudaGetErrorString(e));
        return VQ_ERR_NO_DEVICE;
    }
    if (device < 0 || device >= n) { vq_set_error("device %d out of range [0,%d)", device, n); return VQ_ERR_INVALID_ARG; }
    VQ_CUDA_OK(cudaSetDevice(device));
    cudaDeviceProp prop;
    VQ_CUDA_OK(cudaGetDeviceProperties(&prop, device));
    if (prop.major != 9 || prop.minor != 0) {     // sm_90a code loads on compute capability 9.0 only
        vq_set_error("device %d is sm_%d%d; this library only carries sm_90a code", device, prop.major, prop.minor);
        return VQ_ERR_UNSUPPORTED;
    }
    VqContext* c = new (std::nothrow) VqContext();
    if (!c) return VQ_ERR_OUT_OF_MEMORY;
    c->device = device;
    c->sm_count = prop.multiProcessorCount;
    c->l2_bytes = prop.l2CacheSize;
    if (cudaMalloc(&c->spd_counter, 2 * VQ_SPD_SLOTS * sizeof(uint32_t)) != cudaSuccess) { delete c; vq_set_error("cudaMalloc failed"); return VQ_ERR_OUT_OF_MEMORY; }
    cudaMemset(c->spd_counter, 0, 2 * VQ_SPD_SLOTS * sizeof(uint32_t));
    c->spd_next = new std::atomic<uint32_t>(0u);
    c->mu = new std::recursive_mutex();
    *out_ctx = c;
    return VQ_OK;
}

int vq_ctx_destroy(VqContext* ctx) {
    if (!ctx) return VQ_OK;
    cudaSetDevice(ctx->device);
    if (ctx->streams_ready) {
        for (auto& s : ctx->streams) cudaStreamDestroy(s);
        for (auto& e : ctx->events) cudaEventDestroy(e);
    }
    if (ctx->spd_counter) cudaFree(ctx->spd_counter);
    if (ctx->rv_status) cudaFree(ctx->rv_status);
    if (ctx->rv_cancel_host) cudaFreeHost((void*)ctx->rv_cancel_host);
    delete ctx->spd_next; delete ctx->mu;
    delete ctx;                 // frees the scratch (~VqScratch)
    return VQ_OK;
}

// ---- the rendezvous policy (vqcuda_rendezvous.h) ------------------------------------------------
int vq_ctx_set_rendezvous_deadline(VqContext* ctx, uint64_t ns) {
    VQ_REQUIRE(ctx, "null context");
    VQ_REQUIRE(ns >= 1 && ns <= VQ_RENDEZVOUS_MAX_DEADLINE_NS, "the deadline must be 1 ns..20 s");
    int rc = vq_enter(ctx); if (rc) return rc;
    VqScratchLock lock(ctx);
    if (!ctx->rv_status) {
        cudaFuncAttributes attr;       // a first launch loads its module, which would wait for the signalled kernels running then
        VQ_CUDA_OK(cudaFuncGetAttributes(&attr, rendezvous_clear_kernel));
        void* host = nullptr;
        void* dev = nullptr;
        VqRendezvousStatus* status = nullptr;
        cudaError_t e = cudaHostAlloc(&host, sizeof(uint32_t), cudaHostAllocMapped | cudaHostAllocPortable);
        if (e == cudaSuccess) { *(volatile uint32_t*)host = 0u; e = cudaHostGetDevicePointer(&dev, host, 0); }
        if (e == cudaSuccess) e = cudaMalloc(&status, sizeof(VqRendezvousStatus));
        // the zeroes land before any call of any stream reads them, without waiting for the rest of the device: a stream of its own
        cudaStream_t zs = nullptr;
        if (e == cudaSuccess) e = cudaStreamCreateWithFlags(&zs, cudaStreamNonBlocking);
        if (e == cudaSuccess) e = cudaMemsetAsync(status, 0, sizeof(VqRendezvousStatus), zs);
        if (e == cudaSuccess) e = cudaStreamSynchronize(zs);
        if (zs) cudaStreamDestroy(zs);
        if (e != cudaSuccess) {
            cudaGetLastError();
            if (status) cudaFree(status);
            if (host) cudaFreeHost(host);
            vq_set_error("rendezvous status and cancel word: %s", cudaGetErrorString(e));
            return e == cudaErrorMemoryAllocation ? VQ_ERR_OUT_OF_MEMORY : VQ_ERR_CUDA;
        }
        ctx->rv_cancel_host = (volatile uint32_t*)host;
        ctx->rv_cancel_dev = (const uint32_t*)dev;
        ctx->rv_status = status;
    }
    ctx->rv_deadline_ns.store(ns, std::memory_order_release);
    return VQ_OK;
}

int vq_ctx_cancel_rendezvous(VqContext* ctx) {
    VQ_REQUIRE(ctx, "null context");
    VQ_REQUIRE(ctx->rv_deadline_ns.load(std::memory_order_acquire) != 0, "no rendezvous deadline is registered on this context");
    __atomic_store_n(ctx->rv_cancel_host, 1u, __ATOMIC_RELEASE);
    return VQ_OK;
}

int vq_ctx_rendezvous_status(VqContext* ctx, void* stream, VqRendezvousStatus* out) {
    VQ_REQUIRE(ctx, "null context");
    VQ_REQUIRE(out, "out is null");
    memset(out, 0, sizeof(*out));
    if (ctx->rv_deadline_ns.load(std::memory_order_acquire) == 0) return VQ_OK;
    int rc = vq_enter(ctx); if (rc) return rc;
    VqRendezvousStatus s;          // pageable: the copy has completed when the call returns
    VQ_CUDA_OK(cudaMemcpyAsync(&s, ctx->rv_status, sizeof(s), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    VQ_CUDA_OK(cudaStreamSynchronize((cudaStream_t)stream));
    *out = s;
    return VQ_OK;
}

int vq_ctx_rendezvous_clear(VqContext* ctx, void* stream) {
    VQ_REQUIRE(ctx, "null context");
    if (ctx->rv_deadline_ns.load(std::memory_order_acquire) == 0) return VQ_OK;
    int rc = vq_enter(ctx); if (rc) return rc;
    rendezvous_clear_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(ctx->rv_status, (uint32_t*)ctx->rv_cancel_dev);
    return vq_check_launch("rendezvous_clear");
}

// ---- packed layouts ---------------------------------------------------------------------------
int vq_mip_level_count(uint64_t w, uint64_t h) {   // Image::CalculateMipLevelCount, Image.cpp:231-241
    int mips = 0;
    while (w >= 1 && h >= 1) { ++mips; w >>= 1; h >>= 1; }
    return mips;
}
uint64_t vq_cubemap_texel_count(int res, int mips) {
    uint64_t o = 0;
    for (int m = 0; m < mips; ++m) { const uint64_t r = (uint64_t)(res >> m); o += 6 * r * r; }
    return o;
}
uint64_t vq_cubemap_offset(int res, int mip, int face) {
    const uint64_t r = (uint64_t)(res >> mip);
    return vq_cubemap_texel_count(res, mip) + (uint64_t)face * r * r;
}
int vq_cubemap_row_count(int res, int mips) {
    int n = 0;
    for (int m = 0; m < mips; ++m) n += 6 * (res >> m);
    return n;
}
uint64_t vq_pyramid_texel_count(int width, int height, int levels) {
    uint64_t o = 0;
    for (int l = 0; l < levels; ++l) o += (uint64_t)(width >> l) * (uint64_t)(height >> l);
    return o;
}
uint64_t vq_pyramid_offset(int width, int height, int level) { return vq_pyramid_texel_count(width, height, level); }

// ---- FidelityFX constant setup (host) ------------------------------------------------------------
static inline uint32_t fbits(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

// float -> half bits, truncating, denormal-aware, +-INF/NaN -> +-65504 (the rule behind the
// reference's AU1_AH1_AF1 tables, FSR1.0/ffx_a.h:482-550)
static uint32_t half_bits_trunc(float f) {
    const uint32_t u = fbits(f);
    const uint32_t se = u >> 23, e = se & 0xffu, sign = (se >> 8) << 15;
    uint32_t base, shift;
    if (e < 103u)       { base = 0u;                    shift = 24u; }
    else if (e < 113u)  { base = 0x0400u >> (113u - e); shift = 126u - e; }
    else if (e <= 142u) { base = (e - 112u) << 10;      shift = 13u; }
    else                { base = 0x7bffu;               shift = 24u; }
    return (base | sign) + ((u & 0x7fffffu) >> shift);
}

void vq_fsr_easu_con(uint32_t con[16], float vpw, float vph, float inw, float inh, float outw, float outh) {
    // FsrEasuCon, ffx_fsr1.h:156-202 (ARcpF1(a) = 1.0f/a on the CPU, ffx_a.h:326)
    const float rx = 1.0f / outw, ry = 1.0f / outh, rix = 1.0f / inw, riy = 1.0f / inh;
    con[0] = fbits(vpw * rx);
    con[1] = fbits(vph * ry);
    con[2] = fbits(0.5f * vpw * rx - 0.5f);
    con[3] = fbits(0.5f * vph * ry - 0.5f);
    con[4] = fbits(rix);
    con[5] = fbits(riy);
    con[6] = fbits(1.0f * rix);
    con[7] = fbits(-1.0f * riy);
    con[8] = fbits(-1.0f * rix);
    con[9] = fbits(2.0f * riy);
    con[10] = fbits(1.0f * rix);
    con[11] = fbits(2.0f * riy);
    con[12] = fbits(0.0f * rix);
    con[13] = fbits(4.0f * riy);
    con[14] = con[15] = 0;
}

void vq_fsr_rcas_con(uint32_t con[4], float sharpness_stops) {
    // FsrRcasCon, ffx_fsr1.h:662-672
    const float s = exp2f(-sharpness_stops);
    con[0] = fbits(s);
    con[1] = half_bits_trunc(s) + (half_bits_trunc(s) << 16);
    con[2] = 0; con[3] = 0;
}

void vq_cas_setup(uint32_t con[8], float sharpness, float inw, float inh, float outw, float outh) {
    // CasSetup, ffx_cas.h:375-394; ALerpF1(a,b,c) = b*c + (-a*c + a), ffx_a.h:298
    const float rx = 1.0f / outw, ry = 1.0f / outh;
    con[0] = fbits(inw * rx);
    con[1] = fbits(inh * ry);
    con[2] = fbits(0.5f * inw * rx - 0.5f);
    con[3] = fbits(0.5f * inh * ry - 0.5f);
    const float c = fminf(1.0f, fmaxf(0.0f, sharpness));
    const float l = 5.0f * c + (-8.0f * c + 8.0f);
    const float sharp = -(1.0f / l);
    con[4] = fbits(sharp);
    con[5] = half_bits_trunc(sharp) + (half_bits_trunc(0.0f) << 16);
    con[6] = fbits(8.0f * inw * rx);
    con[7] = 0;
}

void vq_spd_setup(uint32_t dispatch_xy[2], VqSpdConstants* constants, const uint32_t rect[4], int mips) {
    // SpdSetup, ffx_spd.h:327-351
    constants->workGroupOffset[0] = rect[0] / 64;
    constants->workGroupOffset[1] = rect[1] / 64;
    const uint32_t endX = (rect[0] + rect[2] - 1) / 64;
    const uint32_t endY = (rect[1] + rect[3] - 1) / 64;
    dispatch_xy[0] = endX + 1 - constants->workGroupOffset[0];
    dispatch_xy[1] = endY + 1 - constants->workGroupOffset[1];
    constants->numWorkGroups = dispatch_xy[0] * dispatch_xy[1];
    if (mips >= 0) constants->mips = (uint32_t)mips;
    else {
        const uint32_t res = rect[2] > rect[3] ? rect[2] : rect[3];
        constants->mips = (uint32_t)fminf(floorf(log2f((float)res)), 12.0f);
    }
}

}  // extern "C"
