// TEST INFRASTRUCTURE: holds the cross-rank rendezvous of the signalled calls (vq::peer_rendezvous, vq_common.cuh) from the host,
// for tests/test_rendezvous_hold_gpu.py (ctypes, torch stream handles). Never linked into the product.
//
// A world is one allocation of mapped, pinned host memory: PH_ROWS x PH_STRIDE flag words (row q = rank q's flag array; a row is
// wider than any world, so words at index n and above exist and can hold garbage) and a control block. The kernels of the product
// reach the flag words through the device pointer exactly as they reach peer memory (ld.acquire.sys / st.release.sys); the host
// reads and writes them through the host pointer, without any CUDA call.
//   ph_stamp   one thread, queued on a rank's stream right after its call: copies the keeper's release counter into stamp[slot],
//              then sets done[slot]. It runs once the call has finished, so it records how many peers had been released by then
//   ph_watch   one CTA on a second stream: polls one flag word until it EQUALS `epoch` (bounded by %globaltimer, never a trap), then
//              copies up to 8 device byte ranges into snapshot buffers and writes its status (1 seen and copied, 2 timed out)
//   keeper     a std::thread that makes no CUDA call. Held run (rank >= 0): waits until the rank's word in every peer row equals
//              `epoch` and (optionally) the watcher has finished its copy, then releases the rank's own words in the given order,
//              each after a dwell: the release counter is bumped, then the word is stored. Then it waits for `n_stamps` stamps.
//              Watch run (rank < 0): only the last step. On any bound, or when asked to stop, it RESCUES, and counts the rescue:
//              it cycles every word of every row through e and e + 1 for each epoch e the guarded calls may wait on, 25 ms per
//              value, until every stamp has landed or PH_RESCUE_US has passed. One of the two values satisfies an ==, >= or >
//              test, signed or unsigned, of a wait at e on any word a kernel could read, so the calls finish well inside their
//              20 s watchdog, which starts after the keeper: its two waits (PH_BOUND_MAX_US each), its releases and the rescue
//              end within 10 s of its start.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>

#include <atomic>
#include <chrono>
#include <thread>
#include <vector>

namespace {

constexpr int PH_ROWS = 8, PH_STRIDE = 16, PH_SLOTS = 16, PH_EPOCHS = 16;
constexpr long long PH_BOUND_MAX_US = 2000000, PH_RESCUE_US = 5000000, PH_RESCUE_STEP_US = 25000;

struct Ctl {
    uint32_t released;                 // releases begun by the keeper (bumped just before each release store)
    uint32_t rescues;                  // rescues the keeper made
    uint32_t watch;                    // 0 waiting, 1 seen and copied, 2 timed out
    uint32_t pad;
    uint32_t stamp[PH_SLOTS];
    uint32_t done[PH_SLOTS];
};

struct Mapped {
    uint32_t flags[PH_ROWS * PH_STRIDE];
    Ctl ctl;
};

struct Plan {
    int n, rank, wait_watch, n_stamps;
    uint32_t epoch, value;
    std::vector<int> order;
    std::vector<uint32_t> rescue;      // every epoch the guarded calls may wait on
    long long dwell_us, bound_us;
};

struct World {
    Mapped* h = nullptr;               // host view
    Mapped* d = nullptr;               // device view
    std::thread keeper;
    std::atomic<int> stop{0};
};

inline uint32_t ld(const uint32_t* p) { return __atomic_load_n(p, __ATOMIC_ACQUIRE); }
inline void st(uint32_t* p, uint32_t v) { __atomic_store_n(p, v, __ATOMIC_RELEASE); }

using Clock = std::chrono::steady_clock;

// polls `ready` until it holds; false on the bound or a stop request
template <class F>
bool wait_for(World* w, F ready, long long bound_us) {
    const auto t0 = Clock::now();
    for (;;) {
        if (ready()) return true;
        if (w->stop.load()) return false;
        if (std::chrono::duration_cast<std::chrono::microseconds>(Clock::now() - t0).count() > bound_us) return false;
        std::this_thread::sleep_for(std::chrono::microseconds(20));
    }
}

bool stamped(const Mapped* m, int n_stamps) {
    for (int s = 0; s < n_stamps; ++s)
        if (ld(&m->ctl.done[s]) != 1u) return false;
    return true;
}

void rescue(World* w, const Plan& p) {
    st(&w->h->ctl.rescues, ld(&w->h->ctl.rescues) + 1u);
    const auto t0 = Clock::now();
    for (size_t k = 0;; ++k) {
        const uint32_t v = p.rescue[(k / 2) % p.rescue.size()] + (uint32_t)(k % 2);
        for (int i = 0; i < PH_ROWS * PH_STRIDE; ++i) st(&w->h->flags[i], v);
        std::this_thread::sleep_for(std::chrono::microseconds(PH_RESCUE_STEP_US));
        if (stamped(w->h, p.n_stamps)) return;
        if (std::chrono::duration_cast<std::chrono::microseconds>(Clock::now() - t0).count() > PH_RESCUE_US) return;
    }
}

void keep(World* w, Plan p) {
    Mapped* m = w->h;
    bool ok = true;
    if (p.rank >= 0) {
        ok = wait_for(w, [&] {
            for (int q = 0; q < p.n; ++q)
                if (q != p.rank && ld(&m->flags[q * PH_STRIDE + p.rank]) != p.epoch) return false;
            return !p.wait_watch || ld(&m->ctl.watch) != 0;
        }, p.bound_us);
        ok = ok && (!p.wait_watch || ld(&m->ctl.watch) == 1);
        for (size_t k = 0; ok && k < p.order.size(); ++k) {
            std::this_thread::sleep_for(std::chrono::microseconds(p.dwell_us));
            st(&m->ctl.released, ld(&m->ctl.released) + 1u);
            st(&m->flags[p.rank * PH_STRIDE + p.order[k]], p.value);
        }
    }
    ok = ok && wait_for(w, [&] { return stamped(m, p.n_stamps); }, p.bound_us);
    if (!ok) rescue(w, p);
}

__global__ void stamp_kernel(Ctl* c, int slot) {
    uint32_t v;
    asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(&c->released) : "memory");
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(&c->stamp[slot]), "r"(v) : "memory");
    asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(&c->done[slot]), "r"(1u) : "memory");
}

struct Ranges {
    const int4* src[8];
    int4* dst[8];
    unsigned long long n16[8];
    int n;
};

__device__ __forceinline__ unsigned long long now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void __launch_bounds__(1024) watch_kernel(const uint32_t* flag, uint32_t epoch, unsigned long long bound_ns, Ranges R,
                                                     Ctl* c) {
    __shared__ int seen;
    if (threadIdx.x == 0) {
        const unsigned long long t0 = now_ns();
        int ok = 0;
        for (;;) {
            uint32_t v;
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
            if (v == epoch) { ok = 1; break; }
            if (now_ns() - t0 > bound_ns) break;
            __nanosleep(100);
        }
        seen = ok;
    }
    __syncthreads();                   // the acquire, then the barrier: every thread's loads below come after the flag store
    if (seen) {
        unsigned long long most = 0;
        for (int k = 0; k < R.n; ++k) most = R.n16[k] > most ? R.n16[k] : most;
        for (long long i = (long long)most - 1 - threadIdx.x; i >= 0; i -= blockDim.x)
            for (int k = 0; k < R.n; ++k)
                if ((unsigned long long)i < R.n16[k]) R.dst[k][i] = __ldcg(R.src[k] + i);
    }
    __threadfence();                   // every thread's copy is complete before the status says so
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence_system();
        asm volatile("st.release.sys.global.u32 [%0], %1;" :: "l"(&c->watch), "r"(seen ? 1u : 2u) : "memory");
    }
}

}  // namespace

extern "C" {

int ph_new(void** out) {
    World* w = new World();
    void* h = nullptr;
    cudaError_t e = cudaHostAlloc(&h, sizeof(Mapped), cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) { delete w; return (int)e; }
    memset(h, 0, sizeof(Mapped));
    w->h = (Mapped*)h;
    e = cudaHostGetDevicePointer((void**)&w->d, h, 0);
    if (e != cudaSuccess) { cudaFreeHost(h); delete w; return (int)e; }
    *out = w;
    return 0;
}

int ph_free(void* world) {
    World* w = (World*)world;
    if (w->keeper.joinable()) { w->stop = 1; w->keeper.join(); }
    const cudaError_t e = cudaFreeHost(w->h);
    delete w;
    return (int)e;
}

int ph_rows() { return PH_ROWS; }
int ph_stride() { return PH_STRIDE; }
void* ph_host_flags(void* world) { return ((World*)world)->h->flags; }
void* ph_dev_flags(void* world) { return ((World*)world)->d->flags; }
// the control block's host view: released, rescues, watch, pad, stamp[PH_SLOTS], done[PH_SLOTS]
void* ph_host_ctl(void* world) { return &((World*)world)->h->ctl; }

// zeroes the control block except the rescue count; only while no keeper runs and no stamp or watcher is queued
int ph_reset(void* world) {
    World* w = (World*)world;
    if (w->keeper.joinable()) return -1;
    const uint32_t rescues = w->h->ctl.rescues;
    memset(&w->h->ctl, 0, sizeof(Ctl));
    w->h->ctl.rescues = rescues;
    return 0;
}

int ph_stamp(void* world, void* stream, int slot) {
    if (slot < 0 || slot >= PH_SLOTS) return -1;
    stamp_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(&((World*)world)->d->ctl, slot);
    return (int)cudaGetLastError();
}

int ph_watch(void* world, void* stream, int row, int col, uint32_t epoch, unsigned long long bound_ns, int n, const void* const* src,
             void* const* dst, const unsigned long long* bytes) {
    if (n < 0 || n > 8 || row < 0 || row >= PH_ROWS || col < 0 || col >= PH_STRIDE) return -1;
    Ranges R;
    memset(&R, 0, sizeof(R));
    for (int k = 0; k < n; ++k) {
        if (bytes[k] % 16 || (uintptr_t)src[k] % 16 || (uintptr_t)dst[k] % 16) return -1;
        R.src[k] = (const int4*)src[k]; R.dst[k] = (int4*)dst[k]; R.n16[k] = bytes[k] / 16;
    }
    R.n = n;
    World* w = (World*)world;
    watch_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(&w->d->flags[row * PH_STRIDE + col], epoch, bound_ns, R, &w->d->ctl);
    return (int)cudaGetLastError();
}

// starts the keeper (see the top of the file); rank < 0: a watch run (no release). rescue[0..n_rescue): every epoch the calls it
// guards may wait on (at least one); bound_us: at most PH_BOUND_MAX_US, so that a rescue ends well inside the watchdog
int ph_keeper_start(void* world, int n, int rank, uint32_t epoch, uint32_t value, const int* order, int n_order, int wait_watch,
                    int n_stamps, long long dwell_us, long long bound_us, const uint32_t* rescue, int n_rescue) {
    World* w = (World*)world;
    if (w->keeper.joinable() || n < 1 || n > PH_ROWS || rank >= n || n_order < 0 || n_order > PH_STRIDE || n_stamps < 0 ||
        n_stamps > PH_SLOTS || n_rescue < 1 || n_rescue > PH_EPOCHS || bound_us > PH_BOUND_MAX_US)
        return -1;
    Plan p;
    p.n = n; p.rank = rank; p.epoch = epoch; p.value = value; p.wait_watch = wait_watch; p.n_stamps = n_stamps;
    p.dwell_us = dwell_us; p.bound_us = bound_us;
    for (int k = 0; k < n_order; ++k) {
        if (order[k] < 0 || order[k] >= PH_STRIDE) return -1;
        p.order.push_back(order[k]);
    }
    p.rescue.assign(rescue, rescue + n_rescue);
    w->stop = 0;
    w->keeper = std::thread(keep, w, p);
    return 0;
}

// joins the keeper (stop != 0: asks it to rescue now) and returns the world's rescue count
int ph_keeper_join(void* world, int stop) {
    World* w = (World*)world;
    if (stop) w->stop = 1;
    if (w->keeper.joinable()) w->keeper.join();
    return (int)w->h->ctl.rescues;
}

}  // extern "C"
