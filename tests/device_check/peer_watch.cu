// TEST INFRASTRUCTURE: watches the cross-rank rendezvous of the fused gather kernels (vq::peer_rendezvous, vq_common.cuh) from the
// outside, for tests/test_rendezvous_gpu.py (ctypes, raw device pointers, torch stream handles). Never linked into the product.
//   pw_watch       one CTA on the caller's stream: thread 0 acquire-polls one flag word until it EQUALS `epoch` (the tests pre-set
//                  every word to epoch + 1, so "reached or passed" would fire at once), with a %globaltimer bound; once it is seen,
//                  the CTA copies up to 8 device byte ranges into snapshot buffers. status[0] = 1 seen / 2 timed out (never a trap),
//                  status[1] = the %globaltimer of the detection.
//   pw_stamp       one thread writes %globaltimer: queued right after a rank's call, it tells whether the watcher saw the flag while
//                  that call was still running
//   pw_rendezvous  one thread runs vq::peer_rendezvous on a given PeerSync, on flag arrays whose waits are already satisfied
#include "../../vqengine_b200/csrc/vq_common.cuh"

namespace {

struct Ranges {
    const int4* src[8];
    int4* dst[8];
    unsigned long long n16[8];         // 16-byte words of each range
    int n;
};

__device__ __forceinline__ unsigned long long now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void __launch_bounds__(1024) watch_kernel(const uint32_t* flag, uint32_t epoch, unsigned long long bound_ns, Ranges R,
                                                     unsigned long long* status) {
    __shared__ int seen;
    __shared__ unsigned long long when;
    if (threadIdx.x == 0) {
        const unsigned long long t0 = now_ns();
        unsigned long long t = t0;
        int ok = 0;
        for (;;) {
            uint32_t v;
            asm volatile("ld.acquire.sys.global.u32 %0, [%1];" : "=r"(v) : "l"(flag) : "memory");
            t = now_ns();
            if (v == epoch) { ok = 1; break; }
            if (t - t0 > bound_ns) break;
        }
        seen = ok;
        when = t;
    }
    __syncthreads();                   // the acquire, then the barrier: every thread's loads below come after the flag store
    if (seen) {
        // back to front, the ranges interleaved: a persistent CTA's last tile, the one a premature flag would leave unstored, is
        // its highest, so the ends of the ranges are read first
        unsigned long long most = 0;
        for (int k = 0; k < R.n; ++k) most = R.n16[k] > most ? R.n16[k] : most;
        for (long long i = (long long)most - 1 - threadIdx.x; i >= 0; i -= blockDim.x)
            for (int k = 0; k < R.n; ++k)
                if ((unsigned long long)i < R.n16[k]) R.dst[k][i] = __ldcg(R.src[k] + i);
    }
    if (threadIdx.x == 0) {
        status[1] = when;
        status[0] = seen ? 1ull : 2ull;
    }
}

__global__ void stamp_kernel(unsigned long long* out) { *out = now_ns(); }

__global__ void rendezvous_kernel(const PeerSync Y) { vq::peer_rendezvous(Y); }

}  // namespace

extern "C" {

int pw_watch(void* stream, const uint32_t* flag, uint32_t epoch, unsigned long long bound_ns, int n, const void* const* src,
             void* const* dst, const unsigned long long* bytes, unsigned long long* status) {
    if (n < 0 || n > 8) return -1;
    Ranges R;
    memset(&R, 0, sizeof(R));
    for (int k = 0; k < n; ++k) {
        if (bytes[k] % 16 || (uintptr_t)src[k] % 16 || (uintptr_t)dst[k] % 16) return -1;
        R.src[k] = (const int4*)src[k]; R.dst[k] = (int4*)dst[k]; R.n16[k] = bytes[k] / 16;
    }
    R.n = n;
    watch_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(flag, epoch, bound_ns, R, status);
    return (int)cudaGetLastError();
}

int pw_stamp(void* stream, unsigned long long* out) {
    stamp_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(out);
    return (int)cudaGetLastError();
}

int pw_rendezvous(void* stream, uint32_t* const* flags, int n, int my_index, uint32_t epoch) {
    if (n < 2 || n > 8 || my_index < 0 || my_index >= n) return -1;
    PeerSync Y;
    memset(&Y, 0, sizeof(Y));
    for (int k = 0; k < n; ++k) Y.flags[k] = flags[k];
    Y.n = n; Y.myIndex = my_index; Y.epoch = epoch;
    rendezvous_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(Y);
    return (int)cudaGetLastError();
}

}  // extern "C"
