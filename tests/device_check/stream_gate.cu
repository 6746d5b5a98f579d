// TEST INFRASTRUCTURE: a gate that holds a stream, for tests/test_stream_contract_gpu.py (ctypes, torch stream handles). Never
// linked into the product.
//   sg_gate_new     one gate: a control word and a status word in mapped, pinned host memory, so that the host opens the gate and
//                   reads its status without any CUDA call (a CUDA call that waits for the device would wait for the gate too)
//   sg_gate_close   launches one thread on `stream` that polls the control word until the host writes 1, with a %globaltimer bound
//                   of bound_ns; it then writes SG_OPENED or SG_TIMED_OUT to the status word (never a trap). Work enqueued on the
//                   stream after it runs only once the gate has opened
//   sg_stream_*     non-blocking streams created through the runtime (cudaStreamCreateWithFlags), their flags, their destruction
#include <cuda_runtime.h>
#include <stdint.h>

namespace {

enum : uint32_t { SG_ARMED = 1, SG_WAITING = 2, SG_OPENED = 3, SG_TIMED_OUT = 4 };

struct Gate {
    volatile uint32_t* word;           // host view: control word [0], status word [1]
    uint32_t* dword;                   // device view of the same two words
};

__device__ __forceinline__ unsigned long long now_ns() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}

__global__ void gate_kernel(uint32_t* w, unsigned long long bound_ns) {
    volatile uint32_t* v = w;
    v[1] = SG_WAITING;
    __threadfence_system();
    const unsigned long long t0 = now_ns();
    uint32_t status = SG_TIMED_OUT;
    for (;;) {
        if (v[0] == 1u) { status = SG_OPENED; break; }
        if (now_ns() - t0 > bound_ns) break;
        __nanosleep(1000);
    }
    __threadfence_system();
    v[1] = status;
    __threadfence_system();
}

}  // namespace

extern "C" {

int sg_gate_new(void** out_gate) {
    Gate* g = new Gate();
    void* h = nullptr;
    cudaError_t e = cudaHostAlloc(&h, 64, cudaHostAllocMapped | cudaHostAllocPortable);
    if (e != cudaSuccess) { delete g; return (int)e; }
    g->word = (volatile uint32_t*)h;
    g->word[0] = 1u; g->word[1] = 0u;
    e = cudaHostGetDevicePointer((void**)&g->dword, h, 0);
    if (e != cudaSuccess) { cudaFreeHost(h); delete g; return (int)e; }
    *out_gate = g;
    return 0;
}

int sg_gate_free(void* gate) {
    Gate* g = (Gate*)gate;
    const cudaError_t e = cudaFreeHost((void*)g->word);
    delete g;
    return (int)e;
}

// the host's view of the two words: the test reads and writes them with ctypes
void* sg_gate_words(void* gate) { return (void*)((Gate*)gate)->word; }

int sg_gate_close(void* gate, void* stream, unsigned long long bound_ns) {
    Gate* g = (Gate*)gate;
    g->word[0] = 0u;
    g->word[1] = SG_ARMED;
    gate_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(g->dword, bound_ns);
    return (int)cudaGetLastError();
}

int sg_stream_create(void** out) { return (int)cudaStreamCreateWithFlags((cudaStream_t*)out, cudaStreamNonBlocking); }
int sg_stream_flags(void* s, unsigned* flags) { return (int)cudaStreamGetFlags((cudaStream_t)s, flags); }
int sg_stream_destroy(void* s) { return (int)cudaStreamDestroy((cudaStream_t)s); }

}  // extern "C"
