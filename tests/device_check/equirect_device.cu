// TEST INFRASTRUCTURE: the product's equirect sampling header (vqengine_b200/csrc/vq_equirect.cuh) built for sm_90a with the
// flags of build.sh, so that tests/test_ibl_domain_gpu.py can run its pieces one at a time on torch buffers (ctypes, raw device
// pointers). Never linked into the product.
//   dc_atan01_sweep   atan01 on every fp32 bit pattern in [lo, hi) against double atan: per-block max |error| and its argument
//   dc_dir_sweep      dir_to_equirect on n pseudo-random unit directions (seeded hash, fp32-rounded) against double
//                     atan2 / asin of the same fp32 components: per-block max |du| (wrapped) and |dv|
//   dc_dir_list       dir_to_equirect on given directions -> (u, v)
//   dc_sample_list    sample_equirect_level on given (u, v, lod) -> rgb
//   dc_texel_frame    normalize_exact(cube_texel_dir(..)) on given texels -> (N, frame decision fabsf(N.z) < 0.999f)
#include "../../vqengine_b200/csrc/vq_common.cuh"
#include "../../vqengine_b200/csrc/vq_equirect.cuh"

namespace {

constexpr int DC_THREADS = 256;

__device__ __forceinline__ void block_max(double e, uint32_t arg, double* outE, uint32_t* outArg) {
    __shared__ double sE[DC_THREADS];
    __shared__ uint32_t sA[DC_THREADS];
    sE[threadIdx.x] = e; sA[threadIdx.x] = arg;
    __syncthreads();
    for (int s = DC_THREADS / 2; s > 0; s >>= 1) {
        if ((int)threadIdx.x < s && sE[threadIdx.x + s] > sE[threadIdx.x]) { sE[threadIdx.x] = sE[threadIdx.x + s]; sA[threadIdx.x] = sA[threadIdx.x + s]; }
        __syncthreads();
    }
    if (threadIdx.x == 0) { outE[blockIdx.x] = sE[0]; outArg[blockIdx.x] = sA[0]; }
}

__global__ void __launch_bounds__(DC_THREADS) atan01_kernel(uint32_t lo, uint32_t hi, uint32_t perThread, double* outE, uint32_t* outArg) {
    const uint64_t first = (uint64_t)lo + ((uint64_t)blockIdx.x * DC_THREADS + threadIdx.x) * perThread;
    double best = -1.0; uint32_t arg = lo;
    for (uint32_t k = 0; k < perThread; ++k) {
        const uint64_t b = first + k;
        if (b >= hi) break;
        const float q = __uint_as_float((uint32_t)b);
        const double e = fabs((double)atan01(q) - atan((double)q));
        if (e > best) { best = e; arg = (uint32_t)b; }
    }
    block_max(best, arg, outE, outArg);
}

__device__ __forceinline__ uint64_t splitmix(uint64_t x) {
    x += 0x9E3779B97F4A7C15ull;
    x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
    x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
    return x ^ (x >> 31);
}

__device__ __forceinline__ void uv_error(float3 d, double& eu, double& ev) {
    float u, v;
    dir_to_equirect(d, u, v);
    const double ru = atan2((double)d.z, (double)d.x) / (-2.0 * 3.141592653589793) + 0.5;
    const double t = fmin(fmax(-(double)d.y, -1.0), 1.0);
    const double rv = asin(t) / 3.141592653589793 + 0.5;
    eu = fabs((double)u - ru); eu = fmin(eu, fabs(1.0 - eu));         // u = 0 and u = 1 are the same column (WRAP)
    ev = fabs((double)v - rv);
}

__global__ void __launch_bounds__(DC_THREADS) dir_kernel(uint64_t seed, uint64_t n, uint32_t perThread, double* outU, uint32_t* argU,
                                                         double* outV, uint32_t* argV) {
    const uint64_t first = ((uint64_t)blockIdx.x * DC_THREADS + threadIdx.x) * perThread;
    double bu = -1.0, bv = -1.0; uint32_t au = 0, av = 0;
    for (uint32_t k = 0; k < perThread; ++k) {
        const uint64_t i = first + k;
        if (i >= n) break;
        const uint64_t r0 = splitmix(seed ^ (2 * i)), r1 = splitmix(seed ^ (2 * i + 1));
        const double z = 2.0 * ((double)(r0 >> 11) * 0x1.0p-53) - 1.0, ph = 2.0 * 3.141592653589793 * ((double)(r1 >> 11) * 0x1.0p-53);
        const double s = sqrt(fmax(0.0, 1.0 - z * z));
        const float3 d = make_float3((float)(s * cos(ph)), (float)z, (float)(s * sin(ph)));   // y is uniform: every latitude
        double eu, ev;
        uv_error(d, eu, ev);
        if (eu > bu) { bu = eu; au = (uint32_t)i; }
        if (ev > bv) { bv = ev; av = (uint32_t)i; }
    }
    block_max(bu, au, outU, argU);
    __syncthreads();
    block_max(bv, av, outV, argV);
}

__global__ void dir_list_kernel(const float* d, int n, float* uv) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    float u, v;
    dir_to_equirect(make_float3(d[3 * i], d[3 * i + 1], d[3 * i + 2]), u, v);
    uv[2 * i] = u; uv[2 * i + 1] = v;
}

__global__ void sample_list_kernel(const PyrV P, const float* uvl, int n, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float3 c = sample_equirect_level(P, uvl[3 * i], uvl[3 * i + 1], uvl[3 * i + 2]);
    out[3 * i] = c.x; out[3 * i + 1] = c.y; out[3 * i + 2] = c.z;
}

__global__ void texel_frame_kernel(const int* t, int n, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const float3 N = normalize_exact(cube_texel_dir(t[4 * i], t[4 * i + 1], t[4 * i + 2], t[4 * i + 3]));
    out[4 * i] = N.x; out[4 * i + 1] = N.y; out[4 * i + 2] = N.z;
    out[4 * i + 3] = fabsf(N.z) < 0.999f ? 1.0f : 0.0f;       // the tangent-frame rule of specular_texel_warp
}

int finish() { return cudaDeviceSynchronize() == cudaSuccess && cudaGetLastError() == cudaSuccess ? 0 : 1; }

}  // namespace

extern "C" {

// blocks = ceil((hi - lo) / (256 * perThread)); outE / outArg hold one entry per block
int dc_atan01_sweep(uint32_t lo, uint32_t hi, uint32_t perThread, double* outE, uint32_t* outArg) {
    const uint64_t per = (uint64_t)DC_THREADS * perThread;
    const unsigned blocks = (unsigned)(((uint64_t)hi - lo + per - 1) / per);
    atan01_kernel<<<blocks, DC_THREADS>>>(lo, hi, perThread, outE, outArg);
    return finish();
}

int dc_dir_sweep(uint64_t seed, uint64_t n, uint32_t perThread, double* outU, uint32_t* argU, double* outV, uint32_t* argV) {
    const uint64_t per = (uint64_t)DC_THREADS * perThread;
    dir_kernel<<<(unsigned)((n + per - 1) / per), DC_THREADS>>>(seed, n, perThread, outU, argU, outV, argV);
    return finish();
}

int dc_dir_list(const float* d, int n, float* uv) {
    dir_list_kernel<<<(n + 127) / 128, 128>>>(d, n, uv);
    return finish();
}

// pyr: packed levels as vq_pyramid_offset lays them out; off: the level offsets (texels), levels <= 16
int dc_sample_list(const float* pyr, int w, int h, int levels, const uint32_t* off, const float* uvl, int n, float* out) {
    PyrV P; P.p = (const float4*)pyr; P.w = w; P.h = h; P.levels = levels;
    for (int l = 0; l < 16; ++l) P.off[l] = l < levels ? off[l] : 0u;
    sample_list_kernel<<<(n + 127) / 128, 128>>>(P, uvl, n, out);
    return finish();
}

int dc_texel_frame(const int* texels, int n, float* out) {
    texel_frame_kernel<<<(n + 127) / 128, 128>>>(texels, n, out);
    return finish();
}

}  // extern "C"
