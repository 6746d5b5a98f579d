// TEST INFRASTRUCTURE: the device counterpart of tests/host_check/shadow_math_host.cpp — the product's PCF header
// (vqengine_b200/csrc/vq_shadow_math.cuh) built for sm_90a with the flags of build.sh, so that tests/test_shadow_domain_gpu.py can
// run its pieces one at a time on torch buffers (ctypes, raw device pointers). Never linked into the product.
//   dc_pcf_records    pcf_record as shadow_pcf_kernel calls it: 128-thread blocks, whole warps, the last pixel of a row
//                     duplicated past its end, plus the same counts through an array sink ([n][11], -1 = slot not reported)
//   dc_point_paths    per pixel and point caster, no vote: the general count, the axis path's count where
//                     cube_axis_is_certain holds (-1 elsewhere), the axis and the certainty flag
//   dc_sqrt_sweep     sqrt_rn_inrange against __fsqrt_rn on every fp32 of len2_inrange's domain
//   dc_div_sweep      fdiv / fdiv2 / fdiv3 against __fdiv_rn on log-uniform pairs of div_fast_ok's domain
//   dc_div_list       the same three on given operands
#include "../../vqengine_b200/csrc/vq_common.cuh"
#include "../../vqengine_b200/csrc/vq_shadow_math.cuh"

using namespace vqshadow;

namespace {

struct CountSink {
    int c[11];
    __device__ void operator()(int slot, int count) { c[slot] = count; }
};

__global__ void __launch_bounds__(128) records_kernel(const __grid_constant__ ShadowLights L, const float4* pos, const float4* nrm,
                                                     int width, int rows, unsigned long long* rec, int* counts) {
    const int x = blockIdx.x * blockDim.x + threadIdx.x;
    const int cx = min(x, width - 1);                  // as shadow_pcf_kernel: lanes past the row's end re-compute its last pixel
    for (int r = blockIdx.y; r < rows; r += gridDim.y) {
        const float4 p4 = pos[(size_t)r * width + cx], n4 = nrm[(size_t)r * width + cx];
        Px4 p, n;
        p.x = p4.x; p.y = p4.y; p.z = p4.z; p.w = p4.w; n.x = n4.x; n.y = n4.y; n.z = n4.z; n.w = n4.w;
        const unsigned long long v = pcf_record(L, p, n);
        CountSink s;
        for (int k = 0; k < 11; ++k) s.c[k] = -1;
        caster_counts(L, v3(F(p.x), F(p.y), F(p.z)), v3(F(n.x), F(n.y), F(n.z)), s);
        if (x < width) {
            rec[(size_t)r * width + x] = v;
            for (int k = 0; k < 11; ++k) counts[((size_t)r * width + x) * 11 + k] = s.c[k];
        }
    }
}

__global__ void paths_kernel(const __grid_constant__ ShadowLights L, const float4* pos, int n, int4* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    const int pc = blockIdx.y;
    if (i >= n) return;
    const float4 p4 = pos[i];
    const VqPointLight& l = L.pc[pc];
    const V3 Pw = v3(F(p4.x), F(p4.y), F(p4.z));
    const V3 Lw = v3(l.position) - Pw;
    PCF pcf;
    pcf.depthBias = F(l.depthBias);
    pcf.viewDistanceOfPixel = length(Pw - v3(L.cam));
    const float* cube = L.pointCubes + (size_t)pc * 6 * L.pointRes * L.pointRes;
    int axis;
    const bool certain = cube_axis_is_certain(Lw, pcf.viewDistanceOfPixel, F(l.range), axis);
    const int general = OmnidirectionalShadowCount(pcf, cube, L.pointRes, Lw, F(l.range));
    int fast = -1;
    if (certain) {
        if (axis == 0) fast = OmnidirectionalShadowCountAxis<0>(pcf, cube, L.pointRes, Lw, F(l.range));
        else if (axis == 1) fast = OmnidirectionalShadowCountAxis<1>(pcf, cube, L.pointRes, Lw, F(l.range));
        else fast = OmnidirectionalShadowCountAxis<2>(pcf, cube, L.pointRes, Lw, F(l.range));
    }
    out[(size_t)pc * n + i] = make_int4(general, fast, axis, certain ? 1 : 0);
}

// counters: [0] mismatches, [1] first mismatching input (bits), [2] values checked
__global__ void sqrt_kernel(unsigned lo, unsigned hi, unsigned long long* counters, unsigned* first) {
    unsigned long long bad = 0, seen = 0;
    for (unsigned long long b = lo + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; b < hi; b += (unsigned long long)gridDim.x * blockDim.x) {
        const float x = __uint_as_float((unsigned)b);
        if (!vq::len2_inrange(x)) continue;
        ++seen;
        if (__float_as_uint(vq::sqrt_rn_inrange(x)) != __float_as_uint(__fsqrt_rn(x))) { ++bad; atomicMin(first, (unsigned)b); }
    }
    atomicAdd(counters + 0, bad); atomicAdd(counters + 2, seen);
}

__device__ __forceinline__ unsigned long long mix64(unsigned long long z) {        // splitmix64 finaliser
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull; z = (z ^ (z >> 27)) * 0x94d049bb133111ebull; return z ^ (z >> 31);
}
// log-uniform magnitude 2^e, e uniform in [elo, ehi), random sign
__device__ __forceinline__ float loguni(unsigned long long r, float elo, float ehi) {
    const float u = (float)(r >> 40) * (1.0f / 16777216.0f);
    const float m = exp2f(elo + u * (ehi - elo));
    return (r & 1ull) ? -m : m;
}
// per result: exact equality, except where the rounding correction's residual a - q*b falls below the normal range: a subnormal
// quotient (vq_common.cuh) or a numerator under 2^-100 (|residual| ~ |a| 2^-24). Those may be one ulp off: counted apart.
__device__ __forceinline__ void cmp(float a, float got, float want, unsigned long long* c, unsigned* maxd) {
    const unsigned g = __float_as_uint(got), w = __float_as_uint(want);
    const bool sub = fabsf(want) < 1.17549435e-38f, tiny = !sub && fabsf(a) < 0x1p-100f;
    if (sub) ++c[2];
    if (tiny) ++c[3];
    if (g == w) return;
    if ((sub || tiny) && (g >> 31) == (w >> 31)) {
        const unsigned d = g > w ? g - w : w - g;
        atomicMax(maxd + (sub ? 0 : 1), d);
        if (d <= 1) return;
    }
    ++c[0];
}
// counters: [0] mismatches, [1] pairs inside div_fast_ok, [2] subnormal quotients, [3] normal quotients of numerators < 2^-100;
// maxd: the largest ulp difference of [2] and of [3]
__global__ void div_kernel(unsigned long long seed, unsigned long long n, unsigned long long* counters, unsigned* maxd, float* firstbad) {
    unsigned long long c[4] = {0, 0, 0, 0};
    for (unsigned long long i = (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (unsigned long long)gridDim.x * blockDim.x) {
        const unsigned long long r0 = mix64(seed ^ (i * 0x9e3779b97f4a7c15ull)), r1 = mix64(r0), r2 = mix64(r1), r3 = mix64(r2);
        const float b = loguni(r0, -49.8f, 49.8f);                 // |b| in (1e-15, 1e15)
        const float a0 = loguni(r1, -149.0f, 49.8f);               // |a| down to the subnormals: quotients down to 2^-199
        const float a1 = loguni(r2, -60.0f, 49.8f), a2 = loguni(r3, -60.0f, 49.8f);
        const float amax = fmaxf(fmaxf(fabsf(a0), fabsf(a1)), fabsf(a2));
        if (!div_fast_ok(b, amax)) continue;
        ++c[1];
        F q0, q1, q2, p0, p1;
        fdiv3(F(a0), F(a1), F(a2), F(b), q0, q1, q2);
        fdiv2(F(a0), F(a1), F(b), p0, p1);
        const F s = fdiv(F(a0), F(b));
        const unsigned long long before = c[0];
        const float w0 = __fdiv_rn(a0, b), w1 = __fdiv_rn(a1, b), w2 = __fdiv_rn(a2, b);
        cmp(a0, q0.v, w0, c, maxd); cmp(a1, q1.v, w1, c, maxd); cmp(a2, q2.v, w2, c, maxd);
        cmp(a0, p0.v, w0, c, maxd); cmp(a1, p1.v, w1, c, maxd); cmp(a0, s.v, w0, c, maxd);
        if (c[0] != before && atomicCAS((unsigned*)firstbad, 0u, 1u) == 0u) { firstbad[1] = a0; firstbad[2] = b; }
    }
    for (int k = 0; k < 4; ++k) atomicAdd(counters + k, c[k]);
}

__global__ void div_list_kernel(const float* a, const float* b, int n, float* out) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    F q0, q1, q2, p0, p1;
    fdiv3(F(a[i]), F(a[i]), F(a[i]), F(b[i]), q0, q1, q2);
    fdiv2(F(a[i]), F(a[i]), F(b[i]), p0, p1);
    out[4 * i + 0] = fdiv(F(a[i]), F(b[i])).v;
    out[4 * i + 1] = q0.v;
    out[4 * i + 2] = p0.v;
    out[4 * i + 3] = __fdiv_rn(a[i], b[i]);
}

int sync_status() { cudaError_t e = cudaGetLastError(); if (e == cudaSuccess) e = cudaDeviceSynchronize(); return (int)e; }

}  // namespace

extern "C" {

int dc_pcf_records(const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqShadowMaps* sm, const float* pos,
                   const float* nrm, int width, int rows, unsigned long long* rec, int* counts) {
    ShadowLights L;
    fill_shadow_lights(L, *pf, *pv, *sm);
    records_kernel<<<dim3((width + 127) / 128, rows < 65535 ? rows : 65535), 128>>>(L, (const float4*)pos, (const float4*)nrm, width, rows, rec, counts);
    return sync_status();
}

int dc_point_paths(const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqShadowMaps* sm, const float* pos, int n, int* out) {
    ShadowLights L;
    fill_shadow_lights(L, *pf, *pv, *sm);
    paths_kernel<<<dim3((n + 127) / 128, L.nPointCasters), 128>>>(L, (const float4*)pos, n, (int4*)out);
    return sync_status();
}

int dc_sqrt_sweep(unsigned lo, unsigned hi, unsigned long long* counters, unsigned* first) {
    sqrt_kernel<<<132 * 16, 256>>>(lo, hi, counters, first);
    return sync_status();
}

int dc_div_sweep(unsigned long long seed, unsigned long long n, unsigned long long* counters, unsigned* maxd, float* firstbad) {
    div_kernel<<<132 * 16, 256>>>(seed, n, counters, maxd, firstbad);
    return sync_status();
}

int dc_div_list(const float* a, const float* b, int n, float* out) {
    div_list_kernel<<<(n + 255) / 256, 256>>>(a, b, n, out);
    return sync_status();
}

}  // extern "C"
