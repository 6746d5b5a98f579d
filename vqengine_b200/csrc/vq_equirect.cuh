// vq_equirect.cuh — equirectangular HDRI pyramid view + the sampling code shared by the IBL kernels (vq_ibl.cu)
// and the skydome pass (vq_frame.cu). Semantics: SURVEY.md §9 (WRAP in u and v, fp32 weights, trilinear).
#pragma once
#include "vq_common.cuh"

namespace {

struct PyrV { const float4* p; int w, h, levels; uint32_t off[16]; };

inline PyrV make_pyr(const VqPyramid& hd) {
    PyrV v; v.p = (const float4*)hd.ptr; v.w = hd.width; v.h = hd.height; v.levels = hd.levels;
    for (int l = 0; l < 16; ++l) v.off[l] = l < hd.levels ? (uint32_t)vq_pyramid_offset(hd.width, hd.height, l) : 0u;
    return v;
}
inline bool pyr_ok(const VqPyramid& hd) {
    return hd.ptr && hd.width > 0 && hd.height > 0 && hd.levels >= 1 && hd.levels <= 16 &&
           hd.levels <= vq_mip_level_count((uint64_t)hd.width, (uint64_t)hd.height) &&
           vq_pyramid_texel_count(hd.width, hd.height, hd.levels) < (1ull << 32);
}


#ifdef __CUDACC__
using namespace vq;
// =============================================================================================
// shared sampling code (SURVEY.md §9; same rules as oracle/oracle_shading.cpp)
// =============================================================================================
// uv produced by dir_to_equirect lie in [0,1] up to rounding, so the bilinear footprint needs at most one wrap step in
// each direction: branch-free conditional add/sub instead of a modulo.
__device__ __forceinline__ float3 bilinear_wrap(const PyrV& t, int level, float u, float v) {
    const int W = t.w >> level, H = t.h >> level;
    const float4* base = t.p + t.off[level];
    const float x = fmaf(u, (float)W, -0.5f), y = fmaf(v, (float)H, -0.5f);
    const float x0 = floorf(x), y0 = floorf(y);
    const float fx = x - x0, fy = y - y0;
    int ix0 = (int)x0, iy0 = (int)y0;
    ix0 = ix0 < 0 ? ix0 + W : ix0;  ix0 = ix0 >= W ? ix0 - W : ix0;
    iy0 = iy0 < 0 ? iy0 + H : iy0;  iy0 = iy0 >= H ? iy0 - H : iy0;
    ix0 = min(max(ix0, 0), W - 1);  iy0 = min(max(iy0, 0), H - 1);     // safety net for non-finite uv
    const int ix1 = ix0 + 1 == W ? 0 : ix0 + 1, iy1 = iy0 + 1 == H ? 0 : iy0 + 1;
    const uint32_t r0 = (uint32_t)(iy0 * W), r1 = (uint32_t)(iy1 * W);
    const float4 t00 = __ldg(base + (r0 + ix0)), t10 = __ldg(base + (r0 + ix1));
    const float4 t01 = __ldg(base + (r1 + ix0)), t11 = __ldg(base + (r1 + ix1));
    const float3 top = lerp(xyz(t00), xyz(t10), fx), bot = lerp(xyz(t01), xyz(t11), fx);
    return lerp(top, bot, fy);
}

__device__ __forceinline__ float3 sample_equirect_level(const PyrV& t, float u, float v, float lod) {
    lod = fminf(fmaxf(lod, 0.0f), (float)(t.levels - 1));
    const float l0f = floorf(lod);
    const int l0 = (int)l0f;
    const float f = lod - l0f;
    const float3 c0 = bilinear_wrap(t, l0, u, v);
    if (f == 0.0f || l0 + 1 >= t.levels) return c0;
    const float3 c1 = bilinear_wrap(t, l0 + 1, u, v);
    return lerp(c0, c1, f);
}

// atan(q) for q in [0,1]: q * P(q^2), degree-8 minimax fit; |error| <= 1.0e-7 evaluated in fp32 (about 1.7 ulp at pi/4,
// the same class as CUDA's atan2f at ~1/3 of its instruction count). Fitted and checked in tools/fit_atan.py.
__device__ __forceinline__ float atan01(float q) {
    const float z = q * q;
    float p = 0.002456721616908908f;
    p = fmaf(p, z, -0.014401346445083618f);
    p = fmaf(p, z, 0.03978120535612106f);
    p = fmaf(p, z, -0.07234855741262436f);
    p = fmaf(p, z, 0.10498945415019989f);
    p = fmaf(p, z, -0.14161229133605957f);
    p = fmaf(p, z, 0.19985906779766083f);
    p = fmaf(p, z, -0.33332598209381104f);
    p = fmaf(p, z, 0.9999998807907104f);
    return p * q;
}
// atan2(y, x) in [-pi, pi] by octant reduction onto atan01
__device__ __forceinline__ float atan2_fast(float y, float x) {
    const float ax = fabsf(x), ay = fabsf(y);
    const float mx = fmaxf(ax, ay), mn = fminf(ax, ay);
    float r = atan01(mn * rcp_fast(fmaxf(mx, 1e-30f)));
    r = ay > ax ? 1.57079632679f - r : r;
    r = x < 0.0f ? 3.14159265359f - r : r;
    return copysignf(r, y);
}
__device__ __forceinline__ float sqrt_fast(float x) { float r; asm("sqrt.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(x)); return r; }

// DirectionToEquirectUV, ShadingMath.hlsl:70-80:  u = atan2(z,x)/(-2pi) + 0.5,  v = asin(-y)/pi + 0.5.
// asin(-y) = pi/2 - acos(-y) and acos(t) = 2*atan2(sqrt(1-t), sqrt(1+t)), so both angles go through atan01.
__device__ __forceinline__ void dir_to_equirect(float3 d, float& u, float& v) {
    u = fmaf(atan2_fast(d.z, d.x), -1.0f / TWO_PI, 0.5f);
    const float t = fminf(fmaxf(-d.y, -1.0f), 1.0f);           // |d.y| can overshoot 1 by an ulp after an rsqrt-normalise
    const float a = sqrt_fast(1.0f - t), b = sqrt_fast(1.0f + t);   // both >= 0
    const float mx = fmaxf(a, b), mn = fminf(a, b);
    float r = atan01(mn * rcp_fast(mx));                       // atan2(a, b) in [0, pi/2]
    r = a > b ? 1.57079632679f - r : r;
    // asin(t) = pi/2 - 2*atan2(a,b)  ->  v = asin(t)/pi + 0.5 = 1 - 2*r/pi
    v = fmaf(r, -2.0f / PI, 1.0f);
}

// A35: look direction of a cube texel (CubemapUtility.cpp:40-48 + 90-degree projection)
__device__ __forceinline__ float3 cube_texel_dir(int face, int px, int py, int res) {
    const float sx = 2.0f * ((float)px + 0.5f) / (float)res - 1.0f;
    const float sy = 1.0f - 2.0f * ((float)py + 0.5f) / (float)res;
    switch (face) {
        case 0: return f3(1.0f, sy, -sx);
        case 1: return f3(-1.0f, sy, sx);
        case 2: return f3(sx, 1.0f, -sy);
        case 3: return f3(sx, -1.0f, sy);
        case 4: return f3(sx, sy, 1.0f);
        default: return f3(-sx, sy, -1.0f);
    }
}
// exact normalize (v / sqrt(dot)) for the texel basis: it feeds every sample of the texel
__device__ __forceinline__ float3 normalize_exact(float3 v) {
    const float l = sqrtf(dot(v, v));
    return f3(v.x / l, v.y / l, v.z / l);
}

#endif  // __CUDACC__

}  // namespace
