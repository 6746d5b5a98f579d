// vq_ibl.cu — environment-map kernels for sm_90a:
//   K11 HDRI min-filter mip pyramid   (DXGIUtils.cpp:289-317)
//   K2  diffuse irradiance            (CubemapConvolution.hlsl:112-163)
//   K3  specular prefilter            (CubemapConvolution.hlsl:168-223)
//   K4  BRDF integration LUT          (CubemapConvolution.hlsl:227-240, BRDF.hlsl:239-283)
//
// K2/K3: one warp per output texel, lanes stride over the hemisphere samples, partial sums are
// combined with a __shfl_xor butterfly. Everything that does not depend on the texel (the sin/cos of
// the (phi,theta) grid, the tangent-space GGX half vectors of the Hammersley set) is computed once per
// block into shared memory. The HDRI is read through the read-only path (L1/L2): the diffuse integral
// touches half the sphere per texel, so there is no tile to stage; see DESIGN.md for the bound
// (SFU/FP32 + L1, not HBM). K4: one thread per LUT texel (same sequential sum as the HLSL), the
// per-row half-vector table in shared memory is a broadcast read.
#include "vq_common.cuh"
#include "vq_equirect.cuh"
#include <vector>

using namespace vq;

namespace {

// =============================================================================================
// K11: level l+1 = 2x2 MIN of level l (rgb), alpha = 1
// =============================================================================================
__global__ void __launch_bounds__(256) hdri_min_mip_kernel(const float4* __restrict__ src, float4* __restrict__ dst,
                                                           int srcW, int dstW, int dstH) {
    const int x = blockIdx.x * 64 + (threadIdx.x & 63);
    const int y = blockIdx.y * 4 + (threadIdx.x >> 6);
    if (x >= dstW || y >= dstH) return;
    const float4* r0 = src + (size_t)(2 * y) * srcW + 2 * x;
    const float4* r1 = r0 + srcW;
    const float4 a = ld_stream(r0), b = ld_stream(r0 + 1), c = ld_stream(r1), d = ld_stream(r1 + 1);
    // min(rgb[0], min(rgb[1], min(rgb[2], rgb[3]))), samples ordered (0,0),(1,0),(0,1),(1,1)
    float4 o;
    o.x = min4_ref(a.x, b.x, c.x, d.x);
    o.y = min4_ref(a.y, b.y, c.y, d.y);
    o.z = min4_ref(a.z, b.z, c.z, d.z);
    o.w = 1.0f;
    dst[(size_t)y * dstW + x] = o;
}

// =============================================================================================
// K2 diffuse irradiance
// =============================================================================================
constexpr int IBL_THREADS = 256;
constexpr int IBL_WARPS = IBL_THREADS / 32;

struct DiffuseArgs {
    PyrV hdri; int res; int rowBegin; int texels;   // texels = rows * res
    float step; int nPhi, nTheta; int srcMip;
};
// Every texel goes to each of n packed cubemaps (the local one first, then the peers'), and with a rendezvous the last CTA to retire
// runs it (cta_retire). vq_diffuse_irradiance is the band form with one destination and no rendezvous.
struct DiffuseMultiArgs {
    DiffuseArgs a;
    float4* o[8]; int n;
    PeerSync sync;
    uint32_t* ticket;                    // retired-CTA count (zero between launches); sync.n > 1 only
};

// The texels of K2 that this CTA's warps own, each handed to store(texel index, value) by lane 0 of its warp. A texel's bits depend
// only on its own warp (lane-strided sums, then the warp_sum butterfly), not on the CTA or the grid it runs in.
template <class Store>
__device__ __forceinline__ void diffuse_texels(const DiffuseArgs& A, float* smem, Store store) {
    float* sSinP = smem;                 // [nPhi]
    float* sCosP = sSinP + A.nPhi;       // [nPhi]
    float* sSinT = sCosP + A.nPhi;       // [nTheta]
    float* sCosT = sSinT + A.nTheta;     // [nTheta]
    // ---- the (phi, theta) sequences of the HLSL loops (CubemapConvolution.hlsl:129-135) ----
    if (A.step > 0.0f) {
        // float-accumulated loop variable: inherently sequential, so one thread per table walks it
        if (threadIdx.x == 0) { float phi = 0.0f; for (int i = 0; i < A.nPhi; ++i) { sSinP[i] = phi; phi += A.step; } }
        if (threadIdx.x == 32) { float th = 0.0f; for (int j = 0; j < A.nTheta; ++j) { sSinT[j] = th; th += A.step; } }
    } else {
        const float dphi = TWO_PI / (float)A.nPhi, dth = PI_OVER_TWO / (float)A.nTheta;
        for (int i = threadIdx.x; i < A.nPhi; i += IBL_THREADS) sSinP[i] = (float)i * dphi;
        for (int j = threadIdx.x; j < A.nTheta; j += IBL_THREADS) sSinT[j] = (float)j * dth;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < A.nPhi; i += IBL_THREADS) { const float a = sSinP[i]; float s, c; sincosf(a, &s, &c); sSinP[i] = s; sCosP[i] = c; }
    for (int j = threadIdx.x; j < A.nTheta; j += IBL_THREADS) { const float a = sSinT[j]; float s, c; sincosf(a, &s, &c); sSinT[j] = s; sCosT[j] = c; }
    __syncthreads();

    const int lane = threadIdx.x & 31;
    const int warpGlobal = blockIdx.x * IBL_WARPS + (threadIdx.x >> 5);
    const int warpCount = gridDim.x * IBL_WARPS;
    const int nSamples = A.nPhi * A.nTheta;
    for (int tx = warpGlobal; tx < A.texels; tx += warpCount) {
        const int fr = A.rowBegin + tx / A.res, px = tx % A.res;
        const int face = fr / A.res, py = fr % A.res;
        const float3 N = normalize_exact(cube_texel_dir(face, px, py, A.res));
        const float3 right = normalize_exact(cross(f3(0.0f, 1.0f, 0.0f), N));
        const float3 up = normalize_exact(cross(N, right));
        float3 acc = f3(0.0f);
        for (int s = lane; s < nSamples; s += 32) {
            const int ip = s / A.nTheta, it = s - ip * A.nTheta;
            const float sinT = sSinT[it], cosT = sCosT[it], sinP = sSinP[ip], cosP = sCosP[ip];
            const float tsx = sinT * cosP, tsy = sinT * sinP;
            float3 sv = right * tsx + up * tsy + N * cosT;
            sv = normalize(sv);
            float u, v; dir_to_equirect(sv, u, v);
            const float3 Lc = sample_equirect_level(A.hdri, u, v, (float)A.srcMip);
            const float w = cosT * sinT;
            acc.x = fmaf(Lc.x, w, acc.x); acc.y = fmaf(Lc.y, w, acc.y); acc.z = fmaf(Lc.z, w, acc.z);
        }
        acc.x = warp_sum(acc.x); acc.y = warp_sum(acc.y); acc.z = warp_sum(acc.z);
        if (lane == 0) {
            const float n = (float)nSamples;     // numSamples += 1.0f per sample: exact below 2^24
            store((size_t)fr * A.res + px, make_float4(PI * acc.x / n, PI * acc.y / n, PI * acc.z / n, 1.0f));
        }
    }
}

__global__ void __launch_bounds__(IBL_THREADS) diffuse_irradiance_multi_kernel(const __grid_constant__ DiffuseMultiArgs M) {
    extern __shared__ float smem[];
    diffuse_texels(M.a, smem, [&](size_t i, float4 o) {
#pragma unroll
        for (int q = 0; q < 8; ++q)      // constant indices: the pointers stay in the parameter bank
            if (q < M.n) M.o[q][i] = o;
    });
    cta_retire(M);
}

// =============================================================================================
// K3 specular prefilter
// =============================================================================================
__device__ __forceinline__ float radical_inverse_vdc(uint32_t bits) {      // ShadingMath.hlsl:87-95
    return (float)__brev(bits) * 2.3283064365386963e-10f;
}

// One launch covers everything a caller (or a rank) has to prefilter: the flattened (mip, face, row) ranges are cut at mip
// boundaries into SEGMENTS, segments into UNITS of about equal cost, and a persistent grid pulls units off one global ticket:
//   roughness > 0: unit = 8 texels, one warp each, lanes stride the 512 samples          (~19 k warp-instructions)
//   roughness = 0: unit = 256 texels, one thread each (the mip-0 replay below)          (~17 k warp-instructions)
// so there are no per-mip launches, no launch gaps and no per-mip tails (round 1: 9 launches, 81 % efficient at 8 GPUs).
// A CTA sees its units in increasing order, so it rebuilds the tangent-space GGX table only when the mip changes.
// Every finished texel is stored into up to 8 destination cubemaps (the other ranks' buffers over NVLink: fused gather);
// the LAST CTA to retire can then run the cross-rank rendezvous itself (SpecSync), so a step is ONE kernel.
struct SpecSeg { int n, rowBegin, texels; uint32_t unitBegin, mipOff; float roughness; };
constexpr int SPEC_MAX_SEGS = 24;
struct SpecWork {
    PyrV hdri;
    float4* outs[8]; int nOuts;   // packed cubemaps (mip 0 face 0 first): the local one, then the peers'
    SpecSeg seg[SPEC_MAX_SEGS]; int nSeg; uint32_t totalUnits;
    float dimX, dimY; int numSamples;
    uint32_t* ticket;             // [0] next unit, [1] retired CTAs; both zero between launches (the last CTA resets them)
    PeerSync sync;                // optional end-of-pass rendezvous through peer-mapped flag words (n == 0: none)
};
constexpr int SPEC_UNIT_WARP_TEXELS = IBL_WARPS, SPEC_UNIT_THREAD_TEXELS = IBL_THREADS;

__device__ __forceinline__ void spec_store(const SpecWork& W, size_t texel, float4 o) {
    W.outs[0][texel] = o;
    for (int k = 1; k < W.nOuts; ++k) W.outs[k][texel] = o;
}

// Roughness 0 (mip 0): every sample is the same direction (H = N, L = N, source mip 0), so the texel is the
// weighted mean of numSamples IDENTICAL terms. One THREAD per texel samples the HDRI once and then replays the
// HLSL's running sums sequentially (4 independent FADD chains), so their fp32 rounding is reproduced exactly.
__device__ __forceinline__ float4 specular_texel_mip0(const SpecWork& W, int n, int face, int px, int py) {
    const float3 N = normalize_exact(cube_texel_dir(face, px, py, n));
    const float3 H = normalize_exact(N);                       // ImportanceSampleGGX with sinTheta = 0
    const float3 Lv = H * (2.0f * dot(N, H)) - N;              // reflect(-V, H), V = N
    const float NdotL = saturate(dot(N, Lv));
    float4 o = make_float4(0.0f, 0.0f, 0.0f, 1.0f);
    if (NdotL > 0.0f) {
        float u, v; dir_to_equirect(Lv, u, v);
        const float3 c = sample_equirect_level(W.hdri, u, v, 0.0f);
        const float t0 = c.x * NdotL, t1 = c.y * NdotL, t2 = c.z * NdotL;
        float a0 = 0.0f, a1 = 0.0f, a2 = 0.0f, aw = 0.0f;
        for (int i = 0; i < W.numSamples; ++i) {
            a0 = __fadd_rn(a0, t0); a1 = __fadd_rn(a1, t1); a2 = __fadd_rn(a2, t2); aw = __fadd_rn(aw, NdotL);
        }
        const float d = fmaxf(aw, 0.0001f);
        o = make_float4(a0 / d, a1 / d, a2 / d, 1.0f);
    }
    return o;
}

// one warp, one texel: lanes stride the importance samples (sH = tangent-space half vectors of this roughness)
__device__ __forceinline__ float4 specular_texel_warp(const SpecWork& W, const float4* __restrict__ sH, float roughness, int lane,
                                                      int n, int face, int px, int py) {
    // Solid angle of one texel of a 6 x W0 x H0 cube — W0,H0 are the HDRI dims: the reference's quirk
    const float fOmegaP = 4.0f * PI / (6.0f * W.dimX * W.dimY);
    const float fN = (float)W.numSamples;
    const float3 N = normalize_exact(cube_texel_dir(face, px, py, n));   // N = R = V
    // tangent frame (BRDF.hlsl:231-234)
    const float3 upv = fabsf(N.z) < 0.999f ? f3(0, 0, 1) : f3(1, 0, 0);
    const float3 T = normalize_exact(cross(upv, N));
    const float3 B = cross(N, T);
    const float a = roughness * roughness, a2 = a * a;
    float3 acc = f3(0.0f); float wsum = 0.0f;
    for (int i = lane; i < W.numSamples; i += 32) {
        const float4 h = sH[i];
        float3 H = T * h.x + B * h.y + N * h.z;
        H = normalize(H);
        const float VdotH = dot(N, H);
        const float3 Lv = H * (2.0f * VdotH) - N;                          // reflect(-V, H)
        const float NdotL = saturate(dot(N, Lv));
        if (NdotL > 0.0f) {
            const float NdotH = saturate(VdotH);
            const float HdotV = NdotH;
            // NormalDistributionGGX (BRDF.hlsl:65-79)
            const float t = fmaf(NdotH * NdotH, a2 - 1.0f, 1.0f);
            const float dDen = PI * (t * t);
            const float D = dDen < 0.000000000001f ? 1.0f : a2 * rcp_fast(dDen);
            const float pdf = (D * NdotH) * rcp_fast(4.0f * HdotV);
            // 0.5*log2(omegaS/omegaP) - 1 with omegaS = 1/max(N*pdf, 1e-5): one lg2 of the product, no divisions
            const float mip = fmaxf(fmaf(-0.5f, __log2f(fmaxf(fN * pdf, 0.00001f) * fOmegaP), -1.0f), 0.0f);
            float u, v; dir_to_equirect(Lv, u, v);
            const float3 c = sample_equirect_level(W.hdri, u, v, mip);
            acc.x = fmaf(c.x, NdotL, acc.x); acc.y = fmaf(c.y, NdotL, acc.y); acc.z = fmaf(c.z, NdotL, acc.z);
            wsum += NdotL;
        }
    }
    acc.x = warp_sum(acc.x); acc.y = warp_sum(acc.y); acc.z = warp_sum(acc.z); wsum = warp_sum(wsum);
    const float d = fmaxf(wsum, 0.0001f);
    return make_float4(acc.x / d, acc.y / d, acc.z / d, 1.0f);
}

__global__ void __launch_bounds__(IBL_THREADS) specular_persistent_kernel(const __grid_constant__ SpecWork W) {
    extern __shared__ float4 sH[];       // tangent-space half vectors of the current roughness: (cos(phi)*sinT, sin(phi)*sinT, cosT, -)
    __shared__ uint32_t sUnit[2];        // double-buffered: the fetch of unit k+1 overlaps nothing it could race with
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    float tableRoughness = -1.0f;
    int segIdx = 0, it = 0;
    for (;; ++it) {
        if (threadIdx.x == 0) sUnit[it & 1] = atomicAdd(W.ticket, 1u);
        __syncthreads();
        const uint32_t u = sUnit[it & 1];
        if (u >= W.totalUnits) break;
        while (segIdx + 1 < W.nSeg && u >= W.seg[segIdx + 1].unitBegin) ++segIdx;     // units (and so segments) only move forward
        const SpecSeg S = W.seg[segIdx];
        const uint32_t lu = u - S.unitBegin;
        if (S.roughness == 0.0f) {
            const int tx = (int)lu * SPEC_UNIT_THREAD_TEXELS + (int)threadIdx.x;
            if (tx < S.texels) {
                const int fr = S.rowBegin + tx / S.n, px = tx % S.n;
                spec_store(W, (size_t)S.mipOff + (size_t)fr * S.n + px, specular_texel_mip0(W, S.n, fr / S.n, px, fr % S.n));
            }
        } else {
            if (S.roughness != tableRoughness) {          // ImportanceSampleGGX (BRDF.hlsl:217-229): the part that depends only on (i, roughness)
                __syncthreads();                          // nobody still reads the previous table
                for (int i = threadIdx.x; i < W.numSamples; i += IBL_THREADS) {
                    const float xi_x = (float)i / (float)W.numSamples;        // Hammersley, ShadingMath.hlsl:119-127
                    const float xi_y = radical_inverse_vdc((uint32_t)i);
                    const float a = S.roughness * S.roughness;
                    const float phi = 2.0f * PI * xi_x;
                    const float cosTheta = sqrtf((1.0f - xi_y) / (1.0f + (a * a - 1.0f) * xi_y));
                    const float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
                    float sp, cp; sincosf(phi, &sp, &cp);
                    sH[i] = make_float4(cp * sinTheta, sp * sinTheta, cosTheta, 0.0f);
                }
                tableRoughness = S.roughness;
                __syncthreads();
            }
            const int tx = (int)lu * SPEC_UNIT_WARP_TEXELS + warp;
            if (tx < S.texels) {
                const int fr = S.rowBegin + tx / S.n, px = tx % S.n;
                const float4 o = specular_texel_warp(W, sH, S.roughness, lane, S.n, fr / S.n, px, fr % S.n);
                if (lane == 0) spec_store(W, (size_t)S.mipOff + (size_t)fr * S.n + px, o);
            }
        }
    }
    // ---- retire: the last CTA resets the ticket and, when asked to, runs the cross-rank rendezvous ----
    __threadfence_system();                                // this CTA's (peer) stores are ordered before its retirement
    __syncthreads();
    if (threadIdx.x == 0) {
        const uint32_t done = atomicAdd(W.ticket + 1, 1u);
        if (done == gridDim.x - 1) {
            W.ticket[0] = 0u; W.ticket[1] = 0u;            // every CTA has fetched its terminating ticket by now
            __threadfence_system();                        // every CTA's stores happen-before the signals below (cumulativity)
            peer_rendezvous(W.sync);
        }
    }
}

// =============================================================================================
// K4 BRDF integration LUT
// =============================================================================================
struct LutArgs { float2* out; int w, h, pitch2; int rowBegin; int numSamples; };
// The multi-destination form (vq_brdf_integration_lut_multi_signal): n float2 images of one size (the local one first, then the
// peers'), each with its own pitch; the last CTA to retire runs the rendezvous. A.out and A.pitch2 are unused.
struct LutMultiArgs {
    LutArgs a;
    float2* o[8]; int pitch2[8]; int n;
    PeerSync sync;
    uint32_t* ticket;                    // retired-CTA count (zero between launches); sync.n > 1 only
};

// One CTA: texels [256 blockIdx.x, +256) of row rowBegin + blockIdx.y, each handed to store(x, y, value) by its thread
template <class Store>
__device__ __forceinline__ void brdf_lut_texels(const LutArgs& A, float4* sHw, Store store) {
    const int y = A.rowBegin + blockIdx.y;
    const float roughness = ((float)y + 0.5f) / (float)A.h;                  // CubemapConvolution.hlsl:234-236
    for (int i = threadIdx.x; i < A.numSamples; i += 256) {
        const float xi_x = (float)i / (float)A.numSamples;
        const float xi_y = radical_inverse_vdc((uint32_t)i);
        const float a = roughness * roughness;
        const float phi = 2.0f * PI * xi_x;
        const float cosTheta = sqrtf((1.0f - xi_y) / (1.0f + (a * a - 1.0f) * xi_y));
        const float sinTheta = sqrtf(1.0f - cosTheta * cosTheta);
        float sp, cp; sincosf(phi, &sp, &cp);
        // N = (0,0,1): up = (1,0,0), tangent = (0,-1,0), bitangent = (1,0,0)  (BRDF.hlsl:231-236)
        const float3 s = f3(sp * sinTheta, -(cp * sinTheta), cosTheta);
        const float l = sqrtf(dot(s, s));
        sHw[i] = make_float4(s.x / l, s.y / l, s.z / l, 0.0f);
    }
    __syncthreads();
    const int x = blockIdx.x * 256 + threadIdx.x;
    if (x >= A.w) return;
    const float NdotV = ((float)x + 0.5f) / (float)A.w;
    const float3 V = f3(sqrtf(1.0f - NdotV * NdotV), 0.0f, NdotV);          // BRDF.hlsl:241-244
    const float k = (roughness * roughness) * 0.5f, omk = 1.0f - k;         // BRDF.hlsl:110
    const float NVg = fmaxf(0.0f, V.z);
    const float geomNV = NVg / (fmaf(NVg, omk, k) + 0.0001f);
    float F0Scale = 0.0f, F0Bias = 0.0f;
    for (int i = 0; i < A.numSamples; ++i) {
        const float4 h = sHw[i];
        const float3 H = f3(h.x, h.y, h.z);
        const float VdotHr = dot(V, H);
        float3 Lv = H * (2.0f * VdotHr) - V;                                 // reflect(-V, H)
        Lv = normalize(Lv);
        const float NdotL = fmaxf(Lv.z, 0.0f);
        const float NdotH = fmaxf(H.z, 0.0f);
        const float VdotH = fmaxf(VdotHr, 0.0f);
        if (NdotL > 0.0f) {
            const float geomNL = NdotL / (fmaf(NdotL, omk, k) + 0.0001f);
            const float G = geomNV * geomNL;
            const float G_Vis = fmaxf((G * VdotH) / (NdotH * NdotV), 0.0001f);
            const float Fc = pow5(1.0f - VdotH);
            F0Scale = fmaf(1.0f - Fc, G_Vis, F0Scale);
            F0Bias = fmaf(Fc, G_Vis, F0Bias);
        }
    }
    const float n = (float)A.numSamples;
    store(x, y, make_float2(F0Scale / n, F0Bias / n));
}

__global__ void __launch_bounds__(256) brdf_lut_kernel(const __grid_constant__ LutArgs A) {
    extern __shared__ float4 sHw[];      // world-space half vectors for this row's roughness (N = +Z)
    brdf_lut_texels(A, sHw, [&](int x, int y, float2 v) { A.out[(size_t)y * A.pitch2 + x] = v; });
}

__global__ void __launch_bounds__(256) brdf_lut_multi_kernel(const __grid_constant__ LutMultiArgs M) {
    extern __shared__ float4 sHw[];
    brdf_lut_texels(M.a, sHw, [&](int x, int y, float2 v) {
#pragma unroll
        for (int q = 0; q < 8; ++q)
            if (q < M.n) M.o[q][(size_t)y * M.pitch2[q] + x] = v;
    });
    cta_retire(M);        // also the threads past the row's last texel, which left brdf_lut_texels early
}

}  // namespace

// =============================================================================================
// C-ABI
// =============================================================================================
extern "C" int vq_hdri_build_mips(VqContext* ctx, VqPyramid hd, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("EnvironmentMap");
    VQ_REQUIRE(pyr_ok(hd), "bad HDRI pyramid descriptor");
    if (hd.levels == 1) return VQ_OK;
    // one launch for the whole chain when the image fits the SPD kernel (<= 4096^2, <= 12 destination levels)
    if (hd.width <= 4096 && hd.height <= 4096 && hd.levels - 1 <= 12)
        return vq_spd_min_pyramid(ctx, hd, (cudaStream_t)stream);
    float4* base = (float4*)hd.ptr;
    for (int l = 1; l < hd.levels; ++l) {
        const int sw = hd.width >> (l - 1), dw = hd.width >> l, dh = hd.height >> l;
        const dim3 grid((dw + 63) / 64, (dh + 3) / 4);
        hdri_min_mip_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(base + vq_pyramid_offset(hd.width, hd.height, l - 1),
                                                                    base + vq_pyramid_offset(hd.width, hd.height, l), sw, dw, dh);
        rc = vq_check_launch("hdri_build_mips"); if (rc) return rc;
    }
    return VQ_OK;
}

// K2 on rows [row_begin, row_end) into every destination cubemap, with the optional in-kernel rendezvous: the band call, and the
// single call with one destination and no signal. Every argument is checked before the device is touched.
static int diffuse_launch(VqContext* ctx, const VqDiffuseIrradianceParams* p, VqPyramid hd, const VqCubemap* outs, int n_outs,
                          int row_begin, int row_end, const VqPeerSignal* sig, cudaStream_t stream, const char* what) {
    int rc = vq_band_list(outs, n_outs); if (rc) return rc;
    VQ_REQUIRE(p, "params is null");
    VQ_REQUIRE(pyr_ok(hd), "bad HDRI pyramid descriptor");
    const VqCubemap out = outs[0];
    VQ_REQUIRE(out.ptr && out.res >= 2 && out.mips == 1, "diffuse irradiance cubemap must have 1 mip");
    VQ_REQUIRE((out.res & 1) == 0, "cubemap resolution must be even (pole texel, SURVEY.md A32)");
    VQ_REQUIRE(p->src_mip >= 0 && p->src_mip < hd.levels, "src_mip outside the pyramid");
    for (int k = 1; k < n_outs; ++k) {
        VQ_REQUIRE(outs[k].ptr && outs[k].res == outs[0].res && outs[k].mips == outs[0].mips, "every destination cubemap must have the same shape");
        VQ_REQUIRE(outs[k].ptr != outs[0].ptr, "a peer destination must not be the local cubemap outs[0]");
    }
    DiffuseMultiArgs M;
    memset(&M, 0, sizeof(M));
    rc = vq_band_check(ctx, n_outs, 0, 6 * out.res, row_begin, row_end, sig, M.sync); if (rc) return rc;
    int nPhi, nTheta;
    if (p->step > 0.0f) {
        // trip counts of the float-accumulated loops (CubemapConvolution.hlsl:129,133)
        nPhi = 0; for (float phi = 0.0f; phi < 6.28318530718f; phi += p->step) { if (++nPhi > (1 << 20)) break; }
        nTheta = 0; for (float th = 0.0f; th < 1.5707963268f; th += p->step) { if (++nTheta > (1 << 20)) break; }
    } else { nPhi = p->n_phi; nTheta = p->n_theta; }
    VQ_REQUIRE(nPhi >= 1 && nTheta >= 1 && (long long)nPhi * nTheta < (1 << 24), "sample grid out of range");
    const size_t smem = (size_t)(2 * nPhi + 2 * nTheta) * sizeof(float);
    VQ_REQUIRE(smem <= 200 * 1024, "sample grid does not fit shared memory");
    DiffuseArgs& A = M.a;
    A.hdri = make_pyr(hd); A.res = out.res; A.rowBegin = row_begin;
    A.texels = (row_end - row_begin) * out.res;
    A.step = p->step > 0.0f ? p->step : 0.0f; A.nPhi = nPhi; A.nTheta = nTheta; A.srcMip = p->src_mip;
    for (int k = 0; k < n_outs; ++k) M.o[k] = (float4*)outs[k].ptr;
    M.n = n_outs;
    rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("DiffuseIrradianceCubemap");
    if (row_begin == row_end) return VQ_OK;
    M.ticket = vq_band_ticket(ctx, M.sync);
    if (smem > 48 * 1024) VQ_CUDA_OK(cudaFuncSetAttribute(diffuse_irradiance_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    int blocks = (M.a.texels + IBL_WARPS - 1) / IBL_WARPS;         // one warp per texel, at most 8 CTAs per SM (striding the texels)
    if (blocks > ctx->sm_count * 8) blocks = ctx->sm_count * 8;
    diffuse_irradiance_multi_kernel<<<blocks, IBL_THREADS, smem, stream>>>(M);
    return vq_check_launch(what);
}

extern "C" int vq_diffuse_irradiance(VqContext* ctx, const VqDiffuseIrradianceParams* p, VqPyramid hd, VqCubemap out,
                                     int row_begin, int row_end, void* stream) {
    const int rc = vq_enter(ctx); if (rc) return rc;               // the single call refuses a null context first
    return diffuse_launch(ctx, p, hd, &out, 1, row_begin, row_end, nullptr, (cudaStream_t)stream, "diffuse_irradiance");
}

// one rank's band of a multi-GPU prefilter
extern "C" int vq_diffuse_irradiance_multi_signal(VqContext* ctx, const VqDiffuseIrradianceParams* p, VqPyramid hd,
                                                  const VqCubemap* outs, int n_outs, int row_begin, int row_end,
                                                  const VqPeerSignal* signal, void* stream) {
    return diffuse_launch(ctx, p, hd, outs, n_outs, row_begin, row_end, signal, (cudaStream_t)stream, "diffuse_irradiance_multi");
}

// ranges: n_ranges pairs [begin,end) of the flattened (mip, face, row) space, in increasing order and disjoint
static int specular_launch(VqContext* ctx, VqPyramid hd, const VqCubemap* outs, int n_outs, int num_samples,
                           const int* ranges, int n_ranges, const VqPeerSignal* sig, cudaStream_t stream) {
    VQ_REQUIRE(outs && n_outs >= 1 && n_outs <= 8, "1..8 destination cubemaps");
    const VqCubemap out = outs[0];
    VQ_REQUIRE(pyr_ok(hd), "bad HDRI pyramid descriptor");
    VQ_REQUIRE(out.ptr && out.res >= 2 && out.mips >= 2 && out.mips <= 16 && (out.res >> (out.mips - 1)) >= 1, "bad specular cubemap descriptor");
    VQ_REQUIRE((out.res >> (out.mips - 1)) % 2 == 0 || (out.res >> (out.mips - 1)) == 1, "every mip needs an even edge (pole texel)");
    for (int k = 1; k < n_outs; ++k)
        VQ_REQUIRE(outs[k].ptr && outs[k].res == out.res && outs[k].mips == out.mips, "every destination cubemap must have the same shape");
    VQ_REQUIRE(num_samples >= 1 && num_samples <= 8192, "num_samples out of range");
    VQ_REQUIRE(ranges && n_ranges >= 1, "no row ranges");
    const int totalRows = vq_cubemap_row_count(out.res, out.mips);
    SpecWork W;
    memset(&W, 0, sizeof(W));
    int prevEnd = 0;
    uint32_t units = 0;
    for (int r = 0; r < n_ranges; ++r) {
        const int row_begin = ranges[2 * r], row_end = ranges[2 * r + 1];
        VQ_REQUIRE(row_begin >= prevEnd && row_end <= totalRows && row_begin <= row_end, "row ranges must be increasing, disjoint and inside the cubemap");
        prevEnd = row_end;
        int mipRow0 = 0;
        for (int m = 0; m < out.mips; ++m) {
            const int n = out.res >> m, rows = 6 * n;
            const int b = row_begin > mipRow0 ? row_begin : mipRow0;
            const int e = row_end < mipRow0 + rows ? row_end : mipRow0 + rows;
            if (b < e) {
                VQ_REQUIRE(W.nSeg < SPEC_MAX_SEGS, "too many (range, mip) segments for one launch");
                SpecSeg& S = W.seg[W.nSeg++];
                S.n = n; S.rowBegin = b - mipRow0; S.texels = (e - b) * n;
                S.mipOff = (uint32_t)vq_cubemap_offset(out.res, m, 0);
                S.roughness = (float)m / (float)(out.mips - 1);          // EnvironmentMapRendering.cpp:432
                S.unitBegin = units;
                const int per = S.roughness == 0.0f ? SPEC_UNIT_THREAD_TEXELS : SPEC_UNIT_WARP_TEXELS;
                units += (uint32_t)((S.texels + per - 1) / per);
            }
            mipRow0 += rows;
        }
    }
    { const int rcs = vq_fill_peer_sync(ctx, sig, &W.sync); if (rcs) return rcs; }
    if (units == 0 && W.sync.n == 0) return VQ_OK;
    // segments must be visited in increasing unit order with mips that only change forward per CTA: sort is implied by the
    // increasing ranges; roughness 0 segments may sit between others, which only costs a table rebuild
    W.hdri = make_pyr(hd);
    for (int k = 0; k < n_outs; ++k) W.outs[k] = (float4*)outs[k].ptr;
    W.nOuts = n_outs; W.totalUnits = units;
    W.dimX = (float)hd.width; W.dimY = (float)hd.height;     // EnvironmentMapRendering.cpp:433-434
    W.numSamples = num_samples;
    W.ticket = vq_ticket_pair(ctx);
    const size_t smem = (size_t)num_samples * sizeof(float4);
    if (smem > 48 * 1024) VQ_CUDA_OK(cudaFuncSetAttribute(specular_persistent_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    // persistent grid: as many CTAs as fit (8 per SM at 8 KB of table), never more than there are units
    int perSm = 0;
    VQ_CUDA_OK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&perSm, specular_persistent_kernel, IBL_THREADS, smem));
    if (perSm < 1) perSm = 1;
    unsigned blocks = (unsigned)(ctx->sm_count * perSm);
    if (blocks > units) blocks = units > 0 ? units : 1u;
    specular_persistent_kernel<<<blocks, IBL_THREADS, smem, stream>>>(W);
    return vq_check_launch("specular_prefilter");
}

extern "C" int vq_specular_prefilter(VqContext* ctx, VqPyramid hd, VqCubemap out, int num_samples,
                                     int row_begin, int row_end, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("SpecularIrradianceCubemap");
    const int range[2] = {row_begin, row_end};
    if (row_begin == row_end && row_begin >= 0) return VQ_OK;
    return specular_launch(ctx, hd, &out, 1, num_samples, range, 1, nullptr, (cudaStream_t)stream);
}

// K3 fused with the gather of the row blocks (multi-GPU): every prefiltered texel is stored into ALL n_outs cubemaps —
// the local one first, then the other ranks' buffers mapped into this process (NVLink P2P) — while the SMs keep
// integrating (16 bytes of stores per 512-sample texel: the transfer hides completely behind the math).
extern "C" int vq_specular_prefilter_multi(VqContext* ctx, VqPyramid hd, const VqCubemap* outs, int n_outs, int num_samples,
                                           int row_begin, int row_end, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("SpecularIrradianceCubemap");
    const int range[2] = {row_begin, row_end};
    if (row_begin == row_end && row_begin >= 0) return VQ_OK;
    return specular_launch(ctx, hd, outs, n_outs, num_samples, range, 1, nullptr, (cudaStream_t)stream);
}

// Everything one rank prefilters in a step — several row ranges, all destinations, optionally the cross-rank rendezvous —
// as ONE persistent launch.
extern "C" int vq_specular_prefilter_ranges(VqContext* ctx, VqPyramid hd, const VqCubemap* outs, int n_outs, int num_samples,
                                            const int* row_ranges, int n_ranges, const VqPeerSignal* signal, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("SpecularIrradianceCubemap");
    return specular_launch(ctx, hd, outs, n_outs, num_samples, row_ranges, n_ranges, signal, (cudaStream_t)stream);
}

extern "C" int vq_brdf_integration_lut(VqContext* ctx, VqImage out, int num_samples, int row_begin, int row_end, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("CreateBRDFIntegralLUT");
    VQ_REQUIRE(vq_image_ok(out, 8), "bad LUT image descriptor (float2 texels)");
    VQ_REQUIRE(num_samples >= 1 && num_samples <= 8192, "num_samples out of range");
    VQ_REQUIRE(row_begin >= 0 && row_end <= out.height && row_begin <= row_end, "row range out of bounds");
    if (row_begin == row_end) return VQ_OK;
    LutArgs A;
    A.out = (float2*)out.ptr; A.w = out.width; A.h = out.height; A.pitch2 = (int)(out.pitch_bytes / 8);
    A.rowBegin = row_begin; A.numSamples = num_samples;
    const size_t smem = (size_t)num_samples * sizeof(float4);
    if (smem > 48 * 1024) VQ_CUDA_OK(cudaFuncSetAttribute(brdf_lut_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((out.width + 255) / 256, row_end - row_begin);
    brdf_lut_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(A);
    return vq_check_launch("brdf_integration_lut");
}

// K4 on rows [row_begin, row_end) into every destination LUT (one rank's band), with the optional in-kernel rendezvous. Every
// argument is checked before the device is touched.
extern "C" int vq_brdf_integration_lut_multi_signal(VqContext* ctx, const VqImage* outs, int n_outs, int num_samples, int row_begin,
                                                    int row_end, const VqPeerSignal* signal, void* stream) {
    int rc = vq_band_list(outs, n_outs); if (rc) return rc;
    for (int k = 0; k < n_outs; ++k) {
        VQ_REQUIRE(vq_image_ok(outs[k], 8), "bad LUT image descriptor (float2 texels)");
        VQ_REQUIRE(outs[k].width == outs[0].width && outs[k].height == outs[0].height, "every destination must have the size of the first");
        VQ_REQUIRE(k == 0 || outs[k].ptr != outs[0].ptr, "a peer destination must not be the local LUT outs[0]");
    }
    VQ_REQUIRE(num_samples >= 1 && num_samples <= 8192, "num_samples out of range");
    LutMultiArgs M;
    memset(&M, 0, sizeof(M));
    rc = vq_band_check(ctx, n_outs, 0, outs[0].height, row_begin, row_end, signal, M.sync); if (rc) return rc;
    rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("CreateBRDFIntegralLUT");
    if (row_begin == row_end) return VQ_OK;
    M.a.w = outs[0].width; M.a.h = outs[0].height; M.a.rowBegin = row_begin; M.a.numSamples = num_samples;
    for (int k = 0; k < n_outs; ++k) { M.o[k] = (float2*)outs[k].ptr; M.pitch2[k] = (int)(outs[k].pitch_bytes / 8); }
    M.n = n_outs;
    M.ticket = vq_band_ticket(ctx, M.sync);
    const size_t smem = (size_t)num_samples * sizeof(float4);
    if (smem > 48 * 1024) VQ_CUDA_OK(cudaFuncSetAttribute(brdf_lut_multi_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    const dim3 grid((outs[0].width + 255) / 256, row_end - row_begin);
    brdf_lut_multi_kernel<<<grid, 256, smem, (cudaStream_t)stream>>>(M);
    return vq_check_launch("brdf_integration_lut_multi");
}
