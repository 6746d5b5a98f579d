// ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product; never linked into libvqcuda.
//
// oracle_shadow.cpp — SURVEY §8(a) A25 / §8(f).4: the shadow tests of the caster lists and the shadowed PSMain
// (Shaders/Lighting.hlsl:79-272, Shaders/ForwardLighting.hlsl:321-377), restated as scalar C++ over linear R32F shadow
// maps. GROUNDWORK for the (f).4 row: the product path still lights casters with shadow factor 1 (no depth producer
// headless); this file fixes the semantics the CUDA path will have to reproduce once shadow maps are an input.
// PARITY: the reference ships no vectors for it; pinned bit for bit against the reference's own Lighting.hlsl /
// ForwardLighting.hlsl text compiled as C++ (oracle/_ref/libhlslref.so, tests/test_hlsl_ref.py::test_forward_psmain_shadowed_bit_exact).
// Decisions (D3D behaviour that is not in the source), to be kept identical in the kernel:
//   * `PointSampler` is POINT filtering with WRAP addressing (RootSignatures.cpp:148: EDefaultSampler::POINT_WRAP at s1):
//     a 2-D tap reads texel (floor(u*W) mod W, floor(v*H) mod H); the mip is always 0 (shadow maps have one);
//   * a cube tap selects the face as D3D does (largest |component|, ties X > Y > Z: DirectionToCubeFace) and reads
//     texel (min(floor(s*N), N-1), min(floor(t*N), N-1)) of that face;
//   * cbuffer matrices are uploaded as row-major XMMATRIX and declared `matrix` (column-major) in HLSL, so
//     `mul(M, float4(P,1))` (ForwardLighting.hlsl:350,368) is the row vector P times the CPU matrix;
//   * HLSL float literals without suffix (`+0.001`, Lighting.hlsl:160) are fp32.
#include "oracle.h"
#include <cmath>

namespace orc {

namespace {
inline float3 f3(const VqFloat3& v) { return {v.x, v.y, v.z}; }
inline int wrap(int i, int n) { const int r = i % n; return r < 0 ? r + n : r; }
// float -> int as D3D converts (NaN -> 0, saturated): the C++ conversion of NaN is undefined; a NaN coordinate comes from a
// light-space position with x = z = w = 0, whose depth comparisons are all false whichever texel it reads
inline int floor_to_int(float x) {
    const float f = std::floor(x);
    return f != f ? 0 : (f >= 2147483648.0f ? 2147483647 : (f < -2147483648.0f ? (-2147483647 - 1) : (int)f));
}
}  // namespace

// Texture2D(Array).Sample(PointSampler, uv).x on one slice
float SamplePoint2D(const float* map, int w, int h, float u, float v) {
    const int x = wrap(floor_to_int(u * (float)w), w), y = wrap(floor_to_int(v * (float)h), h);
    return map[(size_t)y * w + x];
}
// TextureCubeArray.Sample(PointSampler, float4(dir, index)).x on one cube ([face][y][x])
float SamplePointCube(const float* cube, int res, float3 dir) {
    int face; float sx, sy;
    DirectionToCubeFace(dir, &face, &sx, &sy);                       // ndc coordinates in [-1,1], y up
    const float s = sx * 0.5f + 0.5f, t = -sy * 0.5f + 0.5f;
    const int x = std::min(std::max(floor_to_int(s * (float)res), 0), res - 1);
    const int y = std::min(std::max(floor_to_int(t * (float)res), 0), res - 1);
    return cube[((size_t)face * res + y) * res + x];
}

// Lighting.hlsl:113-165 (NUM_OMNIDIRECTIONAL_PCF_TAPS 20, USE_NORMALIZED_TAP_DIRECTIONS 1)
float OmnidirectionalShadowTestPCF(const ShadowTestPCFData& pcf, const float* cube, int res, float3 lightVectorWorldSpace, float fFarPlane) {
    const float a = 0.5773502691896258f, b = 0.7071067811865475f;
    static const float3 DIRS[20] = {
        {a, a, a}, {a, -a, a}, {-a, -a, a}, {-a, a, a}, {a, a, -a}, {a, -a, -a}, {-a, -a, -a}, {-a, a, -a},
        {b, b, 0}, {b, -b, 0}, {-b, -b, 0}, {-b, b, 0}, {b, 0, b}, {-b, 0, b}, {b, 0, -b}, {-b, 0, -b},
        {0, b, b}, {0, -b, b}, {0, -b, -b}, {0, b, -b}};
    float shadow = 0.0f;
    const float diskRadiusScaleFactor = 1.0f / 8.0f;
    const float diskRadius = (1.0f + (pcf.viewDistanceOfPixel / fFarPlane)) * diskRadiusScaleFactor;
    for (int i = 0; i < 20; ++i) {
        const float3 v = -(lightVectorWorldSpace + DIRS[i] * diskRadius);
        const float closestDepthInLSpace = SamplePointCube(cube, res, v);
        const float closestDepthInWorldSpace = closestDepthInLSpace * fFarPlane;
        shadow += (length(lightVectorWorldSpace) > closestDepthInWorldSpace + pcf.depthBias + 0.001f) ? 1.0f : 0.0f;
    }
    shadow /= 20;
    return 1.0f - shadow;
}

// Lighting.hlsl:168-211: 5x5 PCF on a spot-light shadow map slice; outside the light frustum -> 0 (fully shadowed)
float ShadowTestPCF(const ShadowTestPCFData& pcf, const float* map, int w, int h, float2 shadowMapDimensions) {
    const float3 p = {pcf.lightSpacePos.x / pcf.lightSpacePos.w, pcf.lightSpacePos.y / pcf.lightSpacePos.w, pcf.lightSpacePos.z / pcf.lightSpacePos.w};
    if (p.x < -1.0f || p.x > 1.0f || p.y < -1.0f || p.y > 1.0f || p.z < 0.0f || p.z > 1.0f) return 0.0f;
    const float BIAS = pcf.depthBias * std::tan(std::acos(pcf.NdotL));
    float shadow = 0.0f;
    const float2 texelSize = {1.0f / shadowMapDimensions.x, 1.0f / shadowMapDimensions.y};
    const float2 uv = {0.5f + p.x * 0.5f, 0.5f + p.y * -0.5f};
    for (int x = -2; x <= 2; ++x)
        for (int y = -2; y <= 2; ++y) {
            const float closest = SamplePoint2D(map, w, h, uv.x + (float)x * texelSize.x, uv.y + (float)y * texelSize.y);
            shadow += (p.z - BIAS > closest) ? 1.0f : 0.0f;
        }
    shadow /= 25;
    return 1.0f - shadow;
}

// Lighting.hlsl:215-263: same footprint, constant bias (the LinearDepth values it computes are dead code)
float ShadowTestPCF_Directional(const ShadowTestPCFData& pcf, const float* map, int w, int h, float2 shadowMapDimensions) {
    const float3 p = {pcf.lightSpacePos.x / pcf.lightSpacePos.w, pcf.lightSpacePos.y / pcf.lightSpacePos.w, pcf.lightSpacePos.z / pcf.lightSpacePos.w};
    if (p.x < -1.0f || p.x > 1.0f || p.y < -1.0f || p.y > 1.0f || p.z < 0.0f || p.z > 1.0f) return 0.0f;
    float shadow = 0.0f;
    const float2 texelSize = {1.0f / shadowMapDimensions.x, 1.0f / shadowMapDimensions.y};
    const float2 uv = {0.5f + p.x * 0.5f, 0.5f + p.y * -0.5f};
    for (int x = -2; x <= 2; ++x)
        for (int y = -2; y <= 2; ++y) {
            const float closest = SamplePoint2D(map, w, h, uv.x + (float)x * texelSize.x, uv.y + (float)y * texelSize.y);
            shadow += (p.z - pcf.depthBias > closest) ? 1.0f : 0.0f;
        }
    shadow /= 25;
    return 1.0f - shadow;
}

static float4 mul_row(float3 P, const VqMatrix& M) {               // float4(P,1) * M (row vector, row-major M)
    const float* m = M.m;
    return {P.x * m[0] + P.y * m[4] + P.z * m[8] + m[12], P.x * m[1] + P.y * m[5] + P.z * m[9] + m[13],
            P.x * m[2] + P.y * m[6] + P.z * m[10] + m[14], P.x * m[3] + P.y * m[7] + P.z * m[11] + m[15]};
}

// PSMain with the shadow maps bound (ForwardLighting.hlsl:285-380): identical to ForwardLighting_PSMain except that the
// caster lists and a shadowing directional light are multiplied by their shadow tests.
float4 ForwardLighting_PSMain_Shadowed(const VqPerFrameData& cbPerFrame, const VqPerViewLightingData& cbPerView,
                                       float4 position_ao, float4 normal_roughness, float4 albedo_metalness, const float4* emissive,
                                       const Cubemap& texEnvMapDiff, const Cubemap& texEnvMapSpec, const Image& lut,
                                       const ShadowMaps& sm) {
    // everything that does not involve a caster: evaluate the unshadowed pass on a copy without casters / directional
    VqPerFrameData pf = cbPerFrame;
    pf.Lights.numPointCasters = 0; pf.Lights.numSpotCasters = 0; pf.Lights.directional.enabled = 0;
    const float4 base = ForwardLighting_PSMain(pf, cbPerView, position_ao, normal_roughness, albedo_metalness, emissive,
                                               texEnvMapDiff, texEnvMapSpec, lut);
    float3 I_total = xyz(base);
    BRDF_Surface Surface;
    Surface.N = xyz(normal_roughness); Surface.roughness = normal_roughness.w;
    Surface.diffuseColor = xyz(albedo_metalness); Surface.metalness = albedo_metalness.w;
    Surface.emissiveColor = emissive ? xyz(*emissive) : splat3(0.0f);
    Surface.emissiveIntensity = emissive ? emissive->w : 0.0f;
    const float3 P = xyz(position_ao);
    const float3 cam = f3(cbPerView.CameraPosition);
    const float3 V = normalize(cam - P);
    const VqSceneLighting& L = cbPerFrame.Lights;

    for (int pc = 0; pc < L.numPointCasters; ++pc) {                               // :321-340
        const VqPointLight& l = L.point_casters[pc];
        const float D = length(f3(l.position) - P);
        if (D < l.range) {
            const float3 Ln = normalize(f3(l.position) - P);
            const float3 Lw = f3(l.position) - P;
            ShadowTestPCFData pcf{};
            pcf.depthBias = l.depthBias;
            pcf.NdotL = saturate(dot(Surface.N, Ln));
            pcf.viewDistanceOfPixel = length(P - cam);
            const float s = sm.pointCubes ? OmnidirectionalShadowTestPCF(pcf, sm.pointCubes + (size_t)pc * 6 * sm.pointRes * sm.pointRes,
                                                                         sm.pointRes, Lw, l.range) : 1.0f;
            I_total += CalculatePointLightIllumination(l, Surface, P, V) * s;
        }
    }
    for (int sc = 0; sc < L.numSpotCasters; ++sc) {                                // :343-356
        const VqSpotLight& l = L.spot_casters[sc];
        const float3 Ln = normalize(f3(l.position) - P);
        ShadowTestPCFData pcf{};
        pcf.depthBias = l.depthBias;
        pcf.NdotL = saturate(dot(Surface.N, Ln));
        pcf.lightSpacePos = mul_row(P, L.shadowViews[sc]);
        pcf.viewDistanceOfPixel = length(P - cam);
        const float2 dims = {cbPerFrame.f2SpotLightShadowMapDimensions.x, cbPerFrame.f2SpotLightShadowMapDimensions.y};
        const float s = sm.spotMaps ? ShadowTestPCF(pcf, sm.spotMaps + (size_t)sc * sm.spotW * sm.spotH, sm.spotW, sm.spotH, dims) : 1.0f;
        I_total += CalculateSpotLightIllumination(l, Surface, P, V) * s;
    }
    if (L.directional.enabled) {                                                   // :360-377
        float ShadowingFactor = 1.0f;
        if (L.directional.shadowing && sm.dirMap) {
            const float3 Ln = normalize(-f3(L.directional.lightDirection));
            ShadowTestPCFData pcf{};
            pcf.lightSpacePos = mul_row(P, L.shadowViewDirectional);
            pcf.NdotL = saturate(dot(Surface.N, Ln));
            pcf.depthBias = L.directional.depthBias;
            const float2 dims = {cbPerFrame.f2DirectionalLightShadowMapDimensions.x, cbPerFrame.f2DirectionalLightShadowMapDimensions.y};
            ShadowingFactor = ShadowTestPCF_Directional(pcf, sm.dirMap, sm.dirW, sm.dirH, dims);
        }
        I_total += CalculateDirectionalLightIllumination(L.directional, Surface, V) * ShadowingFactor;
    }
    return make4(I_total, Surface.roughness);
}

// ------------------------------------------------------------------------------------------------
// SURVEY §8(f).4: the hierarchical MIN depth pyramid, DownsampleDepth.hlsl:50-119 = FidelityFX SPD with
// SpdReduce4 = min(min(v0,v1),min(v2,v3)) (:72) over a D3D mip chain. Level 0 is a copy of the depth buffer (:92-103);
// level l is max(1, w>>l) x max(1, h>>l); the shader asks for 1 + floor(log2(max(w,h))) mips (:79-82,:108), i.e. levels up to
// the 1x1 one. SPD works on the 64x64-tile padded domain: source texels outside the image load as 0 (D3D out-of-range Load)
// and stores outside a level are dropped, so level l+1 = 2x2 MIN of the zero-padded level l. With floor-halved sizes no
// padded texel is ever read — except once a dimension has been clamped to 1, where the second row / column of the block
// lies outside and contributes the padded domain's value (0 for the usual depth >= 0: the thin tail of a non-square
// pyramid collapses to 0; kept as is). Pinned against the shader text compiled as C++ (tests/test_hlsl_ref.py).
// `levels` is packed level after level; returns the number of levels written (<= max_levels).
// ------------------------------------------------------------------------------------------------
int DepthMinPyramid(const float* depth, int w, int h, float* levels, int max_levels) {
    int n = 1;
    for (int m = std::max(w, h); m > 1; m >>= 1) ++n;          // 1 + floor(log2(max(w,h)))
    n = std::min(std::min(n, max_levels), 13);                 // SPD: at most 12 mips below level 0
    std::vector<float> cur(depth, depth + (size_t)w * h), next;
    int pw = w, ph = h;                                        // padded-domain size of the current level (ceil-halved)
    float* out = levels;
    for (int l = 0; l < n; ++l) {
        const int lw = std::max(1, w >> l), lh = std::max(1, h >> l);
        for (int y = 0; y < lh; ++y)
            for (int x = 0; x < lw; ++x) out[(size_t)y * lw + x] = (x < pw && y < ph) ? cur[(size_t)y * pw + x] : 0.0f;
        out += (size_t)lw * lh;
        const int nw = (pw + 1) / 2, nh = (ph + 1) / 2;
        next.assign((size_t)nw * nh, 0.0f);
        auto at = [&](int x, int y) { return (x < pw && y < ph) ? cur[(size_t)y * pw + x] : 0.0f; };
        for (int y = 0; y < nh; ++y)
            for (int x = 0; x < nw; ++x)
                next[(size_t)y * nw + x] = std::fmin(std::fmin(at(2 * x, 2 * y), at(2 * x + 1, 2 * y)),
                                                     std::fmin(at(2 * x, 2 * y + 1), at(2 * x + 1, 2 * y + 1)));
        cur.swap(next); pw = nw; ph = nh;
    }
    return n;
}

}  // namespace orc
