// ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product; never linked into libvqcuda.
//
// oracle_surface.cpp — SURVEY.md §8(f).1: the part of PSMain before lighting (ForwardLighting.hlsl:226-283):
// material-texture sampling, sRGB->linear, normal mapping, Has*Map selection, and the RGBA8 mip chain the
// engine builds on the CPU for those textures (DXGIUtils.cpp:250-287).
//
// Decisions (D3D sampler hardware is not in the source; identical in the CUDA kernel, DESIGN.md §3.6):
//   * RGBA8 UNORM texel -> float = byte / 255.0f
//   * Sample()/SampleBias(): implicit derivatives = FINE finite differences inside the pixel's aligned 2x2 quad,
//     ddx = uv(qx+1,y) - uv(qx,y), ddy = uv(x,qy+1) - uv(x,qy) (partner clamped to the image), computed on the RAW uv and
//     scaled by the pixel's own uvScale (helper lanes of a rasteriser run the same material);
//     lod = 0.5*log2(max(|ddx*(W,H)|^2, |ddy*(W,H)|^2)) + bias, clamped to [0, levels-1] (D3D11.3 functional spec 7.18.11,
//     isotropic: the engine's ANISOTROPIC sampler has MaxAnisotropy = 0, RootSignatures.cpp:106-111); trilinear, WRAP
//     (RootSignatures.cpp:147-149), texel-space coordinate u*W - 0.5 with fp32 weights, as for the equirect sampler.
//   * null SRV (missing map, Renderer_Resources.cpp:383-387) reads 0.
//   * texScreenSpaceAO is point-sampled at (SV_Position.xy + 0.5)/ScreenDimensions (ForwardLighting.hlsl:280-281):
//     SV_Position already carries the half-pixel offset, so the fetch lands on texel (x+1, y+1), WRAP (POINT_WRAP,
//     RootSignatures.cpp:148). Restated as is.
#include "oracle.h"
#include <cmath>
#include <algorithm>

namespace orc {

static inline float3 f3(const VqFloat3& v) { return {v.x, v.y, v.z}; }

// ---- VQ_DXGI_UTILS::MipImage, bytesPerPixel == 4 (DXGIUtils.cpp:263-287) -----------------------------------------
// per channel (c00 + c10 + c01 + c11) / 4, integer (truncating). Only complete 2x2 blocks are visited (the reference's
// loops read one texel past odd edges; same decision as the float MIN variant, oracle_ibl.cpp).
void MipImage_Box8(const uint8_t* src, uint8_t* dst, int width, int height) {
    const int dw = width >> 1, dh = height >> 1;
    for (int y = 0; y < dh; ++y)
        for (int x = 0; x < dw; ++x)
            for (int c = 0; c < 4; ++c) {
                unsigned cc = 0;
                cc += src[4 * ((size_t)(2 * y) * width + 2 * x) + c];
                cc += src[4 * ((size_t)(2 * y) * width + 2 * x + 1) + c];
                cc += src[4 * ((size_t)(2 * y + 1) * width + 2 * x) + c];
                cc += src[4 * ((size_t)(2 * y + 1) * width + 2 * x + 1) + c];
                dst[4 * ((size_t)y * dw + x) + c] = (uint8_t)(cc / 4);
            }
}

size_t Texture8::offset(int level) const { return pyramid_texel_count(width, height, level); }

static inline int wrapi(int i, int n) { int r = i % n; return r < 0 ? r + n : r; }
// the device's float -> int conversion (cvt.rzi: NaN -> 0, saturated); the C++ conversion is undefined outside the int range
static inline int to_int_sat(float x) {
    return x != x ? 0 : (x >= 2147483648.0f ? 2147483647 : (x < -2147483648.0f ? (-2147483647 - 1) : (int)x));
}
static inline float4 ld8(const uint8_t* p) {
    return {(float)p[0] / 255.0f, (float)p[1] / 255.0f, (float)p[2] / 255.0f, (float)p[3] / 255.0f};
}

static float4 BilinearWrap8(const Texture8& tex, int level, float2 uv) {
    const int W = tex.w(level), H = tex.h(level);
    const uint8_t* base = tex.data + 4 * tex.offset(level);
    const float x = uv.x * (float)W - 0.5f;
    const float y = uv.y * (float)H - 0.5f;
    const float x0 = std::floor(x), y0 = std::floor(y);
    const float fx = x - x0, fy = y - y0;
    // beyond the int range the floored coordinate saturates, as on the device; a coordinate that is not finite makes fx or fy
    // NaN and the blend NaN (vqcuda.h, VqSurfaceInputs)
    const int ix0 = wrapi(to_int_sat(x0), W), iy0 = wrapi(to_int_sat(y0), H);
    const int ix1 = wrapi(ix0 + 1, W), iy1 = wrapi(iy0 + 1, H);
    const float4 t00 = ld8(base + 4 * ((size_t)iy0 * W + ix0));
    const float4 t10 = ld8(base + 4 * ((size_t)iy0 * W + ix1));
    const float4 t01 = ld8(base + 4 * ((size_t)iy1 * W + ix0));
    const float4 t11 = ld8(base + 4 * ((size_t)iy1 * W + ix1));
    const float4 top = lerp(t00, t10, fx);
    const float4 bot = lerp(t01, t11, fx);
    return lerp(top, bot, fy);
}

float TextureLod(const Texture8& tex, float2 ddx, float2 ddy, float bias) {
    const float W = (float)tex.width, H = (float)tex.height;
    const float ax = ddx.x * W, ay = ddx.y * H, bx = ddy.x * W, by = ddy.y * H;
    const float lx = ax * ax + ay * ay, ly = bx * bx + by * by;
    const float m = std::fmax(lx, ly);
    float lod = (m > 0.0f ? 0.5f * std::log2(m) : -126.0f) + bias;
    const float maxLod = (float)(tex.levels - 1);
    return std::fmin(std::fmax(lod, 0.0f), maxLod);
}

// Texture2D.Sample / SampleBias with the derivatives handed in
float4 SampleTexture8(const Texture8& tex, float2 uv, float2 ddx, float2 ddy, float bias) {
    if (!tex.data) return make4(0, 0, 0, 0);
    const float lod = TextureLod(tex, ddx, ddy, bias);
    const float l0f = std::floor(lod);
    const int l0 = (int)l0f;
    const float f = lod - l0f;
    const float4 c0 = BilinearWrap8(tex, l0, uv);
    if (f == 0.0f || l0 + 1 >= tex.levels) return c0;
    const float4 c1 = BilinearWrap8(tex, l0 + 1, uv);
    return lerp(c0, c1, f);
}

// ShadingMath.hlsl:44-52
float3 UnpackNormal(float3 SampledNormal, float3 worldNormal, float3 worldTangent) {
    SampledNormal = normalize(SampledNormal * 2.0f - splat3(1.0f));
    const float3 T = normalize(worldTangent - worldNormal * dot(worldNormal, worldTangent));
    const float3 N = normalize(worldNormal);
    const float3 B = normalize(cross(T, N));
    // mul(SampledNormal, float3x3(T, B, N)): row vector x matrix whose ROWS are T, B, N
    return T * SampledNormal.x + B * SampledNormal.y + N * SampledNormal.z;
}

static inline int HasBit(int cfg, int bit) { return (cfg & (1 << bit)) > 0 ? 1 : 0; }   // LightingConstantBufferData.h:116-124

// ForwardLighting.hlsl:226-283. Returns false when the ENABLE_ALPHA_MASK variant discards the pixel (237-240).
bool Surface_PSMain(const SurfaceIn& In, float2 uv_ddx_raw, float2 uv_ddy_raw, const VqMaterialData& mat,
                    const MaterialTextures8& tex, float fAmbientLightingFactor, float ssao, bool alphaMask,
                    SurfaceOut* o) {
    const float2 scale = make2(mat.uvScaleOffset.x, mat.uvScaleOffset.y);
    const float2 uv = make2(In.uv.x * scale.x + mat.uvScaleOffset.z, In.uv.y * scale.y + mat.uvScaleOffset.w);   // :226
    const float2 ddx = make2(uv_ddx_raw.x * scale.x, uv_ddx_raw.y * scale.y);
    const float2 ddy = make2(uv_ddy_raw.x * scale.x, uv_ddy_raw.y * scale.y);
    const int TEX_CFG = (int)mat.textureConfig;                                                                   // :227

    float4 AlbedoAlpha = SampleTexture8(tex.diffuse, uv, ddx, ddy, 0.0f);                                         // :229
    const float3 Normal = xyz(SampleTexture8(tex.normals, uv, ddx, ddy, mat.normalMapMipBias));                   // :230
    float3 Emissive = xyz(SampleTexture8(tex.emissive, uv, ddx, ddy, 0.0f));                                      // :231
    const float Metalness = SampleTexture8(tex.metalness, uv, ddx, ddy, 0.0f).x;                                  // :232
    const float Roughness = SampleTexture8(tex.roughness, uv, ddx, ddy, 0.0f).x;                                  // :233
    const float3 OcclRghMtl = xyz(SampleTexture8(tex.occl_rough_metal, uv, ddx, ddy, 0.0f));                      // :234
    const float LocalAO = SampleTexture8(tex.local_ao, uv, ddx, ddy, 0.0f).x;                                     // :235

    if (alphaMask && HasBit(TEX_CFG, 0) && AlbedoAlpha.w < 0.01f) return false;                                   // :237-240

    const float3 albedoLin = SRGBToLinear_pow22(xyz(AlbedoAlpha));                                                // :243
    Emissive = SRGBToLinear_pow22(Emissive);                                                                      // :244

    float ao = fAmbientLightingFactor;                                                                            // :247
    const float3 matDiffuse = f3(mat.diffuse), matEmissive = f3(mat.emissiveColor);
    o->diffuseColor = HasBit(TEX_CFG, 0) ? albedoLin * matDiffuse : matDiffuse;                                   // :249
    o->emissiveColor = HasBit(TEX_CFG, 7) ? Emissive * matEmissive : matEmissive;                                 // :250
    o->emissiveIntensity = mat.emissiveIntensity;                                                                 // :251
    o->roughness = mat.roughness;                                                                                 // :252
    o->metalness = mat.metalness;                                                                                 // :253

    const float3 N = normalize(In.WorldSpaceNormal);                                                              // :265
    const float3 T = normalize(In.WorldSpaceTangent);                                                             // :266
    o->N = length(Normal) < 0.01f ? N : UnpackNormal(Normal, N, T);                                               // :267

    if (HasBit(TEX_CFG, 2) > 0) ao *= LocalAO;                                                                    // :269
    if (HasBit(TEX_CFG, 4) > 0) o->roughness *= Roughness;                                                        // :270
    if (HasBit(TEX_CFG, 5) > 0) o->metalness *= Metalness;                                                        // :271
    if (HasBit(TEX_CFG, 8) > 0) {                                                                                 // :272-277
        o->roughness *= OcclRghMtl.y;
        o->metalness *= OcclRghMtl.z;
    }
    ao *= ssao;                                                                                                   // :280-281
    o->ao = ao;
    o->P = In.WorldSpacePosition;                                                                                 // :284
    return true;
}

}  // namespace orc
