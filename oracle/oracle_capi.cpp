// ORACLE — TEST INFRASTRUCTURE ONLY. Not part of the product; never linked into libvqcuda.
//
// oracle_capi.cpp — extern "C" drivers over the scalar oracle so that tests/ (ctypes) and
// bench.py's cpu_baseline / `--impl reference` leg can run whole passes on host buffers.
// All images are tightly pitched float4 (float2 for the BRDF LUT). `threads` = std::thread count
// (row partition); the per-texel arithmetic is single-threaded scalar code.
#include "oracle.h"

using namespace orc;

namespace {
template <class F>
void par_rows(int n, int threads, F&& f) {
    struct Ctx { F* f; } ctx{&f};
    ParallelRows(n, threads, [](int r, void* u) { (*static_cast<Ctx*>(u)->f)(r); }, &ctx);
}
inline float4 ld(const float* p) { return {p[0], p[1], p[2], p[3]}; }
inline void st(float* p, float4 v) { p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w; }
inline Image img4(const float* d, int w, int h) { return {d, w, h, (size_t)w * 4, 4}; }

// flattened (mip, face, row) -> components
inline void decode_cube_row(int res, int mips, int r, int* mip, int* face, int* row) {
    for (int m = 0; m < mips; ++m) {
        const int n = res >> m;
        if (r < 6 * n) { *mip = m; *face = r / n; *row = r % n; return; }
        r -= 6 * n;
    }
    *mip = -1; *face = 0; *row = 0;
}
}  // namespace

extern "C" {

int orc_mip_level_count(uint64_t w, uint64_t h) { return mip_level_count(w, h); }
uint64_t orc_cubemap_texel_count(int res, int mips) { return cubemap_texel_count(res, mips); }
int orc_cubemap_row_count(int res, int mips) { return cubemap_row_count(res, mips); }
uint64_t orc_pyramid_texel_count(int w, int h, int levels) { return pyramid_texel_count(w, h, levels); }

// ---- K1 ---------------------------------------------------------------------------------------
void orc_forward_lighting(const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                          const float* position_ao, const float* normal_roughness, const float* albedo_metalness,
                          const float* emissive, int width, int height,
                          const float* diff_cube, int diff_res,
                          const float* spec_cube, int spec_res, int spec_mips,
                          const float* lut, int lut_w, int lut_h,
                          float* out, int row_begin, int row_end, int threads) {
    const Cubemap cd{diff_cube, diff_res, 1};
    const Cubemap cs{spec_cube, spec_res, spec_mips};
    const Image lutImg{lut, lut_w, lut_h, (size_t)lut_w * 2, 2};
    (void)height;
    par_rows(row_end - row_begin, threads, [&](int r) {
        const int y = row_begin + r;
        for (int x = 0; x < width; ++x) {
            const size_t o = ((size_t)y * width + x) * 4;
            float4 em;
            if (emissive) em = ld(emissive + o);
            st(out + o, ForwardLighting_PSMain(*pf, *pv, ld(position_ao + o), ld(normal_roughness + o),
                                               ld(albedo_metalness + o), emissive ? &em : nullptr, cd, cs, lutImg));
        }
    });
}

// ---- §8(f).1 surface producer -----------------------------------------------------------------
void orc_texture_build_mips(uint8_t* tex, int w, int h, int levels) {
    const Texture8 t{tex, w, h, levels};
    for (int l = 1; l < levels; ++l)
        MipImage_Box8(tex + 4 * t.offset(l - 1), tex + 4 * t.offset(l), w >> (l - 1), h >> (l - 1));
}

void orc_sample_texture8(const uint8_t* tex, int w, int h, int levels, float u, float v,
                         float dudx, float dvdx, float dudy, float dvdy, float bias, float* out4, float* out_lod) {
    const Texture8 t{tex, w, h, levels};
    st(out4, SampleTexture8(t, make2(u, v), make2(dudx, dvdx), make2(dudy, dvdy), bias));
    if (out_lod) *out_lod = tex ? TextureLod(t, make2(dudx, dvdx), make2(dudy, dvdy), bias) : 0.0f;
}
void orc_unpack_normal(const float* sampled, const float* n, const float* t, float* out3) {
    const float3 r = UnpackNormal(make3(sampled[0], sampled[1], sampled[2]), make3(n[0], n[1], n[2]), make3(t[0], t[1], t[2]));
    out3[0] = r.x; out3[1] = r.y; out3[2] = r.z;
}

// host-side mirror of VqTexture2D / VqMaterialTextures with HOST pointers
struct OrcTexture2D { const uint8_t* ptr; int32_t width, height, levels; };
struct OrcMaterialTextures { OrcTexture2D t[7]; };

void orc_gbuffer_from_materials(const float* position_u, const float* normal_v, const float* tangent_m, const float* ssao,
                                int width, int height, const VqMaterialData* materials, const OrcMaterialTextures* textures,
                                int n_materials, float ambient_factor, int alpha_mask,
                                float* position_ao, float* normal_roughness, float* albedo_metalness, float* emissive,
                                int row_begin, int row_end, int threads) {
    auto tex8 = [](const OrcTexture2D& t) { return Texture8{t.ptr, t.width, t.height, t.levels}; };
    auto rawuv = [&](int x, int y) {
        const size_t o = ((size_t)y * width + x) * 4;
        return make2(position_u[o + 3], normal_v[o + 3]);
    };
    par_rows(row_end - row_begin, threads, [&](int r) {
        const int y = row_begin + r;
        for (int x = 0; x < width; ++x) {
            const size_t o = ((size_t)y * width + x) * 4;
            SurfaceIn in;
            in.WorldSpacePosition = make3(position_u[o], position_u[o + 1], position_u[o + 2]);
            in.WorldSpaceNormal = make3(normal_v[o], normal_v[o + 1], normal_v[o + 2]);
            in.WorldSpaceTangent = make3(tangent_m[o], tangent_m[o + 1], tangent_m[o + 2]);
            in.uv = rawuv(x, y);
            // the device's conversion (cvt.rzi: NaN -> 0, saturated), then clamped; the C++ conversion is undefined there
            const float mf = tangent_m[o + 3];
            int mi = mf != mf ? 0 : (mf >= 2147483648.0f ? 2147483647 : (mf < -2147483648.0f ? (-2147483647 - 1) : (int)mf));
            mi = mi < 0 ? 0 : (mi >= n_materials ? n_materials - 1 : mi);
            // fine derivatives inside the aligned 2x2 quad, partner clamped to the image
            const int qx = x & ~1, qy = y & ~1;
            const int qx1 = qx + 1 < width ? qx + 1 : qx, qy1 = qy + 1 < height ? qy + 1 : qy;
            const float2 a = rawuv(qx, y), b = rawuv(qx1, y), c = rawuv(x, qy), d = rawuv(x, qy1);
            const float2 ddx = make2(b.x - a.x, b.y - a.y), ddy = make2(d.x - c.x, d.y - c.y);
            const OrcMaterialTextures& mt = textures[mi];
            const MaterialTextures8 t8{tex8(mt.t[0]), tex8(mt.t[1]), tex8(mt.t[2]), tex8(mt.t[3]), tex8(mt.t[4]),
                                       tex8(mt.t[5]), tex8(mt.t[6])};
            float ao_ss = 1.0f;
            if (ssao) ao_ss = ssao[(size_t)((y + 1) % height) * width + (x + 1) % width];
            SurfaceOut so;
            if (!Surface_PSMain(in, ddx, ddy, materials[mi], t8, ambient_factor, ao_ss, alpha_mask != 0, &so)) continue;
            st(position_ao + o, make4(so.P, so.ao));
            st(normal_roughness + o, make4(so.N, so.roughness));
            st(albedo_metalness + o, make4(so.diffuseColor, so.metalness));
            if (emissive) st(emissive + o, make4(so.emissiveColor, so.emissiveIntensity));
        }
    });
}

// ---- K11 --------------------------------------------------------------------------------------
void orc_hdri_build_mips(float* pyramid, int w, int h, int levels) {
    Pyramid p{pyramid, w, h, levels};
    for (int l = 1; l < levels; ++l)
        MipImage_MinFilter(pyramid + 4 * p.offset(l - 1), pyramid + 4 * p.offset(l), w >> (l - 1), h >> (l - 1));
}

// ---- K2 ---------------------------------------------------------------------------------------
int orc_diffuse_angle_counts(float step, int n_phi, int n_theta, int* out_phi, int* out_theta) {
    std::vector<float> ph, th;
    DiffuseIrradianceAngles(step, n_phi, n_theta, ph, th);
    *out_phi = (int)ph.size(); *out_theta = (int)th.size();
    return (int)(ph.size() * th.size());
}
void orc_diffuse_irradiance(const float* pyramid, int w, int h, int levels,
                            float step, int n_phi, int n_theta, int src_mip,
                            float* out_cube, int res, int row_begin, int row_end, int threads, int f64_accum) {
    const Pyramid p{pyramid, w, h, levels};
    std::vector<float> phis, thetas;
    DiffuseIrradianceAngles(step, n_phi, n_theta, phis, thetas);
    par_rows(row_end - row_begin, threads, [&](int r) {
        const int fr = row_begin + r, face = fr / res, py = fr % res;
        for (int px = 0; px < res; ++px) {
            const float3 dir = CubeTexelDirection(face, px, py, res);
            st(out_cube + 4 * ((size_t)face * res * res + (size_t)py * res + px),
               DiffuseIrradiance_PSMain(p, dir, phis, thetas, src_mip, f64_accum != 0));
        }
    });
}

// ---- K3 ---------------------------------------------------------------------------------------
void orc_specular_prefilter(const float* pyramid, int w, int h, int levels,
                            float* out_cube, int res, int mips, int num_samples,
                            int row_begin, int row_end, int threads) {
    const Pyramid p{pyramid, w, h, levels};
    const Cubemap cm{out_cube, res, mips};
    par_rows(row_end - row_begin, threads, [&](int r) {
        int mip, face, py;
        decode_cube_row(res, mips, row_begin + r, &mip, &face, &py);
        if (mip < 0) return;
        const int n = res >> mip;
        // EnvironmentMapRendering.cpp:432: Roughness = mip / (NUM_MIPS - 1)
        const float roughness = (float)mip / (float)(mips - 1);
        for (int px = 0; px < n; ++px) {
            const float3 dir = CubeTexelDirection(face, px, py, n);
            st(out_cube + 4 * (cm.offset(mip, face) + (size_t)py * n + px),
               SpecularIrradiance_PSMain(p, dir, roughness, make2((float)w, (float)h), (uint32_t)num_samples));
        }
    });
}

// K3 on an arbitrary texel list (flattened mip-major / face-minor / row-major indices of the packed cube): the same
// per-texel call as orc_specular_prefilter (CubemapConvolution.hlsl:168-223, EnvironmentMapRendering.cpp:413-465), used
// by the full-size parity test that samples 1 % of BASELINE config 5's texels at random. out = n x float4.
void orc_specular_prefilter_texels(const float* pyramid, int w, int h, int levels, int res, int mips, int num_samples,
                                   const int64_t* texels, int n, float* out, int threads) {
    const Pyramid p{pyramid, w, h, levels};
    par_rows(n, threads, [&](int k) {
        int64_t t = texels[k]; int mip = 0;
        for (; mip < mips; ++mip) { const int64_t sz = 6ll * (res >> mip) * (res >> mip); if (t < sz) break; t -= sz; }
        if (mip >= mips) { st(out + 4 * (size_t)k, float4{0, 0, 0, 0}); return; }
        const int nn = res >> mip, face = (int)(t / ((int64_t)nn * nn)), py = (int)((t % ((int64_t)nn * nn)) / nn), px = (int)(t % nn);
        const float roughness = (float)mip / (float)(mips - 1);
        st(out + 4 * (size_t)k, SpecularIrradiance_PSMain(p, CubeTexelDirection(face, px, py, nn), roughness,
                                                          make2((float)w, (float)h), (uint32_t)num_samples));
    });
}

// Conditioning probe for K3 (test infrastructure): how much does the ORACLE's own result move when the texel's (unit) look
// direction is tilted by a few ulps (+- eps ADDED to each component: an absolute tilt of eps radians, also at the poles where a
// relative change of the small components would vanish), or when the length of its un-normalised sample vectors is off by
// 1-4 ulps (the asin(-L.y) of the equirect map is singular at the poles)? out[k] = max over all probes and colour channels
// of |result' - result|. Near the poles of the equirect map (u = atan2(z,x) is singular there) a 1e-7 change of a sample
// direction moves the sample by whole texels, so two correct fp32 implementations cannot agree to 1e-4 on an HDRI that
// carries per-texel detail in its pole rows; the full-size parity test widens its bound by this measured sensitivity.
void orc_specular_prefilter_sensitivity(const float* pyramid, int w, int h, int levels, int res, int mips, int num_samples,
                                        const int64_t* texels, int n, float rel_eps, float* out, int threads) {
    const Pyramid p{pyramid, w, h, levels};
    par_rows(n, threads, [&](int k) {
        int64_t t = texels[k]; int mip = 0;
        for (; mip < mips; ++mip) { const int64_t sz = 6ll * (res >> mip) * (res >> mip); if (t < sz) break; t -= sz; }
        if (mip >= mips) { out[k] = 0.0f; return; }
        const int nn = res >> mip, face = (int)(t / ((int64_t)nn * nn)), py = (int)((t % ((int64_t)nn * nn)) / nn), px = (int)(t % nn);
        const float roughness = (float)mip / (float)(mips - 1);
        const float3 d = normalize(CubeTexelDirection(face, px, py, nn));
        const float2 dim = make2((float)w, (float)h);
        const float4 base = SpecularIrradiance_PSMain(p, d, roughness, dim, (uint32_t)num_samples);
        float s = 0.0f;
        auto upd = [&](const float4& r) {
            s = std::fmax(s, std::fmax(std::fabs(r.x - base.x), std::fmax(std::fabs(r.y - base.y), std::fabs(r.z - base.z))));
        };
        for (int c = 0; c < 3; ++c)
            for (int sgn = -1; sgn <= 1; sgn += 2) {
                float3 e = d;
                const float f = (float)sgn * rel_eps;
                if (c == 0) e.x += f; else if (c == 1) e.y += f; else e.z += f;
                upd(SpecularIrradiance_PSMain(p, e, roughness, dim, (uint32_t)num_samples));
            }
        // the length of the un-normalised sample vectors, +-1, 2 and 4 ulps (see SpecularIrradiance_PSMain)
        for (int k2 = 1; k2 <= 4; k2 *= 2)
            for (int sgn = -1; sgn <= 1; sgn += 2)
                upd(SpecularIrradiance_PSMain(p, d, roughness, dim, (uint32_t)num_samples, 1.0f + (float)(sgn * k2) * 5.9604645e-8f));
        out[k] = s;
    });
}

// ---- K4 ---------------------------------------------------------------------------------------
void orc_brdf_integration_lut(float* out_rg, int w, int h, int samples, int row_begin, int row_end, int threads) {
    par_rows(row_end - row_begin, threads, [&](int r) {
        const int y = row_begin + r;
        for (int x = 0; x < w; ++x) {
            // CubemapConvolution.hlsl:234-239
            const float u = ((float)x + 0.5f) / (float)w, v = ((float)y + 0.5f) / (float)h;
            const float2 sb = IntegrateBRDF(u, v, samples);
            out_rg[((size_t)y * w + x) * 2 + 0] = sb.x;
            out_rg[((size_t)y * w + x) * 2 + 1] = sb.y;
        }
    });
}

// ---- K5 / K6 ----------------------------------------------------------------------------------
void orc_gaussian_blur(const float* in, float* out, int w, int h, int vertical, int threads) {
    const Image I = img4(in, w, h);
    par_rows(h, threads, [&](int y) {
        for (int x = 0; x < w; ++x) st(out + ((size_t)y * w + x) * 4, GaussianBlur_CSMain(I, x, y, vertical != 0, w, h));
    });
}
void orc_tonemap(const VqTonemapperParams* p, const float* in, float* out, int w, int h, int threads) {
    par_rows(h, threads, [&](int y) {
        for (int x = 0; x < w; ++x) {
            const size_t o = ((size_t)y * w + x) * 4;
            st(out + o, Tonemapper_CSMain(*p, ld(in + o)));
        }
    });
}

// ---- K7 / K8 / K9 -----------------------------------------------------------------------------
void orc_cas(const uint32_t c[8], const float* in, float* out, int w, int h, int threads) {
    const Image I = img4(in, w, h);
    par_rows(h, threads, [&](int y) {
        for (int x = 0; x < w; ++x) st(out + ((size_t)y * w + x) * 4, make4(CasFilter_NoScaling(I, x, y, c + 4), 1.0f));
    });
}
void orc_fsr_easu(const uint32_t c[16], int address_mode, const float* in, int in_w, int in_h,
                  float* out, int out_w, int out_h, int threads) {
    const Image I = img4(in, in_w, in_h);
    par_rows(out_h, threads, [&](int y) {
        for (int x = 0; x < out_w; ++x) st(out + ((size_t)y * out_w + x) * 4, make4(FsrEasuF(I, x, y, c, address_mode), 1.0f));
    });
}
void orc_fsr_rcas(const uint32_t c[4], const float* in, float* out, int w, int h, int threads) {
    const Image I = img4(in, w, h);
    par_rows(h, threads, [&](int y) {
        for (int x = 0; x < w; ++x) st(out + ((size_t)y * w + x) * 4, make4(FsrRcasF(I, x, y, c), 1.0f));
    });
}

// ---- K10: dst levels 1..mips packed back to back, level i is (w>>i) x (h>>i) --------------------
void orc_spd_downsample(const float* src, int w, int h, int mips, float* out_packed) {
    Image cur = img4(src, w, h);
    float* o = out_packed;
    for (int l = 1; l <= mips; ++l) {
        const int lw = w >> l, lh = h >> l;
        if (lw < 1 || lh < 1) break;
        MutImage d{o, lw, lh, (size_t)lw * 4, 4};
        SpdDownsampleLevel(cur, d, l);
        cur = d.view();
        o += (size_t)lw * lh * 4;
    }
}

// ---- setup functions --------------------------------------------------------------------------
void orc_cas_setup(uint32_t con[8], float sharpness, float in_w, float in_h, float out_w, float out_h) {
    CasSetup(con, con + 4, sharpness, in_w, in_h, out_w, out_h);
}
void orc_fsr_easu_con(uint32_t con[16], float vp_w, float vp_h, float in_w, float in_h, float out_w, float out_h) {
    FsrEasuCon(con, con + 4, con + 8, con + 12, vp_w, vp_h, in_w, in_h, out_w, out_h);
}
void orc_fsr_rcas_con(uint32_t con[4], float stops) { FsrRcasCon(con, stops); }
void orc_spd_setup(uint32_t dispatch_xy[2], uint32_t wg_offset[2], uint32_t nwg_mips[2], const uint32_t rect[4], int mips) {
    SpdSetup(dispatch_xy, wg_offset, nwg_mips, rect, mips);
}

// ---- scalar probes for known-answer tests -------------------------------------------------------
void orc_brdf(const float N[3], const float V[3], const float Wi[3], const float albedo[3],
              float roughness, float metalness, float out[3]) {
    BRDF_Surface s{};
    s.N = make3(N[0], N[1], N[2]); s.roughness = roughness; s.metalness = metalness;
    s.diffuseColor = make3(albedo[0], albedo[1], albedo[2]);
    const float3 r = BRDF(s, make3(Wi[0], Wi[1], Wi[2]), make3(V[0], V[1], V[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
float orc_ndf_ggx(float NdotH, float roughness) { return NormalDistributionGGX(NdotH, roughness); }
float orc_geometry_smith(const float N[3], const float V[3], const float L[3], float roughness) {
    return Geometry_Smith(make3(N[0], N[1], N[2]), make3(V[0], V[1], V[2]), make3(L[0], L[1], L[2]), roughness);
}
void orc_fresnel_schlick(const float H[3], const float V[3], const float F0[3], float out[3]) {
    const float3 r = Fresnel_Schlick(make3(H[0], H[1], H[2]), make3(V[0], V[1], V[2]), make3(F0[0], F0[1], F0[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
void orc_fresnel_gaussian(const float H[3], const float V[3], const float F0[3], float out[3]) {
    const float3 r = Fresnel_Gaussian(make3(H[0], H[1], H[2]), make3(V[0], V[1], V[2]), make3(F0[0], F0[1], F0[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
void orc_point_light(const VqPointLight* l, const float P[3], const float N[3], const float V[3],
                     const float albedo[3], float roughness, float metalness, float out[3]) {
    BRDF_Surface s{};
    s.N = make3(N[0], N[1], N[2]); s.roughness = roughness; s.metalness = metalness;
    s.diffuseColor = make3(albedo[0], albedo[1], albedo[2]);
    const float3 r = CalculatePointLightIllumination(*l, s, make3(P[0], P[1], P[2]), make3(V[0], V[1], V[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
void orc_spot_light(const VqSpotLight* l, const float P[3], const float N[3], const float V[3],
                    const float albedo[3], float roughness, float metalness, float out[3]) {
    BRDF_Surface s{};
    s.N = make3(N[0], N[1], N[2]); s.roughness = roughness; s.metalness = metalness;
    s.diffuseColor = make3(albedo[0], albedo[1], albedo[2]);
    const float3 r = CalculateSpotLightIllumination(*l, s, make3(P[0], P[1], P[2]), make3(V[0], V[1], V[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
void orc_directional_light(const VqDirectionalLight* l, const float N[3], const float V[3],
                           const float albedo[3], float roughness, float metalness, float out[3]) {
    BRDF_Surface s{};
    s.N = make3(N[0], N[1], N[2]); s.roughness = roughness; s.metalness = metalness;
    s.diffuseColor = make3(albedo[0], albedo[1], albedo[2]);
    const float3 r = CalculateDirectionalLightIllumination(*l, s, make3(V[0], V[1], V[2]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
float orc_spotlight_intensity(const VqSpotLight* l, const float P[3]) { return SpotlightIntensity(*l, make3(P[0], P[1], P[2])); }
void orc_hammersley(uint32_t i, uint32_t n, float out[2]) { const float2 h = Hammersley(i, n); out[0] = h.x; out[1] = h.y; }
void orc_importance_sample_ggx(const float Xi[2], const float N[3], float roughness, float out[3]) {
    const float3 h = ImportanceSampleGGX(make2(Xi[0], Xi[1]), make3(N[0], N[1], N[2]), roughness);
    out[0] = h.x; out[1] = h.y; out[2] = h.z;
}
void orc_integrate_brdf(float NdotV, float roughness, int samples, float out[2]) {
    const float2 r = IntegrateBRDF(NdotV, roughness, samples); out[0] = r.x; out[1] = r.y;
}
void orc_direction_to_equirect_uv(const float d[3], float out[2]) {
    const float2 uv = DirectionToEquirectUV(make3(d[0], d[1], d[2])); out[0] = uv.x; out[1] = uv.y;
}
void orc_cube_texel_direction(int face, int px, int py, int res, float out[3]) {
    const float3 d = CubeTexelDirection(face, px, py, res); out[0] = d.x; out[1] = d.y; out[2] = d.z;
}
void orc_direction_to_cube_face(const float d[3], int* face, float* sx, float* sy) {
    DirectionToCubeFace(make3(d[0], d[1], d[2]), face, sx, sy);
}
void orc_cube_resolve_edge_tap(int N, int face, int i, int j, int out[3]) {
    CubeResolveEdgeTap(N, face, i, j, &out[0], &out[1], &out[2]);
}
void orc_sample_cube(const float* cube, int res, int mips, const float d[3], int mip, float out[4]) {
    const float4 r = SampleCubeLevel(Cubemap{cube, res, mips}, make3(d[0], d[1], d[2]), mip);
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}
// the same over n directions (dirs: n x 3, out: n x 4), one mip each (mips: n ints)
void orc_sample_cube_n(const float* cube, int res, int mips, const float* dirs, const int* mip, int64_t n, float* out) {
    for (int64_t k = 0; k < n; ++k) orc_sample_cube(cube, res, mips, dirs + 3 * k, mip[k], out + 4 * k);
}
void orc_sample_equirect(const float* pyr, int w, int h, int levels, float u, float v, float lod, float out[4]) {
    const float4 r = SampleEquirectLevel(Pyramid{pyr, w, h, levels}, make2(u, v), lod);
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}
void orc_tonemap_pixel(const VqTonemapperParams* p, const float in[4], float out[4]) {
    const float4 r = Tonemapper_CSMain(*p, make4(in[0], in[1], in[2], in[3]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z; out[3] = r.w;
}
float orc_aprx(int which, float a) {
    switch (which) { case 0: return APrxLoSqrtF1(a); case 1: return APrxLoRcpF1(a); case 2: return APrxMedRcpF1(a); default: return APrxLoRsqF1(a); }
}


// ---- A25 / §8(f).4 groundwork: PSMain with shadow maps bound (any map pointer may be null) --------------------------------
void orc_forward_lighting_shadowed(const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                   const float* position_ao, const float* normal_roughness, const float* albedo_metalness,
                                   int width, int height, const float* diff_cube, int diff_res,
                                   const float* spec_cube, int spec_res, int spec_mips, const float* lut, int lut_w, int lut_h,
                                   const float* point_cubes, int point_res, const float* spot_maps, int spot_w, int spot_h,
                                   const float* dir_map, int dir_w, int dir_h, float* out, int threads) {
    const Cubemap cd{diff_cube, diff_res, 1};
    const Cubemap cs{spec_cube, spec_res, spec_mips};
    const Image lutImg{lut, lut_w, lut_h, (size_t)lut_w * 2, 2};
    const ShadowMaps sm{point_cubes, point_res, spot_maps, spot_w, spot_h, dir_map, dir_w, dir_h};
    par_rows(height, threads, [&](int y) {
        for (int x = 0; x < width; ++x) {
            const size_t o = ((size_t)y * width + x) * 4;
            st(out + o, ForwardLighting_PSMain_Shadowed(*pf, *pv, ld(position_ao + o), ld(normal_roughness + o), ld(albedo_metalness + o),
                                                        nullptr, cd, cs, lutImg, sm));
        }
    });
}
float orc_shadow_test_pcf(const float lightSpacePos[4], float depthBias, float NdotL, const float* map, int w, int h, int directional) {
    ShadowTestPCFData pcf{}; pcf.lightSpacePos = {lightSpacePos[0], lightSpacePos[1], lightSpacePos[2], lightSpacePos[3]};
    pcf.depthBias = depthBias; pcf.NdotL = NdotL;
    const float2 dims = {(float)w, (float)h};
    return directional ? ShadowTestPCF_Directional(pcf, map, w, h, dims) : ShadowTestPCF(pcf, map, w, h, dims);
}
float orc_shadow_test_omni(const float Lw[3], float depthBias, float viewDistance, float farPlane, const float* cube, int res) {
    ShadowTestPCFData pcf{}; pcf.depthBias = depthBias; pcf.viewDistanceOfPixel = viewDistance;
    return OmnidirectionalShadowTestPCF(pcf, cube, res, make3(Lw[0], Lw[1], Lw[2]), farPlane);
}

// ---- §8(f).2 Radiance .hdr codec, §8(f).3 skydome / ApplyReflections -----------------------------------------
// decode: call with rgba == nullptr to get the size, then again with a buffer of w*h*4 floats. Returns the stb error class.
int orc_hdr_decode(const uint8_t* file, uint64_t n, int* w, int* h, float* rgba, float* max_luminance) {
    std::vector<float> px;
    const int rc = HdrDecode(file, (size_t)n, w, h, &px);
    if (rc) return rc;
    if (rgba) std::memcpy(rgba, px.data(), px.size() * sizeof(float));
    if (max_luminance) *max_luminance = CalculateMaxLuminance(px.data(), *w, *h);
    return 0;
}
// encode: returns the file size; writes at most `capacity` bytes
uint64_t orc_hdr_encode(const float* rgba, int w, int h, uint8_t* file, uint64_t capacity) {
    std::vector<uint8_t> f;
    HdrEncode(rgba, w, h, &f);
    if (file) std::memcpy(file, f.data(), std::min<uint64_t>(capacity, f.size()));
    return f.size();
}
int orc_resize_downsample(const float* in, int w, int h, float* out, int ow, int oh) { return ResizeFloat4_Downsample(in, w, h, out, ow, oh); }
void orc_linear_to_rgbe(const float* rgba, int n, uint8_t* rgbe) {
    for (int i = 0; i < n; ++i) LinearToRgbe(rgbe + 4 * (size_t)i, rgba + 4 * (size_t)i);
}
void orc_skydome(const float* hdri, int hw, int hh, int levels, const VqMatrix* inv_view_proj,
                 const float* normal_mask /* may be null */, float* scene, int width, int height,
                 int row_begin, int row_end, int threads) {
    const Pyramid py{hdri, hw, hh, levels};
    par_rows(row_end - row_begin, threads, [&](int r) {
        const int y = row_begin + r;
        for (int x = 0; x < width; ++x) {
            const size_t o = ((size_t)y * width + x) * 4;
            if (normal_mask && !(normal_mask[o] == 0.0f && normal_mask[o + 1] == 0.0f && normal_mask[o + 2] == 0.0f)) continue;
            st(scene + o, Skydome_PSMain(py, *inv_view_proj, x, y, width, height));
        }
    });
}
void orc_apply_reflections(float* scene, const float* reflection, const float* bounding_volumes /* may be null */,
                           int width, int height, int threads) {
    par_rows(height, threads, [&](int y) {
        for (int x = 0; x < width; ++x) {
            const size_t o = ((size_t)y * width + x) * 4;
            float4 bv;
            if (bounding_volumes) bv = ld(bounding_volumes + o);
            st(scene + o, ApplyReflections_CSMain(ld(scene + o), ld(reflection + o), bounding_volumes ? &bv : nullptr));
        }
    });
}

// ---- probes used by the compiled-shader pin (tests/test_hlsl_ref.py; oracle/ref_shim/hlsl_ref_shim.cpp) ------------
void orc_sample_lut(const float* lut, int w, int h, float u, float v, float out[2]) {
    const float2 r = SampleLUT(Image{lut, w, h, (size_t)w * 2, 2}, u, v); out[0] = r.x; out[1] = r.y;
}
void orc_sample_lut_n(const float* lut, int w, int h, const float* uv, int64_t n, float* out) {
    for (int64_t k = 0; k < n; ++k) orc_sample_lut(lut, w, h, uv[2 * k], uv[2 * k + 1], out + 2 * k);
}
float orc_sample_point2d(const float* map, int w, int h, float u, float v) { return SamplePoint2D(map, w, h, u, v); }
float orc_sample_point_cube(const float* cube, int res, const float d[3]) { return SamplePointCube(cube, res, make3(d[0], d[1], d[2])); }
void orc_diffuse_irradiance_texel(const float* pyramid, int w, int h, int levels, const float dir[3],
                                  float step, int n_phi, int n_theta, int src_mip, float out[4]) {
    std::vector<float> phis, thetas;
    DiffuseIrradianceAngles(step, n_phi, n_theta, phis, thetas);
    st(out, DiffuseIrradiance_PSMain(Pyramid{pyramid, w, h, levels}, make3(dir[0], dir[1], dir[2]), phis, thetas, src_mip, false));
}
void orc_specular_irradiance_texel(const float* pyramid, int w, int h, int levels, const float dir[3],
                                   float roughness, float dim_x, float dim_y, int num_samples, float out[4]) {
    st(out, SpecularIrradiance_PSMain(Pyramid{pyramid, w, h, levels}, make3(dir[0], dir[1], dir[2]), roughness,
                                      make2(dim_x, dim_y), (uint32_t)num_samples));
}
void orc_skydome_look_direction(const VqMatrix* inv_view_proj, int px, int py, int width, int height, float out[3]) {
    const float3 d = SkydomeLookDirection(*inv_view_proj, px, py, width, height); out[0] = d.x; out[1] = d.y; out[2] = d.z;
}
void orc_environment_brdf(float NdotV, float roughness, float metallic, const float diffuseColor[3], const float diffuseIrradiance[3],
                          const float preFilteredSpecular[3], const float F0ScaleBias[2], float out[3]) {
    const float3 r = EnvironmentBRDF(NdotV, roughness, metallic, make3(diffuseColor[0], diffuseColor[1], diffuseColor[2]),
                                     make3(diffuseIrradiance[0], diffuseIrradiance[1], diffuseIrradiance[2]),
                                     make3(preFilteredSpecular[0], preFilteredSpecular[1], preFilteredSpecular[2]),
                                     make2(F0ScaleBias[0], F0ScaleBias[1]));
    out[0] = r.x; out[1] = r.y; out[2] = r.z;
}
void orc_hdr_curves(const float c[3], float lin_to_srgb[3], float srgb_to_lin[3], float r709_to_2020[3], float r2020_to_709[3], float st2084[3]) {
    const float3 v = make3(c[0], c[1], c[2]);
    auto o3 = [](float* o, float3 r) { o[0] = r.x; o[1] = r.y; o[2] = r.z; };
    o3(lin_to_srgb, LinearToSRGB(v)); o3(srgb_to_lin, SRGBToLinear(v)); o3(r709_to_2020, Rec709ToRec2020(v));
    o3(r2020_to_709, Rec2020ToRec709(v)); o3(st2084, LinearToST2084(v));
}
int orc_depth_min_pyramid(const float* depth, int w, int h, float* levels, int max_levels) { return DepthMinPyramid(depth, w, h, levels, max_levels); }
// the shadowed pass with the emissive plane (orc_forward_lighting_shadowed predates it and passes none)
void orc_forward_lighting_shadowed_e(const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                     const float* position_ao, const float* normal_roughness, const float* albedo_metalness,
                                     const float* emissive, int width, int height, const float* diff_cube, int diff_res,
                                     const float* spec_cube, int spec_res, int spec_mips, const float* lut, int lut_w, int lut_h,
                                     const float* point_cubes, int point_res, const float* spot_maps, int spot_w, int spot_h,
                                     const float* dir_map, int dir_w, int dir_h, float* out, int threads) {
    const Cubemap cd{diff_cube, diff_res, 1};
    const Cubemap cs{spec_cube, spec_res, spec_mips};
    const Image lutImg{lut, lut_w, lut_h, (size_t)lut_w * 2, 2};
    const ShadowMaps sm{point_cubes, point_res, spot_maps, spot_w, spot_h, dir_map, dir_w, dir_h};
    par_rows(height, threads, [&](int y) {
        for (int x = 0; x < width; ++x) {
            const size_t o = ((size_t)y * width + x) * 4;
            float4 em;
            if (emissive) em = ld(emissive + o);
            st(out + o, ForwardLighting_PSMain_Shadowed(*pf, *pv, ld(position_ao + o), ld(normal_roughness + o), ld(albedo_metalness + o),
                                                        emissive ? &em : nullptr, cd, cs, lutImg, sm));
        }
    });
}
}  // extern "C"
