// vq_surface_sample.cuh — the surface producer's per-pixel code: material-texture sampling and the part of PSMain before
// lighting (ForwardLighting.hlsl:226-283) for one pixel of a 2x2 quad. Shared by surface_kernel (vq_surface.cu), which stores
// the result as G-buffer planes, and the fused PSMain kernel (vq_forward.cu), which stages it in shared memory for K1's shading.
#pragma once
#include "vq_common.cuh"

namespace {

using namespace vq;

// device copy of one texture descriptor: 16 B = one LDG.128. Level offsets are recomputed in registers (a short loop over
// the levels below the sampled one) instead of being looked up: a table would add a dependent memory round trip per map.
struct DevTex {
    const uint32_t* p;       // RGBA8 texels, packed levels; nullptr = null SRV
    int32_t w;
    uint32_t h_levels;       // height in bits 0..26, level count in bits 27..31
};
static_assert(sizeof(DevTex) == 16, "DevTex layout");

// One 16-byte RECORD per texel of a material whose maps all have the same size (how shipped material sets look): the bytes
// PSMain reads of every map, interleaved, so that one LDG.128 per trilinear tap fetches the texel of ALL maps:
//   x = diffuse RGBA | y = normal RGB, local-AO R | z = emissive RGB, roughness R | w = metalness R, ORM G, ORM B, 0
// (a null map contributes zeros, which is what a null SRV reads). Built once per table by record_build_kernel from the maps'
// own mip chains, level by level (same packed-level offsets); the K1 sampling copies of the cubemaps are the same idea.
struct DevMaterial {         // 80 + 7*16 + 16 = 208 B
    VqMaterialData c;
    DevTex t[7];
    DevTex rec;              // p = uint4 records (nullptr: this material samples its maps one by one), w, h_levels
};
static_assert(sizeof(DevMaterial) == 208, "DevMaterial layout");

}  // namespace

struct VqMaterialTable {
    DevMaterial* dev;
    int count;
    void* records;           // one allocation holding every material's texel records (nullptr: none)
    size_t record_bytes;
};

namespace {

// ---------------------------------------------------------------------------------------------
// texture sampling
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ int wrap_index(int i, int n) {           // general modulo (uv is unbounded: tiling)
    int r = i % n;
    return r < 0 ? r + n : r;
}

struct TexR { const uint32_t* p; int w, h, levels; };               // a descriptor in registers
__device__ __forceinline__ TexR load_tex(const DevTex* d) {
    const uint4 v = __ldg((const uint4*)d);
    TexR t;
    t.p = (const uint32_t*)(((uint64_t)v.y << 32) | v.x);
    t.w = (int)v.z; t.h = (int)(v.w & 0x07ffffffu); t.levels = (int)(v.w >> 27);
    return t;
}

// Sampler state of one Sample()/SampleBias() call: everything that depends only on (uv, derivatives, texture dimensions,
// bias) — the two mip levels, the trilinear fraction, the four tap offsets (level offset included) and the bilinear
// weights per level. A material's maps are usually all the same size, so consecutive textures reuse it (only the texel
// pointer differs) and the ~70 instructions of address math are paid once per pixel, not once per map.
struct Taps {
    int32_t w, h, levels; float bias;      // key
    uint32_t i[2][4];                      // [level slot][t00, t10, t01, t11]
    float fx[2], fy[2];
    float f;                               // trilinear fraction (0 -> slot 1 repeats slot 0)
};

__device__ __forceinline__ void level_taps(int W, int H, uint32_t o, float u, float v, uint32_t (&idx)[4], float& fx, float& fy) {
    // two roundings, as the oracle writes it: the weights multiply full-contrast byte data, so the coordinate must match
    const float x = __fsub_rn(__fmul_rn(u, (float)W), 0.5f), y = __fsub_rn(__fmul_rn(v, (float)H), 0.5f);
    const float x0 = floorf(x), y0 = floorf(y);
    // (int) is cvt.rzi: NaN -> 0 and saturated beyond the int range, which the oracle spells out. A coordinate that is not
    // finite gives fx or fy = NaN, so that level's blend is NaN (vqcuda.h, VqSurfaceInputs)
    fx = __fsub_rn(x, x0); fy = __fsub_rn(y, y0);
    const bool pow2 = ((W & (W - 1)) | (H & (H - 1))) == 0;
    int ix0, iy0;
    if (pow2) { ix0 = (int)x0 & (W - 1); iy0 = (int)y0 & (H - 1); }
    else      { ix0 = wrap_index((int)x0, W); iy0 = wrap_index((int)y0, H); }
    const int ix1 = ix0 + 1 == W ? 0 : ix0 + 1, iy1 = iy0 + 1 == H ? 0 : iy0 + 1;
    const uint32_t r0 = o + (uint32_t)(iy0 * W), r1 = o + (uint32_t)(iy1 * W);
    idx[0] = r0 + ix0; idx[1] = r0 + ix1; idx[2] = r1 + ix0; idx[3] = r1 + ix1;
}

__device__ __forceinline__ void make_taps(Taps& T, const TexR& t, float u, float v, float dudx, float dvdx, float dudy,
                                          float dvdy, float bias) {
    if (t.w == T.w && t.h == T.h && t.levels == T.levels && bias == T.bias) return;      // same sampler state as the previous map
    T.w = t.w; T.h = t.h; T.levels = t.levels; T.bias = bias;
    const float W = (float)t.w, H = (float)t.h;
    const float ax = dudx * W, ay = dvdx * H, bx = dudy * W, by = dvdy * H;
    const float m = fmaxf(fmaf(ax, ax, ay * ay), fmaf(bx, bx, by * by));
    float lod = (m > 0.0f ? 0.5f * __log2f(m) : -126.0f) + bias;
    lod = fminf(fmaxf(lod, 0.0f), (float)(t.levels - 1));
    const float l0f = floorf(lod);
    const int l0 = (int)l0f;
    T.f = (l0 + 1 < t.levels) ? lod - l0f : 0.0f;
    uint32_t o = 0;                                                   // texel offset of level l0 (vq_pyramid_offset)
    if (t.w == t.h && (t.w & (t.w - 1)) == 0 && t.w <= 16384) {       // square power of two: sum_{l<l0} (w>>l)^2 = 4 (w^2 - (w>>l0)^2) / 3
        const uint32_t wl = (uint32_t)t.w >> l0;
        o = (4u * ((uint32_t)t.w * (uint32_t)t.w - wl * wl)) / 3u;
    } else {
        for (int l = 0; l < l0; ++l) o += (uint32_t)((t.w >> l) * (t.h >> l));
    }
    const int W0 = t.w >> l0, H0 = t.h >> l0;
    level_taps(W0, H0, o, u, v, T.i[0], T.fx[0], T.fy[0]);
    // the second level is fetched unconditionally so that all 8 taps of a Sample() are independent loads in flight at once;
    // when the fraction is 0 it re-reads the first level's taps (L1 hits) and the lerp returns them unchanged
    if (T.f != 0.0f) level_taps(W0 >> 1, H0 >> 1, o + (uint32_t)(W0 * H0), u, v, T.i[1], T.fx[1], T.fy[1]);
    else {
#pragma unroll
        for (int k = 0; k < 4; ++k) T.i[1][k] = T.i[0][k];
        T.fx[1] = T.fx[0]; T.fy[1] = T.fy[0];
    }
}

// byte c of a packed RGBA8 texel as a float in [0,255]: PRMT drops the byte into the mantissa of 2^23 (ALU pipe) and one
// FADD removes the bias — instead of shift/mask + I2F, which issues on the quarter-rate XU pipe (39 % busy before).
template <int C>
__device__ __forceinline__ float byte_to_float(uint32_t texel) {
    return __uint_as_float(__byte_perm(texel, 0x4B000000u, 0x7650 + C)) - 8388608.0f;
}

template <int NCH>
__device__ __forceinline__ void bilinear_lerp(uint32_t t00, uint32_t t10, uint32_t t01, uint32_t t11, float fx, float fy,
                                              float (&out)[NCH]) {
#define VQ_CH(C)                                                                                   \
    if (C < NCH) {                                                                                 \
        const float a = byte_to_float<C>(t00), b = byte_to_float<C>(t10);                          \
        const float d = byte_to_float<C>(t01), e = byte_to_float<C>(t11);                          \
        const float top = fmaf(fx, b - a, a), bot = fmaf(fx, e - d, d);                            \
        out[C < NCH ? C : 0] = fmaf(fy, bot - top, top);                                           \
    }
    VQ_CH(0) VQ_CH(1) VQ_CH(2) VQ_CH(3)
#undef VQ_CH
}

// L2 residency hints (no instruction cost: the policy rides in the LDG/STG descriptor). Material texels are re-read by
// many blocks and should survive in L2; the interpolant planes and the G-buffer are touched exactly once and must not
// push them out (before: 40 % of the texel sectors that missed L1 also missed L2 with a 58 MB texture set).
__device__ __forceinline__ uint64_t l2_policy_evict_last() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_last.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ uint64_t l2_policy_evict_first() {
    uint64_t p; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(p)); return p;
}
__device__ __forceinline__ uint32_t ld_texel(const uint32_t* p, uint64_t pol) {
    uint32_t r; asm volatile("ld.global.nc.L2::cache_hint.b32 %0, [%1], %2;" : "=r"(r) : "l"(p), "l"(pol)); return r;
}
__device__ __forceinline__ float4 ld_once(const float4* p, uint64_t pol) {
    float4 v;
    asm volatile("ld.global.nc.L1::no_allocate.L2::cache_hint.v4.f32 {%0,%1,%2,%3}, [%4], %5;"
                 : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "l"(p), "l"(pol));
    return v;
}
__device__ __forceinline__ void st_once(float4* p, float4 v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// ---- record path: every map of the material in one 16-byte texel record ---------------------------------------------------
// byte C of a texel word as the float 2^23 + byte (PRMT only); differences of two such values are the exact byte differences,
// so only the lerp's base operand needs the bias removed — and the arithmetic runs on channel PAIRS (f2).
template <int C>
__device__ __forceinline__ float byte_biased(uint32_t texel) { return __uint_as_float(__byte_perm(texel, 0x4B000000u, 0x7650 + C)); }

// bilinear blend of channels (C0, C1) of four texel words, in [0,255]; the same operations, in the same order, as bilinear_lerp
template <int C0, int C1>
__device__ __forceinline__ f2 bilinear2(uint32_t t00, uint32_t t10, uint32_t t01, uint32_t t11, f2 fx, f2 fy) {
    const f2 unbias = bc(-8388608.0f);
    const f2 a = mk(byte_biased<C0>(t00), byte_biased<C1>(t00)), b = mk(byte_biased<C0>(t10), byte_biased<C1>(t10));
    const f2 d = mk(byte_biased<C0>(t01), byte_biased<C1>(t01)), e = mk(byte_biased<C0>(t11), byte_biased<C1>(t11));
    const f2 top = fma2(fx, b - a, a + unbias), bot = fma2(fx, e - d, d + unbias);
    return fma2(fy, bot - top, top);
}
// trilinear sample of the four channels of one record word -> [0,1]; w0[] = the word at the four taps of the lower level,
// w1[] = of the upper one (read only when the fraction is not 0: f == 0 returns the lower level's blend unchanged, as sample8 does)
__device__ __forceinline__ void sample_word(const uint32_t (&w0)[4], const uint32_t (&w1)[4], const Taps& T, bool two, float (&out)[4]) {
    f2 lo01 = bilinear2<0, 1>(w0[0], w0[1], w0[2], w0[3], bc(T.fx[0]), bc(T.fy[0]));
    f2 lo23 = bilinear2<2, 3>(w0[0], w0[1], w0[2], w0[3], bc(T.fx[0]), bc(T.fy[0]));
    if (two) {
        const f2 hi01 = bilinear2<0, 1>(w1[0], w1[1], w1[2], w1[3], bc(T.fx[1]), bc(T.fy[1]));
        const f2 hi23 = bilinear2<2, 3>(w1[0], w1[1], w1[2], w1[3], bc(T.fx[1]), bc(T.fy[1]));
        lo01 = fma2(bc(T.f), hi01 - lo01, lo01);
        lo23 = fma2(bc(T.f), hi23 - lo23, lo23);
    }
    lo01 = lo01 * bc(1.0f / 255.0f); lo23 = lo23 * bc(1.0f / 255.0f);
    out[0] = lo01.v.x; out[1] = lo01.v.y; out[2] = lo23.v.x; out[3] = lo23.v.y;
}
__device__ __forceinline__ uint4 ld_record(const uint4* p, uint64_t pol) {
    uint4 r;
    asm volatile("ld.global.nc.L2::cache_hint.v4.u32 {%0,%1,%2,%3}, [%4], %5;" : "=r"(r.x), "=r"(r.y), "=r"(r.z), "=r"(r.w) : "l"(p), "l"(pol));
    return r;
}

// Texture2D.Sample / SampleBias of ONE RGBA8 map: isotropic trilinear, WRAP; channels in [0,1]. Two or more channels are
// filtered as packed pairs (bilinear2); the operations per channel are those of bilinear_lerp either way.
template <int NCH>
__device__ __forceinline__ void sample8(Taps& T, const TexR& t, float u, float v, float dudx, float dvdx, float dudy,
                                        float dvdy, float bias, float (&out)[NCH]) {
    make_taps(T, t, u, v, dudx, dvdx, dudy, dvdy, bias);
    const uint32_t* p = t.p;
    const uint64_t keep = l2_policy_evict_last();
    uint32_t q[8];
#pragma unroll
    for (int k = 0; k < 4; ++k) { q[k] = ld_texel(p + T.i[0][k], keep); q[4 + k] = ld_texel(p + T.i[1][k], keep); }
    if (NCH == 1) {
        float lo[1], hi[1];
        bilinear_lerp<1>(q[0], q[1], q[2], q[3], T.fx[0], T.fy[0], lo);
        bilinear_lerp<1>(q[4], q[5], q[6], q[7], T.fx[1], T.fy[1], hi);
        out[0] = fmaf(T.f, hi[0] - lo[0], lo[0]) * (1.0f / 255.0f);
    } else {
        const uint32_t w0[4] = {q[0], q[1], q[2], q[3]}, w1[4] = {q[4], q[5], q[6], q[7]};
        float o[4];
        sample_word(w0, w1, T, true, o);                             // f == 0: the upper level repeats the lower one's taps
#pragma unroll
        for (int c = 0; c < NCH; ++c) out[c] = o[c];
    }
}

// what PSMain's Sample() calls return for one pixel (zeros where a map is not sampled or its SRV is null)
struct Sampled {
    float d[4];              // diffuse RGBA
    float n[3];              // tangent-space normal RGB
    float e[3];              // emissive RGB
    float ao, rg, mt;        // local AO .r, roughness .r, metalness .r
    float og, ob;            // ORM .g, .b
    bool nrm;                // a normal map is bound
};

__device__ __forceinline__ float pow22(float c) {                   // SRGBToLinear, ShadingMath.hlsl:65; c in [0,1]
    // lg2.approx / ex2.approx (2 ulp each) without exp2f()'s scaling for denormal results: c^2.2 of a sampled byte blend is either 0
    // (log2(0) = -inf -> ex2 = 0) or >= (1/255/2^20)^2.2, far above the denormal range
    float r; asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(2.2f * __log2f(c))); return r;
}

struct SurfArgs {
    ImgV posU, nrmV, tanM;
    const float* ssao; int ssaoPitch;       // floats
    ImgV outPos, outNrm, outAlb, outEmi;    // outEmi.p == nullptr -> no emissive plane
    const DevMaterial* mats; int nMats;
    float ambient;
    int alphaMask;
    int rowBegin, rowEnd, tileY0;           // tileY0 = rowBegin & ~1 (quads are aligned to absolute even rows)
};

// One pixel of PSMain before lighting, from its interpolants (pu, nv, tm), its material index and the fine quad derivatives of
// the raw uv. The result goes to sink({P, ao}, {N, roughness}, {albedo, metalness}, {emissive, intensity}), laid out as the
// G-buffer planes (VqGBuffer). Early returns = the alpha-mask discard: the sink is not called.
template <class Sink>
__device__ __forceinline__ void shade_surface_pixel(const SurfArgs& A, int mi, float4 pu, float4 nv, float4 tm, float ssao,
                                                    float dRawUdx, float dRawVdx, float dRawUdy, float dRawVdy, Sink&& sink) {
    const float ru = pu.w, rv = nv.w;
    const DevMaterial& M = A.mats[mi];
    const float4 c0 = __ldg((const float4*)&M.c), c1 = __ldg((const float4*)&M.c + 1);
    const float4 c2 = __ldg((const float4*)&M.c + 2), c3 = __ldg((const float4*)&M.c + 3), c4 = __ldg((const float4*)&M.c + 4);
    const uint4 rd = __ldg((const uint4*)&M.rec);                   // texel records of this material (pointer 0: none)
    // c0 = diffuse.rgb, alpha | c1 = emissiveColor.rgb, emissiveIntensity | c2 = specular.rgb, normalMapMipBias
    // c3 = uvScaleOffset | c4 = roughness, metalness, displacement, textureConfig
    const int cfg = (int)c4.w;

    const float u = __fadd_rn(__fmul_rn(ru, c3.x), c3.z), v = __fadd_rn(__fmul_rn(rv, c3.y), c3.w);   // :226
    const float dudx = dRawUdx * c3.x, dvdx = dRawVdx * c3.y, dudy = dRawUdy * c3.x, dvdy = dRawVdy * c3.y;

    Sampled S;
    S.d[0] = S.d[1] = S.d[2] = S.d[3] = 0.0f; S.n[0] = S.n[1] = S.n[2] = 0.0f; S.e[0] = S.e[1] = S.e[2] = 0.0f;
    S.ao = S.rg = S.mt = S.og = S.ob = 0.0f; S.nrm = false;
    Taps T;
    T.w = T.h = T.levels = -1; T.bias = 0.0f; T.f = 0.0f;

    if (rd.x | rd.y) {
        // ---- record path: the maps share one size, so ONE sampler state and 8 x LDG.128 serve every Sample() of the pixel ----
        TexR tr;
        tr.p = nullptr; tr.w = (int)(rd.z & 0x00ffffffu); tr.h = (int)(rd.w & 0x07ffffffu); tr.levels = (int)(rd.w >> 27);
        const uint4* R = (const uint4*)(((uint64_t)rd.y << 32) | rd.x);
        const uint32_t present = rd.z >> 24;                                // bit k: map k is bound
        S.nrm = (present & 2u) != 0u;
        make_taps(T, tr, u, v, dudx, dvdx, dudy, dvdy, 0.0f);
        const uint64_t keep = l2_policy_evict_last();
        const bool two = T.f != 0.0f;
        uint4 q[8];
#pragma unroll
        for (int k = 0; k < 4; ++k) q[k] = ld_record(R + T.i[0][k], keep);
        if (two) {
#pragma unroll
            for (int k = 0; k < 4; ++k) q[4 + k] = ld_record(R + T.i[1][k], keep);
        } else {
#pragma unroll
            for (int k = 0; k < 4; ++k) q[4 + k] = q[k];
        }
        const bool biasedNormal = S.nrm && c2.w != 0.0f;                    // SampleBias with its own LOD: a second set of taps
        uint32_t nq[8];
        Taps TN;
        bool twoN = false;
        if (biasedNormal) {
            TN.w = -1; TN.h = TN.levels = -1; TN.bias = 0.0f; TN.f = 0.0f;
            make_taps(TN, tr, u, v, dudx, dvdx, dudy, dvdy, c2.w);
            twoN = TN.f != 0.0f;
            const uint32_t* Rw = (const uint32_t*)R + 1;                    // word y of a record
#pragma unroll
            for (int k = 0; k < 4; ++k) { nq[k] = ld_texel(Rw + 4 * (size_t)TN.i[0][k], keep); nq[4 + k] = ld_texel(Rw + 4 * (size_t)TN.i[1][k], keep); }
        }
        float o[4];
        if (cfg & VQ_TEXCFG_DIFFUSE) {
            const uint32_t w0[4] = {q[0].x, q[1].x, q[2].x, q[3].x}, w1[4] = {q[4].x, q[5].x, q[6].x, q[7].x};
            sample_word(w0, w1, T, two, o);
            S.d[0] = o[0]; S.d[1] = o[1]; S.d[2] = o[2]; S.d[3] = o[3];
        }
        if ((S.nrm && !biasedNormal) || (cfg & VQ_TEXCFG_AO)) {
            const uint32_t w0[4] = {q[0].y, q[1].y, q[2].y, q[3].y}, w1[4] = {q[4].y, q[5].y, q[6].y, q[7].y};
            sample_word(w0, w1, T, two, o);
            S.n[0] = o[0]; S.n[1] = o[1]; S.n[2] = o[2]; S.ao = o[3];
        }
        if (biasedNormal) {
            const uint32_t w0[4] = {nq[0], nq[1], nq[2], nq[3]}, w1[4] = {nq[4], nq[5], nq[6], nq[7]};
            sample_word(w0, w1, TN, twoN, o);
            S.n[0] = o[0]; S.n[1] = o[1]; S.n[2] = o[2];
        }
        if (cfg & (VQ_TEXCFG_EMISSIVE | VQ_TEXCFG_ROUGHNESS)) {
            const uint32_t w0[4] = {q[0].z, q[1].z, q[2].z, q[3].z}, w1[4] = {q[4].z, q[5].z, q[6].z, q[7].z};
            sample_word(w0, w1, T, two, o);
            S.e[0] = o[0]; S.e[1] = o[1]; S.e[2] = o[2]; S.rg = o[3];
        }
        if (cfg & (VQ_TEXCFG_METALLIC | VQ_TEXCFG_ORM)) {
            const uint32_t w0[4] = {q[0].w, q[1].w, q[2].w, q[3].w}, w1[4] = {q[4].w, q[5].w, q[6].w, q[7].w};
            sample_word(w0, w1, T, two, o);
            S.mt = o[0]; S.og = o[1]; S.ob = o[2];
        }
    } else {
        // ---- one map at a time (maps of different sizes): a Sample() = 8 x LDG.32 ----
        // (one looped copy of the sampler instead of these seven inlined ones shrinks the kernel from 92 KB to 36 KB of code but
        //  executes more instructions — four channels for every map, routing by slot: measured slower, not kept)
        if (cfg & VQ_TEXCFG_DIFFUSE) {
            const TexR tDiff = load_tex(&M.t[0]);
            if (tDiff.p) {
                if (A.alphaMask) sample8<4>(T, tDiff, u, v, dudx, dvdx, dudy, dvdy, 0.0f, S.d);
                else { float s3[3]; sample8<3>(T, tDiff, u, v, dudx, dvdx, dudy, dvdy, 0.0f, s3); S.d[0] = s3[0]; S.d[1] = s3[1]; S.d[2] = s3[2]; }
            }
            if (A.alphaMask && S.d[3] < 0.01f) return;                                                // discard before the other maps are read
        }
        if (cfg & VQ_TEXCFG_EMISSIVE) {
            const TexR tEmi = load_tex(&M.t[2]);
            if (tEmi.p) sample8<3>(T, tEmi, u, v, dudx, dvdx, dudy, dvdy, 0.0f, S.e);
        }
        const TexR tNrm = load_tex(&M.t[1]);                                                          // sampled whatever the config says
        if (tNrm.p) { S.nrm = true; sample8<3>(T, tNrm, u, v, dudx, dvdx, dudy, dvdy, c2.w, S.n); }
        if (cfg & VQ_TEXCFG_AO)        { float s[1] = {0.f}; const TexR t = load_tex(&M.t[6]); if (t.p) sample8<1>(T, t, u, v, dudx, dvdx, dudy, dvdy, 0.0f, s); S.ao = s[0]; }
        if (cfg & VQ_TEXCFG_ROUGHNESS) { float s[1] = {0.f}; const TexR t = load_tex(&M.t[4]); if (t.p) sample8<1>(T, t, u, v, dudx, dvdx, dudy, dvdy, 0.0f, s); S.rg = s[0]; }
        if (cfg & VQ_TEXCFG_METALLIC)  { float s[1] = {0.f}; const TexR t = load_tex(&M.t[3]); if (t.p) sample8<1>(T, t, u, v, dudx, dvdx, dudy, dvdy, 0.0f, s); S.mt = s[0]; }
        if (cfg & VQ_TEXCFG_ORM) {
            float s[3] = {0.f, 0.f, 0.f};
            const TexR t = load_tex(&M.t[5]);
            if (t.p) sample8<3>(T, t, u, v, dudx, dvdx, dudy, dvdy, 0.0f, s);
            S.og = s[1]; S.ob = s[2];
        }
    }

    // --- diffuse (+alpha for the ENABLE_ALPHA_MASK variant, :237-240) ---
    float3 diffuseColor = f3(c0.x, c0.y, c0.z);
    if (cfg & VQ_TEXCFG_DIFFUSE) {
        if (A.alphaMask && S.d[3] < 0.01f) return;                                                    // discard
        diffuseColor = f3(pow22(S.d[0]) * c0.x, pow22(S.d[1]) * c0.y, pow22(S.d[2]) * c0.z);          // :243,249
    }
    // --- emissive ---
    float3 emissiveColor = f3(c1.x, c1.y, c1.z);
    if (cfg & VQ_TEXCFG_EMISSIVE) emissiveColor = f3(pow22(S.e[0]) * c1.x, pow22(S.e[1]) * c1.y, pow22(S.e[2]) * c1.z);   // :244,250
    float roughness = c4.x, metalness = c4.y;                                                         // :252-253
    float ao = A.ambient;                                                                             // :247

    // --- normal: N / T from the interpolants, tangent-space normal whenever the sample is not ~0 (:265-267) ---
    const float3 Nw = f3(nv.x, nv.y, nv.z), Tw = f3(tm.x, tm.y, tm.z);
    const float3 N = Nw * rsqrtf(dot(Nw, Nw));
    float3 Nout = N;
    if (S.nrm) {
        const float* s = S.n;
        if (!(sqrtf(s[0] * s[0] + s[1] * s[1] + s[2] * s[2]) < 0.01f)) {                          // :267 as written: NaN unpacks
            const float3 T0 = Tw * rsqrtf(dot(Tw, Tw));
            float3 sn = f3(s[0] * 2.0f - 1.0f, s[1] * 2.0f - 1.0f, s[2] * 2.0f - 1.0f);               // ShadingMath.hlsl:46
            sn = sn * rsqrtf(dot(sn, sn));
            float3 T = T0 - N * dot(N, T0);                                                           // :47
            T = T * rsqrtf(dot(T, T));
            const float3 Nn = N * rsqrtf(dot(N, N));                                                  // :48 (N is already unit)
            float3 B = cross(T, Nn);                                                                  // :49
            B = B * rsqrtf(dot(B, B));
            Nout = T * sn.x + B * sn.y + Nn * sn.z;                                                   // :50-51
        }
    }
    if (cfg & VQ_TEXCFG_AO)        ao *= S.ao;                                                        // :269
    if (cfg & VQ_TEXCFG_ROUGHNESS) roughness *= S.rg;                                                 // :270
    if (cfg & VQ_TEXCFG_METALLIC)  metalness *= S.mt;                                                 // :271
    if (cfg & VQ_TEXCFG_ORM) { roughness *= S.og; metalness *= S.ob; }                                // :272-277
    ao *= ssao;                                                                                       // :280-281 (1 when no SSAO plane is bound)

    sink(make_float4(pu.x, pu.y, pu.z, ao), make_float4(Nout.x, Nout.y, Nout.z, roughness),
         make_float4(diffuseColor.x, diffuseColor.y, diffuseColor.z, metalness), make_float4(emissiveColor.x, emissiveColor.y, emissiveColor.z, c1.w));
}

// Pixel (x, y) of a warp that covers a 16x2 strip of aligned 2x2 quads (lane & 15 = column, lane >> 4 = row): loads its
// interpolants, takes the quad derivatives by shuffles (every lane of the warp must call this) and, for a pixel inside the
// image and the row range, runs shade_surface_pixel into `sink`. `once`: the L2 evict-first policy of the interpolant loads.
template <class Sink>
__device__ __forceinline__ void surface_quad_pixel(const SurfArgs& A, int x, int y, int lane, uint64_t once, Sink&& sink) {
    const int W = A.posU.w, H = A.posU.h;
    // threads outside the image re-read the clamped texel: their uv equals the in-image partner's -> derivative 0,
    // exactly the oracle's "partner clamped to the image"
    const int cx = min(x, W - 1), cy = min(y, H - 1);
    const float4 pu = ld_once(A.posU.row(cy) + cx, once);
    const float4 nv = ld_once(A.nrmV.row(cy) + cx, once);
    const float4 tm = ld_once(A.tanM.row(cy) + cx, once);
    // the SSAO texel (x+1, y+1, WRAP; :280-281) depends on nothing but the pixel: fetched with the interpolants, not at the point
    // of use after the whole sampling chain (where it was 17 % of the kernel's long-scoreboard stalls)
    float ssao = 1.0f;
    if (A.ssao) {
        const int sxp = cx + 1 == W ? 0 : cx + 1, syp = cy + 1 == H ? 0 : cy + 1;
        ssao = __ldg(A.ssao + (size_t)syp * A.ssaoPitch + sxp);
    }
    const float ru = pu.w, rv = nv.w;
    // fine quad derivatives of the RAW uv: horizontal partner = lane^1, vertical = lane^16
    const float ruX = __shfl_xor_sync(0xffffffffu, ru, 1), rvX = __shfl_xor_sync(0xffffffffu, rv, 1);
    const float ruY = __shfl_xor_sync(0xffffffffu, ru, 16), rvY = __shfl_xor_sync(0xffffffffu, rv, 16);
    const float sx = (lane & 1) ? -1.0f : 1.0f, sy = (lane & 16) ? -1.0f : 1.0f;   // (odd - even) regardless of which I am
    const float dRawUdx = (ruX - ru) * sx, dRawVdx = (rvX - rv) * sx;
    const float dRawUdy = (ruY - ru) * sy, dRawVdy = (rvY - rv) * sy;
    if (x < W && y < H && y >= A.rowBegin && y < A.rowEnd) {
        const int mi = min(max((int)tm.w, 0), A.nMats - 1);
        shade_surface_pixel(A, mi, pu, nv, tm, ssao, dRawUdx, dRawVdx, dRawUdy, dRawVdy, sink);
    }
}

// Checks the caller's interpolant planes, SSAO plane and material table and fills every field of A but the G-buffer outputs.
int surface_inputs(const VqSurfaceInputs* in, const VqMaterialTable* table, float ambient_factor, int alpha_mask,
                          int row_begin, int row_end, SurfArgs& A) {
    VQ_REQUIRE(in && table, "null argument");
    const int W = in->position_u.width, H = in->position_u.height;
    VQ_REQUIRE(vq_image_ok(in->position_u) && vq_image_ok(in->normal_v) && vq_image_ok(in->tangent_m), "bad attribute plane");
    VQ_REQUIRE(in->normal_v.width == W && in->normal_v.height == H && in->tangent_m.width == W && in->tangent_m.height == H,
               "attribute planes differ in size");
    if (in->ssao.ptr)
        VQ_REQUIRE(vq_image_ok(in->ssao, 4) && in->ssao.width == W && in->ssao.height == H, "bad SSAO plane");
    VQ_REQUIRE(row_begin >= 0 && row_end <= H && row_begin <= row_end, "row range out of bounds");
    VQ_REQUIRE(table->dev && table->count >= 1, "empty material table");
    A.posU = make_view(in->position_u); A.nrmV = make_view(in->normal_v); A.tanM = make_view(in->tangent_m);
    A.ssao = (const float*)in->ssao.ptr; A.ssaoPitch = in->ssao.ptr ? (int)(in->ssao.pitch_bytes / 4) : 0;
    A.mats = table->dev; A.nMats = table->count;
    A.ambient = ambient_factor; A.alphaMask = alpha_mask;
    A.rowBegin = row_begin; A.rowEnd = row_end; A.tileY0 = row_begin & ~1;
    return VQ_OK;
}

}  // namespace
