// vq_forward.cu — K1 forward PBR lighting for sm_90a.
//
// Replaces VQRenderer::RenderSceneColor (SceneRendering.cpp:1619-1851) + PSMain
// (ForwardLighting.hlsl:285-380) over a G-buffer of three float4 planes (+ optional emissive):
//   64 B/pixel of HBM traffic: the three planes arrive as 4 KB row segments through a TMA (cp.async.bulk) /
//   mbarrier ring in shared memory, the result leaves as one STG.128 per pixel; one thread shades TWO pixels (two
//   independent dependency chains through the light loop); the light array is staged once per
//   CTA into shared memory; the IBL cubemaps and the BRDF LUT are gathered from L2-resident sampling copies
//   (bordered texels / LUT column pairs, 51 MB at the reference sizes) with five 32-byte gathers per pixel, each read by
//   two neighbouring lanes together (see "lane-pair record gathers"), because the L1 data pipe — one wavefront per distinct
//   line of a divergent gather — is what bounds this kernel (DESIGN.md §4).
// The math is PSMain's with per-pixel invariants hoisted out of the light loops (N, V, N.V, the
// Smith-G term of V, F0, kD factors). Discontinuities are evaluated exactly as the oracle does:
//   * `D < l.range` uses an unfused |L-P|^2 and a per-light threshold on the squared distance that is
//     equivalent to the correctly-rounded sqrt compare;
//   * the specular mip is int(roughness * MAX_LOD) (one fp32 multiply);
//   * cubemap taps are seamless across face edges, so face selection is not a discontinuity.
#include "vq_common.cuh"
#include "vq_surface_sample.cuh"
#include "vq_shadow_math.cuh"
#include <stdlib.h>

using namespace vq;

namespace {


// Sampling copy of a cubemap. Every face of every mip is a (N+2)x(N+2) grid of bordered texel positions, the 1-texel
// border holding the neighbouring faces' edge texels (corners: the mean of the three texels that meet there), so
// that the seamless bilinear footprint never leaves the face. One float4 per position: a bilinear footprint is two rows of two
// adjacent texels, {t(i,j), t(i+1,j)} and {t(i,j+1), t(i+1,j+1)}, 32 contiguous bytes each, instead of four scattered texels.
// A gather whose lanes go to unrelated texels costs one L1 wavefront per distinct 128-byte line it touches, so the number
// of distinct lines per pixel is what the layout and the loads minimise: lanes 2q and 2q+1 read each other's footprint rows
// together (cube_issue / ldg_pair), the even lane t(i) and the odd lane t(i+1), so one instruction touches at most 16 places
// (a row crosses a line boundary once in 8 positions). mipOffset[] are position offsets of face 0 per mip.
struct CubeV { const float4* p; int res, mips; uint32_t mipOffset[16]; };
// Column-pair copy of the BRDF LUT: a (W+2) x (H+1) grid of 16-byte texels, texel (c,cy) = {p(xc,y0), p(xc,y1)} with
// xc = clamp(c-1, 0, W-1), y0 = clamp(cy-1, 0, H-1), y1 = clamp(cy, 0, H-1). The CLAMP-addressed bilinear footprint of (x0,y0) is
// then texels c = x0+1 and x0+2 of row cy = y0+1: 32 contiguous bytes, read by a lane pair exactly like a row of a cube footprint.
// 16 bytes per footprint position keep the copies small enough for L2 to hold most of them (DESIGN.md §9).
struct LutV { const float4* p; int w, h; };
struct F8 { float4 a, b; };

struct SPoint { float3 pos; float d2Limit; float3 color; float brightness; };
struct SDir { float3 wi; float pad0; float3 radiance; float pad1; };
struct SSpot { float3 pos; float outer; float3 color; float brightness; float3 dir; float inner; float invCone; float cosLo, cosHi; float pad; };
constexpr int FWD_MAX_POINT = VQ_NUM_LIGHTS_POINT + VQ_NUM_SHADOWING_LIGHTS_POINT, FWD_MAX_SPOT = VQ_NUM_LIGHTS_SPOT + VQ_NUM_SHADOWING_LIGHTS_SPOT;

struct FwdParams {
    // the frame's lights, conditioned on the host (exact range thresholds, normalised directions, radiance) and read by the kernel
    // straight from the constant bank with warp-uniform indices: no shared-memory staging, no LDS in the light loop (the L1/MIO
    // pipe that the environment gathers keep busy is left alone)
    SPoint pts[FWD_MAX_POINT];         // point lights, then (unshadowed) point casters
    SSpot spots[FWD_MAX_SPOT];         // spot lights, then spot casters
    SDir dir;
    int numPoint, numSpot, dirEnabled;
    float3 cam;
    float cosB, sinB;                  // GetHDRIRotationMatrix (Lighting.hlsl:348-358), cos/sin(-offset)
    int maxLod;                        // int(MaxEnvMapLODLevels)
    int diffuseOnly;
    int hasEmissive;
    ImgV pos, nrm, alb, emi;
    ImgV outs[8];                      // destinations: the local frame and, for the fused gather, the peers' frames (NVLink P2P)
    int nOut, dstRowOffset;            // every shaded pixel goes to row dstRowOffset+y of every destination
    CubeV diff, spec;
    LutV lut;
    PeerSync sync;                     // MULTI: optional end-of-pass rendezvous run by the last CTA (n == 0: none)
    uint32_t* ticket;                  // MULTI: retired-CTA count (zero between launches)
    float diffHalfN;                   // res/2 of the diffuse cube
    uint32_t diffMaxRec, specMaxRec;   // last record a footprint may start at (address clamp for non-finite directions)
    int rowBegin, rows, width;
    // SHADOWED instantiation only (vq_forward_lighting_shadowed): PCF tap counts per pixel and caster; the caster lights are the
    // LAST nPointCasters / nSpotCasters entries of pts[] / spots[]
    ShadowRecV shadow;
};

// ---------------------------------------------------------------------------------------------
// cubemap sampling: bilinear, seamless (SURVEY.md §9; identical rule in oracle/oracle_shading.cpp)
// ---------------------------------------------------------------------------------------------
// D3D face selection (largest |component|; ties X > Y > Z as in the oracle) written with selects so that a warp never
// diverges on it:  face, and the face-plane coordinates sx (right), sy (up) in [-1,1]
//   +X: (-z, y)  -X: (z, y)  +Y: (x, -z)  -Y: (x, z)  +Z: (x, y)  -Z: (-x, y), each over |major|
// The sign choices ride on the SIGNED reciprocal of the major component: rcp.approx is odd, so (+-c) * rcp(|m|) ==
// c' * rcp(m) bit for bit with c' = -z on X and Y, x on Z (a zero or NaN product is the same zero or NaN downstream).
__device__ __forceinline__ void dir_to_face(float3 d, int& face, float& sx, float& sy) {
    const float ax = fabsf(d.x), ay = fabsf(d.y), az = fabsf(d.z);
    const bool isX = ax >= ay && ax >= az;
    const bool isY = !isX && ay >= az;
    const float mv = isX ? d.x : (isY ? d.y : d.z);          // signed major component
    const float r = rcp_fast(mv), ra = fabsf(r);             // rcp(|mv|) == |rcp(mv)|
    sx = (isX ? -d.z : d.x) * (isY ? ra : r);
    sy = (isY ? -d.z : d.y) * (isY ? r : ra);
    face = (isX ? 0 : (isY ? 2 : 4)) + (mv > 0.0f ? 0 : 1);
}

// integer-only neighbour lookup for a tap one texel outside the face (see DESIGN.md "cube edges"); used only by
// the border-padding kernel, never per pixel
__device__ void cube_resolve_edge(int N, int face, int i, int j, int& of, int& oi, int& oj) {
    const int A = 2 * i + 1 - N, B = N - 1 - 2 * j, C = N;
    int dx, dy, dz;
    switch (face) {
        case 0: dx = C;  dy = B;  dz = -A; break;
        case 1: dx = -C; dy = B;  dz = A;  break;
        case 2: dx = A;  dy = C;  dz = -B; break;
        case 3: dx = A;  dy = -C; dz = B;  break;
        case 4: dx = A;  dy = B;  dz = C;  break;
        default: dx = -A; dy = B; dz = -C; break;
    }
    const int M = N + 1;
    int nsx, nsy;
    if (dx == M)       { of = 0; nsx = -dz; nsy = dy; }
    else if (dx == -M) { of = 1; nsx = dz;  nsy = dy; }
    else if (dy == M)  { of = 2; nsx = dx;  nsy = -dz; }
    else if (dy == -M) { of = 3; nsx = dx;  nsy = dz; }
    else if (dz == M)  { of = 4; nsx = dx;  nsy = dy; }
    else               { of = 5; nsx = -dx; nsy = dy; }
    oi = min(max(((nsx + M) * N) / (2 * M), 0), N - 1);
    oj = min(max(((M - nsy) * N) / (2 * M), 0), N - 1);
}

// value of bordered position `idx` (flattened over mips, faces, (N+2)^2 positions) of a packed cube
__device__ float4 bordered_texel(const float4* __restrict__ src, int res, int mips, uint32_t idx) {
    uint32_t rem = idx, srcOff = 0; int m = 0, N = res;
    for (; m < mips; ++m) {
        N = res >> m;
        const uint32_t sz = 6u * (uint32_t)(N + 2) * (uint32_t)(N + 2);
        if (rem < sz) break;
        rem -= sz; srcOff += 6u * (uint32_t)N * (uint32_t)N;
    }
    const int P = N + 2;
    const int face = (int)(rem / (uint32_t)(P * P));
    const int r2 = (int)(rem % (uint32_t)(P * P));
    const int i = r2 % P - 1, j = r2 / P - 1;           // face-relative texel, -1..N
    const float4* sm = src + srcOff;
    auto fetch = [&](int f, int x, int y) { return __ldg(sm + (size_t)f * N * N + (size_t)y * N + x); };
    auto edge = [&](int x, int y) { int f2, i2, j2; cube_resolve_edge(N, face, x, y, f2, i2, j2); return fetch(f2, i2, j2); };
    const bool oi = (i < 0 || i >= N), oj = (j < 0 || j >= N);
    if (!oi && !oj) return fetch(face, i, j);
    if (oi != oj) return edge(i, j);
    // cube corner: mean of the three texels meeting there (own corner + the two edge neighbours)
    const int ci = i < 0 ? 0 : N - 1, cj = j < 0 ? 0 : N - 1;
    const float4 a = fetch(face, ci, cj), b = edge(i, cj), c = edge(ci, j);
    return make_float4((a.x + b.x + c.x) * (1.0f / 3.0f), (a.y + b.y + c.y) * (1.0f / 3.0f),
                       (a.z + b.z + c.z) * (1.0f / 3.0f), (a.w + b.w + c.w) * (1.0f / 3.0f));
}
// packed cube (mip-major / face-minor, N x N faces) -> sampling copy: one texel per bordered position
__global__ void __launch_bounds__(256) cube_pad_kernel(const float4* __restrict__ src, float4* __restrict__ dst,
                                                        int res, int mips, uint32_t totalPadded) {
    for (uint32_t idx = blockIdx.x * 256u + threadIdx.x; idx < totalPadded; idx += gridDim.x * 256u)
        dst[idx] = bordered_texel(src, res, mips, idx);
}

// BRDF LUT (float2, pitched) -> column pairs (see LutV): (W+2) x (H+1) texels of 16 bytes
__global__ void __launch_bounds__(256) lut_pair_kernel(const float2* __restrict__ src, int pitch2, int W, int H, float4* __restrict__ dst) {
    const uint32_t total = (uint32_t)(W + 2) * (uint32_t)(H + 1);
    for (uint32_t idx = blockIdx.x * 256u + threadIdx.x; idx < total; idx += gridDim.x * 256u) {
        const int c = (int)(idx % (uint32_t)(W + 2)), cy = (int)(idx / (uint32_t)(W + 2));
        const int xc = min(max(c - 1, 0), W - 1), y0 = max(cy - 1, 0), y1 = min(cy, H - 1);
        const float2 p0 = __ldg(src + (size_t)y0 * pitch2 + xc), p1 = __ldg(src + (size_t)y1 * pitch2 + xc);
        dst[idx] = make_float4(p0.x, p0.y, p1.x, p1.y);
    }
}

// ---------------------------------------------------------------------------------------------
// pixel pairs
// ---------------------------------------------------------------------------------------------
// One thread shades TWO pixels and every quantity of the light loop is a pair {pixel A, pixel B} (vq_common.cuh: f2):
// lane .x of every f2 is pixel A (column x0 + tid), lane .y pixel B (column x0 + 128 + tid).

// ---------------------------------------------------------------------------------------------
// per-pixel-pair shading state with everything that does not depend on the light hoisted
// ---------------------------------------------------------------------------------------------
struct Px2 {
    float3 PA, PB;                // positions of the two pixels (scalar: every use is a first-touch subtraction)
    f2 Nx, Ny, Nz;                // normalize(Ns)                                   (BRDF.hlsl:167)
    f2 Vx, Vy, Vz;                // normalize(cam - P)                              (ForwardLighting.hlsl:285)
    f2 nsLen;                     // |Ns|: dot(Ns,Wi) = nsLen * dot(Nn,Wi)           (Lighting.hlsl:316 uses the raw s.N)
    f2 nv, nv4;                   // dot(Nn,V), 4*saturate(dot(Nn,V))
    f2 a2m1;                      // roughness^4 - 1 (unfused, feeds the exact t)
    f2 a2gV, gV;                  // a2 * G1(V), G1(V) = Smith-Schlick-GGX of the view vector (BRDF.hlsl:82-97)
    f2 k4, omk;                   // k + 0.0001, 1 - k with k = (roughness+1)^2 / 8
    uint32_t texA, texB;          // shared-memory addresses of the two pixels' position texels (planes follow at FWD_PLANE)
    uint64_t recA, recB;          // SHADOWED forward_kernel only: the two pixels' PCF records (ShadowRecV, vq_common.cuh)
};
struct Acc2 { f2 ax, ay, az, bx, by, bz, cx, cy, cz; };   // sum over lights of w*col * {(1-fc), fc*spec, spec}

// ---- exact re-evaluation of N.H -------------------------------------------------------------------
// GGX's t = nh2*(a2-1)+1 cancels catastrophically near a highlight on a smooth surface (t ~ a2 ~ 1e-5),
// so D amplifies a 1-ulp difference in N.H by up to 1e4. Where t is small the kernel therefore recomputes
// N.H with the oracle's exact operation sequence (correctly rounded div/sqrt, no FMA contraction): V, Wo,
// N, Wi, H as BRDF.hlsl:166-169 / Lighting.hlsl:312 write them. T_EXACT = 0.02 bounds the fast path's
// relative error in D by 2*dt/t <= 2*5e-7/0.02 = 5e-5; the slow path runs for < 1 % of pixel-light pairs.
constexpr float T_EXACT = 0.02f;

// dot_u, sqrt_rn_inrange, rcp_rn_prepare / div_rn_inrange, len2_inrange: vq_common.cuh (shared with the PCF kernel)
// v / sqrt(dot(v,v)) with correctly rounded sqrt and divisions (== the oracle's normalize)
__device__ __noinline__ float3 normalize_u_generic(float3 v) {
    const float l = __fsqrt_rn(dot_u(v, v));
    return f3(__fdiv_rn(v.x, l), __fdiv_rn(v.y, l), __fdiv_rn(v.z, l));
}
__device__ __forceinline__ float3 normalize_inrange(float3 v, float d) {
    const RcpRn r = rcp_rn_prepare(sqrt_rn_inrange(d));
    return f3(div_rn_inrange(v.x, r), div_rn_inrange(v.y, r), div_rn_inrange(v.z, r));
}
__device__ __forceinline__ float3 normalize_u(float3 v) {
    const float d = dot_u(v, v);
    if (!len2_inrange(d)) return normalize_u_generic(v);                          // never taken for sane geometry
    return normalize_inrange(v, d);
}
// normalize_u of the result of a normalize_u: that is a unit vector (|v|^2 within a few ulp of 1), or a zero vector or one
// with NaN components (zero or non-finite sources), which both sequences turn into all-NaN: no range check needed
__device__ __forceinline__ float3 renormalize_u(float3 v) { return normalize_inrange(v, dot_u(v, v)); }

constexpr int FWD_THREADS = 128;
constexpr int FWD_TILE = 2 * FWD_THREADS;          // pixels per tile: 256 consecutive pixels of one row (4 KB per G-buffer plane)
constexpr uint32_t FWD_PLANE = FWD_TILE * 16u;     // bytes between the planes of one stage

// posTexel: the pixel's position texel in the shared-memory stage, its raw {N.xyz, roughness} texel one plane further (still
// valid: the stage is released after the pixel is finished). Reading P there rather than taking it as arguments keeps the
// call sites in the light loop short.
__device__ __noinline__ float exact_ndoth(float3 cam, uint32_t posTexel, float3 wiSrc, float wiLenSq) {
    float4 pa, nr;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(pa.x), "=f"(pa.y), "=f"(pa.z), "=f"(pa.w) : "r"(posTexel));
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(nr.x), "=f"(nr.y), "=f"(nr.z), "=f"(nr.w) : "r"(posTexel + FWD_PLANE));
    const float3 Ns = f3(nr.x, nr.y, nr.z);
    const float3 Vv = f3(__fsub_rn(cam.x, pa.x), __fsub_rn(cam.y, pa.y), __fsub_rn(cam.z, pa.z));
    const float3 V = normalize_u(Vv);                 // ForwardLighting.hlsl:285
    const float3 Wo = renormalize_u(V);               // BRDF.hlsl:166
    const float3 N = normalize_u(Ns);                 // BRDF.hlsl:167
    float3 Wi;                                        // Lighting.hlsl:312: Lv / length(Lv)
    if (len2_inrange(wiLenSq)) {
        const RcpRn r = rcp_rn_prepare(sqrt_rn_inrange(wiLenSq));
        Wi = f3(div_rn_inrange(wiSrc.x, r), div_rn_inrange(wiSrc.y, r), div_rn_inrange(wiSrc.z, r));
    } else {
        const float w2 = __fsqrt_rn(wiLenSq);
        Wi = f3(__fdiv_rn(wiSrc.x, w2), __fdiv_rn(wiSrc.y, w2), __fdiv_rn(wiSrc.z, w2));
    }
    const float3 Hs = f3(__fadd_rn(Wo.x, Wi.x), __fadd_rn(Wo.y, Wi.y), __fadd_rn(Wo.z, Wi.z));
    const float3 H = normalize_u(Hs);                 // BRDF.hlsl:168
    return saturate(dot_u(N, H));
}

// ---- exact re-evaluation of N.V ---------------------------------------------------------------------
// `denom = max(4*NdotV*NdotL, 0.0001)` (BRDF.hlsl:186): once the clamp is active the specular term is PROPORTIONAL to NdotV
// (the G1(V) factor no longer cancels) with a gain of 1e4, and NdotV ~ 0 comes out of a cancellation: a 2e-7 difference in
// dot(N, Wo) is a 2e-3 difference in D*G*F/denom. Found by the full-frame parity test at 1920x1080 (4 pixels in 2 M, all with
// |N.V| < 5e-5; tests/diag_fullsize.py). Grazing pixels therefore recompute N.V with the oracle's operation sequence.
constexpr float NV_EXACT = 1e-3f;
__device__ __noinline__ float exact_nv(float3 cam, float3 P, uint32_t nrmTexel) {
    float4 nr;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(nr.x), "=f"(nr.y), "=f"(nr.z), "=f"(nr.w) : "r"(nrmTexel));
    const float3 Vv = f3(__fsub_rn(cam.x, P.x), __fsub_rn(cam.y, P.y), __fsub_rn(cam.z, P.z));
    const float3 Wo = renormalize_u(normalize_u(Vv));               // ForwardLighting.hlsl:285, BRDF.hlsl:166
    const float3 N = normalize_u(f3(nr.x, nr.y, nr.z));             // BRDF.hlsl:167
    return dot_u(N, Wo);
}

// ---- exact re-evaluation of a spot's cosine near its axis ------------------------------------------------------------
// SpotlightIntensity (Lighting.hlsl:57-73) takes acos of dot(normalize(P - Lpos), spotDir). Near the axis dtheta = dcos / sin(theta),
// so the few ulp by which the fast cosine (rsqrt.approx, FMA contraction) differs from the oracle's move theta by up to 5e-4 rad there,
// and the ramp multiplies that by 1/(outer - inner). Where that product can exceed 2^-5 * (cosine difference) / sin(theta), i.e. for
// sin(theta) < 2^-5 * invCone, and theta can lie on the ramp, the kernel recomputes the cosine with the oracle's operation sequence.
// The band [cosLo, cosHi] of cosines that need it is per light (condition_lights); it is empty for cones whose ramp starts beyond
// that angle, as in every scene of bench.py.
__device__ __noinline__ float exact_spot_cos(float3 P, float3 lpos, float3 dir) {
    const float3 d = f3(__fsub_rn(P.x, lpos.x), __fsub_rn(P.y, lpos.y), __fsub_rn(P.z, lpos.z));
    return dot_u(normalize_u(d), dir);
}

// One light for the pixel pair: accumulates BRDF(s, Wi, V) * radiance * NdotL (BRDF.hlsl:163-194, Lighting.hlsl:308-345) in the
// factored form  r = K1*(1-fc) + omF0*(fc*spec) + F0*spec  with  F = F0 + (1-F0)*fc.
//   L, d2 : un-normalised light vector and its squared length (Wi = L/sqrt(d2)),  invD = 1/sqrt(d2)
//   scale : attenuation * brightness * spot intensity (0 when the light is out of range);  col : light colour
// H = normalize(V+Wi) is never formed: |V+Wi|^2 = 2+2c with c = V.Wi, so N.H = (N.V+N.Wi)*rh and
// H.V = (1+c)*rh with rh = rsqrt(2+2c).
// The body is branch-free (a light that does not contribute gets weight 0); only the rare exact-N.H slow path branches.
// TINY: the `denom < EPSILON -> D = 1` escape of NormalDistributionGGX (BRDF.hlsl:77) can only trigger when
// PI*(1+min(a2-1,0))^2 < 1e-12, i.e. roughness < (1e-12/PI)^(1/8) = 0.0274 (in fp32 at N.H = 1: t = (a2-1)+1 is a multiple
// of 2^-24 and the escape holds up to t = 9*2^-24); the caller votes with 2e-12 (roughness < 0.0298) and picks the instantiation per warp, so ordinary
// materials never pay for the selects.
template <bool TINY>
__device__ __forceinline__ void shade_light2(const Px2& s, Acc2& acc, float3 cam, f2 Lx, f2 Ly, f2 Lz, f2 d2, f2 invD,
                                             f2 scale, float3 col) {
    const f2 nl = dot3(s.Nx, s.Ny, s.Nz, Lx, Ly, Lz) * invD;
    const f2 c = dot3(s.Vx, s.Vy, s.Vz, Lx, Ly, Lz) * invD;
    const f2 rh = rsq2(max2(fma2(bc(2.0f), c, bc(2.0f)), 1e-12f));
    f2 NdotH = mulsat2(s.nv + nl, rh);
    const f2 HV = mulsat2(bc(1.0f) + c, rh);              // (1+c)*rh = cos of the half angle: in [0,1] up to rounding
    const f2 omh = bc(1.0f) - HV;
    const f2 omh2 = omh * omh;
    const f2 fc = omh2 * omh2 * omh;                      // Fresnel_Schlick (BRDF.hlsl:132-136)
    f2 t = fma2(NdotH * NdotH, s.a2m1, bc(1.0f));         // NormalDistributionGGX (BRDF.hlsl:65-79)
    const f2 NL = sat2(nl);                               // saturate(N.L) == max(0,N.L) for unit vectors
    const f2 w = mulsat2(s.nsLen, nl) * scale;            // NdotL of the raw s.N (Lighting.hlsl:316) * radiance scale
    if (fminf(t.v.x, t.v.y) < T_EXACT) {                  // < 1 % of pixel-light pairs
        if (t.v.x < T_EXACT && w.v.x > 0.0f) {
            const float nh = exact_ndoth(cam, s.texA, f3(Lx.v.x, Ly.v.x, Lz.v.x), d2.v.x);
            t.v.x = __fadd_rn(__fmul_rn(__fmul_rn(nh, nh), s.a2m1.v.x), 1.0f);
        }
        if (t.v.y < T_EXACT && w.v.y > 0.0f) {
            const float nh = exact_ndoth(cam, s.texB, f3(Lx.v.y, Ly.v.y, Lz.v.y), d2.v.y);
            t.v.y = __fadd_rn(__fmul_rn(__fmul_rn(nh, nh), s.a2m1.v.y), 1.0f);
        }
    }
    f2 dDen = bc(PI) * (t * t);
    const f2 gDen = fma2(NL, s.omk, s.k4);                // Geometry_Smiths_SchlickGGX of L (BRDF.hlsl:82-97)
    const f2 sDen = max2(s.nv4 * NL, 0.0001f);            // max(4*NdotV*NdotL, 0.0001)
    f2 num;
    if (TINY) {                                           // `denom < EPSILON -> D = 1` (BRDF.hlsl:77)
        const bool ta = dDen.v.x < 0.000000000001f, tb = dDen.v.y < 0.000000000001f;
        num = mk(ta ? s.gV.v.x : s.a2gV.v.x, tb ? s.gV.v.y : s.a2gV.v.y) * NL;
        dDen = mk(ta ? 1.0f : dDen.v.x, tb ? 1.0f : dDen.v.y);
    } else {
        num = s.a2gV * NL;
    }
    const f2 spec = num * rcp2(dDen * gDen * sDen);       // D*G/denom with ONE reciprocal (den >= 1e-20)
    const f2 wa = (bc(1.0f) - fc) * w, wc = spec * w, wb = fc * wc;
    const f2 cr = bc(col.x), cg = bc(col.y), cb = bc(col.z);
    acc.ax = fma2(wa, cr, acc.ax); acc.ay = fma2(wa, cg, acc.ay); acc.az = fma2(wa, cb, acc.az);
    acc.bx = fma2(wb, cr, acc.bx); acc.by = fma2(wb, cg, acc.by); acc.bz = fma2(wb, cb, acc.bz);
    acc.cx = fma2(wc, cr, acc.cx); acc.cy = fma2(wc, cg, acc.cy); acc.cz = fma2(wc, cb, acc.cz);
}

// un-normalised light vector of a positional light and its squared length, |L-P|^2 exactly as the oracle's dot():
// (x*x + y*y) + z*z with every operation rounded
struct LightVec2 { f2 x, y, z, d2, invD; };
__device__ __forceinline__ LightVec2 light_vector2(const Px2& s, float3 pos) {
    LightVec2 L;
    // two scalar subtractions write straight into a register pair: cheaper than packing P once more per light
    L.x = mk(pos.x - s.PA.x, pos.x - s.PB.x); L.y = mk(pos.y - s.PA.y, pos.y - s.PB.y); L.z = mk(pos.z - s.PA.z, pos.z - s.PB.z);
    L.d2 = add_rn2(add_rn2(mul_rn2(L.x, L.x), mul_rn2(L.y, L.y)), mul_rn2(L.z, L.z));
    L.invD = rsq2(L.d2 + bc(1e-30f));                     // == rsqrt(d2) for every d2 >= 1e-22; finite at d2 = 0
    return L;
}

// REC_SMEM (psmain_kernel): the pixels' PCF records are not in Px2 but in shared memory, PS_REC_PLANE bytes past each pixel's
// position texel (a fifth plane of the stage, 8 of its 16 bytes used), and are read where a caster needs them: two LDS.64 per
// caster light instead of four registers live across the whole light loop, which the fused kernel's budget has no room for.
constexpr uint32_t PS_REC_PLANE = 4u * FWD_PLANE;
__device__ __forceinline__ uint64_t lds64(uint32_t addr) {       // volatile: read at the point of use, not hoisted out of the loop
    uint64_t r; asm volatile("ld.shared.u64 %0, [%1];" : "=l"(r) : "r"(addr) : "memory"); return r;
}

// SHADOWED: the shadow factor pair {pixel A, pixel B} of caster slot c = 1 - taps/n (Lighting.hlsl:162-164, :207-209), taps from the
// pixels' PCF records; a continuous factor of the light's weight, so one FMA instead of the reference's division
template <bool REC_SMEM>
__device__ __forceinline__ f2 shadow_factor2(const Px2& s, int slot, float invTaps) {
    const uint64_t ra = REC_SMEM ? lds64(s.texA + PS_REC_PLANE) : s.recA, rb = REC_SMEM ? lds64(s.texB + PS_REC_PLANE) : s.recB;
    const float ca = (float)((uint32_t)(ra >> (5 * slot)) & 31u), cb = (float)((uint32_t)(rb >> (5 * slot)) & 31u);
    return fma2(mk(ca, cb), bc(-invTaps), bc(1.0f));
}

// every light of the frame for one pixel pair, in PSMain's order
template <bool TINY, bool SHADOWED, bool REC_SMEM>
__device__ __forceinline__ void shade_all_lights(const Px2& s, Acc2& acc, const FwdParams& P) {
    const float3 cam = P.cam;
    const int numPoint = P.numPoint, numSpot = P.numSpot;
    // ---- point lights, then point casters (Lighting.hlsl:308-322; PSMain :310-313,321-340):
    //      in range <=> d2 < d2Limit (== length(Lw-P) < l.range, exactly) ----
#pragma unroll 1
    for (int i = 0; i < numPoint; ++i) {
        const SPoint l = P.pts[i];                                       // constant bank, warp-uniform index
        const LightVec2 L = light_vector2(s, l.pos);
        const f2 att = (L.invD * L.invD) * bc(l.brightness);               // AttenuationBRDF = 1/D^2
        f2 scale = mk(L.d2.v.x < l.d2Limit ? att.v.x : 0.0f, L.d2.v.y < l.d2Limit ? att.v.y : 0.0f);
        if (SHADOWED) {                                                   // OmnidirectionalShadowTestPCF: 20 taps
            const int c = i - (numPoint - P.shadow.nPointCasters);
            if (c >= 0) scale = scale * shadow_factor2<REC_SMEM>(s, c, 1.0f / 20.0f);
        }
        shade_light2<TINY>(s, acc, cam, L.x, L.y, L.z, L.d2, L.invD, scale, l.color);
    }
    // ---- spot lights, then spot casters (Lighting.hlsl:57-73,323-333) ----
    for (int k = 0; k < numSpot; ++k) {
        const SSpot l = P.spots[k];
        const LightVec2 L = light_vector2(s, l.pos);
        const f2 cosT = dot3(L.x, L.y, L.z, bc(l.dir.x), bc(l.dir.y), bc(l.dir.z)) * L.invD;   // pixel direction = -Wi
        float cq[2] = {-cosT.v.x, -cosT.v.y};
        if (l.cosLo < 1.5f) {                                            // warp-uniform: most cones have no exact band
            if (cq[0] > l.cosLo && cq[0] < l.cosHi) cq[0] = exact_spot_cos(s.PA, l.pos, l.dir);   // near the axis, on the ramp
            if (cq[1] > l.cosLo && cq[1] < l.cosHi) cq[1] = exact_spot_cos(s.PB, l.pos, l.dir);
        }
        float inten[2];
#pragma unroll
        for (int q = 0; q < 2; ++q) {
            // clamped: a cosine that rounds outside [-1, 1] gives the on-axis (or opposite) angle, where the reference's acos is NaN
            const float theta = acosf(fminf(fmaxf(cq[q], -1.0f), 1.0f));
            const float lin = 1.0f - (theta - l.inner) * l.invCone;
            inten[q] = theta > l.outer ? 0.0f : (theta <= l.inner ? 1.0f : lin);
        }
        f2 scale = mk(inten[0], inten[1]) * bc(l.brightness) * (L.invD * L.invD);
        if (SHADOWED) {                                                   // ShadowTestPCF: 5x5 taps
            const int c = k - (numSpot - P.shadow.nSpotCasters);
            if (c >= 0) scale = scale * shadow_factor2<REC_SMEM>(s, P.shadow.nPointCasters + c, 1.0f / 25.0f);
        }
        shade_light2<TINY>(s, acc, cam, L.x, L.y, L.z, L.d2, L.invD, scale, l.color);
    }
    // ---- directional (PSMain :360-377; ShadowingFactor = 1 unless SHADOWED and the light casts) ----
    if (P.dirEnabled) {
        const SDir d = P.dir;
        f2 scale = bc(1.0f);
        if (SHADOWED) { if (P.shadow.dirSlot >= 0) scale = shadow_factor2<REC_SMEM>(s, P.shadow.dirSlot, 1.0f / 25.0f); }
        shade_light2<TINY>(s, acc, cam, bc(d.wi.x), bc(d.wi.y), bc(d.wi.z), bc(1.0f), bc(1.0f), scale, d.radiance);
    }
}

// ---------------------------------------------------------------------------------------------
// TMA (bulk async copy) + mbarrier plumbing, raw PTX for sm_90a
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" :: "r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t done;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    } while (!done);
}
// single-thread waits (the producer on an empty[] barrier): 128 ns of sleep between polls, so as not to steal issue slots
__device__ __forceinline__ void mbar_wait_backoff(uint32_t bar, uint32_t parity) {
    uint32_t done;
    for (;;) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(done) : "r"(bar), "r"(parity) : "memory");
        if (done) break;
        __nanosleep(128);
    }
}
__device__ __forceinline__ uint64_t l2_evict_first_policy() {
    uint64_t pol; asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(pol)); return pol;
}
// one contiguous row segment global -> shared through the TMA unit; completion is counted in bytes on `bar`
__device__ __forceinline__ void tma_load_row(uint32_t dst, const void* src, uint32_t bytes, uint32_t bar, uint64_t pol) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.L2::cache_hint [%0], [%1], %2, [%3], %4;"
                 :: "r"(dst), "l"(src), "r"(bytes), "r"(bar), "l"(pol) : "memory");
}
__device__ __forceinline__ float4 lds128(uint32_t addr) {       // volatile: the load stays where it is written (register diet)
    float4 r;
    asm volatile("ld.shared.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "r"(addr) : "memory");
    return r;
}
__device__ __forceinline__ float lds32(uint32_t addr) {
    float r; asm volatile("ld.shared.f32 %0, [%1];" : "=f"(r) : "r"(addr) : "memory"); return r;
}
__device__ __forceinline__ void st_stream_hint(float4* p, float4 v, uint64_t pol) {
    asm volatile("st.global.L1::no_allocate.L2::cache_hint.v4.f32 [%0], {%1,%2,%3,%4}, %5;"
                 :: "l"(p), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w), "l"(pol) : "memory");
}

// K1 is a persistent kernel: FWD_CTAS_PER_SM CTAs of 128 threads per SM, each walking the tile list
// (tile = 256 consecutive pixels of one row = one 4 KB row segment per G-buffer plane; two pixels per thread) with stride
// gridDim.y over the rows. The G-buffer arrives through a FWD_STAGES-deep TMA pipeline in shared memory: thread 0 issues one bulk
// copy per plane for the tile FWD_AHEAD iterations ahead (full[] mbarriers count the bytes), every thread reads
// ITS texels back with LDS when it needs them and releases the stage (empty[] mbarriers) when its pixels are
// stored. Nothing of the G-buffer is live in registers across the light loop: albedo/metalness/ao, the raw
// normal and the emissive texel are (re-)read from the stage after it. 3 CTAs per SM measured 8 % slower (DESIGN.md §9).
constexpr int FWD_STAGES = 2;          // shared-memory stages
constexpr int FWD_AHEAD = 1;           // tiles requested ahead of the one being shaded (< FWD_STAGES)
constexpr int FWD_CTAS_PER_SM = 4;
static_assert(FWD_AHEAD >= 1 && FWD_AHEAD < FWD_STAGES, "the lookahead must leave at least one stage for the tile being shaded");

// ---- environment taps -----------------------------------------------------------------------------------
// per (mip, face) constants of the specular sampling copy, staged once per CTA: one LDS.128 replaces the shifts, the
// int->float conversions and the mipOffset[] constant-bank indexing of a per-pixel mip
struct FaceRec { uint32_t base; uint32_t P; float halfN; float c0; };     // first record of the face, row stride, N/2, N/2 - 0.5
static_assert(sizeof(FaceRec) == 16, "one LDS.128");

// Every gather allocates in L1: a lane pair reads its two pixels' footprints in consecutive instructions, and neighbouring
// pixels' footprints often share lines (L1::no_allocate measured 3-12 % slower, DESIGN.md §9).
__device__ __forceinline__ float4 ldg128(const float4* p) {
    float4 r;
    asm("ld.global.nc.v4.f32 {%0,%1,%2,%3}, [%4];" : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
    return r;
}
// ---- lane-pair record gathers ----
// A record here is the 32 bytes one bilinear row needs: two adjacent texels of a cube or of the LUT's column pairs. sm_90 has no
// 256-bit load, so a record takes two LDG.128. If every lane read its own record with both, each instruction would touch up to 32
// unrelated lines and every line would be paid for twice. So lanes 2q and 2q+1 read their two records TOGETHER: in one
// instruction both read the even lane's record (the even lane its half .a, the odd lane its half .b), in the other both read the
// odd lane's record (the even lane .b, the odd lane .a). Each instruction touches at most 16 places and each lane still issues
// two loads per record. Every lane then holds the .a half of its own record and the .b half of its partner's, and one shuffle
// per component swaps the .b halves. Every lane of the warp takes part (pixels off a ragged row are aliased, never masked off),
// so the shuffles use the full mask.
__device__ __forceinline__ bool odd_lane() { return (threadIdx.x & 1u) != 0u; }
// record k = texel k and its right neighbour.
// iE, iO: float4 indices of what this lane reads of the even lane's record (.a on an even lane, .b on an odd one) and of the odd
// lane's record (.b on an even lane, .a on an odd one), given this lane's record `mine`
__device__ __forceinline__ void pair_halves(uint32_t mine, uint32_t& iE, uint32_t& iO) {
    const uint32_t other = __shfl_xor_sync(0xffffffffu, mine, 1) + 1u;          // the partner's record, second half
    const bool odd = odd_lane();
    iE = odd ? other : mine; iO = odd ? mine : other;
}
struct HalfPair { float4 e, o; };          // what this lane read of the even lane's record and of the odd lane's record
__device__ __forceinline__ HalfPair ldg_pair(const float4* __restrict__ base, uint32_t iE, uint32_t iO) {
    HalfPair h; h.e = ldg128(base + iE); h.o = ldg128(base + iO); return h;
}
// this lane's own record: its .a half is the one this lane read, its .b half comes from the partner. Only the first N components
// of each half are exchanged (a cube blend reads rgb); the rest are zero.
template <int N>
__device__ __forceinline__ F8 own_record(const HalfPair& h) {
    const bool odd = odd_lane();
    const float he[4] = {h.e.x, h.e.y, h.e.z, h.e.w}, ho[4] = {h.o.x, h.o.y, h.o.z, h.o.w};
    float a[4] = {0.0f, 0.0f, 0.0f, 0.0f}, b[4] = {0.0f, 0.0f, 0.0f, 0.0f};
#pragma unroll
    for (int k = 0; k < N; ++k) {
        a[k] = odd ? ho[k] : he[k];
        b[k] = __shfl_xor_sync(0xffffffffu, odd ? he[k] : ho[k], 1);        // send the partner's .b, receive our own
    }
    F8 rec; rec.a = make_float4(a[0], a[1], a[2], a[3]); rec.b = make_float4(b[0], b[1], b[2], b[3]);
    return rec;
}

struct CubeLoad { HalfPair r0, r1; float fx, fy; };               // rows j0 and j0+1: {t(i0), t(i0+1)} each
// A gather is split into "issue" (addresses + the loads) and "finish" (the exchange and the lerps) so that the loads of several
// gathers are in flight before the first one is consumed.
// maxRec: last position a footprint may start at (clamps the address for NaN/inf directions: no surface => no normal)
// UNIFORM_P: the row stride f.P is the same for every lane (the diffuse cube has one mip), so only the first row's offset is exchanged
template <bool UNIFORM_P>
__device__ __forceinline__ CubeLoad cube_issue(const float4* __restrict__ texels, FaceRec f, uint32_t maxRec, float sx, float sy) {
    const float x = fmaf(sx, f.halfN, f.c0), y = fmaf(-sy, f.halfN, f.c0);       // texel space: (s*0.5+0.5)*N - 0.5
    const float xf = floorf(x), yf = floorf(y);                                  // in [-1, N-1] for every finite direction
    CubeLoad L;
    L.fx = x - xf; L.fy = y - yf;
    const uint32_t off = min(f.base + (uint32_t)((int)yf + 1) * f.P + (uint32_t)((int)xf + 1), maxRec);
    uint32_t e0, o0, e1, o1;
    pair_halves(off, e0, o0);
    L.r0 = ldg_pair(texels, e0, o0);
    if (UNIFORM_P) {                                          // the second row from a row-shifted base: no per-lane adds
        L.r1 = ldg_pair(texels + f.P, e0, o0);
    } else {
        pair_halves(off + f.P, e1, o1);
        L.r1 = ldg_pair(texels, e1, o1);
    }
    return L;
}
// bilinear blend of the footprint as pairs {x,y}, {z,w} of one pixel
__device__ __forceinline__ float3 cube_finish(const CubeLoad& L) {
    const F8 q0 = own_record<3>(L.r0), q1 = own_record<3>(L.r1);
    const f2 fx = bc(L.fx), fy = bc(L.fy);
    const f2 a0 = mk(q0.a.x, q0.a.y), a1 = mk(q0.a.z, q0.a.w), b0 = mk(q0.b.x, q0.b.y), b1 = mk(q0.b.z, q0.b.w);
    const f2 c0 = mk(q1.a.x, q1.a.y), c1 = mk(q1.a.z, q1.a.w), d0 = mk(q1.b.x, q1.b.y), d1 = mk(q1.b.z, q1.b.w);
    const f2 t0 = fma2(fx, b0 - a0, a0), t1 = fma2(fx, b1 - a1, a1);
    const f2 u0 = fma2(fx, d0 - c0, c0), u1 = fma2(fx, d1 - c1, c1);
    const f2 r0 = fma2(fy, u0 - t0, t0), r1 = fma2(fy, u1 - t1, t1);
    return f3(r0.v.x, r0.v.y, r1.v.x);
}
struct LutLoad { HalfPair q; float fx, fy; };
__device__ __forceinline__ LutLoad lut_issue(const LutV& l, float u, float v) {   // bilinear, CLAMP
    const float x = fmaf(u, (float)l.w, -0.5f), y = fmaf(v, (float)l.h, -0.5f);
    const float x0 = floorf(x), y0 = floorf(y);
    LutLoad L;
    L.fx = x - x0; L.fy = y - y0;
    // clamped per axis: the footprint's two texels lie inside the copy for every input, NaN and inf included
    const int cx = min(max((int)x0 + 1, 0), l.w), cy = min(max((int)y0 + 1, 0), l.h);
    uint32_t e, o;
    pair_halves((uint32_t)(cy * (l.w + 2) + cx), e, o);
    L.q = ldg_pair(l.p, e, o);
    return L;
}
__device__ __forceinline__ float2 lut_finish(const LutLoad& L) {    // record = {p00, p01 | p10, p11} as float2 each
    const F8 q = own_record<4>(L.q);
    const f2 fx = bc(L.fx), fy = bc(L.fy);
    const f2 p00 = mk(q.a.x, q.a.y), p01 = mk(q.a.z, q.a.w), p10 = mk(q.b.x, q.b.y), p11 = mk(q.b.z, q.b.w);
    const f2 t = fma2(fx, p10 - p00, p00), u = fma2(fx, p11 - p01, p01);
    return fma2(fy, u - t, t).v;
}

// The environment lookups of one pixel, split into "issue" (the five record gathers: diffuse cube x2, specular cube x2, LUT, with
// their bilinear weights) and "compose" (the blends + the final composition), so that the kernel puts BOTH pixels' gathers in
// flight before it consumes either: a thread then waits for the L2/HBM latency once per pair instead of once per pixel.
//   V/nsnv : normalize(cam-P), saturate(dot(s.N, V))
//   Ns : the surface normal as normalize(Ns)*|Ns| (within an ulp of the raw texel; it only steers the two cube lookups)
struct EnvLoads { CubeLoad D, S; LutLoad L; };
template <bool ROT, bool SPEC>
__device__ __forceinline__ void env_issue(EnvLoads& E, const FwdParams& P, const FaceRec* __restrict__ sFace, float3 V, float nsnv, float3 Ns, float roughness) {
    const float3 Nr = ROT ? f3(Ns.x * P.cosB - Ns.z * P.sinB, Ns.y, Ns.x * P.sinB + Ns.z * P.cosB) : Ns;
    int face; float sx, sy;
    dir_to_face(Nr, face, sx, sy);
    FaceRec fd; fd.P = (uint32_t)P.diff.res + 2u; fd.base = (uint32_t)face * fd.P * fd.P; fd.halfN = P.diffHalfN; fd.c0 = P.diffHalfN - 0.5f;
    E.D = cube_issue<true>(P.diff.p, fd, P.diffMaxRec, sx, sy);
    if (SPEC) {
        const float3 R0 = reflect(-V, Ns);
        const float3 R = ROT ? f3(R0.x * P.cosB - R0.z * P.sinB, R0.y, R0.x * P.sinB + R0.z * P.cosB) : R0;
        dir_to_face(R, face, sx, sy);
        const int mip = min(max((int)(roughness * (float)P.maxLod), 0), P.spec.mips - 1);
        E.S = cube_issue<false>(P.spec.p, sFace[face * 16 + mip], P.specMaxRec, sx, sy);
        E.L = lut_issue(P.lut, nsnv, roughness);                                 // (saturate(dot(s.N, V)), roughness)
    }
}
// the final composition of the pixel (PSMain :290-293, Lighting.hlsl:360-395, BRDF.hlsl:177-207)
//   texel : shared-memory address of the pixel's position texel,  nsnv : saturate(dot(s.N, V))
//   la/lb/lc : the light sums  sum w*col*{(1-fc), fc*spec, spec}
__device__ __forceinline__ float4 compose_values(const FwdParams& P, uint32_t texel, float nsnv, float roughness, float ao,
                                                 float3 la, float3 lb, float3 lc, float3 diffIrr, float3 specCol, float2 sb) {
    // ---- the rest of the G-buffer texel comes out of the stage only now ----
    const float4 am = lds128(texel + 2u * FWD_PLANE);
    const float3 albedo = xyz(am);
    const float metalness = am.w;
    float3 I = albedo * ao;                                  // ForwardLighting.hlsl:290-293 (the ambient factor rides in position.w)
    if (P.hasEmissive) {
        const float4 em = lds128(texel + 3u * FWD_PLANE);
        I += xyz(em) * em.w;
    }
    const float3 F0 = lerp(f3(0.04f), albedo, metalness);    // BRDF.hlsl:177
    {   // K1 = (1-F0)*(1-metal)*albedo/PI (BRDF.hlsl:189-191)
        const float3 omF0 = f3(1.0f) - F0;
        const float3 K1 = omF0 * albedo * ((1.0f - metalness) * (1.0f / PI));
        I.x += fmaf(K1.x, la.x, fmaf(omF0.x, lb.x, F0.x * lc.x));
        I.y += fmaf(K1.y, la.y, fmaf(omF0.y, lb.y, F0.y * lc.y));
        I.z += fmaf(K1.z, la.z, fmaf(omF0.z, lb.z, F0.z * lc.z));
    }
    {   // ---- EnvironmentBRDF (BRDF.hlsl:196-207) on the gathered taps ----
        const float fr = pow5(1.0f - nsnv);                      // FresnelWithRoughness(saturate(dot(s.N, V))), BRDF.hlsl:152-156
        const float omr = 1.0f - roughness;
        const float3 Ks = f3(fmaf(fmaxf(omr, F0.x) - F0.x, fr, F0.x),
                             fmaf(fmaxf(omr, F0.y) - F0.y, fr, F0.y),
                             fmaf(fmaxf(omr, F0.z) - F0.z, fr, F0.z));
        const float om = 1.0f - metalness;
        I.x += (1.0f - Ks.x) * om * (diffIrr.x * albedo.x) + specCol.x * fmaf(Ks.x, sb.x, sb.y);
        I.y += (1.0f - Ks.y) * om * (diffIrr.y * albedo.y) + specCol.y * fmaf(Ks.y, sb.x, sb.y);
        I.z += (1.0f - Ks.z) * om * (diffIrr.z * albedo.z) + specCol.z * fmaf(Ks.z, sb.x, sb.y);
    }
    return make_float4(I.x, I.y, I.z, roughness);                // :380
}
template <bool SPEC>
__device__ __forceinline__ float4 compose_pixel(const FwdParams& P, uint32_t texel, float nsnv, float roughness, float ao,
                                                float3 la, float3 lb, float3 lc, const EnvLoads& E) {
    float3 specCol = f3(0.0f); float2 sb = make_float2(0.0f, 0.0f);
    if (SPEC) { specCol = cube_finish(E.S); sb = lut_finish(E.L); }
    const float3 diffIrr = cube_finish(E.D);
    return compose_values(P, texel, nsnv, roughness, ao, la, lb, lc, diffIrr, specCol, sb);
}

// everything after the light loop for the pixel pair: environment taps, composition, stores (pixel A to (yA, xA), B to (yB, xB))
template <bool MULTI, bool ROT, bool SPEC>
__device__ __forceinline__ void finish_pair(const FwdParams& P, const FaceRec* __restrict__ sFace, const Px2& s, const Acc2& acc, f2 roughness, f2 ao,
                                            int yA, int xA, int yB, int xB, bool validA, bool validB) {
    const f2 nsnv = mulsat2(s.nsLen, s.nv);                      // saturate(dot(s.N, V)) of the raw normal
    const f2 Nrx = s.Nx * s.nsLen, Nry = s.Ny * s.nsLen, Nrz = s.Nz * s.nsLen;
    EnvLoads eA, eB;
    env_issue<ROT, SPEC>(eA, P, sFace, f3(s.Vx.v.x, s.Vy.v.x, s.Vz.v.x), nsnv.v.x, f3(Nrx.v.x, Nry.v.x, Nrz.v.x), roughness.v.x);
    env_issue<ROT, SPEC>(eB, P, sFace, f3(s.Vx.v.y, s.Vy.v.y, s.Vz.v.y), nsnv.v.y, f3(Nrx.v.y, Nry.v.y, Nrz.v.y), roughness.v.y);
    const float4 oA = compose_pixel<SPEC>(P, s.texA, nsnv.v.x, roughness.v.x, ao.v.x, f3(acc.ax.v.x, acc.ay.v.x, acc.az.v.x),
                                          f3(acc.bx.v.x, acc.by.v.x, acc.bz.v.x), f3(acc.cx.v.x, acc.cy.v.x, acc.cz.v.x), eA);
    if (validA) {   // one STG.128 per destination; peer destinations are mapped NVLink addresses (fused compute + gather)
        if (MULTI) { for (int q = 0; q < P.nOut; ++q) st_stream(P.outs[q].row(P.dstRowOffset + yA) + xA, oA); }
        else st_stream_hint(P.outs[0].row(P.dstRowOffset + yA) + xA, oA, l2_evict_first_policy());
    }
    const float4 oB = compose_pixel<SPEC>(P, s.texB, nsnv.v.y, roughness.v.y, ao.v.y, f3(acc.ax.v.y, acc.ay.v.y, acc.az.v.y),
                                          f3(acc.bx.v.y, acc.by.v.y, acc.bz.v.y), f3(acc.cx.v.y, acc.cy.v.y, acc.cz.v.y), eB);
    if (validB) {
        if (MULTI) { for (int q = 0; q < P.nOut; ++q) st_stream(P.outs[q].row(P.dstRowOffset + yB) + xB, oB); }
        else st_stream_hint(P.outs[0].row(P.dstRowOffset + yB) + xB, oB, l2_evict_first_policy());
    }
}

// per-pixel-pair set-up (everything the lights share) and the light loops: fills s, acc, roughness, ao from the staged texels
template <bool SHADOWED, bool REC_SMEM = false>
__device__ __forceinline__ void shade_pair_lights(const FwdParams& P, Px2& s, Acc2& acc, f2& roughness, f2& ao) {
    {
        const float4 pa = lds128(s.texA), pb = lds128(s.texB);
        ao = mk(pa.w, pb.w);
        const float4 na = lds128(s.texA + FWD_PLANE), nb = lds128(s.texB + FWD_PLANE);
        s.PA = xyz(pa); s.PB = xyz(pb);
        const f2 Nsx = mk(na.x, nb.x), Nsy = mk(na.y, nb.y), Nsz = mk(na.z, nb.z);
        roughness = mk(na.w, nb.w);
        const f2 Vx = mk(P.cam.x - pa.x, P.cam.x - pb.x), Vy = mk(P.cam.y - pa.y, P.cam.y - pb.y), Vz = mk(P.cam.z - pa.z, P.cam.z - pb.z);
        const f2 rv = rsq2(dot3(Vx, Vy, Vz, Vx, Vy, Vz));
        s.Vx = Vx * rv; s.Vy = Vy * rv; s.Vz = Vz * rv;          // ForwardLighting.hlsl:285
        const f2 n2 = dot3(Nsx, Nsy, Nsz, Nsx, Nsy, Nsz), rn = rsq2(n2);
        s.Nx = Nsx * rn; s.Ny = Nsy * rn; s.Nz = Nsz * rn;       // BRDF.hlsl:167
        s.nsLen = n2 * rn;
    }
    const f2 a = roughness * roughness;
    const f2 a2 = mul_rn2(a, a);
    s.a2m1 = add_rn2(a2, bc(-1.0f));                             // no contraction: feeds the exact t
    const f2 rp1 = roughness + bc(1.0f);
    const f2 k = (rp1 * rp1) * bc(0.125f);
    s.omk = bc(1.0f) - k; s.k4 = k + bc(0.0001f);
    s.nv = dot3(s.Nx, s.Ny, s.Nz, s.Vx, s.Vy, s.Vz);
    if (fminf(fabsf(s.nv.v.x), fabsf(s.nv.v.y)) < NV_EXACT) {     // grazing view: ~0.1 % of pixels
        if (fabsf(s.nv.v.x) < NV_EXACT) s.nv.v.x = exact_nv(P.cam, s.PA, s.texA + FWD_PLANE);
        if (fabsf(s.nv.v.y) < NV_EXACT) s.nv.v.y = exact_nv(P.cam, s.PB, s.texB + FWD_PLANE);
    }
    const f2 NdotV = sat2(s.nv);
    s.gV = NdotV * rcp2(fma2(NdotV, s.omk, s.k4));
    s.a2gV = a2 * s.gV;
    s.nv4 = NdotV * bc(4.0f);

    acc.ax = acc.ay = acc.az = acc.bx = acc.by = acc.bz = acc.cx = acc.cy = acc.cz = bc(0.0f);
    // can `PI*t*t < 1e-12` ever hold for one of this warp's pixels?  t >= 1 + min(a2-1, 0), rounding is monotone
    const f2 tmin = bc(1.0f) + mk(fminf(s.a2m1.v.x, 0.0f), fminf(s.a2m1.v.y, 0.0f));
    const f2 dmin = bc(PI) * (tmin * tmin);
    if (__any_sync(0xffffffffu, fminf(dmin.v.x, dmin.v.y) < 2e-12f))
        shade_all_lights<true, SHADOWED, REC_SMEM>(s, acc, P);
    else
        shade_all_lights<false, SHADOWED, REC_SMEM>(s, acc, P);
}

// entry i = face*16 + mip of the specular cube's face table, staged once per CTA: the lanes of a warp mostly share the face and
// differ in the mip (per-pixel roughness), so the entries they read are ADJACENT 16-byte words in different banks (mip*8+face
// measured 19 wavefronts per LDS.128, ideal 4)
__device__ __forceinline__ FaceRec face_rec(const FwdParams& P, int i) {
    const int mip = i & 15, face = i >> 4;
    FaceRec f; f.base = 0u; f.P = 3u; f.halfN = 0.5f; f.c0 = 0.0f;
    if (!P.diffuseOnly && mip < P.spec.mips && face < 6) {
        const int N = P.spec.res >> mip;
        f.P = (uint32_t)N + 2u; f.base = P.spec.mipOffset[mip] + (uint32_t)face * f.P * f.P;
        f.halfN = 0.5f * (float)N; f.c0 = f.halfN - 0.5f;
    }
    return f;
}

template <bool MULTI, bool ROT, bool SHADOWED = false>
__global__ void __launch_bounds__(FWD_THREADS, FWD_CTAS_PER_SM) forward_kernel(const __grid_constant__ FwdParams P) {
    extern __shared__ __align__(128) unsigned char smemRaw[];
    const int nPl = P.hasEmissive ? 4 : 3;
    const int tid = threadIdx.x;
    // shared-memory layout: [FWD_STAGES][nPl][FWD_TILE] float4 | full[S], empty[S] mbarriers | FaceRec[8*16]
    const uint32_t stageBytes = (uint32_t)nPl * FWD_PLANE;
    uint64_t* bars = (uint64_t*)(smemRaw + FWD_STAGES * stageBytes);
    FaceRec* sFace = (FaceRec*)(bars + 2 * FWD_STAGES);
    const uint32_t stage0 = smem_u32(smemRaw), bar0 = smem_u32(bars);
    auto fullBar = [&](int st) { return bar0 + 8u * (uint32_t)st; };
    auto emptyBar = [&](int st) { return bar0 + 8u * (uint32_t)(FWD_STAGES + st); };

    // ---- tile schedule: the grid is (tiles per row) x (row groups); a CTA keeps its column and strides rows, so the
    //      only loop state is the row, the stage index and the stage's use count ----
    const int x0 = (int)blockIdx.x * FWD_TILE;
    const int rowStep = (int)gridDim.y;
    const uint32_t tileBytes = (uint32_t)min(FWD_TILE, P.width - x0) * 16u;
    // thread 0: request the tile of row `r` into stage `sIdx`, which has been used `useCount` times before
    auto request = [&](int r, int sIdx, uint32_t useCount) {
        if (r >= P.rows) return;
        if (useCount > 0) mbar_wait_backoff(emptyBar(sIdx), (useCount - 1u) & 1u);   // every thread is done with the previous use
        const uint64_t pol = l2_evict_first_policy();                 // the G-buffer is touched once: first out of L2
        const uint32_t dst = stage0 + (uint32_t)sIdx * stageBytes, bar = fullBar(sIdx);
        const size_t y = (size_t)(P.rowBegin + r);
        mbar_expect_tx(bar, tileBytes * (uint32_t)nPl);
        tma_load_row(dst, P.pos.p + y * P.pos.pitch4 + x0, tileBytes, bar, pol);
        tma_load_row(dst + FWD_PLANE, P.nrm.p + y * P.nrm.pitch4 + x0, tileBytes, bar, pol);
        tma_load_row(dst + 2u * FWD_PLANE, P.alb.p + y * P.alb.pitch4 + x0, tileBytes, bar, pol);
        if (nPl == 4) tma_load_row(dst + 3u * FWD_PLANE, P.emi.p + y * P.emi.pitch4 + x0, tileBytes, bar, pol);
    };
    if (tid == 0) {
        for (int s = 0; s < FWD_STAGES; ++s) { mbar_init(fullBar(s), 1u); mbar_init(emptyBar(s), (uint32_t)FWD_THREADS); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        for (int s = 0; s < FWD_AHEAD; ++s) request((int)blockIdx.y + s * rowStep, s, 0u);   // prologue: FWD_AHEAD tiles in flight
    }

    for (int i = tid; i < 16 * 8; i += FWD_THREADS) sFace[i] = face_rec(P, i);     // the specular cube's face table
    __syncthreads();                                              // face table staged, mbarriers initialised

    int st = 0; uint32_t use = 0;                                 // stage of the current tile, completed uses of that stage
    const int xA = x0 + tid, xB = xA + FWD_THREADS;
    const bool validA = xA < P.width, validB = xB < P.width;      // a ragged last tile: B (or both) fall off the row
    for (int row = (int)blockIdx.y; row < P.rows; row += rowStep) {
        if (tid == 0) {                                           // request the tile FWD_AHEAD iterations ahead
            const int ps = st + FWD_AHEAD;
            if (ps < FWD_STAGES) request(row + FWD_AHEAD * rowStep, ps, use);
            else request(row + FWD_AHEAD * rowStep, ps - FWD_STAGES, use + 1u);
        }
        mbar_wait(fullBar(st), use & 1u);                         // this tile has landed
        const int y = P.rowBegin + row;
        {   // every lane shades (the warp votes below need whole warps): pixels off the end of a ragged row are aliased to the
            // row's last pixel and simply not stored
            Px2 s;
            const uint32_t stageBase = stage0 + (uint32_t)st * stageBytes;
            s.texA = stageBase + (uint32_t)(min(xA, P.width - 1) - x0) * 16u;
            s.texB = stageBase + (uint32_t)(min(xB, P.width - 1) - x0) * 16u;
            f2 roughness, ao;
            Acc2 acc;
            if (SHADOWED) {                                       // the pair's PCF records: two coalesced 8-byte loads, consumed in the light loop
                const uint2* rr = P.shadow.p + (size_t)row * P.shadow.pitch;
                const uint2 ra = __ldg(rr + min(xA, P.width - 1)), rb = __ldg(rr + min(xB, P.width - 1));
                s.recA = ((uint64_t)ra.y << 32) | ra.x; s.recB = ((uint64_t)rb.y << 32) | rb.x;
            }
            shade_pair_lights<SHADOWED>(P, s, acc, roughness, ao);
            if (P.diffuseOnly) finish_pair<MULTI, ROT, false>(P, sFace, s, acc, roughness, ao, y, xA, y, xB, validA, validB);
            else finish_pair<MULTI, ROT, true>(P, sFace, s, acc, roughness, ao, y, xA, y, xB, validA, validB);
        }
        mbar_arrive(emptyBar(st));                               // this thread is done with the stage
        if (++st == FWD_STAGES) { st = 0; ++use; }
    }
    if (MULTI && P.sync.n > 1) {       // fused gather: the last CTA to retire signals the peers and waits for theirs (one kernel = one step)
        __threadfence_system();        // this CTA's peer stores are ordered before its retirement
        __syncthreads();
        if (tid == 0) {
            const uint32_t done = atomicAdd(P.ticket, 1u);
            if (done == gridDim.x * gridDim.y - 1u) {
                *P.ticket = 0u;
                __threadfence_system();
                peer_rendezvous(P.sync);
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------
// PSMain end to end: the surface producer and K1 fused, with the G-buffer in shared memory instead of HBM
// ---------------------------------------------------------------------------------------------
struct PsParams {
    FwdParams F;                       // K1's frame (outs[0..nOut) = the destinations; no G-buffer planes; SHADOWED: F.shadow holds the
                                       // caster counts and dirSlot, its record pointer stays null)
    SurfArgs S;                        // the surface producer's inputs (no G-buffer outputs)
    vqshadow::ShadowLights L;          // SHADOWED only: what the PCF tests read besides the pixel (last, so that the unshadowed
                                       // instantiations read F and S at the same offsets)
};
__device__ __forceinline__ void sts128(uint32_t addr, float4 v) {
    asm volatile("st.shared.v4.f32 [%0], {%1,%2,%3,%4};" :: "r"(addr), "f"(v.x), "f"(v.y), "f"(v.z), "f"(v.w) : "memory");
}
// The PCF record of a staged pixel: exactly what shadow_pcf_kernel computes from the G-buffer texels the stage holds (position =
// plane 0 .xyz, the normal-mapped normal = plane 1 .xyz). Every lane of the warp must call it (pcf_record votes across the warp).
__device__ __forceinline__ uint64_t staged_pcf_record(const vqshadow::ShadowLights& L, uint32_t texel) {
    const float4 p = lds128(texel), n = lds128(texel + FWD_PLANE);
    vqshadow::Px4 p4, n4;
    p4.x = p.x; p4.y = p.y; p4.z = p.z; p4.w = p.w;
    n4.x = n.x; n4.y = n.y; n4.z = n.z; n4.w = n.w;
    return vqshadow::pcf_record(L, p4, n4);
}

// A persistent CTA walks tiles of 2 rows x FWD_THREADS columns (rows aligned to absolute even rows, as the surface producer's
// quads are), keeping its column and striding the row pairs by gridDim.y. Per tile, two phases separated by CTA barriers:
//   producer: warp w runs the surface producer's per-pixel code for the 16x2 strips w and w+4 of the tile and writes the four
//             G-buffer texels of each pixel into a shared-memory stage with K1's layout (plane k of stage pixel p at
//             k*FWD_PLANE + 16p; row 0 of the tile is stage pixels 0..127, row 1 is 128..255), plus a flag saying whether the
//             pixel was produced (inside the image and the row range, not discarded by the alpha mask);
//   shading:  thread t shades the pixel pair (row 0, column t), (row 1, column t) with K1's code on the stage and stores the
//             pixels that were produced. The lane-pair gathers pair neighbouring columns of one row, as in K1.
//             SHADOWED: first the PCF records of both pixels from the stage (all 128 threads: a warp is 32 consecutive columns of
//             one row, as in shadow_pcf_kernel), then the shadowed light loop on them.
// The phases stay sequential: a warp-specialised K1 measured slower (DESIGN.md §4).
// MULTI: every produced pixel goes to row dstRowOffset + y of each of the F.nOut destinations, and with a VqPeerSignal the last CTA
// to retire runs the cross-rank rendezvous, as in forward_kernel.
template <bool ROT, bool SHADOWED, bool MULTI = false>
__global__ void __launch_bounds__(FWD_THREADS, FWD_CTAS_PER_SM) psmain_kernel(const __grid_constant__ PsParams Q) {
    const FwdParams& P = Q.F;
    const SurfArgs& A = Q.S;
    __shared__ __align__(128) float4 sStage[(SHADOWED ? 5 : 4) * FWD_TILE];       // SHADOWED: + the PCF records (PS_REC_PLANE)
    __shared__ FaceRec sFace[16 * 8];
    __shared__ uint8_t sProduced[FWD_TILE];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const uint32_t stage0 = smem_u32(sStage);
    // the stage starts zeroed: a pixel that is not produced is still shaded (whole warps take part in the votes and exchanges)
    // but never stored, and it reads defined values
    for (int i = tid; i < 4 * FWD_TILE; i += FWD_THREADS) sStage[i] = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
    for (int i = tid; i < 16 * 8; i += FWD_THREADS) sFace[i] = face_rec(P, i);
    const int x0 = (int)blockIdx.x * FWD_THREADS;
    const int xA = x0 + tid;
    const bool inRow = xA < P.width;
    const int pairs = (A.rowEnd - A.tileY0 + 1) / 2;
    for (int t = (int)blockIdx.y; t < pairs; t += (int)gridDim.y) {
        const int y0 = A.tileY0 + 2 * t;
        __syncthreads();                                          // the previous tile's shading is done with the stage
#pragma unroll 1
        for (int k = 0; k < 2; ++k) {
            const int c = (warp + 4 * k) * 16 + (lane & 15), r = lane >> 4;
            const uint32_t px = (uint32_t)(r * FWD_THREADS + c);
            bool produced = false;
            surface_quad_pixel(A, x0 + c, y0 + r, lane, l2_policy_evict_first(), [&](float4 posAo, float4 nrmRough, float4 albMetal, float4 emi) {
                const uint32_t texel = stage0 + px * 16u;
                sts128(texel, posAo);
                sts128(texel + FWD_PLANE, nrmRough);
                sts128(texel + 2u * FWD_PLANE, albMetal);
                sts128(texel + 3u * FWD_PLANE, emi);
                produced = true;
            });
            sProduced[px] = produced ? 1 : 0;
        }
        __syncthreads();                                          // the tile is staged
        Px2 s;
        s.texA = stage0 + (uint32_t)(min(xA, P.width - 1) - x0) * 16u;   // a ragged tile: columns off the row alias its last pixel
        s.texB = s.texA + FWD_THREADS * 16u;
        f2 roughness, ao;
        Acc2 acc;
        if (SHADOWED) {                                           // one copy of the PCF code, run for pixel A then pixel B
            // lanes off a ragged row alias its last pixel and store the same record there (the axis path gives the general
            // count, so the warp a lane sits in does not change it); a record is only read by the threads that stored it
#pragma unroll 1
            for (int k = 0; k < 2; ++k) {
                const uint32_t texel = k ? s.texB : s.texA;
                const uint64_t rec = staged_pcf_record(Q.L, texel);
                asm volatile("st.shared.u64 [%0], %1;" :: "r"(texel + PS_REC_PLANE), "l"(rec) : "memory");
            }
        }
        shade_pair_lights<SHADOWED, SHADOWED>(P, s, acc, roughness, ao);
        const bool validA = inRow && sProduced[tid] != 0, validB = inRow && sProduced[FWD_THREADS + tid] != 0;
        if (P.diffuseOnly) finish_pair<MULTI, ROT, false>(P, sFace, s, acc, roughness, ao, y0, xA, y0 + 1, xA, validA, validB);
        else finish_pair<MULTI, ROT, true>(P, sFace, s, acc, roughness, ao, y0, xA, y0 + 1, xA, validA, validB);
    }
    // forward_kernel's retirement block, copied: as a shared helper it changed the register allocation of every forward_kernel
    if (MULTI && P.sync.n > 1) {       // fused gather: the last CTA to retire signals the peers and waits for theirs (one kernel = one step)
        __threadfence_system();        // this CTA's peer stores are ordered before its retirement
        __syncthreads();
        if (tid == 0) {
            const uint32_t done = atomicAdd(P.ticket, 1u);
            if (done == gridDim.x * gridDim.y - 1u) {
                *P.ticket = 0u;
                __threadfence_system();
                peer_rendezvous(P.sync);
            }
        }
    }
}

uint64_t padded_texels(int res, int mips) {
    uint64_t n = 0;
    for (int m = 0; m < mips; ++m) { const uint64_t p = (uint64_t)(res >> m) + 2; n += 6 * p * p; }
    return n;
}
// bytes of a sampling copy: the texels plus one mip-0 row and a texel of slack, so that a footprint whose first position was
// clamped to the last position (a non-finite direction: pixels without a surface carry a zero normal) still reads inside the
// allocation
size_t padded_bytes(int res, int mips) { return (size_t)(padded_texels(res, mips) + (uint64_t)res + 3u) * 16u; }
bool cube_desc_ok(const VqCubemap& c) {
    return c.ptr && c.res >= 1 && c.mips >= 1 && c.mips <= 16 && (c.res >> (c.mips - 1)) >= 1 &&
           padded_texels(c.res, c.mips) < (1ull << 30);
}
// builds the sampling copy of `c` into `dst` (padded_texels() texels of 16 bytes) on `stream`
int pad_cube(const VqCubemap& c, float4* dst, cudaStream_t stream) {
    const uint32_t total = (uint32_t)padded_texels(c.res, c.mips);
    unsigned blocks = (total + 255u) / 256u;
    if (blocks > 148u * 16u) blocks = 148u * 16u;
    cube_pad_kernel<<<blocks, 256, 0, stream>>>((const float4*)c.ptr, dst, c.res, c.mips, total);
    return vq_check_launch("cube_pad");
}
void fill_cube_view(const VqCubemap& c, const float4* padded, CubeV& v) {
    v.p = padded; v.res = c.res; v.mips = c.mips;
    uint32_t off = 0;
    for (int m = 0; m < 16; ++m) {
        v.mipOffset[m] = m < c.mips ? off : 0u;
        if (m < c.mips) { const uint32_t p = (uint32_t)(c.res >> m) + 2u; off += 6u * p * p; }
    }
}
bool same_cube(const VqCubemap& a, const VqCubemap& b) { return a.ptr == b.ptr && a.res == b.res && a.mips == b.mips; }
bool same_image(const VqImage& a, const VqImage& b) { return a.ptr == b.ptr && a.width == b.width && a.height == b.height && a.pitch_bytes == b.pitch_bytes; }
// no slack needed: lut_issue clamps both coordinates, so no footprint can start past texel (W, H) of the copy
size_t lut_pair_bytes(const VqImage& lut) { return (size_t)(lut.width + 2) * (size_t)(lut.height + 1) * 16; }
// builds the column-pair copy of the BRDF LUT into `dst` on `stream`
int pair_lut(const VqImage& lut, float4* dst, cudaStream_t stream) {
    const uint32_t total = (uint32_t)(lut.width + 2) * (uint32_t)(lut.height + 1);
    unsigned blocks = (total + 255u) / 256u;
    if (blocks > 148u * 16u) blocks = 148u * 16u;
    lut_pair_kernel<<<blocks, 256, 0, stream>>>((const float2*)lut.ptr, (int)(lut.pitch_bytes / 8), lut.width, lut.height, dst);
    return vq_check_launch("lut_pair");
}

// K1's sampling copies of one environment share ONE buffer: diffuse | specular | LUT column pairs, each part 256-byte aligned
// (the specular cube and the LUT only when asked). Points the views into the buffer at `base` and returns its size.
size_t sampling_views(const VqEnvironmentMaps& env, bool withSpec, bool withLut, uintptr_t base, CubeV& diff, CubeV& spec, LutV& lut) {
    auto up = [](size_t b) { return (b + 255) & ~(size_t)255; };
    const size_t bD = up(padded_bytes(env.irradiance_diffuse.res, env.irradiance_diffuse.mips));
    const size_t bS = withSpec ? up(padded_bytes(env.irradiance_specular.res, env.irradiance_specular.mips)) : 0;
    fill_cube_view(env.irradiance_diffuse, (const float4*)base, diff);
    if (withSpec) fill_cube_view(env.irradiance_specular, (const float4*)(base + bD), spec);
    if (withLut) lut.p = (const float4*)(base + bD + bS);
    return bD + bS + (withLut ? up(lut_pair_bytes(env.brdf_lut)) : 0);
}
// grows `s` to that layout, builds the copies of `env` into it on `stream` and points the views at them
int build_sampling_copies(VqScratch& s, const VqEnvironmentMaps& env, bool withSpec, bool withLut, cudaStream_t stream,
                          CubeV& diff, CubeV& spec, LutV& lut) {
    int rc = vq_scratch_reserve(s, sampling_views(env, withSpec, withLut, 0, diff, spec, lut), "sampling copies"); if (rc) return rc;
    sampling_views(env, withSpec, withLut, (uintptr_t)s.p, diff, spec, lut);
    rc = pad_cube(env.irradiance_diffuse, (float4*)diff.p, stream);
    if (!rc && withSpec) rc = pad_cube(env.irradiance_specular, (float4*)spec.p, stream);
    if (!rc && withLut) rc = pair_lut(env.brdf_lut, (float4*)lut.p, stream);
    return rc;
}

}  // namespace

// Scene::GatherLightData's arrays -> what the kernel reads per light, on the host in IEEE fp32 (every operation rounded on its
// own: the same bits the oracle's normalize() / length() produce):
//   point: smallest d2 with sqrt_rn(d2) >= range, so that (d2 < limit) == (sqrt_rn(d2) < range) exactly  (Lighting.hlsl:308-322)
//   spot : normalize(l.spotDir) (Lighting.hlsl:60), 1/(outer - inner);  directional: Wi = normalize(-dir), radiance = color*brightness
static void normalize_host(const float v[3], float out[3]) {
    volatile float xx = v[0] * v[0], yy = v[1] * v[1], zz = v[2] * v[2];
    volatile float s = xx + yy; s = s + zz;
    const float l = sqrtf(s);
    out[0] = v[0] / l; out[1] = v[1] / l; out[2] = v[2] / l;
}
static void condition_lights(const VqSceneLighting& L, FwdParams& P) {
    const int nP = L.numPointLights, nPC = L.numPointCasters, nS = L.numSpotLights, nSC = L.numSpotCasters;
    P.numPoint = nP + nPC; P.numSpot = nS + nSC;
    for (int i = 0; i < P.numPoint; ++i) {
        const VqPointLight& l = i < nP ? L.point_lights[i] : L.point_casters[i - nP];
        SPoint& s = P.pts[i];
        s.pos = make_float3(l.position.x, l.position.y, l.position.z);
        s.color = make_float3(l.color.x, l.color.y, l.color.z);
        s.brightness = l.brightness;
        volatile float lim = l.range * l.range;
        if (!(l.range > 0.0f)) lim = 0.0f;
        else {
            auto bits = [](float f) { uint32_t u; memcpy(&u, &f, 4); return u; };
            auto flt = [](uint32_t u) { float f; memcpy(&f, &u, 4); return f; };
            while (sqrtf(lim) >= l.range && lim > 0.0f) lim = flt(bits(lim) - 1u);
            while (sqrtf(lim) < l.range) lim = flt(bits(lim) + 1u);
        }
        s.d2Limit = lim;
    }
    for (int i = 0; i < P.numSpot; ++i) {
        const VqSpotLight& l = i < nS ? L.spot_lights[i] : L.spot_casters[i - nS];
        SSpot& s = P.spots[i];
        s.pos = make_float3(l.position.x, l.position.y, l.position.z);
        s.color = make_float3(l.color.x, l.color.y, l.color.z);
        s.brightness = l.brightness;
        const float d[3] = {l.spotDir.x, l.spotDir.y, l.spotDir.z};
        float n[3]; normalize_host(d, n);
        s.dir = make_float3(n[0], n[1], n[2]);
        s.outer = l.outerConeAngle; s.inner = l.innerConeAngle;
        s.invCone = 1.0f / (l.outerConeAngle - l.innerConeAngle);
        // the band of cosines recomputed exactly (exact_spot_cos): theta in [inner, min(asin(2^-5 * invCone), outer)], widened by
        // 2e-6 on both sides (more than the fast cosine's error); empty (cosLo = 2) when the ramp is unreachable or starts beyond it
        const double ic = 1.0 / ((double)l.outerConeAngle - (double)l.innerConeAngle);
        s.cosLo = 2.0f; s.cosHi = 2.0f;
        if (ic > 0.0) {
            const double thB = ic * 0x1p-5 >= 1.0 ? 1.5707963267948966 : asin(ic * 0x1p-5);
            const double thX = fmin(thB, (double)l.outerConeAngle);
            if (thX >= (double)l.innerConeAngle) {
                s.cosLo = (float)(cos(thX) - 2e-6);
                s.cosHi = l.innerConeAngle > 0.0f ? (float)(cos((double)l.innerConeAngle) + 2e-6) : 2.0f;
            }
        }
    }
    P.dirEnabled = L.directional.enabled != 0;
    if (P.dirEnabled) {
        const float d[3] = {-L.directional.lightDirection.x, -L.directional.lightDirection.y, -L.directional.lightDirection.z};
        float n[3]; normalize_host(d, n);
        P.dir.wi = make_float3(n[0], n[1], n[2]);
        P.dir.radiance = make_float3(L.directional.color.x * L.directional.brightness, L.directional.color.y * L.directional.brightness,
                                     L.directional.color.z * L.directional.brightness);
    }
}

static bool light_counts_ok(const VqSceneLighting& L) {
    return L.numPointLights >= 0 && L.numPointLights <= VQ_NUM_LIGHTS_POINT && L.numSpotLights >= 0 && L.numSpotLights <= VQ_NUM_LIGHTS_SPOT &&
           L.numPointCasters >= 0 && L.numPointCasters <= VQ_NUM_SHADOWING_LIGHTS_POINT &&
           L.numSpotCasters >= 0 && L.numSpotCasters <= VQ_NUM_SHADOWING_LIGHTS_SPOT;
}

// What K1 reads of the frame but the surface: lights, camera, HDRI yaw, environment (its sampling copies: the registered ones
// when they match, else built now on `stream`). Call with the context's scratch locked.
static int frame_params(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqEnvironmentMaps* env,
                        cudaStream_t stream, FwdParams& P) {
    condition_lights(pf->Lights, P);
    P.cam = make_float3(pv->CameraPosition.x, pv->CameraPosition.y, pv->CameraPosition.z);
    P.cosB = cosf(-pf->fHDRIOffsetInRadians);
    P.sinB = sinf(-pf->fHDRIOffsetInRadians);
    P.maxLod = (int)pv->MaxEnvMapLODLevels;
    P.diffuseOnly = pv->EnvironmentMapDiffuseOnlyIllumination != 0;
    VQ_REQUIRE(cube_desc_ok(env->irradiance_diffuse), "bad cubemap descriptor (irradiance_diffuse)");
    if (!P.diffuseOnly) {
        VQ_REQUIRE(cube_desc_ok(env->irradiance_specular), "bad cubemap descriptor (irradiance_specular)");
        VQ_REQUIRE(vq_image_ok(env->brdf_lut, 8), "bad BRDF LUT descriptor");
        VQ_REQUIRE(env->brdf_lut.width <= 8192 && env->brdf_lut.height <= 8192, "BRDF LUT larger than 8192^2");
        P.lut.w = env->brdf_lut.width; P.lut.h = env->brdf_lut.height;
    }
    // bordered sampling copies: from the prepared environment when it matches (the descriptors checked above are non-null, so
    // a match also means the registration holds every part this call reads), else built now on this stream
    const bool full = !P.diffuseOnly;
    const bool prepared = ctx->env_valid && same_cube(ctx->env_key.irradiance_diffuse, env->irradiance_diffuse) &&
                          (P.diffuseOnly || (same_cube(ctx->env_key.irradiance_specular, env->irradiance_specular) &&
                                             same_image(ctx->env_key.brdf_lut, env->brdf_lut)));
    if (prepared) sampling_views(*env, full, full, (uintptr_t)ctx->env_prepared.p, P.diff, P.spec, P.lut);
    else {
        const int rc = build_sampling_copies(ctx->env_per_call, *env, full, full, stream, P.diff, P.spec, P.lut); if (rc) return rc;
    }
    P.diffHalfN = 0.5f * (float)env->irradiance_diffuse.res;
    P.diffMaxRec = (uint32_t)padded_texels(env->irradiance_diffuse.res, 1) - 1u;      // K1 samples mip 0 of the diffuse cube only
    P.specMaxRec = P.diffuseOnly ? 0u : (uint32_t)padded_texels(env->irradiance_specular.res, env->irradiance_specular.mips) - 1u;
    return VQ_OK;
}

// The forward passes' band destinations over a W x H source (G-buffer or attribute planes): frames as wide as the source that
// hold dst_row_offset + H rows, between the shared band checks. Fills `sync` from `sig`.
static int forward_band_check(const VqContext* ctx, const VqImage* outs, int n_outs, int W, int H, int dst_row_offset, int row_begin,
                              int row_end, const VqPeerSignal* sig, PeerSync& sync) {
    int rc = vq_band_list(outs, n_outs); if (rc) return rc;
    for (int k = 0; k < n_outs; ++k)
        VQ_REQUIRE(vq_image_ok(outs[k]) && outs[k].width == W && outs[k].height >= dst_row_offset + H,
                   "every destination must be as wide as the G-buffer and hold dst_row_offset + height rows");
    return vq_band_check(ctx, n_outs, dst_row_offset, H, row_begin, row_end, sig, sync);
}

int vq_forward_check(const VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqGBuffer* gb,
                     const VqEnvironmentMaps* env, const VqImage* outs, int n_outs, int dst_row_offset, int row_begin, int row_end,
                     const VqPeerSignal* sig, PeerSync& sync) {
    VQ_REQUIRE(pf && pv && gb && env && outs, "null parameter block");
    VQ_REQUIRE(vq_image_ok(gb->position_ao) && vq_image_ok(gb->normal_roughness) && vq_image_ok(gb->albedo_metalness), "bad image descriptor");
    const int W = gb->position_ao.width, H = gb->position_ao.height;
    VQ_REQUIRE(gb->normal_roughness.width == W && gb->albedo_metalness.width == W &&
               gb->normal_roughness.height == H && gb->albedo_metalness.height == H, "G-buffer planes must have the same size");
    if (gb->emissive.ptr)
        VQ_REQUIRE(vq_image_ok(gb->emissive) && gb->emissive.width == W && gb->emissive.height == H, "bad emissive plane");
    return forward_band_check(ctx, outs, n_outs, W, H, dst_row_offset, row_begin, row_end, sig, sync);
}

int vq_forward_launch_multi(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                            const VqGBuffer* gb, const VqEnvironmentMaps* env, const VqImage* outs, int n_outs,
                            int dst_row_offset, int row_begin, int row_end, const PeerSync& sync, cudaStream_t stream,
                            const ShadowRecV* shadow) {
    const int W = gb->position_ao.width;
    const VqSceneLighting& L = pf->Lights;
    VQ_REQUIRE(light_counts_ok(L), "light counts exceed the cbuffer arrays");
    if (row_begin == row_end) return VQ_OK;
    VqScratchLock lock(ctx);           // the registered environment and the per-call sampling copies are the context's

    FwdParams P;
    memset(&P, 0, sizeof(P));
    P.pos = make_view(gb->position_ao); P.nrm = make_view(gb->normal_roughness); P.alb = make_view(gb->albedo_metalness);
    for (int k = 0; k < n_outs; ++k) P.outs[k] = make_view(outs[k]);
    P.nOut = n_outs; P.dstRowOffset = dst_row_offset;
    P.hasEmissive = gb->emissive.ptr != nullptr;
    if (P.hasEmissive) P.emi = make_view(gb->emissive);
    int rc = frame_params(ctx, pf, pv, env, stream, P); if (rc) return rc;
    P.rowBegin = row_begin; P.rows = row_end - row_begin; P.width = W;
    const bool shadowed = shadow && shadow->p;
    if (shadowed) {
        VQ_REQUIRE(shadow->nPointCasters == L.numPointCasters && shadow->nSpotCasters == L.numSpotCasters && shadow->pitch >= W,
                   "PCF records do not match the frame's caster lists");
        P.shadow = *shadow;
    }
    P.sync = sync;

    // persistent grid: x = the row's 256-pixel tiles, y = row groups striding the rows
    const unsigned gx = (unsigned)((W + FWD_TILE - 1) / FWD_TILE);
    unsigned gy = (unsigned)(ctx->sm_count * FWD_CTAS_PER_SM) / gx;
    if (gy < 1) gy = 1;
    if (gy > (unsigned)P.rows) gy = (unsigned)P.rows;
    VQ_REQUIRE(gy <= 65535u, "frame too tall for the launch grid");
    const int nPl = P.hasEmissive ? 4 : 3;
    const size_t smem = (size_t)FWD_STAGES * nPl * FWD_PLANE + 2 * FWD_STAGES * sizeof(uint64_t) + 16 * 8 * sizeof(FaceRec);
    const bool rot = P.sinB != 0.0f || P.cosB != 1.0f;            // yaw offset 0 is the common case: compiled out
    static std::atomic<bool> attrSet{false};                      // process-wide and idempotent: every instantiation, once
    if (!attrSet.load(std::memory_order_acquire)) {
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<true, false>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<false, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<false, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<true, false, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        VQ_CUDA_OK(cudaFuncSetAttribute(forward_kernel<true, true, true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 96 * 1024));
        attrSet.store(true, std::memory_order_release);
    }
    auto launch = [&](auto kernel) -> int {
        cudaLaunchConfig_t cfg;
        memset(&cfg, 0, sizeof(cfg));
        cfg.gridDim = dim3(gx, gy); cfg.blockDim = dim3(FWD_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = stream;
        VQ_CUDA_OK(cudaLaunchKernelEx(&cfg, kernel, P));
        return VQ_OK;
    };
    VQ_REQUIRE(smem <= 96 * 1024, "stage layout exceeds the shared-memory budget");
    P.ticket = vq_band_ticket(ctx, P.sync);
    if (shadowed && n_outs > 1) rc = rot ? launch(forward_kernel<true, true, true>) : launch(forward_kernel<true, false, true>);
    else if (shadowed) rc = rot ? launch(forward_kernel<false, true, true>) : launch(forward_kernel<false, false, true>);
    else if (n_outs > 1) rc = rot ? launch(forward_kernel<true, true>) : launch(forward_kernel<true, false>);
    else rc = rot ? launch(forward_kernel<false, true>) : launch(forward_kernel<false, false>);
    if (rc) return rc;
    return vq_check_launch("forward_lighting");
}

// the G-buffer pass without shadow maps: checked, then launched
static int forward_call(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqGBuffer* gb,
                        const VqEnvironmentMaps* env, const VqImage* outs, int n_outs, int dst_row_offset, int row_begin, int row_end,
                        const VqPeerSignal* sig, cudaStream_t stream) {
    PeerSync sync;
    const int rc = vq_forward_check(ctx, pf, pv, gb, env, outs, n_outs, dst_row_offset, row_begin, row_end, sig, sync); if (rc) return rc;
    return vq_forward_launch_multi(ctx, pf, pv, gb, env, outs, n_outs, dst_row_offset, row_begin, row_end, sync, stream);
}

int vq_forward_launch(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                      const VqGBuffer* gb, const VqEnvironmentMaps* env, VqImage out,
                      int row_begin, int row_end, cudaStream_t stream) {
    VQ_REQUIRE(gb && vq_image_ok(out) && out.height == gb->position_ao.height, "G-buffer planes and output must have the same size");
    return forward_call(ctx, pf, pv, gb, env, &out, 1, 0, row_begin, row_end, nullptr, stream);
}

extern "C" int vq_forward_lighting(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                   const VqGBuffer* gb, const VqEnvironmentMaps* env, VqImage out,
                                   int row_begin, int row_end, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("RenderSceneColor");
    return vq_forward_launch(ctx, pf, pv, gb, env, out, row_begin, row_end, (cudaStream_t)stream);
}

extern "C" int vq_forward_lighting_multi(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                         const VqGBuffer* gb, const VqEnvironmentMaps* env, const VqImage* outs, int n_outs,
                                         int dst_row_offset, int row_begin, int row_end, void* stream) {
    return vq_forward_lighting_multi_signal(ctx, pf, pv, gb, env, outs, n_outs, dst_row_offset, row_begin, row_end, nullptr, stream);
}

// the same, with the cross-rank rendezvous run by the kernel's last CTA (VqPeerSignal): one kernel = shade + gather + barrier
extern "C" int vq_forward_lighting_multi_signal(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                                const VqGBuffer* gb, const VqEnvironmentMaps* env, const VqImage* outs, int n_outs,
                                                int dst_row_offset, int row_begin, int row_end, const VqPeerSignal* signal, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("RenderSceneColor");
    return forward_call(ctx, pf, pv, gb, env, outs, n_outs, dst_row_offset, row_begin, row_end, signal, (cudaStream_t)stream);
}

// PSMain from interpolants and materials in one launch (psmain_kernel): what vq_gbuffer_from_materials with an emissive plane
// followed by vq_forward_lighting (sm == nullptr) or vq_forward_lighting_shadowed computes, without the G-buffer. `multi`: the
// multi-destination call (outs[0..n_outs), rows offset by dst_row_offset, optional rendezvous); otherwise outs[0] is the one output,
// of the attribute planes' size. The arguments are checked before the device is touched.
static int psmain_launch(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv, const VqSurfaceInputs* in,
                         const VqMaterialTable* table, int alpha_mask, const VqEnvironmentMaps* env, const VqShadowMaps* sm,
                         bool multi, const VqImage* outs, int n_outs, int dst_row_offset, int row_begin, int row_end,
                         const VqPeerSignal* sig, void* stream) {
    VQ_REQUIRE(pf && pv && env && in && outs, "null argument");
    const int W = in->position_u.width, H = in->position_u.height;
    static_assert(sizeof(PsParams) <= 32764, "kernel parameter space");
    PsParams Q;
    memset(&Q, 0, sizeof(Q));
    int rc;
    if (multi) {
        rc = forward_band_check(ctx, outs, n_outs, W, H, dst_row_offset, row_begin, row_end, sig, Q.F.sync); if (rc) return rc;
        // the surface producer's quads sit on even rows of the attribute planes: an even offset keeps them on even rows of the frame
        VQ_REQUIRE((dst_row_offset & 1) == 0, "dst_row_offset must be even (quads are aligned to even rows)");
    } else {
        VQ_REQUIRE(vq_image_ok(outs[0]) && outs[0].width == W && outs[0].height == H, "the output must have the size of the attribute planes");
    }
    bool shadowed = false;                                        // does any PCF test run?
    if (sm) {
        rc = vq_shadow_maps_check(pf->Lights, *sm); if (rc) return rc;
        shadowed = vq_shadow_slots(pf->Lights, *sm, Q.F.shadow);  // no test runs: every factor is 1, the unshadowed kernel
        if (shadowed) vqshadow::fill_shadow_lights(Q.L, *pf, *pv, *sm);
    }
    rc = surface_inputs(in, table, pf->fAmbientLightingFactor, alpha_mask, row_begin, row_end, Q.S); if (rc) return rc;
    VQ_REQUIRE(light_counts_ok(pf->Lights), "light counts exceed the cbuffer arrays");
    rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("RenderSceneColor");
    if (row_begin == row_end) return VQ_OK;
    VqScratchLock lock(ctx);           // the registered environment and the per-call sampling copies are the context's
    FwdParams& P = Q.F;
    rc = frame_params(ctx, pf, pv, env, (cudaStream_t)stream, P); if (rc) return rc;
    P.hasEmissive = 1;
    for (int k = 0; k < n_outs; ++k) P.outs[k] = make_view(outs[k]);
    P.nOut = n_outs; P.dstRowOffset = dst_row_offset;
    P.ticket = vq_band_ticket(ctx, P.sync);
    P.rowBegin = row_begin; P.rows = row_end - row_begin; P.width = W;
    // persistent grid: x = the row's 128-column tiles, y = groups striding the row pairs
    const unsigned gx = (unsigned)((W + FWD_THREADS - 1) / FWD_THREADS);
    const unsigned pairs = (unsigned)((row_end - Q.S.tileY0 + 1) / 2);
    unsigned gy = (unsigned)(ctx->sm_count * FWD_CTAS_PER_SM) / gx;
    if (gy < 1) gy = 1;
    if (gy > pairs) gy = pairs;
    const bool rot = P.sinB != 0.0f || P.cosB != 1.0f;
    void (*kernel)(PsParams);          // one destination: the single-destination kernels, as vq_forward_launch_multi picks them
    if (shadowed) kernel = n_outs > 1 ? (rot ? psmain_kernel<true, true, true> : psmain_kernel<false, true, true>)
                                      : (rot ? psmain_kernel<true, true> : psmain_kernel<false, true>);
    else kernel = n_outs > 1 ? (rot ? psmain_kernel<true, false, true> : psmain_kernel<false, false, true>)
                             : (rot ? psmain_kernel<true, false> : psmain_kernel<false, false>);
    kernel<<<dim3(gx, gy), FWD_THREADS, 0, (cudaStream_t)stream>>>(Q);
    return vq_check_launch(multi ? "forward_lighting_from_materials_multi"
                                 : sm ? "forward_lighting_shadowed_from_materials" : "forward_lighting_from_materials");
}

extern "C" int vq_forward_lighting_from_materials(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                                  const VqSurfaceInputs* in, const VqMaterialTable* table, int alpha_mask,
                                                  const VqEnvironmentMaps* env, VqImage out, int row_begin, int row_end, void* stream) {
    return psmain_launch(ctx, pf, pv, in, table, alpha_mask, env, nullptr, false, &out, 1, 0, row_begin, row_end, nullptr, stream);
}

// The same with the shadow maps bound: the PCF tests run inside psmain_kernel on the staged positions and normals, so there are no
// PCF records in device memory and no context scratch beyond what the unshadowed call uses.
extern "C" int vq_forward_lighting_shadowed_from_materials(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                                           const VqSurfaceInputs* in, const VqMaterialTable* table, int alpha_mask,
                                                           const VqEnvironmentMaps* env, const VqShadowMaps* sm, VqImage out,
                                                           int row_begin, int row_end, void* stream) {
    VQ_REQUIRE(sm, "null shadow maps");
    return psmain_launch(ctx, pf, pv, in, table, alpha_mask, env, sm, false, &out, 1, 0, row_begin, row_end, nullptr, stream);
}

// Both with every pixel stored into each of n_outs frames at row dst_row_offset + y and the optional rendezvous (shadow_maps NULL:
// unshadowed), as vq_forward_lighting_multi_signal does for the G-buffer pass.
extern "C" int vq_forward_lighting_from_materials_multi_signal(VqContext* ctx, const VqPerFrameData* pf, const VqPerViewLightingData* pv,
                                                               const VqSurfaceInputs* in, const VqMaterialTable* table, int alpha_mask,
                                                               const VqEnvironmentMaps* env, const VqShadowMaps* sm, const VqImage* outs,
                                                               int n_outs, int dst_row_offset, int row_begin, int row_end,
                                                               const VqPeerSignal* signal, void* stream) {
    return psmain_launch(ctx, pf, pv, in, table, alpha_mask, env, sm, true, outs, n_outs, dst_row_offset, row_begin, row_end, signal,
                         stream);
}

// The IBL cubemaps and the BRDF LUT are sampled from footprint-friendly copies (see CubeV, LutV).
// vq_environment_prepare builds them once and registers them in the context: the analogue of the RENDER_TARGET -> PIXEL_SHADER_RESOURCE transition the engine
// records after prefiltering (EnvironmentMapRendering.cpp:466-472). Call it again whenever the maps' contents change.
// Without it vq_forward_lighting rebuilds the copies on every call (always correct, slower: see tools/perf_forward.py).
extern "C" int vq_environment_prepare(VqContext* ctx, const VqEnvironmentMaps* env, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("TransitionForSceneRendering");
    VQ_REQUIRE(env, "env is null");
    VQ_REQUIRE(cube_desc_ok(env->irradiance_diffuse), "bad cubemap descriptor (irradiance_diffuse)");
    VqScratchLock lock(ctx);
    ctx->env_valid = 0;
    const bool hasSpec = env->irradiance_specular.ptr != nullptr, hasLut = env->brdf_lut.ptr != nullptr;
    if (hasSpec) VQ_REQUIRE(cube_desc_ok(env->irradiance_specular), "bad cubemap descriptor (irradiance_specular)");
    if (hasLut) VQ_REQUIRE(vq_image_ok(env->brdf_lut, 8) && env->brdf_lut.width <= 8192 && env->brdf_lut.height <= 8192, "bad BRDF LUT descriptor");
    CubeV diff, spec; LutV lut;        // not kept: a call that matches the registration points its own views (sampling_views)
    rc = build_sampling_copies(ctx->env_prepared, *env, hasSpec, hasLut, (cudaStream_t)stream, diff, spec, lut); if (rc) return rc;
    ctx->env_key = *env;
    ctx->env_valid = 1;
    return VQ_OK;
}
extern "C" int vq_environment_invalidate(VqContext* ctx) {
    if (!ctx) { vq_set_error("null context"); return VQ_ERR_INVALID_ARG; }
    VqScratchLock lock(ctx);
    ctx->env_valid = 0;    return VQ_OK;
}
