// vq_surface.cu — SURVEY.md §8(f).1: the part of PSMain BEFORE lighting (ForwardLighting.hlsl:226-283) as a kernel that
// fills the G-buffer K1 consumes, plus the RGBA8 box mip chain the engine builds on the CPU for material textures
// (DXGIUtils.cpp:250-287).
//
// Bound: HBM. Algorithmic bytes per pixel = 3 float4 attribute planes in + 3 (4 with emissive) float4 G-buffer planes out
// = 96 (112) B/px (+4 with the SSAO plane); material textures are L2-resident side data (like K1's cubemaps).
//
// Sampling semantics (identical in oracle/oracle_surface.cpp, DESIGN.md §3.6): implicit derivatives = fine finite
// differences inside the pixel's aligned 2x2 quad, exchanged with warp shuffles (a warp shades a 16x2 pixel strip, so
// lane^1 is the horizontal and lane^16 the vertical quad partner); isotropic trilinear, WRAP; texel = byte/255.
#include "vq_common.cuh"
#include "vq_surface_sample.cuh"
#include <stdlib.h>

using namespace vq;

namespace {

// ---------------------------------------------------------------------------------------------
// RGBA8 2x2 box, per channel (a+b+c+d)/4 truncating.  One thread = 4 destination texels (16 B store, two 32 B loads).
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t box4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) {
    // per-byte sums need 10 bits: split even/odd bytes into 16-bit lanes
    const uint32_t lo = (a & 0x00ff00ffu) + (b & 0x00ff00ffu) + (c & 0x00ff00ffu) + (d & 0x00ff00ffu);
    const uint32_t hi = ((a >> 8) & 0x00ff00ffu) + ((b >> 8) & 0x00ff00ffu) + ((c >> 8) & 0x00ff00ffu) + ((d >> 8) & 0x00ff00ffu);
    return ((lo >> 2) & 0x00ff00ffu) | (((hi >> 2) & 0x00ff00ffu) << 8);
}

// Six levels per launch: a block reduces one 64x64 tile of the source level all the way to 1x1 (levels +1 .. +6), so a
// 4096^2 chain is 2 launches instead of 12 and every level is read at most once from HBM. Floor-halved level sizes keep
// the hierarchy tile-local: a valid texel of level k only depends on valid texels of level k-1 (2X+1 < 2*(w>>k) <= w>>(k-1)).
struct MipArgs {
    const uint32_t* src; int sw, sh;       // source level
    uint32_t* dst[6]; int n;               // destination levels (n <= 6), level j is (sw >> (j+1)) x (sh >> (j+1))
};

__global__ void __launch_bounds__(256) tex_mip6_kernel(const __grid_constant__ MipArgs A) {
    __shared__ uint32_t sm[2][16][16];
    const int t = threadIdx.x, px = t & 15, py = t >> 4;
    const int x0 = blockIdx.x * 64 + px * 4, y0 = blockIdx.y * 64 + py * 4;          // 4x4 source patch of this thread
    const int w1 = A.sw >> 1, h1 = A.sh >> 1;
    uint32_t l1[2][2] = {{0u, 0u}, {0u, 0u}};
    const bool vec = ((A.sw & 3) == 0) && (((uintptr_t)A.src & 15) == 0) && x0 + 4 <= A.sw && y0 + 4 <= A.sh;
    if (vec) {
        uint4 r[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) r[k] = __ldg((const uint4*)(A.src + (size_t)(y0 + k) * A.sw + x0));
        l1[0][0] = box4(r[0].x, r[0].y, r[1].x, r[1].y); l1[0][1] = box4(r[0].z, r[0].w, r[1].z, r[1].w);
        l1[1][0] = box4(r[2].x, r[2].y, r[3].x, r[3].y); l1[1][1] = box4(r[2].z, r[2].w, r[3].z, r[3].w);
    } else {
#pragma unroll
        for (int j = 0; j < 2; ++j)
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int X = (x0 >> 1) + i, Y = (y0 >> 1) + j;
                if (X < w1 && Y < h1) {
                    const uint32_t* q = A.src + (size_t)(2 * Y) * A.sw + 2 * X;
                    l1[j][i] = box4(__ldg(q), __ldg(q + 1), __ldg(q + A.sw), __ldg(q + A.sw + 1));
                }
            }
    }
    {   // level +1: 2x2 texels per thread
        const int X = x0 >> 1, Y = y0 >> 1;
#pragma unroll
        for (int j = 0; j < 2; ++j) {
            if (Y + j >= h1) continue;
            uint32_t* d = A.dst[0] + (size_t)(Y + j) * w1 + X;
            if (X + 1 < w1 && (((uintptr_t)d) & 7) == 0) *(uint2*)d = make_uint2(l1[j][0], l1[j][1]);
            else { if (X < w1) d[0] = l1[j][0]; if (X + 1 < w1) d[1] = l1[j][1]; }
        }
    }
    if (A.n < 2) return;
    uint32_t v = box4(l1[0][0], l1[0][1], l1[1][0], l1[1][1]);                       // level +2: one texel per thread
    {
        const int w2 = A.sw >> 2, h2 = A.sh >> 2, X = x0 >> 2, Y = y0 >> 2;
        if (X < w2 && Y < h2) A.dst[1][(size_t)Y * w2 + X] = v;
    }
    sm[0][py][px] = v;
    // levels +3 .. +6: 8x8, 4x4, 2x2, 1x1 texels of this tile, ping-pong through shared memory
    int side = 8, cur = 0;
#pragma unroll
    for (int lvl = 2; lvl < 6; ++lvl, side >>= 1, cur ^= 1) {
        if (lvl >= A.n) return;                                                      // uniform across the block
        __syncthreads();
        if (t < side * side) {
            const int qx = t % side, qy = t / side;
            v = box4(sm[cur][2 * qy][2 * qx], sm[cur][2 * qy][2 * qx + 1], sm[cur][2 * qy + 1][2 * qx], sm[cur][2 * qy + 1][2 * qx + 1]);
            sm[cur ^ 1][qy][qx] = v;
            const int wl = A.sw >> (lvl + 1), hl = A.sh >> (lvl + 1);
            const int X = blockIdx.x * side + qx, Y = blockIdx.y * side + qy;
            if (X < wl && Y < hl) A.dst[lvl][(size_t)Y * wl + X] = v;
        }
    }
}


// block = 256 threads = 8 warps; a warp shades 16x2 pixels (one row of 2x2 quads), a block 32x8.
// Four restructurings of this launch were measured slower and NOT kept: queueing a warp's minority-material pixels for a second
// pass inside the block or for a second small launch — the majority paths dominate the instruction count, not the stray lanes;
// a persistent kernel with the interpolant planes on a TMA / mbarrier ring like K1's — the waits are on the texel and SSAO
// loads, not on the interpolants; and several 32x8 tiles per block with the next tile's interpolants and SSAO texel requested
// before the current tile is shaded — the extra live registers cost more in spills than the overlap returns.
constexpr int SURF_MIN_BLOCKS = 4;
__global__ void __launch_bounds__(256, SURF_MIN_BLOCKS) surface_kernel(const __grid_constant__ SurfArgs A) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int x = blockIdx.x * 32 + (warp & 1) * 16 + (lane & 15);
    const int y = A.tileY0 + blockIdx.y * 8 + (warp >> 1) * 2 + (lane >> 4);
    const uint64_t once = l2_policy_evict_first();
    surface_quad_pixel(A, x, y, lane, once, [&](float4 posAo, float4 nrmRough, float4 albMetal, float4 emi) {
        st_once(A.outPos.row(y) + x, posAo, once);
        st_once(A.outNrm.row(y) + x, nrmRough, once);
        st_once(A.outAlb.row(y) + x, albMetal, once);
        if (A.outEmi.p) st_once(A.outEmi.row(y) + x, emi, once);
    });
}

// interleaves the texels of a material's seven maps (same size, same level count; nullptr = null SRV = zeros) into records
struct RecBuildArgs { const uint32_t* src[7]; uint4* dst; uint32_t n; };
__global__ void __launch_bounds__(256) record_build_kernel(const __grid_constant__ RecBuildArgs A) {
    const uint32_t i = blockIdx.x * 256u + threadIdx.x;
    if (i >= A.n) return;
    uint32_t t[7];
#pragma unroll
    for (int k = 0; k < 7; ++k) t[k] = A.src[k] ? __ldg(A.src[k] + i) : 0u;
    // slots: 0 diffuse, 1 normals, 2 emissive, 3 metalness, 4 roughness, 5 occl_rough_metal, 6 local_ao
    A.dst[i] = make_uint4(t[0], (t[1] & 0x00ffffffu) | (t[6] << 24), (t[2] & 0x00ffffffu) | (t[4] << 24), (t[3] & 0xffu) | (t[5] & 0x00ffff00u));
}

static bool tex_ok(const VqTexture2D& t) {
    if (!t.ptr) return true;     // null SRV
    return t.width > 0 && t.height > 0 && t.levels >= 1 && t.levels <= vq_mip_level_count((uint64_t)t.width, (uint64_t)t.height) &&
           t.levels <= 31 && t.height < (1 << 27) && ((uintptr_t)t.ptr % 4) == 0;
}

}  // namespace

extern "C" int vq_texture_build_mips(VqContext* ctx, VqTexture2D tex, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_REQUIRE(tex.ptr && tex_ok(tex), "bad texture descriptor");
    uint32_t* base = (uint32_t*)tex.ptr;
    for (int l0 = 0; l0 + 1 < tex.levels; l0 += 6) {                   // source level l0 -> levels l0+1 .. l0+6
        MipArgs A;
        A.src = base + vq_pyramid_offset(tex.width, tex.height, l0);
        A.sw = tex.width >> l0; A.sh = tex.height >> l0;
        A.n = tex.levels - 1 - l0 < 6 ? tex.levels - 1 - l0 : 6;
        for (int j = 0; j < 6; ++j) A.dst[j] = j < A.n ? base + vq_pyramid_offset(tex.width, tex.height, l0 + 1 + j) : nullptr;
        const dim3 grid((A.sw + 63) / 64, (A.sh + 63) / 64);
        tex_mip6_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A);
        rc = vq_check_launch("texture_build_mips"); if (rc) return rc;
    }
    return VQ_OK;
}

extern "C" int vq_material_table_create(VqContext* ctx, const VqMaterialData* materials, const VqMaterialTextures* textures,
                                        int count, VqMaterialTable** out_table) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_REQUIRE(materials && textures && out_table, "null argument");
    VQ_REQUIRE(count >= 1 && count <= (1 << 20), "material count out of range");
    DevMaterial* host = (DevMaterial*)calloc((size_t)count, sizeof(DevMaterial));
    if (!host) { vq_set_error("out of host memory"); return VQ_ERR_OUT_OF_MEMORY; }
    for (int i = 0; i < count; ++i) {
        // the kernel converts textureConfig with (int): defined, and the same on host and device, only inside [0, 2^31)
        const float cfg = materials[i].textureConfig;
        if (!(cfg >= 0.0f && cfg < 2147483648.0f)) {
            free(host); vq_set_error("invalid argument: material %d textureConfig %g outside [0, 2^31)", i, (double)cfg); return VQ_ERR_INVALID_ARG;
        }
        host[i].c = materials[i];
        const VqTexture2D* src = &textures[i].diffuse;     // 7 consecutive descriptors
        for (int k = 0; k < 7; ++k) {
            if (!tex_ok(src[k])) { free(host); vq_set_error("invalid argument: material %d texture %d descriptor", i, k); return VQ_ERR_INVALID_ARG; }
            DevTex& d = host[i].t[k];
            if (!src[k].ptr) continue;                                  // null SRV: p = nullptr, reads 0
            if (vq_pyramid_texel_count(src[k].width, src[k].height, src[k].levels) > 0xffffffffull) {
                free(host); vq_set_error("invalid argument: texture too large for 32-bit texel offsets"); return VQ_ERR_INVALID_ARG;
            }
            d.p = (const uint32_t*)src[k].ptr; d.w = src[k].width;
            d.h_levels = (uint32_t)src[k].height | ((uint32_t)src[k].levels << 27);
        }
    }
    // texel records (see DevMaterial): a material qualifies when at least two maps are bound and every bound map has the same
    // width, height and level count. VQ_SURFACE_RECORDS=0 in the environment keeps every material on the map-by-map path.
    const char* recEnv = getenv("VQ_SURFACE_RECORDS");
    const bool wantRecords = !(recEnv && recEnv[0] == '0');
    uint64_t recTexels = 0;
    uint64_t* recOffset = (uint64_t*)calloc((size_t)count, sizeof(uint64_t));
    uint64_t* recCount = (uint64_t*)calloc((size_t)count, sizeof(uint64_t));
    if (!recOffset || !recCount) { free(host); free(recOffset); free(recCount); vq_set_error("out of host memory"); return VQ_ERR_OUT_OF_MEMORY; }
    for (int i = 0; wantRecords && i < count; ++i) {
        const VqTexture2D* src = &textures[i].diffuse;
        int bound = 0, first = -1; bool same = true;
        for (int k = 0; k < 7; ++k) {
            if (!src[k].ptr) continue;
            if (first < 0) first = k;
            else same = same && src[k].width == src[first].width && src[k].height == src[first].height && src[k].levels == src[first].levels;
            ++bound;
        }
        if (bound < 2 || !same || src[first].width >= (1 << 24)) continue;
        recOffset[i] = recTexels;
        recCount[i] = vq_pyramid_texel_count(src[first].width, src[first].height, src[first].levels);
        recTexels += recCount[i];
    }
    VqMaterialTable* t = (VqMaterialTable*)calloc(1, sizeof(VqMaterialTable));
    if (!t) { free(host); free(recOffset); free(recCount); vq_set_error("out of host memory"); return VQ_ERR_OUT_OF_MEMORY; }
    // blocking: ordered after all device work enqueued before the call, on any stream (mip chains may still be in flight on the
    // caller's streams, and the sampling copies below read them)
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess && recTexels) {
        // a sampling copy is an optimisation: when it does not fit, the materials simply stay on the map-by-map path
        if (cudaMalloc(&t->records, (size_t)recTexels * 16) != cudaSuccess) { cudaGetLastError(); t->records = nullptr; recTexels = 0; }
        else t->record_bytes = (size_t)recTexels * 16;
    }
    if (e == cudaSuccess && t->records) {
        for (int i = 0; e == cudaSuccess && i < count; ++i) {
            if (!recCount[i]) continue;
            const VqTexture2D* src = &textures[i].diffuse;
            RecBuildArgs B;
            uint32_t present = 0; int first = -1;
            for (int k = 0; k < 7; ++k) { B.src[k] = (const uint32_t*)src[k].ptr; if (src[k].ptr) { present |= 1u << k; if (first < 0) first = k; } }
            B.dst = (uint4*)t->records + recOffset[i]; B.n = (uint32_t)recCount[i];
            record_build_kernel<<<(unsigned)((recCount[i] + 255) / 256), 256>>>(B);
            vq_count_launch();
            e = cudaGetLastError();
            host[i].rec.p = (const uint32_t*)B.dst;
            host[i].rec.w = src[first].width | (int32_t)(present << 24);
            host[i].rec.h_levels = (uint32_t)src[first].height | ((uint32_t)src[first].levels << 27);
        }
        if (e == cudaSuccess) e = cudaDeviceSynchronize();
    }
    free(recOffset); free(recCount);
    if (e == cudaSuccess) e = cudaMalloc(&t->dev, (size_t)count * sizeof(DevMaterial));
    if (e == cudaSuccess) e = cudaMemcpy(t->dev, host, (size_t)count * sizeof(DevMaterial), cudaMemcpyHostToDevice);
    free(host);
    if (e != cudaSuccess) {
        if (t->dev) cudaFree(t->dev);
        if (t->records) cudaFree(t->records);
        free(t);
        vq_set_error("material table upload failed: %s", cudaGetErrorString(e));
        return e == cudaErrorMemoryAllocation ? VQ_ERR_OUT_OF_MEMORY : VQ_ERR_CUDA;
    }
    t->count = count;
    *out_table = t;
    return VQ_OK;
}

extern "C" int vq_material_table_destroy(VqContext* ctx, VqMaterialTable* table) {
    int rc = vq_enter(ctx); if (rc) return rc;
    if (!table) return VQ_OK;
    if (table->dev) cudaFree(table->dev);
    if (table->records) cudaFree(table->records);
    free(table);
    return VQ_OK;
}

extern "C" int vq_gbuffer_from_materials(VqContext* ctx, const VqSurfaceInputs* in, const VqMaterialTable* table,
                                         float ambient_factor, int alpha_mask, const VqGBuffer* out,
                                         int row_begin, int row_end, void* stream) {
    int rc = vq_enter(ctx); if (rc) return rc;
    VQ_MARK("Geometry");
    VQ_REQUIRE(out, "null argument");
    SurfArgs A;
    rc = surface_inputs(in, table, ambient_factor, alpha_mask, row_begin, row_end, A); if (rc) return rc;
    const int W = in->position_u.width, H = in->position_u.height;
    VQ_REQUIRE(vq_image_ok(out->position_ao) && vq_image_ok(out->normal_roughness) && vq_image_ok(out->albedo_metalness), "bad G-buffer plane");
    VQ_REQUIRE(out->position_ao.width == W && out->position_ao.height == H && out->normal_roughness.width == W &&
               out->normal_roughness.height == H && out->albedo_metalness.width == W && out->albedo_metalness.height == H,
               "G-buffer planes differ in size from the attribute planes");
    if (out->emissive.ptr)
        VQ_REQUIRE(vq_image_ok(out->emissive) && out->emissive.width == W && out->emissive.height == H, "bad emissive plane");
    if (row_begin == row_end) return VQ_OK;

    A.outPos = make_view(out->position_ao); A.outNrm = make_view(out->normal_roughness); A.outAlb = make_view(out->albedo_metalness);
    if (out->emissive.ptr) A.outEmi = make_view(out->emissive); else { A.outEmi.p = nullptr; A.outEmi.w = A.outEmi.h = A.outEmi.pitch4 = 0; }
    const dim3 grid((W + 31) / 32, (row_end - A.tileY0 + 7) / 8);
    surface_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(A);
    return vq_check_launch("gbuffer_from_materials");
}
