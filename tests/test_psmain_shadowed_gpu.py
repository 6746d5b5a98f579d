"""-m gpu: vq_forward_lighting_shadowed_from_materials, shadowed PSMain end to end in one launch. It must equal, bit for bit, the
composition it replaces (vq_gbuffer_from_materials with an emissive plane, then vq_forward_lighting_shadowed): the PCF tests read the
same fp32 positions and normals from shared memory instead of the G-buffer. Pixels the alpha mask discards and rows outside the range
stay untouched; with no test to run it is the unshadowed fused call; it drives the in-kernel PCF tests over the whole domain of
tests/shadow_domain.py; it agrees with the reference's shader text as the two-pass path does; the host mirror's new overloads call it."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import light_domain as ld
import shadow_domain as shd
import vqengine_b200 as vq
from envmaps import small_env
from gpu_util import TOL, assert_scaled, dev, host, report
from shader_cases import _pixel_scene, _shadow_setup
from test_psmain_fused_gpu import GB_INIT, SENTINEL, _env_maps, _scene, _spot_band_frame, _table, check_equal

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KINDS = ("point", "spot", "dir")


def _maps(kw, bind=KINDS):
    """shader_cases._shadow_setup's numpy maps -> forward_lighting_shadowed's keyword arguments, only the kinds in `bind`"""
    return {"point_cubes": kw["point_cubes"] if "point" in bind else None,
            "spot_maps": kw["spot_maps"] if "spot" in bind else None,
            "directional_map": kw["dir_map"] if "dir" in bind else None}


def _inputs(planes):
    dp = [dev(p) for p in planes]
    si = vq.SurfaceInputs(vq.image_of(dp[0]), vq.image_of(dp[1]), vq.image_of(dp[2]),
                          vq.image_of(dp[3], 1) if len(dp) > 3 else vq.null_image())
    return si, dp


def run_both(ctx, planes, mats, chains, env, pf, pv, maps, *, alpha_mask=False, rows=None, records=True, monkeypatch=None,
             prepare=True):
    """(fused output, two-pass output, produced mask) on the same inputs; both outputs start as SENTINEL"""
    if monkeypatch is not None:
        monkeypatch.setenv("VQ_SURFACE_RECORDS", "1" if records else "0")
    h, w = planes[0].shape[:2]
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    if prepare:
        ctx.environment_prepare(em)
    else:
        ctx.environment_invalidate()
    si, dp = _inputs(planes)
    dm = {k: (dev(v) if v is not None else None) for k, v in maps.items()}
    rb, re = rows or (0, h)
    gbt = [dev(np.full((h, w, 4), GB_INIT, np.float32)) for _ in range(4)]
    gb = vq.GBuffer(*(vq.image_of(t) for t in gbt))
    two = dev(np.full((h, w, 4), SENTINEL, np.float32))
    ctx.gbuffer_from_materials(si, table, pf.fAmbientLightingFactor, gb, alpha_mask=alpha_mask, row_begin=rb, row_end=re)
    ctx.forward_lighting_shadowed(pf, pv, gb, em, two, row_begin=rb, row_end=re, **dm)
    fused = dev(np.full((h, w, 4), SENTINEL, np.float32))
    ctx.forward_lighting_shadowed_from_materials(pf, pv, si, table, em, fused, alpha_mask=alpha_mask, row_begin=rb, row_end=re, **dm)
    got, want, g0 = host(fused), host(two), host(gbt[0])
    table.close()
    ctx.environment_invalidate()
    produced = ~(g0 == GB_INIT).all(-1)
    return got, want, produced


def run_fused(ctx, planes, mats, chains, env, pf, pv, maps=None):
    """the fused call once (maps None: the unshadowed vq_forward_lighting_from_materials); -> (output, launches)"""
    h, w = planes[0].shape[:2]
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    ctx.environment_prepare(em)
    si, dp = _inputs(planes)
    out = dev(np.full((h, w, 4), SENTINEL, np.float32))
    dm = {k: (dev(v) if v is not None else None) for k, v in (maps or {}).items()}
    before = vq.launch_count()
    if maps is None:
        ctx.forward_lighting_from_materials(pf, pv, si, table, em, out)
    else:
        ctx.forward_lighting_shadowed_from_materials(pf, pv, si, table, em, out, **dm)
    launches = vq.launch_count() - before
    got = host(out)
    table.close()
    ctx.environment_invalidate()
    return got, launches


def _shadow_scene(w, h, *, uv_scale=0.05, seed=21, **lights):
    """test_psmain_fused_gpu's material scene with casters (2 point, 2 spot by default) and shader_cases' shadow views and maps"""
    lights.setdefault("n_spot", 2)
    planes, mats, chains, env, pf, pv = _scene(w, h, uv_scale=uv_scale, seed=seed, casters=True, **lights)
    kw = _shadow_setup(pf, seed + 100)
    assert pf.Lights.numPointCasters > 0 and pf.Lights.numSpotCasters > 0
    return planes, mats, chains, env, pf, pv, kw


# ---- 1. equals the two passes ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,uv_scale", [(96, 54, 0.05), (130, 7, 0.1), (37, 19, 0.5), (1, 1, 0.1), (257, 9, 0.05), (200, 33, 0.2)])
@pytest.mark.parametrize("records", [True, False])
def test_equals_two_pass(ctx, w, h, uv_scale, records, monkeypatch):
    """record and map-by-map materials (VQ_SURFACE_RECORDS=0), ragged widths, odd heights, 1x1"""
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(w, h, uv_scale=uv_scale)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, _maps(kw), records=records, monkeypatch=monkeypatch)
    assert produced.all()
    check_equal(f"{w}x{h}@{uv_scale}/records={records}", got, want, produced)


@pytest.mark.parametrize("records", [True, False])
def test_alpha_mask_leaves_discarded_pixels_untouched(ctx, records, monkeypatch):
    env, mats, chains, planes, pf, pv = _pixel_scene(96, 48, 7, casters=True)
    kw = _shadow_setup(pf, 110)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, _maps(kw), alpha_mask=True, records=records,
                                   monkeypatch=monkeypatch)
    assert not produced.all(), "the scene has no discarded pixels"
    check_equal(f"alpha mask/records={records}", got, want, produced)


@pytest.mark.parametrize("rows", [(0, 1), (1, 2), (5, 6), (1, 30), (7, 33), (32, 33), (12, 12)])
@pytest.mark.parametrize("alpha_mask", [False, True])
def test_row_ranges(ctx, rows, alpha_mask):
    """ranges from odd rows and of length 1, the last row of an odd height, an empty range; rows outside stay untouched"""
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(150, 33)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, _maps(kw), alpha_mask=alpha_mask, rows=rows)
    outside = np.ones(33, bool)
    outside[rows[0]:rows[1]] = False
    assert (got[outside] == SENTINEL).all()
    if rows[0] == rows[1]:
        assert (got == SENTINEL).all()
        return
    check_equal(f"rows {rows}/alpha={alpha_mask}", got, want, produced)


def test_tiled_rows_compose_the_frame(ctx):
    """row ranges that tile the image (odd boundaries) give the whole-image call's result"""
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(140, 41)
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    si, dp = _inputs(planes)
    dm = {k: dev(v) for k, v in _maps(kw).items()}
    whole = dev(np.full((41, 140, 4), SENTINEL, np.float32))
    tiled = dev(np.full((41, 140, 4), SENTINEL, np.float32))
    ctx.forward_lighting_shadowed_from_materials(pf, pv, si, table, em, whole, **dm)
    for rb, re in ((0, 7), (7, 8), (8, 23), (23, 41)):
        ctx.forward_lighting_shadowed_from_materials(pf, pv, si, table, em, tiled, row_begin=rb, row_end=re, **dm)
    assert np.array_equal(host(whole).view(np.uint32), host(tiled).view(np.uint32))
    table.close()


@pytest.mark.parametrize("kind", ["rotated", "diffuse only", "maximum", "spot band", "not prepared"])
def test_frame_settings(ctx, kind):
    """HDRI yaw != 0 (the ROT instantiation), the diffuse-only flag, the ABI's maximum light set (100 + 5 point, 20 + 5 spot and a
    shadowing directional light), spot casters in the exact-cosine band, and an environment that is not registered"""
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(300, 40, uv_scale=0.03)
    if kind == "rotated":
        pf.fHDRIOffsetInRadians = 0.7
    elif kind == "diffuse only":
        pv.EnvironmentMapDiffuseOnlyIllumination = 1
    elif kind == "maximum":
        m = ld.mixed_frame("maximum", 3)
        pf, pv2 = m["pf"], m["pv"]
        pf.fAmbientLightingFactor = 0.3
        pv.CameraPosition = pv2.CameraPosition
        L = pf.Lights
        assert (L.numPointLights, L.numPointCasters, L.numSpotLights, L.numSpotCasters) == (100, 5, 20, 5) and L.directional.enabled
        kw = _shadow_setup(pf, 120)
    elif kind == "spot band":
        pf, pv2 = _spot_band_frame(env["spec_mips"])
        pf.fAmbientLightingFactor = 0.3
        pv.CameraPosition = pv2.CameraPosition
        L = pf.Lights
        for i in range(L.numSpotLights):                       # the narrow cones become the casters
            L.spot_casters[i] = L.spot_lights[i]
        L.numSpotCasters, L.numSpotLights = L.numSpotLights, 0
        L.point_casters[0] = L.point_lights[0]
        L.numPointCasters = 1
        kw = _shadow_setup(pf, 121)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, _maps(kw), prepare=(kind != "not prepared"))
    if kind == "rotated":
        # the yaw rotation of the two cube lookups is free FMA contraction, which the compiler may place differently in the two
        # kernels: a few pixels differ in their last bits, within the parity bar
        assert produced.all() and (got != SENTINEL).all(-1).all()
        print(assert_scaled(kind, got, want))
        assert (got != want).any(-1).mean() < 0.01
        return
    check_equal(kind, got, want, produced)


# ---- 2. caster configurations -------------------------------------------------------------------------------------------
SUBSETS = [("point",), ("spot",), ("dir",), ("point", "spot"), ("point", "dir"), ("spot", "dir")]


@pytest.mark.parametrize("bind", SUBSETS, ids=["+".join(b) for b in SUBSETS])
def test_caster_configurations(ctx, bind):
    """each map type bound alone and every pair: equal to the two passes; with every map at 'nothing in front' equal to the
    unshadowed fused call, and at 'everything in front' equal to the fused call without the bound types' casters (the caster lists
    emptied, the directional light off), as test_shadow_gpu's nothing / everything occluded tests ask of the two-pass path"""
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(160, 36)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, _maps(kw, bind))
    assert produced.all()
    check_equal("+".join(bind), got, want, produced)
    assert (got != run_fused(ctx, planes, mats, chains, env, pf, pv)[0]).any(), "the bound maps shadow nothing"

    ones = {k: np.ones_like(v) for k, v in kw.items() if isinstance(v, np.ndarray)}
    got, launches = run_fused(ctx, planes, mats, chains, env, pf, pv, _maps(ones, bind))
    ref, _ = run_fused(ctx, planes, mats, chains, env, pf, pv)
    assert launches == 1
    r = report("unoccluded", got, ref)
    assert r["max_scaled"] <= TOL, r
    print("unoccluded", r, "bit-identical pixels", float((got == ref).all(-1).mean()))

    zeros = {k: np.zeros_like(v) for k, v in kw.items() if isinstance(v, np.ndarray)}
    got, _ = run_fused(ctx, planes, mats, chains, env, pf, pv, _maps(zeros, bind))
    L = pf.Lights
    saved = (L.numPointCasters, L.numSpotCasters, L.directional.enabled)
    if "point" in bind:
        L.numPointCasters = 0
    if "spot" in bind:
        L.numSpotCasters = 0
    if "dir" in bind:
        L.directional.enabled = 0
    ref, _ = run_fused(ctx, planes, mats, chains, env, pf, pv)
    L.numPointCasters, L.numSpotCasters, L.directional.enabled = saved
    r = report("occluded", got, ref)
    assert r["max_scaled"] <= TOL, r
    print("occluded", r, "bit-identical pixels", float((got == ref).all(-1).mean()))


@pytest.mark.parametrize("case", ["no maps", "cubes without point casters", "maps without spot casters", "directional not shadowing"])
def test_no_test_runs_is_the_unshadowed_call(ctx, case):
    """no map bound, or maps bound for no caster present: bit for bit the unshadowed fused call, in one launch"""
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(96, 20)
    L = pf.Lights
    bind = ()
    if case == "cubes without point casters":
        L.numPointCasters, bind = 0, ("point",)
    elif case == "maps without spot casters":
        L.numSpotCasters, bind = 0, ("spot",)
    elif case == "directional not shadowing":
        L.directional.shadowing, bind = 0, ("dir",)
    got, launches = run_fused(ctx, planes, mats, chains, env, pf, pv, _maps(kw, bind))
    ref, _ = run_fused(ctx, planes, mats, chains, env, pf, pv)
    assert launches == 1
    assert np.array_equal(got.view(np.uint32), ref.view(np.uint32))


# ---- 3. the PCF domain through the fused kernel ---------------------------------------------------------------------------
@pytest.fixture(scope="module")
def domain_scenes():
    return shd.scenes()


def _plain_material():
    m = vq.MaterialData()
    m.diffuse.x, m.diffuse.y, m.diffuse.z = 0.6, 0.5, 0.4
    m.alpha = 1.0
    m.roughness, m.metalness = 0.5, 0.3
    m.uvScaleOffset.x, m.uvScaleOffset.y = 1.0, 1.0
    m.textureConfig = 0.0
    return m


@pytest.mark.parametrize("idx", range(len(shd.SIZES)))
def test_pcf_domain(ctx, domain_scenes, idx):
    """every scene of tests/shadow_domain.py, its G-buffer positions and normals passed in as interpolants with a material without
    maps (the producer writes the position unchanged and renormalises the normal): perspective w = 0 and NaN quotients, cube edges
    and corners, whole-warp axis paths and mixed-axis warps, exact directional texel boundaries, in the warps they were built for
    (a fused warp is 32 consecutive columns of one row, and the scenes' rows are 128 pixels)"""
    s = domain_scenes[idx]
    pos, nrm = s.planes[0], s.planes[1]
    h, w = pos.shape[:2]
    pu = np.zeros((h, w, 4), np.float32); nv = np.zeros((h, w, 4), np.float32); tm = np.zeros((h, w, 4), np.float32)
    pu[..., :3], nv[..., :3] = pos[..., :3], nrm[..., :3]
    tm[..., 0] = 1.0
    maps = {"point_cubes": s.cubes, "spot_maps": s.spots, "directional_map": s.dmap}
    got, want, produced = run_both(ctx, [pu, nv, tm], [_plain_material()], [{}], small_env(), s.pf, s.pv, maps)
    assert produced.all()
    check_equal(f"shadow domain scene {idx}", got, want, produced)


# ---- 4. the reference's shader text -----------------------------------------------------------------------------------------
def test_agrees_with_the_reference_shader_text(ctx):
    """the shadowed whole-PSMain case of tests/shader_cases.py: the fused call gives the two-pass result bit for bit, so it agrees
    with the shader text within the bounds the two-pass path meets on it, measured here on the two-pass output"""
    golden = np.load(os.path.join(ROOT, "tests", "golden", "shader_golden.npz"))
    ref = golden["psmain_shadowed"]
    env, mats, chains, planes, pf, pv = _pixel_scene(48, 24, 5, casters=True)
    kw = _shadow_setup(pf, 110)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, _maps(kw))
    check_equal("psmain_shadowed", got, want, produced)
    assert produced.all() and np.isfinite(ref).all()
    two, fused = report("two-pass", want, ref), report("fused", got, ref)
    print(two, fused)
    assert fused["max_scaled"] <= two["max_scaled"] and fused["frac_abs_le_tol"] >= two["frac_abs_le_tol"]
    d = np.abs(got.astype(np.float64) - ref) / np.maximum(1.0, np.abs(ref.astype(np.float64)))
    bad_two = (np.abs(want.astype(np.float64) - ref) / np.maximum(1.0, np.abs(ref.astype(np.float64))) > 2e-4).any(-1)
    assert ((d > 2e-4).any(-1) <= bad_two).all(), "the fused call misses the shader text where the two-pass path meets it"


# ---- 5. launches ------------------------------------------------------------------------------------------------------------
def test_one_call_is_one_launch(ctx):
    planes, mats, chains, env, pf, pv, kw = _shadow_scene(64, 32)
    got, launches = run_fused(ctx, planes, mats, chains, env, pf, pv, _maps(kw))
    assert launches == 1
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    ctx.environment_prepare(em)
    si, dp = _inputs(planes)
    gbt = [dev(np.zeros((32, 64, 4), np.float32)) for _ in range(4)]
    gb = vq.GBuffer(*(vq.image_of(t) for t in gbt))
    ctx.gbuffer_from_materials(si, table, pf.fAmbientLightingFactor, gb)
    out = dev(np.zeros((32, 64, 4), np.float32))
    dm = {k: dev(v) for k, v in _maps(kw).items()}
    before = vq.launch_count()
    ctx.forward_lighting_shadowed(pf, pv, gb, em, out, **dm)
    assert vq.launch_count() - before == 2
    torch.cuda.synchronize()
    table.close()
    ctx.environment_invalidate()


# ---- 6. the host mirror -----------------------------------------------------------------------------------------------------
HOST_PROGRAM = r'''
#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>
#include "vq_renderer.hpp"

static float frand(unsigned& s) { s = s * 1664525u + 1013904223u; return (float)(s >> 8) / 16777216.0f; }
static void upload(vq::FTexture2D& t, const std::vector<float>& v, int w, int h) { t.Create(w, h); cudaMemcpy(t.mem.ptr, v.data(), v.size() * 4, cudaMemcpyHostToDevice); }
static std::vector<float> download(const VqImage& im) {
    std::vector<float> v((size_t)im.width * im.height * 4);
    cudaMemcpy(v.data(), im.ptr, v.size() * 4, cudaMemcpyDeviceToHost);
    return v;
}
static size_t differ(const std::vector<float>& a, const std::vector<float>& b) {
    size_t n = 0;
    for (size_t i = 0; i < a.size(); i += 4) n += std::memcmp(&a[i], &b[i], 16) != 0;
    return n;
}

int main() {
    const int W = 70, H = 37;
    unsigned seed = 0x5EED0007u;
    vq::VQRenderer r;
    if (!r.Initialize(0) || !r.LoadDefaultResources()) return 2;
    std::vector<float> hdri(64 * 32 * 4);
    for (size_t i = 0; i < hdri.size(); ++i) hdri[i] = (i % 4 == 3) ? 1.0f : 0.2f + 1.5f * frand(seed);
    vq::FEnvironmentMapRenderingResources env;
    if (!env.CreateRenderingResources(r, vq::FEnvironmentMapDescriptor{hdri.data(), 64, 32, 0.0f}, 16, 32)) return 3;
    if (!r.PreFilterEnvironmentMap(env, 0.1f) || !r.OnWindowSizeChanged(W, H, W, H)) return 3;

    // interpolants of a height field, one material without maps
    std::vector<float> pu((size_t)W * H * 4), nv(pu.size()), tm(pu.size());
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const size_t o = ((size_t)y * W + x) * 4;
            const float fx = -20.f + 40.f * x / W, fz = 20.f - 40.f * y / H;
            pu[o] = fx; pu[o + 1] = 2.0f * std::sin(0.3f * fx) * std::cos(0.25f * fz); pu[o + 2] = fz; pu[o + 3] = 0.05f * fx;
            nv[o] = -0.6f * std::cos(0.3f * fx); nv[o + 1] = 1.0f + 0.2f * frand(seed); nv[o + 2] = 0.5f * std::sin(0.25f * fz); nv[o + 3] = 0.05f * fz;
            tm[o] = 1.0f; tm[o + 1] = 0.0f; tm[o + 2] = 0.1f; tm[o + 3] = 0.0f;
        }
    vq::FTexture2D tpu, tnv, ttm;
    upload(tpu, pu, W, H); upload(tnv, nv, W, H); upload(ttm, tm, W, H);
    const VqSurfaceInputs si{tpu.View(), tnv.View(), ttm.View(), VqImage{nullptr, 0, 0, 0}};
    VqMaterialData mat; std::memset(&mat, 0, sizeof(mat));
    mat.diffuse = {0.7f, 0.6f, 0.5f}; mat.alpha = 1.0f; mat.emissiveColor = {0.1f, 0.0f, 0.05f}; mat.emissiveIntensity = 0.5f;
    mat.roughness = 0.45f; mat.metalness = 0.3f; mat.uvScaleOffset = {1.0f, 1.0f, 0.0f, 0.0f};
    VqMaterialTextures tex; std::memset(&tex, 0, sizeof(tex));
    VqMaterialTable* table = nullptr;
    if (vq_material_table_create(r.Context(), &mat, &tex, 1, &table) != VQ_OK) return 4;

    // lights: a point light, a point caster, a spot caster and a shadowing directional light
    vq::FSceneView view;
    view.cameraPosition = {0.0f, 5.0f, -17.0f};
    view.sceneRenderOptions.fAmbientLightingFactor = 0.3f;
    VqSceneLighting& L = view.GPULightingData;
    L.numPointLights = 1;
    L.point_lights[0].position = {5.0f, 9.0f, 3.0f}; L.point_lights[0].range = 60.0f; L.point_lights[0].brightness = 600.0f; L.point_lights[0].color = {1, 0.9f, 0.8f};
    L.numPointCasters = 1;
    L.point_casters[0].position = {-4.0f, 7.0f, -2.0f}; L.point_casters[0].range = 40.0f; L.point_casters[0].brightness = 900.0f;
    L.point_casters[0].color = {0.9f, 1, 0.7f}; L.point_casters[0].depthBias = 0.01f;
    L.numSpotCasters = 1;
    VqSpotLight& s = L.spot_casters[0];
    s.position = {2.0f, 12.0f, 1.0f}; s.spotDir = {0.1f, -1.0f, 0.2f}; s.innerConeAngle = 0.4f; s.outerConeAngle = 0.8f;
    s.brightness = 1200.0f; s.color = {1, 0.8f, 0.6f}; s.range = 100.0f; s.depthBias = 0.002f;
    const float M[16] = {1 / 25.f, 0.01f, 0, 0,  -0.02f, 1 / 25.f, 0, 0,  0, 0, 0, 0,  0.1f, 0, 0.5f, 1};
    std::memcpy(L.shadowViews[0].m, M, sizeof(M)); std::memcpy(L.shadowViewDirectional.m, M, sizeof(M));
    L.directional.enabled = 1; L.directional.shadowing = 1; L.directional.brightness = 1.5f; L.directional.color = {1, 1, 1};
    L.directional.lightDirection = {-0.5f, -0.83f, 0.25f}; L.directional.depthBias = 0.001f;

    // maps of sizes other than the engine's, so that the dimensions the overloads pass matter
    const int PR = 8, SW = 20, SH = 12, DW = 24, DH = 16;
    std::vector<float> cube(6 * PR * PR), spot(SW * SH), dir(DW * DH);
    for (float& v : cube) v = 1.2f * frand(seed);
    for (float& v : spot) v = 0.3f + 0.4f * frand(seed);
    for (float& v : dir) v = 0.3f + 0.4f * frand(seed);
    void *dc, *ds, *dd;
    cudaMalloc(&dc, cube.size() * 4); cudaMalloc(&ds, spot.size() * 4); cudaMalloc(&dd, dir.size() * 4);
    cudaMemcpy(dc, cube.data(), cube.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(ds, spot.data(), spot.size() * 4, cudaMemcpyHostToDevice);
    cudaMemcpy(dd, dir.data(), dir.size() * 4, cudaMemcpyHostToDevice);
    const VqShadowMaps maps{dc, PR, ds, SW, SH, dd, DW, DH};

    vq::FPostProcessParameters pp; pp.SceneRTWidth = W; pp.SceneRTHeight = H;
    vq::FGraphicsSettings gfx;
    if (!r.RenderSceneColorFromMaterials(nullptr, view, pp, si, table, env, gfx, false, maps)) { std::fprintf(stderr, "%s\n", vq::LastError()); return 5; }
    const std::vector<float> fusedMirror = download(r.SceneColor().View());

    // the same frame through the C-ABI: the constant blocks the engine uploads, with the bound maps' dimensions
    VqPerFrameData pf; std::memset(&pf, 0, sizeof(pf));
    pf.Lights = L; pf.fAmbientLightingFactor = 0.3f; pf.fHDRIOffsetInRadians = 0.0f;
    pf.f2PointLightShadowMapDimensions = {(float)PR, (float)PR};
    pf.f2SpotLightShadowMapDimensions = {(float)SW, (float)SH};
    pf.f2DirectionalLightShadowMapDimensions = {(float)DW, (float)DH};
    VqPerViewLightingData pv; std::memset(&pv, 0, sizeof(pv));
    pv.CameraPosition = view.cameraPosition; pv.ScreenDimensions = {(float)W, (float)H};
    pv.MaxEnvMapLODLevels = (float)env.GetNumSpecularIrradianceCubemapLODLevels();
    const VqEnvironmentMaps em{env.DiffuseBlurred(), env.Specular(), r.BRDFIntegrationLUT().View()};
    vq::FTexture2D abi; abi.Create(W, H);
    if (vq_forward_lighting_shadowed_from_materials(r.Context(), &pf, &pv, &si, table, 0, &em, &maps, abi.View(), 0, H, nullptr) != VQ_OK) return 6;
    const std::vector<float> fusedAbi = download(abi.View());

    // and the G-buffer overload on the G-buffer of the same interpolants
    vq::FTexture2D g0, g1, g2, g3;
    g0.Create(W, H); g1.Create(W, H); g2.Create(W, H); g3.Create(W, H);
    const VqGBuffer gb{g0.View(), g1.View(), g2.View(), g3.View()};
    if (vq_gbuffer_from_materials(r.Context(), &si, table, pf.fAmbientLightingFactor, 0, &gb, 0, H, nullptr) != VQ_OK) return 7;
    if (!r.RenderSceneColor(nullptr, view, pp, gb, env, gfx, false, maps)) return 8;
    const std::vector<float> twoPassMirror = download(r.SceneColor().View());
    if (cudaDeviceSynchronize() != cudaSuccess) return 9;

    size_t shadowedPx = 0, finite = 1;
    {   // the same frame unshadowed: the maps must change the result
        VqShadowMaps none; std::memset(&none, 0, sizeof(none));
        if (!r.RenderSceneColorFromMaterials(nullptr, view, pp, si, table, env, gfx, false, none)) return 10;
        shadowedPx = differ(download(r.SceneColor().View()), fusedAbi);
    }
    for (float v : fusedAbi) finite &= std::isfinite(v) ? 1u : 0u;
    std::printf("%zu %zu %zu %zu\n", differ(fusedMirror, fusedAbi), differ(twoPassMirror, fusedAbi), shadowedPx, finite);
    vq_material_table_destroy(r.Context(), table);
    cudaFree(dc); cudaFree(ds); cudaFree(dd);
    env.DestroyRenderingResources();
    return 0;
}
'''


def test_host_mirror_shadowed_overloads(tmp_path):
    """VQRenderer's shadowed overloads: RenderSceneColorFromMaterials equals the C-ABI call with the bound maps' dimensions bit for
    bit, and RenderSceneColor on the G-buffer of the same interpolants equals it too (every pixel is produced)"""
    host_dir = os.path.join(ROOT, "vqengine_b200", "host")
    if not shutil.which("g++") or not os.path.exists(os.path.join(host_dir, "libvqhost.so")):
        pytest.skip("g++ / libvqhost.so not available")
    src = tmp_path / "shadowed.cpp"
    src.write_text(HOST_PROGRAM)
    exe = str(tmp_path / "shadowed")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["g++", "-std=c++17", str(src), "-I", host_dir, "-I", os.path.join(cuda, "include"), "-L", host_dir, "-lvqhost",
                           "-L", os.path.join(ROOT, "vqengine_b200"), "-lvqcuda", "-L", os.path.join(cuda, "lib64"), "-lcudart",
                           f"-Wl,-rpath,{host_dir}", f"-Wl,-rpath,{os.path.join(ROOT, 'vqengine_b200')}",
                           f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}", "-o", exe])
    res = subprocess.run([exe], capture_output=True, text=True, timeout=300)
    assert res.returncode == 0, (res.returncode, res.stdout, res.stderr)
    mirror_vs_abi, two_pass_vs_abi, shadowed_px, finite = (int(v) for v in res.stdout.split())
    assert finite == 1
    assert mirror_vs_abi == 0 and two_pass_vs_abi == 0, res.stdout
    assert shadowed_px > 0, "the shadow maps changed nothing"
