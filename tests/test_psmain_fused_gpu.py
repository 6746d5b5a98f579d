"""-m gpu: vq_forward_lighting_from_materials, PSMain end to end in one launch. It must equal, bit for bit, the two-pass composition
it replaces (vq_gbuffer_from_materials with an emissive plane, then vq_forward_lighting): the same fp32 G-buffer values pass
through shared memory instead of device memory. Pixels the alpha mask discards and rows outside the range stay untouched, and it
agrees with the reference's shader text (tests/golden/shader_golden.npz) to the parity bar."""
import os

import numpy as np
import pytest
import torch

import light_domain as ld
import surface_domain as sd
import vqengine_b200 as vq
from envmaps import small_env
from gpu_util import dev, host, assert_scaled
from shader_cases import _pixel_scene
from surface_util import material_set
from vqengine_b200 import synth
from vqengine_b200.shader_data import TEXCFG_EMISSIVE

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0          # output texels the call must not write
GB_INIT = -7.0              # G-buffer texels the surface producer did not write (two-pass side)


def _env_maps(env):
    dd, ds, dl = (torch.from_numpy(np.ascontiguousarray(env[k])).cuda() for k in ("diff", "spec", "lut"))
    em = vq.EnvironmentMaps(vq.cubemap_of(dd, env["diff_res"], 1), vq.cubemap_of(ds, env["spec_res"], env["spec_mips"]),
                            vq.image_of(dl, 2))
    return em, (dd, ds, dl)


def _table(ctx, mats, chains):
    keep, tex = [], []
    for d in chains:
        mt = vq.MaterialTextures()
        for slot in vq.MATERIAL_TEXTURE_SLOTS:
            e = d.get(slot)
            if e is not None:
                buf, w, h, levels = e
                t = torch.from_numpy(buf).cuda()
                keep.append(t)
                setattr(mt, slot, vq.texture_of(t, w, h, levels))
        tex.append(mt)
    return ctx.material_table(mats, tex), keep


def run_both(ctx, planes, mats, chains, env, pf, pv, *, alpha_mask=False, rows=None, records=True, monkeypatch=None,
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
    dp = [dev(p) for p in planes]
    si = vq.SurfaceInputs(vq.image_of(dp[0]), vq.image_of(dp[1]), vq.image_of(dp[2]),
                          vq.image_of(dp[3], 1) if len(dp) > 3 else vq.null_image())
    rb, re = rows or (0, h)
    gbt = [dev(np.full((h, w, 4), GB_INIT, np.float32)) for _ in range(4)]
    gb = vq.GBuffer(*(vq.image_of(t) for t in gbt))
    two = dev(np.full((h, w, 4), SENTINEL, np.float32))
    ctx.gbuffer_from_materials(si, table, pf.fAmbientLightingFactor, gb, alpha_mask=alpha_mask, row_begin=rb, row_end=re)
    ctx.forward_lighting(pf, pv, gb, em, two, row_begin=rb, row_end=re)
    fused = dev(np.full((h, w, 4), SENTINEL, np.float32))
    ctx.forward_lighting_from_materials(pf, pv, si, table, em, fused, alpha_mask=alpha_mask, row_begin=rb, row_end=re)
    got, want, g0 = host(fused), host(two), host(gbt[0])
    table.close()
    ctx.environment_invalidate()
    produced = ~(g0 == GB_INIT).all(-1)
    return got, want, produced


def check_equal(tag, got, want, produced):
    """bit for bit where the surface was produced, SENTINEL everywhere else"""
    assert produced.any(), f"{tag}: nothing produced"
    g, t = got[produced].view(np.uint32), want[produced].view(np.uint32)
    bad = np.argwhere((g != t).any(-1))
    assert bad.size == 0, f"{tag}: {len(bad)} produced pixels differ from the two-pass result, first {np.argwhere(produced)[bad[0, 0]]}"
    assert (got[~produced] == SENTINEL).all(), f"{tag}: wrote {int((got[~produced] != SENTINEL).any(-1).sum())} pixels it did not produce"


def _scene(w, h, *, n=4, tex_res=64, uv_scale=0.05, seed=21, uniform=False, emissive=True, **lights):
    mats, _, chains = material_set(n, tex_res, uniform=uniform)
    if not emissive:
        for m in mats:
            m.textureConfig = float(int(m.textureConfig) & ~TEXCFG_EMISSIVE)
            m.emissiveColor.x = m.emissiveColor.y = m.emissiveColor.z = 0.0
    env = small_env()
    planes = synth.surface_inputs(w, h, n, seed=seed, uv_scale=uv_scale)
    pf, pv = synth.scene_constants(w, h, env["spec_mips"], seed=seed, **lights)
    pf.fAmbientLightingFactor = 0.3
    return planes, mats, chains, env, pf, pv


@pytest.mark.parametrize("w,h,uv_scale", [(96, 54, 0.05), (256, 64, 0.02), (130, 7, 0.1), (37, 19, 0.5), (1, 1, 0.1),
                                          (257, 9, 0.05), (128, 2, 0.004), (200, 33, 0.2)])
@pytest.mark.parametrize("records", [True, False])
def test_equals_two_pass(ctx, w, h, uv_scale, records, monkeypatch):
    """record and map-by-map materials (VQ_SURFACE_RECORDS=0), materials mixed inside warps, ragged widths, odd heights"""
    planes, mats, chains, env, pf, pv = _scene(w, h, uv_scale=uv_scale, n_spot=2)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, records=records, monkeypatch=monkeypatch)
    assert produced.all()
    check_equal(f"{w}x{h}@{uv_scale}/records={records}", got, want, produced)


@pytest.mark.parametrize("records", [True, False])
@pytest.mark.parametrize("emissive", [True, False])
def test_uniform_map_sizes_and_emissive(ctx, records, emissive, monkeypatch):
    """materials whose maps share one size take the texel-record path unless VQ_SURFACE_RECORDS=0; emissive maps and colours
    on and off"""
    planes, mats, chains, env, pf, pv = _scene(192, 108, tex_res=128, uniform=True, emissive=emissive)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, records=records, monkeypatch=monkeypatch)
    check_equal(f"uniform/emissive={emissive}/records={records}", got, want, produced)


@pytest.mark.parametrize("records", [True, False])
def test_alpha_mask_leaves_discarded_pixels_untouched(ctx, records, monkeypatch):
    env, mats, chains, planes, pf, pv = _pixel_scene(96, 48, 7, casters=False)
    pf.Lights.directional.shadowing = 0
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, alpha_mask=True, records=records, monkeypatch=monkeypatch)
    assert not produced.all(), "the scene has no discarded pixels"
    check_equal(f"alpha mask/records={records}", got, want, produced)


@pytest.mark.parametrize("rows", [(0, 1), (1, 2), (3, 4), (5, 6), (1, 30), (2, 31), (7, 33), (32, 33), (0, 33), (12, 12)])
@pytest.mark.parametrize("alpha_mask", [False, True])
def test_row_ranges(ctx, rows, alpha_mask):
    """ranges from odd rows and of length 1 (the quad partner row is read, not written), the last row of an odd height, an
    empty range; rows outside the range stay untouched"""
    planes, mats, chains, env, pf, pv = _scene(150, 33)
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, alpha_mask=alpha_mask, rows=rows)
    outside = np.ones(33, bool)
    outside[rows[0]:rows[1]] = False
    assert (got[outside] == SENTINEL).all()
    if rows[0] == rows[1]:
        assert (got == SENTINEL).all()
        return
    check_equal(f"rows {rows}/alpha={alpha_mask}", got, want, produced)


def test_tiled_rows_compose_the_frame(ctx):
    """row ranges that tile the image (odd boundaries) give the whole-image call's result"""
    planes, mats, chains, env, pf, pv = _scene(140, 41)
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    dp = [dev(p) for p in planes]
    si = vq.SurfaceInputs(vq.image_of(dp[0]), vq.image_of(dp[1]), vq.image_of(dp[2]), vq.image_of(dp[3], 1))
    whole = dev(np.full((41, 140, 4), SENTINEL, np.float32))
    tiled = dev(np.full((41, 140, 4), SENTINEL, np.float32))
    ctx.forward_lighting_from_materials(pf, pv, si, table, em, whole)
    for rb, re in ((0, 7), (7, 8), (8, 23), (23, 41)):
        ctx.forward_lighting_from_materials(pf, pv, si, table, em, tiled, row_begin=rb, row_end=re)
    assert np.array_equal(host(whole).view(np.uint32), host(tiled).view(np.uint32))
    table.close()


def _spot_band_frame(env_mips):
    """spot lights with narrow cones aimed straight down at the field: their cosines near the axis fall in the exact-cosine band"""
    spots = [dict(pos=(x, 12.0, z), dir=(0.0, -1.0, 0.0), inner=inner, outer=outer, brightness=900.0, color=(1.0, 0.8, 0.6))
             for (x, z, inner, outer) in ((0.0, 0.0, 0.0, 0.05), (3.0, -2.0, 0.0, 0.1), (-4.0, 1.0, 0.02, 0.08))]
    pts = [dict(pos=(2.0, 9.0, 1.0), range=60.0, brightness=500.0, color=(0.9, 0.9, 1.0))]
    return ld.scene(ld.CAM, points=pts, spots=spots, directional=dict(dir=(0.3, -1.0, 0.4), brightness=1.5, color=(1.0, 0.5, 0.7)),
                    max_lod=env_mips)


@pytest.mark.parametrize("kind", ["rotated", "diffuse only", "maximum", "spot band", "not prepared"])
def test_frame_settings(ctx, kind):
    """HDRI yaw != 0 (the ROT instantiation), the diffuse-only flag, the ABI's maximum light set (100 + 5 point, 20 + 5 spot,
    directional), spot lights in the exact-cosine band, and an environment that is not registered (copies built per call)"""
    planes, mats, chains, env, pf, pv = _scene(300, 40, uv_scale=0.03)
    if kind == "rotated":
        pf.fHDRIOffsetInRadians = 0.7
    elif kind == "diffuse only":
        pv.EnvironmentMapDiffuseOnlyIllumination = 1
    elif kind == "maximum":
        m = ld.mixed_frame("maximum", 3)
        pf, pv2 = m["pf"], m["pv"]
        pf.fAmbientLightingFactor = 0.3
        pv.CameraPosition = pv2.CameraPosition
        assert pf.Lights.numPointLights == 100 and pf.Lights.numSpotLights == 20
    elif kind == "spot band":
        pf, pv2 = _spot_band_frame(env["spec_mips"])
        pf.fAmbientLightingFactor = 0.3
        pv.CameraPosition = pv2.CameraPosition
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, prepare=(kind != "not prepared"))
    if kind == "rotated":
        # the yaw rotation of the two cube lookups (env_issue<ROT>) is free FMA contraction, which the compiler may place
        # differently in the two kernels: a few pixels differ in their last bits, within the parity bar
        assert produced.all() and (got != SENTINEL).all(-1).all()
        print(assert_scaled(kind, got, want))
        assert (got != want).any(-1).mean() < 0.01
        return
    check_equal(kind, got, want, produced)


CASES = [c for c in sd.sampler_cases() if c[1] * c[2] <= 1 << 16]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_surface_domain_inputs(ctx, case, monkeypatch):
    """the sampler probes of tests/surface_domain.py (every texture shape, level count and texel kind, derivatives from
    magnified to fully minified) shaded end to end, on both sampling paths"""
    name, w, h, levels, kind, seed = case
    level0, ru, rv = sd.build_sampler_case(w, h, levels, kind, seed)
    maps = sd.probe_maps(level0, levels)
    planes = sd.planes_from_uv(ru, rv)
    ph, pw = ru.shape
    env = small_env()
    pf, pv = synth.scene_constants(pw, ph, env["spec_mips"], seed=seed % 1000)
    pf.fAmbientLightingFactor = 1.0
    for records in (True, False):
        got, want, produced = run_both(ctx, planes, [sd.probe_material()], [maps], env, pf, pv, records=records, monkeypatch=monkeypatch)
        check_equal(f"{name}/records={records}", got, want, produced)


@pytest.mark.parametrize("kind", ["unshadowed", "diffuse_only", "alpha_mask"])
def test_agrees_with_the_reference_shader_text(ctx, kind):
    """the whole-PSMain cases of tests/shader_cases.py (interpolants + materials through the reference's shader text): the fused
    call gives the two-pass result bit for bit, so it agrees with the shader text exactly as the two-pass path does (largest
    scaled |delta| about 1.1e-4 on these cases: each half stays within 1e-4 of its oracle, and the halves' errors compose), with
    more than 99.8 % of the values within the strict 1e-4; discarded pixels untouched"""
    golden = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "shader_golden.npz"))
    ref = golden["psmain_" + kind]
    w, h, seed = (96, 48, 7) if kind == "alpha_mask" else (48, 24, 5)
    env, mats, chains, planes, pf, pv = _pixel_scene(w, h, seed, casters=False)
    pf.Lights.directional.shadowing = 0
    if kind == "diffuse_only":
        pv.EnvironmentMapDiffuseOnlyIllumination = 1
    got, want, produced = run_both(ctx, planes, mats, chains, env, pf, pv, alpha_mask=(kind == "alpha_mask"))
    check_equal(f"psmain_{kind}", got, want, produced)
    disc = np.isnan(ref).any(-1)
    assert np.array_equal(disc, ~produced)
    if kind == "alpha_mask":
        assert disc.any()
    print(assert_scaled(f"psmain_{kind}", got[~disc], ref[~disc], tol=2e-4, min_frac_strict=0.998))


def test_one_call_is_one_launch(ctx):
    planes, mats, chains, env, pf, pv = _scene(64, 32)
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    ctx.environment_prepare(em)
    dp = [dev(p) for p in planes]
    si = vq.SurfaceInputs(vq.image_of(dp[0]), vq.image_of(dp[1]), vq.image_of(dp[2]), vq.image_of(dp[3], 1))
    out = dev(np.zeros((32, 64, 4), np.float32))
    before = vq.launch_count()
    ctx.forward_lighting_from_materials(pf, pv, si, table, em, out)
    assert vq.launch_count() - before == 1
    torch.cuda.synchronize()
    table.close()
    ctx.environment_invalidate()


def test_invalid_arguments_launch_nothing(ctx):
    planes, mats, chains, env, pf, pv = _scene(64, 32)
    table, keep = _table(ctx, mats, chains)
    em, env_keep = _env_maps(env)
    dp = [dev(p) for p in planes]
    small = dev(np.zeros((31, 64, 4), np.float32))
    si = vq.SurfaceInputs(vq.image_of(dp[0]), vq.image_of(dp[1]), vq.image_of(dp[2]), vq.image_of(dp[3], 1))
    bad_si = vq.SurfaceInputs(vq.image_of(dp[0]), vq.image_of(small), vq.image_of(dp[2]), vq.image_of(dp[3], 1))
    out = dev(np.full((32, 64, 4), SENTINEL, np.float32))
    before = vq.launch_count()
    for call in (lambda: ctx.forward_lighting_from_materials(pf, pv, bad_si, table, em, out),
                 lambda: ctx.forward_lighting_from_materials(pf, pv, si, table, em, small),
                 lambda: ctx.forward_lighting_from_materials(pf, pv, si, table, em, out, row_begin=0, row_end=33),
                 lambda: ctx.forward_lighting_from_materials(pf, pv, si, table, em, out, row_begin=-1, row_end=2),
                 lambda: ctx.forward_lighting_from_materials(pf, pv, si, table, em, out, row_begin=5, row_end=4)):
        with pytest.raises(vq.VqError) as e:
            call()
        assert e.value.code == vq.VQ_ERR_INVALID_ARG
    import ctypes as C
    rc = vq.lib.vq_forward_lighting_from_materials(ctx._h, C.byref(pf), C.byref(pv), C.byref(si), None, 0, C.byref(em),
                                                   vq.image_of(out), 0, 32, None)
    assert rc == vq.VQ_ERR_INVALID_ARG
    assert vq.launch_count() == before
    assert (host(out) == SENTINEL).all()
    table.close()
