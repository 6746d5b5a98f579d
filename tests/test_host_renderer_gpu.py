"""-m gpu: the C++ host layer (vq::VQRenderer, libvqhost.so) entry point by entry point, through tests/host_check/renderer_driver.cpp
on a non-default stream, against references that do not go through the layer.

The layer is pure plumbing: it fills the engine's constant blocks and binds resources, and every kernel underneath is proven by its
own tests. So each stage here is fed, in the reference, the DEVICE's previous stage (the pyramid, the unblurred diffuse cube, the
blurred cube, the specular cube, the LUT and the scene colour the layer produced), and the bound of every comparison is the one the
kernel's own test already justifies. What the tests pin is what the layer decides. The expected constants are written here from the
rules the layer cites (SceneRendering.cpp:429-467, EnvironmentMapRendering.cpp:63 and 181-472, Renderer.cpp:1026-1032, as quoted in
vq_renderer.cpp, INTEGRATION.md and vqcuda.h); nothing is read back from the layer:

  - HDRIMips = mip_level_count(W, H); K2 samples HDRI mip (3 < HDRIMips ? 3 : HDRIMips - 1) with the given step;
    SpecMips = mip_level_count(SpecRes, SpecRes) - 1 ("2x2 for the last mip level"); MaxEnvMapLODLevels = SpecMips;
  - the diffuse cube is blurred per face, X then Y; PSMain binds the BLURRED diffuse cube;
  - ambient x 0.005 on an HDR display; EnvironmentMapDiffuseOnlyIllumination under SSR; the HDRI yaw; the camera position;
    ScreenDimensions = the render size; shadow-map sizes 1024 (point, spot) and 2048 (directional) unless a map of that kind is bound;
  - RenderPostProcess: optional blur, then CAS only when CAS is enabled, FSR is off and Sharpness > 0, or FSR (display size), or
    the tonemapper alone (render size);
  - LoadDefaultResources: a 1024^2 RG32F LUT at 2048 samples; MaxContentLightLevel = (int) Image::MaxLuminance.

One reading had to be chosen: the engine's EnvironmentMapRendering.cpp:63 comment "2x2 for the last mip level" is taken as the
count rule above (a 32^2 specular cube has 5 mips, 32 .. 2), which is also what vqcuda.h documents."""
import ctypes as C

import numpy as np
import pytest
import torch

import host_driver as hd
from gpu_util import dev, host, assert_abs, assert_scaled, report, TOL

pytestmark = pytest.mark.gpu

DIFF_STEP = 0.05


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    assert hd.available(), "host layer not built"
    return hd.build(tmp_path_factory.mktemp("driver"))


def _bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def spot_hdri(w, h, spot=200.0):
    """equirect radiance with one compact bright spot at mid latitude over a smooth sky that is flat towards the poles (so the
    specular prefilter's pole sensitivity stays tiny), alpha 1. The spot makes the blurred diffuse cube differ from the unblurred
    one, and the source mip of K2 and the specular roughness of every mip visible."""
    v, u = np.meshgrid((np.arange(h) + 0.5) / h, (np.arange(w) + 0.5) / w, indexing="ij")
    sky = 0.3 + 0.4 * np.sin(np.pi * v) ** 4 * (1.0 + 0.5 * np.cos(2 * np.pi * u))
    du = np.minimum(np.abs(u - 0.3), 1.0 - np.abs(u - 0.3))
    s = spot * np.exp(-(du ** 2 + (v - 0.42) ** 2) / (2 * 0.05 ** 2))
    img = np.ones((h, w, 4), np.float32)
    for c, (a, b) in enumerate(((1.0, 1.0), (0.9, 0.8), (0.8, 0.6))):
        img[..., c] = sky * a + s * b
    return img


def expected_src_mip(levels):
    return 3 if 3 < levels else levels - 1


def expected_spec_mips(vq, spec_res):
    return vq.mip_level_count(spec_res, spec_res) - 1


def expected_constants(vq, lights, w, h, spec_mips, cam=(0.0, 0.0, 0.0), yaw=0.0, ambient=0.055, hdr=False, ssr=False, dims=None):
    """CopyPerFrameConstantBufferData / CopyPerViewConstantBufferData (SceneRendering.cpp:429-467) restated"""
    pf = vq.PerFrameData()
    C.memset(C.byref(pf), 0, C.sizeof(pf))
    pf.Lights = lights
    amb = np.float32(ambient)
    pf.fAmbientLightingFactor = float(amb * np.float32(0.005)) if hdr else float(amb)
    pf.f2PointLightShadowMapDimensions.x = pf.f2PointLightShadowMapDimensions.y = 1024.0
    pf.f2SpotLightShadowMapDimensions.x = pf.f2SpotLightShadowMapDimensions.y = 1024.0
    pf.f2DirectionalLightShadowMapDimensions.x = pf.f2DirectionalLightShadowMapDimensions.y = 2048.0
    for kind, (dw, dh) in (dims or {}).items():
        d = getattr(pf, f"f2{kind}LightShadowMapDimensions")
        d.x, d.y = float(dw), float(dh)
    pf.fHDRIOffsetInRadians = yaw
    pv = vq.PerViewLightingData()
    C.memset(C.byref(pv), 0, C.sizeof(pv))
    pv.CameraPosition.x, pv.CameraPosition.y, pv.CameraPosition.z = cam
    pv.ScreenDimensions.x, pv.ScreenDimensions.y = float(w), float(h)
    pv.MaxEnvMapLODLevels = float(spec_mips)
    pv.EnvironmentMapDiffuseOnlyIllumination = 1 if ssr else 0
    return pf, pv


def check_spec(orc, vq, got, pyr, hw, hh, levels, res, mips, name):
    """C5's bound: |delta| <= 1e-4 max(1, |ref|) + 2 S, S the oracle's own few-ulp sensitivity (tiny on a pole-flat HDRI)"""
    ids = np.arange(vq.cubemap_texel_count(res, mips), dtype=np.int64)
    ref = orc.specular_prefilter_texels(pyr, hw, hh, levels, res, mips, ids)
    sens = orc.specular_prefilter_sensitivity(pyr, hw, hh, levels, res, mips, ids)
    d = np.abs(got.astype(np.float64) - ref).max(axis=1)
    scale = np.maximum(1.0, np.abs(ref).max(axis=1))
    bound = 1e-4 * scale + 2.0 * sens
    assert (d <= bound).all(), f"{name}: {int((d > bound).sum())} texels outside the bound ({report(name, got, ref)})"
    assert float((d <= 1e-4 * scale).mean()) >= 0.995, name
    return ref


def lights_for(vq, w, h, spec_mips, shadowing=False):
    from vqengine_b200 import synth
    pf, _ = synth.scene_constants(w, h, spec_mips, seed=synth.SEED_BASE + 41, n_point=2, n_spot=1, directional=True)
    L = pf.Lights
    if shadowing:
        m = np.zeros(16, np.float32); m[0] = 1 / 25; m[5] = 1 / 25; m[14] = 0.5; m[15] = 1.0; m[1] = 0.01; m[4] = -0.02; m[12] = 0.1
        for k in range(16):
            L.shadowViewDirectional.m[k] = float(m[k])
        L.directional.shadowing = 1
        L.directional.depthBias = 0.001
    return L


def gbuffer_planes(w, h, seed):
    """synth's G-buffer with roughness over all of [0, 1]: exact 0 and 1 on some pixels, so MaxEnvMapLODLevels and every
    specular mip show"""
    from vqengine_b200 import synth
    planes = synth.gbuffer(w, h, seed=seed, emissive=True)
    rng = np.random.default_rng(seed)
    r = planes[1][..., 3]
    r[:] = rng.uniform(0.0, 1.0, r.shape)
    r[rng.uniform(0, 1, r.shape) < 0.1] = 0.0
    r[rng.uniform(0, 1, r.shape) < 0.1] = 1.0
    return planes


def constant_materials(n):
    from vqengine_b200 import synth
    mats, _ = synth.materials(n, tex_res=16, seed=synth.SEED_BASE + 43)
    for m in mats:
        m.textureConfig = 0.0
    return mats


def _env_lines(kind, hdri_name, w, h, diff, spec, maxcll=None):
    if kind == "texels":
        return [f"env_texels file={hdri_name} w={w} h={h} diff={diff} spec={spec} out=pyr.bin" + (f" maxcll={maxcll!r}" if maxcll else "")]
    return [f"env_hdr file={hdri_name} diff={diff} spec={spec} out=pyr.bin"]


def _env_info(out):
    line = [l for l in out if l.startswith("env ")]
    assert len(line) == 1, out
    return [int(x) for x in line[0].split()[1:]]


# ---- environment map: CreateRenderingResources + PreFilterEnvironmentMap ---------------------------------------------------------
@pytest.mark.parametrize("hw,hh,diff,spec", [(4, 2, 16, 32), (7, 3, 16, 32), (64, 32, 16, 32), (128, 64, 64, 64)],
                         ids=["4x2", "7x3", "64x32", "128x64"])
def test_prefilter_environment_map(driver, tmp_path, vq, orc, hw, hh, diff, spec):
    """the pyramid bit for bit, the unblurred diffuse cube (documented src_mip, the given step) against a float64-accumulated K2,
    each face's blur X then Y against the oracle on the device's unblurred face, every specular mip against K3 on the device
    pyramid with SpecMips = mip_level_count(SpecRes) - 1. HDRIs with <= 3 mips take the src_mip = HDRIMips - 1 branch."""
    img = spot_hdri(hw, hh)
    hd.put(tmp_path, "hdri.bin", img)
    out = hd.run(driver, tmp_path, ["init"] + _env_lines("texels", "hdri.bin", hw, hh, diff, spec, maxcll=1234.75) +
                 [f"prefilter step={DIFF_STEP!r} diff=diff.bin blurred=blurred.bin spec=spec.bin"])
    levels, spec_mips = vq.mip_level_count(hw, hh), expected_spec_mips(vq, spec)
    assert _env_info(out) == [hw, hh, levels, diff, spec, spec_mips, 1234]
    pyr = hd.get(tmp_path, "pyr.bin").reshape(-1, 4)
    assert np.array_equal(_bits(pyr), _bits(orc.hdri_build_mips(img, levels))), "pyramid"

    src = expected_src_mip(levels)
    got = hd.get(tmp_path, "diff.bin").reshape(-1, 4)
    ref = orc.diffuse_irradiance(pyr, hw, hh, levels, diff, step=DIFF_STEP, n_phi=0, n_theta=0, src_mip=src, f64_accum=True)
    print(assert_scaled(f"diffuse src_mip {src}", got, ref))
    if levels > 3:   # the rule matters: the neighbouring source mips give other cubes
        for other in (src - 1, src + 1):
            alt = orc.diffuse_irradiance(pyr, hw, hh, levels, diff, step=DIFF_STEP, n_phi=0, n_theta=0, src_mip=other, f64_accum=True)
            assert np.abs(alt - ref).max() > 100 * TOL, f"src_mip {other} is indistinguishable from {src}"

    blurred = hd.get(tmp_path, "blurred.bin").reshape(6, diff, diff, 4)
    faces = got.reshape(6, diff, diff, 4)
    for f in range(6):
        # two passes of the blur bound (1e-5 scaled each; the Y weights sum to 1, so X's error passes through unscaled)
        want = orc.gaussian_blur(orc.gaussian_blur(faces[f], False), True)
        d = np.abs(blurred[f].astype(np.float64) - want) / np.maximum(1.0, np.abs(want))
        assert np.isfinite(blurred[f]).all() and d.max() <= 2e-5, f"blurred face {f}: {d.max():.3e}"

    spec_got = hd.get(tmp_path, "spec.bin").reshape(-1, 4)
    assert spec_got.shape[0] == vq.cubemap_texel_count(spec, spec_mips)
    check_spec(orc, vq, spec_got, pyr, hw, hh, levels, spec, spec_mips, f"specular {spec}^2 x {spec_mips}")


def test_environment_from_hdr_file(driver, tmp_path, vq, orc):
    """CreateRenderingResourcesFromHDRFile: level 0 is the decoded file, the pyramid is built on it, MaxContentLightLevel is
    (int) of the file's maximum luminance"""
    img = spot_hdri(96, 48, spot=23.0)
    data = orc.hdr_encode(img)
    hd.put_bytes(tmp_path, "env.hdr", data)
    out = hd.run(driver, tmp_path, ["init"] + _env_lines("hdr", "env.hdr", 96, 48, 8, 16))
    rc, dec, lum = orc.hdr_decode(data)
    assert rc == 0 and lum > 1.0 and lum != int(lum)
    levels = vq.mip_level_count(96, 48)
    assert _env_info(out) == [96, 48, levels, 8, 16, expected_spec_mips(vq, 16), int(lum)]
    pyr = hd.get(tmp_path, "pyr.bin").reshape(-1, 4)
    assert np.array_equal(_bits(pyr[:96 * 48]), _bits(dec.reshape(-1, 4))), "level 0"
    assert np.array_equal(_bits(pyr), _bits(orc.hdri_build_mips(dec, levels))), "pyramid"


def test_load_default_resources_lut(driver, tmp_path, ctx, vq, orc):
    """LoadDefaultResources: a 1024^2 RG32F LUT at 2048 samples, bit for bit the C-ABI call; rows 0, 1, 511, 1023 at 1e-4 against
    the oracle"""
    out = hd.run(driver, tmp_path, ["init", "lut out=lut.bin"])
    assert "lut 1024 1024 8" in out
    got = hd.get(tmp_path, "lut.bin", (1024, 1024, 2))
    want = torch.zeros((1024, 1024, 2), dtype=torch.float32, device="cuda")
    ctx.brdf_integration_lut(want, 2048)
    assert np.array_equal(_bits(got), _bits(host(want)))
    for r in (0, 1, 511, 1023):
        ref = orc.brdf_integration_lut(1024, 1024, 2048, row_begin=r, row_end=r + 1)[r]
        assert_abs(f"lut row {r}", got[r], ref)


# ---- the scene passes -------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def scene_run(driver, tmp_path_factory, vq):
    """one renderer: 64x32 spot HDRI -> 8^2 diffuse (8 texels per face make the blur visible through the forward pass) / 32^2 specular, the LUT, a 70x37 window (display 140x74), then every
    RenderSceneColor overload and setting, the skydome and the reflection composites"""
    d = tmp_path_factory.mktemp("scene")
    hw, hh, w, h = 64, 32, 70, 37
    from vqengine_b200 import synth
    hd.put(d, "hdri.bin", spot_hdri(hw, hh))
    spec_mips = expected_spec_mips(vq, 32)
    L, Ls = lights_for(vq, w, h, spec_mips), lights_for(vq, w, h, spec_mips, shadowing=True)
    hd.put_bytes(d, "lights.bin", bytes(L))
    hd.put_bytes(d, "lights_sh.bin", bytes(Ls))
    planes = gbuffer_planes(w, h, seed=51)
    for i, p in enumerate(planes):
        hd.put(d, f"g{i}.bin", p)
    surf = synth.surface_inputs(w, h, 3, seed=synth.SEED_BASE + 52, ssao=False)
    for i, p in enumerate(surf):
        hd.put(d, f"s{i}.bin", p)
    mats = constant_materials(3)
    hd.put_bytes(d, "mats.bin", b"".join(bytes(m) for m in mats))
    rng = np.random.default_rng(53)
    dmap = rng.uniform(0.3, 0.7, (24, 16)).astype(np.float32)
    hd.put(d, "dir.bin", dmap)
    # RenderEnvironmentMap: the G-buffer normals with a third of the pixels cleared (no surface there)
    normal = planes[1].copy()
    normal[rng.uniform(0, 1, (h, w)) < 0.35, :3] = 0.0
    hd.put(d, "normal.bin", normal)
    vp, inv = synth.sky_view_proj(0.8, -0.3, 1.1, w / h)
    hd.put(d, "vp.bin", vp.astype(np.float32))
    hd.put(d, "singular.bin", np.zeros(16, np.float32))
    refl = rng.uniform(0.0, 2.0, (h, w, 4)).astype(np.float32)
    bv = rng.uniform(0.0, 1.0, (h, w, 4)).astype(np.float32)
    hd.put(d, "refl.bin", refl)
    hd.put(d, "bv.bin", bv)
    cam, yaw = (3.5, 6.0, -14.0), 0.7
    sc = f"lights=lights.bin cam={cam[0]},{cam[1]},{cam[2]} yaw={yaw} ambient=0.055"
    lines = ["init", "lut out=lut.bin", f"env_texels file=hdri.bin w={hw} h={hh} diff=8 spec=32 out=pyr.bin",
             f"prefilter step={DIFF_STEP!r} diff=diff.bin blurred=blurred.bin spec=spec.bin", f"window w={w} h={h} dw={2 * w} dh={2 * h}",
             f"scene planes=g0.bin,g1.bin,g2.bin,g3.bin {sc} out=gb.bin",
             f"scene planes=g0.bin,g1.bin,g2.bin,g3.bin {sc} ssr=1 out=gb_ssr.bin",
             f"scene planes=g0.bin,g1.bin,g2.bin,g3.bin {sc} hdr=1 out=gb_hdr.bin",
             f"scene_materials surface=s0.bin,s1.bin,s2.bin materials=mats.bin {sc} out=mat.bin",
             f"scene_materials surface=s0.bin,s1.bin,s2.bin materials=mats.bin {sc} hdr=1 out=mat_hdr.bin",
             f"scene planes=g0.bin,g1.bin,g2.bin {sc.replace('lights.bin', 'lights_sh.bin')} dir=dir.bin dir_w=16 dir_h=24 out=gb_sh.bin",
             f"scene_materials surface=s0.bin,s1.bin,s2.bin materials=mats.bin {sc.replace('lights.bin', 'lights_sh.bin')} "
             "dir=dir.bin dir_w=16 dir_h=24 out=mat_sh.bin",
             "sky vp=singular.bin normal=normal.bin out=unused.bin expect=fail",
             "sky vp=vp.bin normal=normal.bin out=sky.bin",
             "reflect refl=refl.bin out=refl_out.bin",
             "reflect refl=refl.bin bv=bv.bin out=refl_bv_out.bin"]
    out = hd.run(driver, d, lines)
    return dict(dir=d, out=out, hw=hw, hh=hh, w=w, h=h, L=L, Ls=Ls, planes=planes, surf=surf, mats=mats, dmap=dmap, normal=normal,
                vp=vp, inv=inv, refl=refl, bv=bv, cam=cam, yaw=yaw, spec_mips=spec_mips,
                pyr=hd.get(d, "pyr.bin").reshape(-1, 4), lut=hd.get(d, "lut.bin", (1024, 1024, 2)),
                diff=hd.get(d, "diff.bin").reshape(-1, 4), blurred=hd.get(d, "blurred.bin").reshape(-1, 4),
                spec=hd.get(d, "spec.bin").reshape(-1, 4))


def _forward_ref(orc, s, pf, pv, planes, cube="blurred"):
    return orc.forward_lighting(pf, pv, planes, s[cube], 8, s["spec"], 32, s["spec_mips"], s["lut"])


@pytest.mark.parametrize("kind", ["plain", "ssr", "hdr"])
def test_render_scene_color_gbuffer(scene_run, vq, orc, kind):
    """RenderSceneColor (G-buffer overload): the blurred diffuse cube, MaxEnvMapLODLevels = SpecMips, the yaw, the camera, the
    SSR diffuse-only flag. On the G-buffer path the ambient term rides in position.w, so an HDR display changes nothing there."""
    s = scene_run
    pf, pv = expected_constants(vq, s["L"], s["w"], s["h"], s["spec_mips"], cam=s["cam"], yaw=s["yaw"], hdr=kind == "hdr",
                                ssr=kind == "ssr")
    got = hd.get(s["dir"], {"plain": "gb.bin", "ssr": "gb_ssr.bin", "hdr": "gb_hdr.bin"}[kind], (s["h"], s["w"], 4))
    ref = _forward_ref(orc, s, pf, pv, s["planes"])
    print(assert_scaled(f"RenderSceneColor {kind}", got, ref))
    if kind == "plain":   # every constant the test pins is observable in this scene
        wrong = [("unblurred diffuse cube", pf, pv, "diff")]
        for field, value in (("MaxEnvMapLODLevels", s["spec_mips"] - 1), ("EnvironmentMapDiffuseOnlyIllumination", 1)):
            _, pv2 = expected_constants(vq, s["L"], s["w"], s["h"], s["spec_mips"], cam=s["cam"], yaw=s["yaw"])
            setattr(pv2, field, value)
            wrong.append((field, pf, pv2, "blurred"))
        pf2, _ = expected_constants(vq, s["L"], s["w"], s["h"], s["spec_mips"], cam=s["cam"], yaw=0.0)
        wrong.append(("yaw 0", pf2, pv, "blurred"))
        _, pv3 = expected_constants(vq, s["L"], s["w"], s["h"], s["spec_mips"], cam=(0.0, 0.0, 0.0), yaw=s["yaw"])
        wrong.append(("camera at the origin", pf, pv3, "blurred"))
        for name, a, b, cube in wrong:
            alt = _forward_ref(orc, s, a, b, s["planes"], cube)
            assert (np.abs(alt - ref) > 10 * TOL * np.maximum(1.0, np.abs(ref))).any(), f"{name} is not observable"


@pytest.mark.parametrize("hdr", [False, True], ids=["sdr", "hdr"])
def test_render_scene_color_from_materials(scene_run, vq, orc, hdr):
    """RenderSceneColorFromMaterials: gbuffer_from_materials with ambient 0.055 (SDR) or 0.055 x 0.005 (HDR display), then the
    forward pass with the blurred cube"""
    s = scene_run
    pf, pv = expected_constants(vq, s["L"], s["w"], s["h"], s["spec_mips"], cam=s["cam"], yaw=s["yaw"], hdr=hdr)
    gb = orc.gbuffer_from_materials(s["surf"], s["mats"], [{} for _ in s["mats"]], pf.fAmbientLightingFactor)
    got = hd.get(s["dir"], "mat_hdr.bin" if hdr else "mat.bin", (s["h"], s["w"], 4))
    ref = _forward_ref(orc, s, pf, pv, gb)
    print(assert_scaled(f"RenderSceneColorFromMaterials hdr={hdr}", got, ref))
    other = orc.gbuffer_from_materials(s["surf"], s["mats"], [{} for _ in s["mats"]], 0.055 if hdr else 0.055 * 0.005)
    assert (np.abs(_forward_ref(orc, s, pf, pv, other) - ref) > 10 * TOL * np.maximum(1.0, np.abs(ref))).any(), \
        "the ambient factor is not observable"


@pytest.mark.parametrize("path", ["gbuffer", "materials"])
def test_render_scene_color_shadowed(scene_run, vq, orc, path):
    """the shadowed overloads with only a directional map bound (16 x 24): its size replaces 2048, the point and spot kinds keep 1024"""
    s = scene_run
    pf, pv = expected_constants(vq, s["Ls"], s["w"], s["h"], s["spec_mips"], cam=s["cam"], yaw=s["yaw"], dims={"Directional": (16, 24)})
    # the G-buffer run binds no emissive plane; the materials pass produces one
    planes = s["planes"][:3] if path == "gbuffer" else orc.gbuffer_from_materials(s["surf"], s["mats"], [{} for _ in s["mats"]],
                                                                                  pf.fAmbientLightingFactor)
    def ref_with(pf_):
        return orc.forward_lighting_shadowed_e(pf_, pv, planes, s["blurred"], 8, s["spec"], 32, s["spec_mips"], s["lut"], dir_map=s["dmap"])
    got = hd.get(s["dir"], "gb_sh.bin" if path == "gbuffer" else "mat_sh.bin", (s["h"], s["w"], 4))
    ref = ref_with(pf)
    # test_shadow_gpu's PCF bound: a PCF tap may flip on the last ulp of tan / acos / pow, so count the pixels, not their size
    over = (np.abs(got.astype(np.float64) - ref) > TOL * np.maximum(1.0, np.abs(ref))).any(axis=-1)
    assert np.isfinite(got).all() and over.mean() <= 2e-3, f"shadowed {path}: {int(over.sum())} pixels outside ({report(path, got, ref)})"
    pf2, _ = expected_constants(vq, s["Ls"], s["w"], s["h"], s["spec_mips"], cam=s["cam"], yaw=s["yaw"])
    assert (np.abs(ref_with(pf2) - ref) > 10 * TOL * np.maximum(1.0, np.abs(ref))).any(axis=-1).mean() > 0.01, \
        "the directional map's size is not observable"


def test_render_environment_map(scene_run, vq, orc):
    """RenderEnvironmentMap: the skydome through the inverse of EnvironmentMapViewProj (float64 here, rounded to fp32) on level 0,
    only where the normal plane is 0, within frame_ref's ray bound; a singular matrix is refused with the documented error"""
    import frame_ref as fr
    s = scene_run
    assert any(l.startswith("refused sky:") and "EnvironmentMapViewProj is singular" in l for l in s["out"]), s["out"]
    h, w = s["h"], s["w"]
    before = hd.get(s["dir"], "mat_sh.bin", (h, w, 4))
    got = hd.get(s["dir"], "sky.bin", (h, w, 4))
    inv32 = np.linalg.inv(s["vp"].astype(np.float32).astype(np.float64)).astype(np.float32)
    lvl0 = s["pyr"][: s["hw"] * s["hh"]].reshape(s["hh"], s["hw"], 4)
    ref, bound, written, _ = fr.sky_ref(inv32.reshape(16), w, h, lvl0, None, s["normal"], before)
    assert written.any() and (~written).any()
    assert np.array_equal(_bits(got[~written]), _bits(before[~written])), "pixels with a surface changed"
    d = np.abs(got[..., :3].astype(np.float64) - ref[..., :3])
    assert (d <= bound).all(), f"skydome: {int((d > bound).sum())} values outside the bound, max excess {float((d - bound).max()):.3e}"
    o = orc.skydome(lvl0, s["hw"], s["hh"], 1, inv32.reshape(16), before.copy(), normal_mask=s["normal"])
    assert (np.abs(got[..., :3].astype(np.float64) - o[..., :3]) <= 2 * bound + 1e-6).all()
    # the transposed inverse looks elsewhere
    alt, _, _, _ = fr.sky_ref(inv32.T.reshape(16), w, h, lvl0, None, s["normal"], before)
    assert (np.abs(alt[..., :3] - ref[..., :3]) > 10 * bound + 1e-3).any()


def test_apply_reflections(scene_run, orc):
    """ApplyReflections with and without bounding volumes, on the layer's own scene colour, bit for bit"""
    s = scene_run
    h, w = s["h"], s["w"]
    sky = hd.get(s["dir"], "sky.bin", (h, w, 4))
    one = hd.get(s["dir"], "refl_out.bin", (h, w, 4))
    assert np.array_equal(_bits(one), _bits(orc.apply_reflections(sky.copy(), s["refl"])))
    two = hd.get(s["dir"], "refl_bv_out.bin", (h, w, 4))
    assert np.array_equal(_bits(two), _bits(orc.apply_reflections(one.copy(), s["refl"], s["bv"])))


def test_apply_reflections_pass(driver, tmp_path, orc):
    """ApplyReflectionsPass::RecordCommands: the variant without bounding volumes when SRVBoundingVolumes is null, with them
    otherwise; iSceneRT sizes that do not match the target are refused"""
    w, h = 33, 9
    rng = np.random.default_rng(61)
    tgt, refl, bv = (rng.uniform(0.0, 3.0, (h, w, 4)).astype(np.float32) for _ in range(3))
    bv[..., 3] = rng.uniform(0.0, 1.0, (h, w))
    for n, a in (("t.bin", tgt), ("r.bin", refl), ("b.bin", bv)):
        hd.put(tmp_path, n, a)
    out = hd.run(driver, tmp_path, ["init", f"reflect_pass target=t.bin refl=r.bin w={w} h={h} rtw={w} rth={h} out=o1.bin",
                                    f"reflect_pass target=t.bin refl=r.bin bv=b.bin w={w} h={h} rtw={w} rth={h} out=o2.bin",
                                    f"reflect_pass target=t.bin refl=r.bin w={w} h={h} rtw={w + 1} rth={h} out=o3.bin expect=fail"])
    assert any(l.startswith("refused reflect_pass:") and "do not match" in l for l in out), out
    assert np.array_equal(_bits(hd.get(tmp_path, "o1.bin", (h, w, 4))), _bits(orc.apply_reflections(tgt.copy(), refl)))
    assert np.array_equal(_bits(hd.get(tmp_path, "o2.bin", (h, w, 4))), _bits(orc.apply_reflections(tgt.copy(), refl, bv)))


# ---- RenderPostProcess ----------------------------------------------------------------------------------------------------------
def _post_abi(ctx, vq, orc, scene, mode, dw, dh, blur=False, sharpness=0.8, stops=0.2, check_stages=True):
    """the same post chain through the C-ABI with constants built here from the engine's rules: vq_post_process and the separate
    calls agree bit for bit, and each separate stage is within the C4 bound of the oracle on the device's previous stage"""
    from vqengine_b200 import synth
    h, w = scene.shape[:2]
    tm = synth.default_tonemapper()
    src = dev(scene)
    if blur:
        a, b = torch.empty_like(src), torch.empty_like(src)
        ctx.gaussian_blur(src, a, False)
        ctx.gaussian_blur(a, b, True)
        src = b
    cas = vq.cas_setup(sharpness, w, h, w, h) if mode == "cas" and sharpness > 0 else None
    easu = vq.fsr_easu_con(w, h, w, h, dw, dh) if mode == "fsr" else None
    rcas = vq.fsr_rcas_con(stops) if mode == "fsr" else None
    out = torch.empty((dh, dw, 4) if mode == "fsr" else (h, w, 4), dtype=torch.float32, device="cuda")
    ctx.post_process(tm, src, out, cas=cas, easu=easu, rcas=rcas)
    fused = host(out)
    t = torch.empty_like(src)
    ctx.tonemap(tm, src, t)
    ht = host(t)
    if check_stages:
        assert_abs("tonemap", ht, orc.tonemap(tm, host(src)))
    want = ht
    if cas is not None:
        c = torch.empty_like(t)
        ctx.cas(cas, t, c)
        want = host(c)
        if check_stages:
            assert_abs("cas", want, orc.cas(orc.cas_setup(sharpness, w, h, w, h), ht))
    if easu is not None:
        e = torch.empty((dh, dw, 4), dtype=torch.float32, device="cuda")
        ctx.fsr_easu(easu, t, e)
        r = torch.empty_like(e)
        ctx.fsr_rcas(rcas, e, r)
        he, want = host(e), host(r)
        if check_stages:
            assert_abs("easu", he, orc.fsr_easu(orc.fsr_easu_con(w, h, w, h, dw, dh), ht, dw, dh, 0))
            assert_abs("rcas", want, orc.fsr_rcas(orc.fsr_rcas_con(stops), he))
    assert np.array_equal(_bits(fused), _bits(want)), "vq_post_process and the separate calls differ"
    return fused


POST_CASES = [("none", 1.0, False, 0.8), ("none", 1.0, True, 0.8), ("cas", 1.0, False, 0.8), ("cas", 1.0, False, 0.0),
              ("fsr", 2.0, False, 0.8), ("fsr", 1.5, False, 0.8), ("fsr", 2.0, True, 0.8)]


@pytest.mark.parametrize("mode,ratio,blur,sharpness", POST_CASES,
                         ids=["none", "blur", "cas", "cas-sharpness0", "fsr2x", "fsr1.5x-quality", "blur-fsr2x"])
def test_render_post_process(driver, tmp_path, ctx, vq, orc, mode, ratio, blur, sharpness):
    """RenderPostProcess's branch and target: the display frame is the C-ABI chain's bit for bit, at display size with FSR (mRCASOut)
    and render size otherwise (mPostOut); CAS runs only with Sharpness > 0"""
    from vqengine_b200 import synth
    w, h = 70, 37
    dw, dh = int(w * ratio), int(h * ratio)
    planes = gbuffer_planes(w, h, seed=71)
    for i, p in enumerate(planes):
        hd.put(tmp_path, f"g{i}.bin", p)
    hd.put(tmp_path, "hdri.bin", spot_hdri(16, 8))
    hd.put_bytes(tmp_path, "lights.bin", bytes(lights_for(vq, w, h, 3)))
    out = hd.run(driver, tmp_path, ["init", "lut out=lut.bin", "env_texels file=hdri.bin w=16 h=8 diff=8 spec=8 out=pyr.bin",
                                    "prefilter step=0.1 diff=d.bin blurred=b.bin spec=s.bin", f"window w={w} h={h} dw={dw} dh={dh}",
                                    "scene planes=g0.bin,g1.bin,g2.bin,g3.bin lights=lights.bin cam=1,5,-12 out=scene.bin",
                                    f"post mode={mode} blur={int(blur)} sharpness={sharpness!r} out=post.bin"])
    ow, oh = (dw, dh) if mode == "fsr" else (w, h)
    assert f"post {ow} {oh}" in out, out
    scene = hd.get(tmp_path, "scene.bin", (h, w, 4))
    got = hd.get(tmp_path, "post.bin", (oh, ow, 4))
    want = _post_abi(ctx, vq, orc, scene, mode, ow, oh, blur=blur, sharpness=sharpness)
    assert np.array_equal(_bits(got), _bits(want)), f"{mode}: the layer's display frame differs from the C-ABI chain"
    if mode == "cas" and sharpness == 0.0:
        tm_only = _post_abi(ctx, vq, orc, scene, "none", w, h, check_stages=False)
        assert np.array_equal(_bits(got), _bits(tm_only))


def test_window_resizes_between_frames(driver, tmp_path, ctx, vq, orc):
    """OnWindowSizeChanged to a smaller and then a larger size between frames: each frame's scene colour and display frame have
    the new sizes and every row is the new frame's (no stale rows from the previous, larger or smaller, targets)"""
    sizes = [(70, 37), (40, 21), (96, 50)]
    hd.put(tmp_path, "hdri.bin", spot_hdri(16, 8))
    L = lights_for(vq, 70, 37, 3)
    hd.put_bytes(tmp_path, "lights.bin", bytes(L))
    lines = ["init", "lut out=lut.bin", "env_texels file=hdri.bin w=16 h=8 diff=8 spec=8 out=pyr.bin",
             "prefilter step=0.1 diff=d.bin blurred=b.bin spec=s.bin"]
    all_planes = []
    for k, (w, h) in enumerate(sizes):
        planes = gbuffer_planes(w, h, seed=80 + k)
        all_planes.append(planes)
        names = [hd.put(tmp_path, f"g{k}_{i}.bin", p) for i, p in enumerate(planes)]
        lines += [f"window w={w} h={h} dw={2 * w} dh={2 * h}",
                  f"scene planes={','.join(names)} lights=lights.bin cam=1,5,-12 out=scene{k}.bin",
                  f"post mode=fsr out=post{k}.bin"]
    out = hd.run(driver, tmp_path, lines)
    assert [l for l in out if l.startswith("post ")] == [f"post {2 * w} {2 * h}" for w, h in sizes]
    spec_mips = expected_spec_mips(vq, 8)
    lut = hd.get(tmp_path, "lut.bin", (1024, 1024, 2))
    blurred, spec = hd.get(tmp_path, "b.bin").reshape(-1, 4), hd.get(tmp_path, "s.bin").reshape(-1, 4)
    for k, (w, h) in enumerate(sizes):
        pf, pv = expected_constants(vq, L, w, h, spec_mips, cam=(1.0, 5.0, -12.0))
        scene = hd.get(tmp_path, f"scene{k}.bin", (h, w, 4))
        assert_scaled(f"scene {w}x{h}", scene, orc.forward_lighting(pf, pv, all_planes[k], blurred, 8, spec, 8, spec_mips, lut))
        got = hd.get(tmp_path, f"post{k}.bin", (2 * h, 2 * w, 4))
        want = _post_abi(ctx, vq, orc, scene, "fsr", 2 * w, 2 * h, check_stages=False)
        assert np.array_equal(_bits(got), _bits(want)), f"frame {k} ({w}x{h})"


# ---- file images ---------------------------------------------------------------------------------------------------------------
def test_save_and_downsize_hdr_file_images(driver, tmp_path, vq, orc):
    """SaveToHDRFileImage equals orc.hdr_encode of the same pixels; CreateEnvironmentMapFileImageFromHiRes equals decode -> Mitchell
    downsize -> encode in the oracle, byte for byte; a target larger than the source is refused"""
    img = spot_hdri(64, 32, spot=9.0)
    hd.put_bytes(tmp_path, "hi.hdr", orc.hdr_encode(img))
    rng = np.random.default_rng(91)
    g = [rng.uniform(0.0, 4.0, (9, 13, 4)).astype(np.float32) for _ in range(3)]
    names = [hd.put(tmp_path, f"g{i}.bin", p) for i, p in enumerate(g)]
    hd.put(tmp_path, "hdri.bin", spot_hdri(8, 4))
    hd.put_bytes(tmp_path, "lights.bin", bytes(lights_for(vq, 13, 9, 3)))
    out = hd.run(driver, tmp_path, ["init", "lut out=lut.bin", "env_texels file=hdri.bin w=8 h=4 diff=4 spec=8 out=pyr.bin",
                                    "prefilter step=0.1 diff=d.bin blurred=b.bin spec=s.bin", "window w=13 h=9 dw=13 dh=9",
                                    f"scene planes={','.join(names)} lights=lights.bin out=scene.bin", "save src=scene out=scene.hdr",
                                    "hires file=hi.hdr w=40 h=20 out=lo.hdr", "hires file=hi.hdr w=64 h=32 out=same.hdr",
                                    "hires file=hi.hdr w=65 h=32 out=x.hdr expect=fail"])
    assert any(l.startswith("refused hires:") and "must not be larger than the source" in l for l in out), out
    scene = hd.get(tmp_path, "scene.bin", (9, 13, 4))
    assert hd.get_bytes(tmp_path, "scene.hdr") == orc.hdr_encode(scene)
    rc, dec, _ = orc.hdr_decode(orc.hdr_encode(img))
    assert rc == 0
    assert hd.get_bytes(tmp_path, "lo.hdr") == orc.hdr_encode(orc.resize_downsample(dec, 40, 20))
    assert hd.get_bytes(tmp_path, "same.hdr") == orc.hdr_encode(orc.resize_downsample(dec, 64, 32))


# ---- IRenderPass objects -------------------------------------------------------------------------------------------------------
SPD_SIZES = [(64, 64), (70, 37), (1024, 4), (4, 1024), (1, 1), (1, 7), (4096, 2)]


@pytest.mark.parametrize("w,h", SPD_SIZES, ids=[f"{w}x{h}" for w, h in SPD_SIZES])
def test_single_pass_downsampler_pass(driver, tmp_path, vq, orc, w, h):
    """SinglePassDownsamplerPass: as many mips as SPD's count allows before a side reaches 0 (non-square and tiny inputs truncate
    early), each bit for bit the oracle's"""
    img = np.random.default_rng(w * 31 + h).uniform(0.0, 4.0, (h, w, 4)).astype(np.float32)
    hd.put(tmp_path, "in.bin", img)
    out = hd.run(driver, tmp_path, ["init", f"spd file=in.bin w={w} h={h} out=mips.bin"])
    _, c = vq.spd_setup(w, h)
    want_n = 0
    for l in range(1, c.mips + 1):
        if (w >> l) < 1 or (h >> l) < 1:
            break
        want_n = l
    line = [l for l in out if l.startswith("spd ")][0].split()
    assert int(line[1]) == want_n and line[2:] == [f"{w >> l}x{h >> l}" for l in range(1, want_n + 1)], line
    got = hd.get(tmp_path, "mips.bin").reshape(-1, 4)
    ref = orc.spd_downsample(img, want_n) if want_n else []
    assert got.shape[0] == sum(r.shape[0] * r.shape[1] for r in ref)
    o = 0
    for l, r in enumerate(ref, start=1):
        n = r.shape[0] * r.shape[1]
        assert np.array_equal(_bits(got[o:o + n]), _bits(r.reshape(-1, 4))), f"mip {l}"
        o += n


def test_single_pass_downsampler_refuses_4097_wide(driver, tmp_path):
    """a source wider than SPD's 4096 is refused by the C-ABI, and RecordCommands surfaces it through LastError"""
    hd.put(tmp_path, "in.bin", np.ones((2, 4097, 4), np.float32))
    out = hd.run(driver, tmp_path, ["init", "spd file=in.bin w=4097 h=2 out=mips.bin expect=fail"])
    assert any(l.startswith("refused spd:") and "SinglePassDownsamplerPass" in l and "4096" in l for l in out), out


@pytest.mark.parametrize("w,h", [(16, 16), (70, 37), (1, 5)])
def test_gaussian_blur_pass(driver, tmp_path, orc, w, h):
    """GaussianBlurPass: X into its own temporary, Y into the target, at the blur bound against the oracle on each pass"""
    img = np.random.default_rng(w + h).uniform(0.0, 6.0, (h, w, 4)).astype(np.float32)
    hd.put(tmp_path, "in.bin", img)
    hd.run(driver, tmp_path, ["init", f"blur_pass file=in.bin w={w} h={h} out=o.bin"])
    got = hd.get(tmp_path, "o.bin", (h, w, 4))
    want = orc.gaussian_blur(orc.gaussian_blur(img, False), True)
    d = np.abs(got.astype(np.float64) - want) / np.maximum(1.0, np.abs(want))
    assert np.isfinite(got).all() and d.max() <= 2e-5, d.max()


# ---- one engine frame ----------------------------------------------------------------------------------------------------------
def test_engine_frame_end_to_end(driver, tmp_path, ctx, vq, orc):
    """.hdr file image -> CreateRenderingResourcesFromHDRFile -> PreFilterEnvironmentMap -> LoadDefaultResources ->
    RenderSceneColorFromMaterials -> RenderEnvironmentMap -> ApplyReflections -> RenderPostProcess (FSR 2x) -> SaveToHDRFileImage,
    every stage held to its reference on the device's previous stage"""
    import frame_ref as fr
    from vqengine_b200 import synth
    hw, hh, w, h = 64, 32, 70, 37
    img = spot_hdri(hw, hh, spot=30.0)
    data = orc.hdr_encode(img)
    hd.put_bytes(tmp_path, "env.hdr", data)
    spec_mips = expected_spec_mips(vq, 32)
    L = lights_for(vq, w, h, spec_mips)
    hd.put_bytes(tmp_path, "lights.bin", bytes(L))
    surf = synth.surface_inputs(w, h, 3, seed=synth.SEED_BASE + 101, ssao=False)
    for i, p in enumerate(surf):
        hd.put(tmp_path, f"s{i}.bin", p)
    mats = constant_materials(3)
    hd.put_bytes(tmp_path, "mats.bin", b"".join(bytes(m) for m in mats))
    rng = np.random.default_rng(102)
    normal = surf[1].copy()
    normal[rng.uniform(0, 1, (h, w)) < 0.3, :3] = 0.0
    hd.put(tmp_path, "normal.bin", normal)
    vp, _ = synth.sky_view_proj(-1.2, 0.2, 1.0, w / h)
    hd.put(tmp_path, "vp.bin", vp.astype(np.float32))
    refl = rng.uniform(0.0, 1.0, (h, w, 4)).astype(np.float32)
    hd.put(tmp_path, "refl.bin", refl)
    out = hd.run(driver, tmp_path, [
        "init", "env_hdr file=env.hdr diff=16 spec=32 out=pyr.bin",
        f"prefilter step={DIFF_STEP!r} diff=diff.bin blurred=blurred.bin spec=spec.bin", "lut out=lut.bin",
        f"window w={w} h={h} dw={2 * w} dh={2 * h}",
        "scene_materials surface=s0.bin,s1.bin,s2.bin materials=mats.bin lights=lights.bin cam=2,4,-15 yaw=-0.4 out=scene.bin",
        "sky vp=vp.bin normal=normal.bin out=sky.bin", "reflect refl=refl.bin out=refl.out.bin", "post mode=fsr out=display.bin",
        "save src=post out=display.hdr"])
    # 1-2: the file image's pyramid and light level
    rc, dec, lum = orc.hdr_decode(data)
    levels = vq.mip_level_count(hw, hh)
    assert rc == 0 and _env_info(out) == [hw, hh, levels, 16, 32, spec_mips, int(lum)]
    pyr = hd.get(tmp_path, "pyr.bin").reshape(-1, 4)
    assert np.array_equal(_bits(pyr), _bits(orc.hdri_build_mips(dec, levels)))
    # 3: the prefilter
    diff = hd.get(tmp_path, "diff.bin").reshape(-1, 4)
    assert_scaled("diffuse", diff, orc.diffuse_irradiance(pyr, hw, hh, levels, 16, step=DIFF_STEP, n_phi=0, n_theta=0,
                                                          src_mip=expected_src_mip(levels), f64_accum=True))
    blurred = hd.get(tmp_path, "blurred.bin").reshape(-1, 4)
    faces = diff.reshape(6, 16, 16, 4)
    bref = np.concatenate([orc.gaussian_blur(orc.gaussian_blur(f, False), True).reshape(-1, 4) for f in faces])
    assert (np.abs(blurred.astype(np.float64) - bref) / np.maximum(1.0, np.abs(bref))).max() <= 2e-5
    spec = hd.get(tmp_path, "spec.bin").reshape(-1, 4)
    check_spec(orc, vq, spec, pyr, hw, hh, levels, 32, spec_mips, "specular")
    # 4: the LUT (bit for bit the C-ABI call's)
    lut = hd.get(tmp_path, "lut.bin", (1024, 1024, 2))
    want = torch.zeros((1024, 1024, 2), dtype=torch.float32, device="cuda")
    ctx.brdf_integration_lut(want, 2048)
    assert np.array_equal(_bits(lut), _bits(host(want)))
    # 5: the materials pass
    pf, pv = expected_constants(vq, L, w, h, spec_mips, cam=(2.0, 4.0, -15.0), yaw=-0.4)
    gb = orc.gbuffer_from_materials(surf, mats, [{} for _ in mats], pf.fAmbientLightingFactor)
    scene = hd.get(tmp_path, "scene.bin", (h, w, 4))
    assert_scaled("scene", scene, orc.forward_lighting(pf, pv, gb, blurred, 16, spec, 32, spec_mips, lut))
    # 6: the skydome where no surface is
    sky = hd.get(tmp_path, "sky.bin", (h, w, 4))
    inv32 = np.linalg.inv(vp.astype(np.float32).astype(np.float64)).astype(np.float32)
    ref, bound, written, _ = fr.sky_ref(inv32.reshape(16), w, h, pyr[: hw * hh].reshape(hh, hw, 4), None, normal, scene)
    assert np.array_equal(_bits(sky[~written]), _bits(scene[~written]))
    assert (np.abs(sky[..., :3].astype(np.float64) - ref[..., :3]) <= bound).all()
    # 7: the reflections
    composite = hd.get(tmp_path, "refl.out.bin", (h, w, 4))
    assert np.array_equal(_bits(composite), _bits(orc.apply_reflections(sky.copy(), refl)))
    # 8: the post chain, FSR 2x
    assert f"post {2 * w} {2 * h}" in out
    display = hd.get(tmp_path, "display.bin", (2 * h, 2 * w, 4))
    assert np.array_equal(_bits(display), _bits(_post_abi(ctx, vq, orc, composite, "fsr", 2 * w, 2 * h)))
    # 9: the saved file image
    assert hd.get_bytes(tmp_path, "display.hdr") == orc.hdr_encode(display)
