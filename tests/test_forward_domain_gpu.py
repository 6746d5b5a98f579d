"""-m gpu: K1 over the whole domain of its inputs (tests/forward_domain.py): sampler probes against the float64 sampling
rules and the oracle, and whole-pixel parity on adversarial G-buffers against the oracle."""
import math

import numpy as np
import pytest
import torch

import forward_domain as fd
import sampling_ref as sr
from gpu_util import dev, host, assert_scaled

pytestmark = pytest.mark.gpu


def _env(vq, env):
    t = {k: dev(env[k]) for k in ("diff", "spec", "lut")}
    em = vq.EnvironmentMaps(vq.cubemap_of(t["diff"], env["diff_res"], env["diff_mips"]),
                            vq.cubemap_of(t["spec"], env["spec_res"], env["spec_mips"]), vq.image_of(t["lut"], 2))
    return em, t


def _gbuffer(vq, planes):
    d = [dev(p) for p in planes]
    gb = vq.GBuffer(vq.image_of(d[0]), vq.image_of(d[1]), vq.image_of(d[2]), vq.image_of(d[3]) if len(d) > 3 else vq.null_image())
    return gb, d


def _shade(ctx, vq, pf, pv, planes, env, rows=None):
    """K1 with sampling copies built per call and from vq_environment_prepare: the two must agree bit for bit (pixels
    without a surface shade to NaN in both: the skydome pass fills them)"""
    h, w = planes[0].shape[:2]
    gb, keep = _gbuffer(vq, planes)
    em, tk = _env(vq, env)
    rb, re = rows or (0, h)
    outs = []
    for prepared in (False, True):
        ctx.environment_invalidate()
        if prepared:
            ctx.environment_prepare(em)
        out = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        ctx.forward_lighting(pf, pv, gb, em, out, rb, re)
        outs.append(host(out))
    ctx.environment_invalidate()
    assert np.array_equal(outs[0], outs[1], equal_nan=True), "prepared sampling copies differ from the per-call ones"
    return outs[0]


def _oracle(orc, pf, pv, planes, env, rows=None):
    h = planes[0].shape[0]
    rb, re = rows or (0, h)
    return orc.forward_lighting(pf, pv, planes, env["diff"], env["diff_res"], env["spec"], env["spec_res"], env["spec_mips"],
                                env["lut"], rb, re)


def _probe_check(name, got, ref, p):
    """|K1 - float64| within the probe's per-pixel bound, and |K1 - oracle| within twice it (the oracle is itself inside
    the bound, test_forward_domain.py)"""
    assert np.isfinite(got).all(), name
    e64 = np.abs(got[..., :3].astype(np.float64) - p["want"]).max(-1)
    eor = np.abs(got[..., :3].astype(np.float64) - ref[..., :3]).max(-1)
    r64, ror = float((e64 / p["tol"]).max()), float((eor / (2 * p["tol"])).max())
    print(f"{name}: max |K1 - float64| = {e64.max():.2e} ({r64:.3f} of the bound), max |K1 - oracle| = {eor.max():.2e}")
    assert r64 <= 1.0 and ror <= 1.0, (name, r64, ror, np.unravel_index(np.argmax(e64 / p["tol"]), e64.shape))
    assert (got[..., 3] == p["planes"][1][..., 3]).all()


N_UNIFORM = 30_000


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_specular_probe(ctx, vq, orc, res):
    """specular sample at reflect(-V, N) and mip int(roughness * MAX_LOD), every mip of a cube with random texels,
    MaxEnvMapLODLevels in {mips, mips-2, mips+3, 4.7, 0}"""
    env = fd.probe_env("spec", fd.make_env(5, res, (20, 48), seed=res))
    mips = env["spec_mips"]
    for max_lod, offset in ((mips, 0.0), (mips - 2, 0.0), (mips + 3, 0.0), (4.7, 0.0), (0, 0.0), (mips, 0.7)):
        p = fd.specular_probe(env, max_lod, N_UNIFORM, seed=res * 31 + int(max_lod * 10), offset=offset)
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)
        _probe_check(f"spec res {res} lod {max_lod} offset {offset}", got, _oracle(orc, p["pf"], p["pv"], p["planes"], env), p)


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_diffuse_probe(ctx, vq, orc, res):
    """(1 - 0.04f) * diffuse sample at the (rotated) raw normal; the diffuse cube carries its whole mip chain and K1 must
    read mip 0"""
    env = fd.probe_env("diff", fd.make_env(res, 2, (20, 48), seed=res))
    for offset in (0.0, 0.7, math.pi):
        p = fd.diffuse_probe(env, N_UNIFORM, seed=res * 13 + int(offset * 10), offset=offset)
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)
        _probe_check(f"diff res {res} offset {offset:.3f}", got, _oracle(orc, p["pf"], p["pv"], p["planes"], env), p)


@pytest.mark.parametrize("wh", sr.LUT_SIZES)
def test_lut_probe(ctx, vq, orc, wh):
    """each LUT channel on its own at (saturate(dot(N, V)), roughness), N.V from back-facing to exactly 1"""
    for ch in (0, 1):
        env = fd.probe_env("lut", fd.make_env(2, 5, wh, seed=wh[0] + wh[1]), channel=ch)
        p = fd.lut_probe(env, ch, 2 * N_UNIFORM, seed=wh[0] * 7 + ch)
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)
        _probe_check(f"lut {wh} channel {ch}", got, _oracle(orc, p["pf"], p["pv"], p["planes"], env), p)


# ---- whole pixels -------------------------------------------------------------------------------------------------
CAM = (0.0, 5.0, -17.0)
# (w, h, rows, diffuse res, specular res, LUT (W, H), HDRI offset, emissive, MaxEnvMapLODLevels (None: mips), diffuse-only)
CASES = [
    (515, 37, None, 16, 33, (48, 20), 0.0, False, None, False),
    (515, 37, None, 33, 5, (20, 48), 0.7, True, "mips+3", False),
    (256, 8, None, 5, 16, (1, 1), -0.0, False, 4.7, False),
    (256, 8, None, 2, 2, (48, 20), 1e-8, True, "mips-2", False),
    (130, 21, (5, 18), 1, 33, (20, 48), math.pi, False, 0, False),
    (515, 37, None, 16, 16, (48, 20), 0.7, True, None, True),
]


def _case_inputs(case, seed, sky_frac=0.0):
    w, h, rows, dres, sres, lut, off, emissive, lod, diff_only = case
    env = fd.make_env(dres, sres, lut, seed=seed)
    mips = env["spec_mips"]
    max_lod = {None: mips, "mips+3": mips + 3, "mips-2": mips - 2}.get(lod, lod)
    planes, sky = fd.adversarial_gbuffer(w, h, seed, CAM, emissive=emissive, sky_frac=sky_frac)
    pf, pv = fd.constants(CAM, max_lod, off, lights=fd.lights(w, h, seed, off), diffuse_only=diff_only)
    return env, planes, sky, pf, pv, rows


@pytest.mark.parametrize("k", range(len(CASES)))
def test_forward_adversarial_parity(ctx, vq, orc, k):
    env, planes, _, pf, pv, rows = _case_inputs(CASES[k], seed=500 + k)
    got = _shade(ctx, vq, pf, pv, planes, env, rows)
    ref = _oracle(orc, pf, pv, planes, env, rows)
    rb, re = rows or (0, planes[0].shape[0])
    print(assert_scaled(f"adversarial case {k}", got[rb:re], ref[rb:re]))
    assert (got[:rb] == 0).all() and (got[re:] == 0).all()


def test_forward_mirror_kat(ctx, vq, orc):
    """roughness 0 and 0.01, N = +Y, P = 0, camera (-4, 4, 0), point light (2, 2, 0): V and Wi are mirror images with
    bit-identical components, so H = N exactly, N.H = 1, GGX's t = 0 and the `denom < EPSILON -> D = 1` escape decides the
    highlight. Environment maps and ao are zero, so the output is BRDF * radiance * N.L alone, computed here in float64."""
    a, b = 4.0, 2.0
    pf, pv = fd.constants((-a, a, 0.0), 1)
    L = pf.Lights
    L.numPointLights = 1
    l = L.point_lights[0]
    l.position.x, l.position.y, l.position.z = b, b, 0.0
    l.range, l.brightness = 100.0, 50.0
    l.color.x, l.color.y, l.color.z = 1.0, 0.5, 0.25
    rough = np.array([0.0, 0.01], np.float32)
    pos = np.zeros((1, 2, 4), np.float32)
    nrm = np.zeros((1, 2, 4), np.float32); nrm[..., 1] = 1.0; nrm[0, :, 3] = rough
    alb = np.zeros((1, 2, 4), np.float32); alb[..., :3] = (0.5, 0.25, 0.75)
    env = fd.make_env(2, 2, (2, 2), seed=9, diff=np.zeros((30, 4), np.float32), spec=np.zeros((30, 4), np.float32),
                      lut=np.zeros((2, 2, 2), np.float32))
    got = _shade(ctx, vq, pf, pv, [pos, nrm, alb], env)
    ref = _oracle(orc, pf, pv, [pos, nrm, alb], env)
    c = 1.0 / math.sqrt(2.0)                          # N.V = N.L = H.V
    col = np.array([1.0, 0.5, 0.25])
    alb64 = np.array([0.5, 0.25, 0.75])
    F = 0.04 + 0.96 * (1.0 - c) ** 5                  # F0 = 0.04 (metalness 0); Fresnel_Schlick(H, V)
    want = []
    for r in rough.astype(np.float64):
        k = (r + 1.0) ** 2 / 8.0
        G = (c / (c * (1 - k) + k + 1e-4)) ** 2
        spec = F * 1.0 * G / max(4 * c * c, 1e-4)     # D = 1
        diff = (1.0 - F) * alb64 / math.pi
        want.append((diff + spec) * col * 50.0 / (2 * b * b) * c)
    want = np.array(want)
    print("mirror KAT", got[0, :, :3], want)
    assert np.isfinite(got).all()
    assert np.abs(got[0, :, :3] - want).max() <= 1e-5 * np.abs(want).max()
    assert_scaled("mirror KAT vs oracle", got, ref)


def test_forward_sky_pixels_do_not_touch_neighbours(ctx, vq, orc):
    """~10 % all-zero texels (no surface) interleaved with surface pixels: the surface pixels meet the parity bound, and
    they are bit-identical to a frame whose holes hold surface pixels of roughness 0 (every warp votes for the TINY loop
    in both, as a cleared texel has roughness 0)"""
    case = CASES[0]
    env, planes, sky, pf, pv, _ = _case_inputs(case, seed=77, sky_frac=0.1)
    assert 0.05 < sky.mean() < 0.15
    got = _shade(ctx, vq, pf, pv, planes, env)
    ref = _oracle(orc, pf, pv, planes, env)
    surf = ~sky
    print(assert_scaled("sky frame, surface pixels", got[surf], ref[surf]))
    full, _ = fd.adversarial_gbuffer(case[0], case[1], 78, CAM, emissive=case[7])
    filled = [p.copy() for p in planes]
    for p, q in zip(filled, full):
        p[sky] = q[sky]
    filled[1][sky, 3] = 0.0
    got2 = _shade(ctx, vq, pf, pv, filled, env)
    assert np.array_equal(got[surf], got2[surf])


def test_forward_multi_rotated_equals_single(ctx, vq, orc):
    """forward_kernel<MULTI=1, ROT=1>: the fused multi-destination store with a rotated HDRI equals the single-destination
    call bit for bit"""
    env, planes, _, pf, pv, _ = _case_inputs(CASES[1][:7] + (False, None, False), seed=91)
    assert pf.fHDRIOffsetInRadians == np.float32(0.7)
    h, w = planes[0].shape[:2]
    single = _shade(ctx, vq, pf, pv, planes, env)
    gb, keep = _gbuffer(vq, planes)
    em, tk = _env(vq, env)
    frames = [torch.zeros((h + 3, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    ctx.forward_lighting_multi(pf, pv, gb, em, [vq.image_of(f) for f in frames], dst_row_offset=3)
    for f in frames:
        got = host(f)
        assert np.array_equal(got[3:], single) and (got[:3] == 0).all()
