"""-m gpu: K1's domain (tests/forward_domain.py, tests/light_domain.py) through the one-pass PSMain kernels, with the inputs in the
fused kernel's form (tests/psmain_domain.py), unfolded and folded onto psmain's warps.

For every probe family: without yaw, vq_forward_lighting_from_materials equals vq_gbuffer_from_materials -> vq_forward_lighting
bit for bit; with or without yaw, it meets the domain's own float64 check re-evaluated on the G-buffer the producer made (the
probe bound, the fp32 range rule, the spot interval, the escape decision, HDR parity with the oracle). With yaw (the ROT
instantiations) the two paths may differ in the last bits of the rotated lookup direction; the difference is bounded by what a
2^-21 relative change of both cube directions can do to the samples. The shadowed kernel with +Inf shadow cubes and a dark caster
equals the unshadowed one, the multi-destination kernel equals the single call, and odd row ranges store nothing outside them."""
import math

import numpy as np
import pytest
import torch

import forward_domain as fd
import light_domain as ld
import light_ref as lr
import psmain_domain as pd
import sampling_ref as sr
from gpu_util import assert_scaled, dev, host
from test_forward_domain_gpu import CASES, _case_inputs, _env, _probe_check
from test_light_domain_gpu import parity, term, zenv

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0
GB_INIT = -7.0
N_UNIFORM = 8_000
ROT_REL = 2.0 ** -21            # relative change of a rotated lookup direction the ROT bound allows


def _pf1(pf):
    """the frame with fAmbientLightingFactor = 1: the producer's ao is 1 * ssao, exact"""
    q = ld.copy_pf(pf)
    q.fAmbientLightingFactor = 1.0
    return q


def _inputs(vq, planes):
    sp, mats = pd.adapt(planes)
    d = [dev(p) for p in sp]
    si = vq.SurfaceInputs(vq.image_of(d[0]), vq.image_of(d[1]), vq.image_of(d[2]), vq.image_of(d[3], 1))
    return si, mats, d


def run(ctx, vq, planes, pf, pv, env, rows=None, shadowed=False, multi=None):
    """(fused, two-pass, produced G-buffer planes) on the adapted inputs under the frame's own lights; outputs start as SENTINEL.
    shadowed: the frame with a dark point caster appended (ld.with_dark_caster) through the fused kernel and through the shadowed
    kernel with +Inf point cubes, asserted equal; multi: destination counts (>= 2: the MULTI instantiation) for
    forward_lighting_from_materials_multi at row offset 2, asserted equal to the fused call"""
    assert all(n >= 2 for n in multi or ()), "one destination launches the single-destination kernel"
    pf = _pf1(pf)
    h, w = planes[0].shape[:2]
    rb, re = rows or (0, h)
    si, mats, keep = _inputs(vq, planes)
    table = ctx.material_table(mats, [vq.MaterialTextures() for _ in mats])
    em, tk = _env(vq, env)
    ctx.environment_prepare(em)
    gbt = [dev(np.full((h, w, 4), GB_INIT, np.float32)) for _ in range(4)]
    gb = vq.GBuffer(*(vq.image_of(t) for t in gbt))
    ctx.gbuffer_from_materials(si, table, 1.0, gb, row_begin=rb, row_end=re)
    two = dev(np.full((h, w, 4), SENTINEL, np.float32))
    ctx.forward_lighting(pf, pv, gb, em, two, row_begin=rb, row_end=re)
    fused = dev(np.full((h, w, 4), SENTINEL, np.float32))
    ctx.forward_lighting_from_materials(pf, pv, si, table, em, fused, row_begin=rb, row_end=re)
    got = host(fused)
    if shadowed:
        pfc = ld.with_dark_caster(pf)
        plain = dev(np.full((h, w, 4), SENTINEL, np.float32))
        ctx.forward_lighting_from_materials(pfc, pv, si, table, em, plain, row_begin=rb, row_end=re)
        cubes = dev(np.full((pfc.Lights.numPointCasters, 6, 2, 2), np.inf, np.float32))
        sh = dev(np.full((h, w, 4), SENTINEL, np.float32))
        ctx.forward_lighting_shadowed_from_materials(pfc, pv, si, table, em, sh, point_cubes=cubes, row_begin=rb, row_end=re)
        assert np.array_equal(host(sh).view(np.uint32), host(plain).view(np.uint32)), "shadowed fused kernel differs from the plain one"
    for n in multi or ():
        frames = [torch.full((h + 2, w, 4), SENTINEL, dtype=torch.float32, device="cuda") for _ in range(n)]
        ctx.forward_lighting_from_materials_multi(pf, pv, si, table, em, [vq.image_of(f) for f in frames], dst_row_offset=2,
                                                  row_begin=rb, row_end=re)
        for f in frames:
            g = host(f)
            assert np.array_equal(g[2:].view(np.uint32), got.view(np.uint32)) and (g[:2] == SENTINEL).all(), f"multi x{n}"
    want = host(two)
    gbp = [host(t) for t in gbt]
    table.close()
    ctx.environment_invalidate()
    return got, want, gbp


def _rotated(pf):
    return float(pf.fHDRIOffsetInRadians) != 0.0


def equal_or_rot_bound(name, got, want, pf, env):
    """bit for bit without yaw; with yaw, report and bound the differences: a rotated direction off by ROT_REL moves the diffuse
    sample (weight <= 1) and the specular sample (weight Ks * LUT.x + LUT.y <= 2) by fd._cube_tol each, plus a few ulp"""
    diff = (got.view(np.uint32) != want.view(np.uint32)).any(-1)
    if not _rotated(pf):
        assert not diff.any(), f"{name}: {int(diff.sum())} pixels differ from the two-pass result, first {np.argwhere(diff)[0]}"
        return 0, 0.0
    d = np.abs(got[..., :3].astype(np.float64) - want[..., :3]).max(-1)
    span = lambda a: float(a.max() - a.min())
    bound = (fd._cube_tol(float(env["diff_res"]), ROT_REL, span(env["diff"])) +
             2 * fd._cube_tol(float(env["spec_res"]), ROT_REL, span(env["spec"])) + 16 * fd.U24 * np.abs(want[..., :3]).max(-1))
    ratio = float((d / bound).max())
    print(f"{name}: yaw: {int(diff.sum())} of {diff.size} pixels differ from the two-pass result, largest {d.max():.2e} "
          f"({ratio:.3f} of the bound)")
    assert ratio <= 1.0, (name, ratio)
    return int(diff.sum()), float(d.max())


def _variants(p):
    """the probe unfolded and folded (cropped to a multiple of 256 columns first when it is wider)"""
    yield p
    w = p["planes"][0].shape[1]
    if w >= pd.TILE:
        q = pd.crop(p, w - w % pd.TILE) if w % pd.TILE else p
        yield pd.fold_probe(q)


def _record(family, ratio):
    print(f"family {family}: {ratio:.3f} of its bound")


# ---- forward-domain sampler probes --------------------------------------------------------------------------------------
def _sampler(ctx, vq, orc, family, p, env, expect):
    for q in _variants(dict(p, name=family)):
        got, want, gb = run(ctx, vq, q["planes"], q["pf"], q["pv"], env, shadowed=True)
        equal_or_rot_bound(q["name"], got, want, q["pf"], env)
        w64, tol = expect(gb)
        ref = orc.forward_lighting(_pf1(q["pf"]), q["pv"], gb, env["diff"], env["diff_res"], env["spec"], env["spec_res"],
                                   env["spec_mips"], env["lut"])
        _probe_check(q["name"], got, ref, dict(planes=gb, want=w64, tol=tol))
        _record(family.split(" ")[0], float((np.abs(got[..., :3] - w64).max(-1) / tol).max()))


def _cam(pv):
    return (pv.CameraPosition.x, pv.CameraPosition.y, pv.CameraPosition.z)


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_specular_probe(ctx, vq, orc, res):
    env = fd.probe_env("spec", fd.make_env(5, res, (20, 48), seed=res))
    mips = env["spec_mips"]
    for max_lod, offset in ((mips, 0.0), (mips - 2, 0.0), (mips + 3, 0.0), (4.7, 0.0), (0, 0.0), (mips, 0.7)):
        p = fd.specular_probe(env, max_lod, N_UNIFORM, seed=res * 31 + int(max_lod * 10), offset=offset)
        _sampler(ctx, vq, orc, f"specular res {res} lod {max_lod} offset {offset}", p, env,
                 lambda gb: fd.specular_expect(env, gb, _cam(p["pv"]), max_lod, offset))


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_diffuse_probe(ctx, vq, orc, res):
    env = fd.probe_env("diff", fd.make_env(res, 2, (20, 48), seed=res))
    for offset in (0.0, 0.7, math.pi):
        p = fd.diffuse_probe(env, N_UNIFORM, seed=res * 13 + int(offset * 10), offset=offset)
        _sampler(ctx, vq, orc, f"diffuse res {res} offset {offset:.3f}", p, env, lambda gb: fd.diffuse_expect(env, gb, offset))


@pytest.mark.parametrize("wh", sr.LUT_SIZES)
def test_lut_probe(ctx, vq, orc, wh):
    for ch in (0, 1):
        env = fd.probe_env("lut", fd.make_env(2, 5, wh, seed=wh[0] + wh[1]), channel=ch)
        p = fd.lut_probe(env, ch, 2 * N_UNIFORM, seed=wh[0] * 7 + ch)
        _sampler(ctx, vq, orc, f"lut{ch} {wh}", p, env, lambda gb: fd.lut_expect(env, ch, gb, _cam(p["pv"])))


@pytest.mark.parametrize("k", range(len(CASES)))
def test_adversarial_cases(ctx, vq, orc, k):
    """the adversarial G-buffers (diffuse-only, emissive and a row range from an odd row included): HDR parity with the oracle
    on the produced G-buffer inside the range, nothing stored outside it; the shadowed kernel equals the plain one; cases 0, 1 and
    4 also through the multi-destination kernel"""
    env, planes, _, pf, pv, rows = _case_inputs(CASES[k], seed=500 + k)
    p = dict(name=f"adversarial case {k}", planes=planes, pf=pf, pv=pv)
    for q in _variants(p):
        rb, re = rows or (0, q["planes"][0].shape[0])
        got, want, gb = run(ctx, vq, q["planes"], q["pf"], q["pv"], env, rows=(rb, re), shadowed=True,
                            multi=(2, 3) if k in (0, 1, 4) else ())
        equal_or_rot_bound(q["name"], got, want, q["pf"], env)
        assert (got[:rb] == SENTINEL).all() and (got[re:] == SENTINEL).all(), q["name"]
        ref = orc.forward_lighting(_pf1(q["pf"]), q["pv"], gb, env["diff"], env["diff_res"], env["spec"], env["spec_res"],
                                   env["spec_mips"], env["lut"], rb, re)
        r = assert_scaled(q["name"], got[rb:re], ref[rb:re])
        _record("adversarial", r["max_scaled"] / 1e-4)
        print(r)


# ---- light-domain families ----------------------------------------------------------------------------------------------
def _light(ctx, vq, orc, p, shadowed=True, multi=()):
    env = p.get("env") or zenv()
    got, want, gb = run(ctx, vq, p["planes"], p["pf"], p["pv"], env, shadowed=shadowed, multi=multi)
    equal_or_rot_bound(p["name"], got, want, p["pf"], env)
    ref = orc.forward_lighting(_pf1(p["pf"]), p["pv"], gb, env["diff"], env["diff_res"], env["spec"], env["spec_res"],
                               env["spec_mips"], env["lut"])
    return got, ref, gb


def _rec(r, family):
    _record(family, r["max_scaled"] / 1e-4)


def test_range(ctx, vq, orc):
    """lit exactly where the fp32 range rule says (positions reach the kernel bit for bit), a pixel at the light adds 0, and the
    oracle is non-finite exactly at lit pixels at the light"""
    for p0 in ld.range_probes():
        for p in _variants(p0):
            got, ref, _ = _light(ctx, vq, orc, p, multi=(2,) if p0 is not p else ())
            t, at = term(got), p["at_light"]
            assert np.array_equal(t[~at] != 0, p["lit"][~at]), p["name"]
            assert (got[at][:, :3] == 0).all(), p["name"]
            assert np.array_equal(~np.isfinite(ref).all(-1), at & p["lit"]), p["name"]
            _rec(parity(p["name"], got, ref, at), "range")


def test_spot(ctx, vq, orc):
    """fused(spot) / fused(point light at the spot's position) inside the float64 interval; parity where decided"""
    for p0 in ld.spot_probes():
        for p in _variants(p0):
            got, ref, _ = _light(ctx, vq, orc, p)
            pt, _, _ = _light(ctx, vq, orc, dict(p, pf=p["point"][0], pv=p["point"][1]), shadowed=False)
            ts, tp = term(got), term(pt)
            at = p["at_light"]
            obs = ~at & (tp > 0)
            ratio = ts[obs] / tp[obs]
            bad = (ratio < p["lo"][obs] - 8 * lr.U24) | (ratio > p["hi"][obs] + 8 * lr.U24)
            assert not bad.any(), (p["name"], ratio[bad][:4])
            nanc = (np.abs(p["cos32"]) > 1) | np.isnan(p["cos32"])
            assert np.array_equal(~np.isfinite(ref).all(-1), nanc | at), p["name"]
            _rec(parity(p["name"], got, ref, nanc | at | ~lr.decided(p["lo"], p["hi"])), "spot")


def test_escape(ctx, vq, orc):
    """N = H bit for bit (axis normals pass the producer's renormalisation unchanged): D = 1 exactly where the fp32 rule escapes"""
    for p0 in ld.mirror_probes():
        for p in _variants(p0):
            got, ref, gb = _light(ctx, vq, orc, p)
            assert np.array_equal(gb[1][..., :3], p["planes"][1][..., :3]), "axis normals changed in the producer"
            g = got[..., :3].astype(np.float64)
            de = np.abs(g - p["want_escape"]).max(-1) / np.abs(p["want_escape"]).max(-1)
            with np.errstate(invalid="ignore"):                   # want_ggx is Inf/Inf where t = 0
                dg = np.nan_to_num(np.abs(g - p["want_ggx"]).max(-1) / np.abs(p["want_ggx"]).max(-1), nan=np.inf)
            assert np.array_equal(de < dg, p["escape"]), p["name"]
            assert np.minimum(de, dg).max() <= 2e-5, p["name"]
            _rec(parity(p["name"], got[..., :3], ref[..., :3]), "escape")


def _other():
    return ld.distance_probes() + ld.directional_probe() + [ld.t_sweep_probe(), ld.view_probe()]


def test_other_probes(ctx, vq, orc):
    """distance, directional, t sweep and view: parity with the oracle and the documented deviations (tests/test_light_domain_gpu.py:
    a light exactly at the pixel adds 0; where d2 is denormal the oracle overflows and the fused kernel stays finite, the point
    light lit; for 1e-26 > d2 >= FLT_MIN the fused light is never brighter than the oracle's; the camera at the pixel is NaN);
    counts of pixels on the exact-N.V path reported"""
    for p0 in _other():
        for p in _variants(p0):
            got, ref, gb = _light(ctx, vq, orc, p, multi=(2, 3) if p0["name"] == "t sweep" else ())
            skip = None
            if p.get("d2") is not None:
                d2 = p["d2"].astype(np.float64)
                skip = d2 < 1e-26
                assert (got[d2 == 0][:, :3] == 0).all(), p["name"]
                den = (d2 > 0) & (d2 < np.finfo(np.float32).tiny)
                assert den.any() and not np.isfinite(ref[den][:, :3]).all(-1).any(), p["name"]
                assert (term(got)[den] > 0).all() if p0["name"] == "near point" else (term(got)[den] >= 0).all(), p["name"]
                mid = (d2 >= np.finfo(np.float32).tiny) & skip
                assert (term(got)[mid] >= 0).all() and (term(got)[mid] <= term(ref)[mid]).all(), p["name"]
            if "at_cam" in p:
                at = p["at_cam"]
                assert at.any() and np.isnan(got[at][:, :3]).all() and np.isfinite(ref[at]).all(), p["name"]
                skip = at
            fam = p0["name"].split(" ")[0]
            _rec(parity(p["name"], got, ref, skip), fam)
            if fam == "view":
                P = gb[0][..., :3].astype(np.float64)
                V = np.asarray(_cam(p["pv"])) - P
                with np.errstate(all="ignore"):
                    nv = (gb[1][..., :3] * V).sum(-1) / np.linalg.norm(V, axis=-1)
                print(f"{p['name']}: {int((np.abs(nv) < 1e-3).sum())} pixels on the exact-N.V path")


@pytest.mark.parametrize("kind", ld.MIXED)
def test_mixed(ctx, vq, orc, kind):
    p0 = ld.mixed_frame(kind, seed=700 + ld.MIXED.index(kind))
    for p in _variants(p0):
        got, ref, gb = _light(ctx, vq, orc, p, multi=(2, 3) if kind in ("maximum", "rotated") else ())
        r = assert_scaled(p["name"], got, ref, min_frac_strict=0.0 if kind == "bright" else 0.99)
        _rec(r, "mixed " + kind)
        tiny = pd.tiny_pixels(gb)
        warps = pd.ps_warps(tiny.shape) if p is not p0 else pd.k1_warps(tiny.shape)
        print(f"{p['name']}: {int(tiny.sum())} TINY-vote pixels, {int((pd.per_warp(tiny, warps) > 0).sum())} TINY warps")


# ---- row ranges ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows", [(1, 2), (1, 14), (3, 15), (14, 15), (0, 15)])
def test_odd_rows_of_folded_frames(ctx, vq, rows):
    """folded frames of odd height (15 rows) and odd row ranges: the last tile's second row is shaded from the zeroed or stale
    stage and must not be stored; rows outside the range keep SENTINEL"""
    p = pd.fold_probe(pd.crop(ld.mixed_frame("one of each", seed=701), 512))
    planes = [np.ascontiguousarray(x[:15]) for x in p["planes"]]
    got, want, _ = run(ctx, vq, planes, p["pf"], p["pv"], p["env"], rows=rows, shadowed=True, multi=(2,))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    out = np.ones(15, bool)
    out[rows[0]:rows[1]] = False
    assert (got[out] == SENTINEL).all() and (got[~out] != SENTINEL).all()



@pytest.mark.parametrize("rows", [(0, 301), (1, 300), (3, 298), (0, 2), (299, 301)])
def test_stale_stage_frames(ctx, vq, rows):
    """a frame with more row pairs than psmain's grid has CTAs per column (301 rows, 512 wide: 4 tile columns of at most 132 CTAs
    on an H100): every CTA shades a second tile from a stage that still holds the first tile's texels, and the last tile's
    second row lies past the odd height. Two-pass equality, the shadowed and the multi-destination kernel, nothing stored outside
    the range"""
    planes, env, pf, pv = tall_frame(301)
    h = planes[0].shape[0]
    gy = pd.ps_ctas_per_column(512, torch.cuda.get_device_properties(0).multi_processor_count)
    if rows[1] - rows[0] > 2:
        assert (rows[1] - (rows[0] & ~1) + 1) // 2 > gy, "the frame must give some CTA a second tile"
    got, want, _ = run(ctx, vq, planes, pf, pv, env, rows=rows, shadowed=True, multi=(2,))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    out = np.ones(h, bool)
    out[rows[0]:rows[1]] = False
    assert (got[out] == SENTINEL).all() and (got[~out] != SENTINEL).all()


def tall_frame(h, seed=33):
    """an adversarial G-buffer 512 wide and h rows tall (emissive plane, no holes) under the 4 point + 3 spot lights, casters and
    the directional light of forward_domain.lights"""
    cam = (0.0, 5.0, -17.0)
    planes, _ = fd.adversarial_gbuffer(512, h, seed, cam, emissive=True)
    env = fd.make_env(8, 16, (48, 20), seed=seed)
    pf, pv = fd.constants(cam, env["spec_mips"], 0.0, lights=fd.lights(512, h, seed, 0.0))
    return planes, env, pf, pv
