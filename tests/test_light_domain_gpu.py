"""-m gpu: K1's light loop over the whole domain of its inputs (tests/light_domain.py, bounds from tests/light_ref.py):
range and escape decisions recovered from the radiance against the fp32 rules, the spot intensity K1(spot) / K1(point)
against the float64 interval, whole-pixel parity with the oracle on every probe frame and on mixed frames, and the SHADOWED,
MULTI and ROT instantiations against the plain pass.

Deviations from the oracle, decided and asserted here (DESIGN.md §5):
  * a spot cosine that rounds outside [-1, 1] (on the axis, directly behind the light): the oracle's acos is NaN, K1 clamps
    and gives the on-axis (or opposite) intensity, which lies inside the float64 interval;
  * a pixel exactly at a positional light (d2 = 0): the oracle is NaN (Wi = 0/0, 1/0 attenuation), K1's light adds exactly 0;
  * d2 below 1e-26 (a pixel closer than 1e-13 to a light): K1 scales the light vector by 1/sqrt(d2 + 1e-30), so the light is
    dimmer than the oracle's; where d2 is denormal the oracle's 1/d2 overflows and K1 stays finite;
  * the camera exactly at the pixel (V = 0/0): the oracle's saturates drop the NaN, K1's pixel is NaN."""
import math

import numpy as np
import pytest
import torch

import light_domain as ld
import light_ref as lr
from gpu_util import assert_scaled, dev, host
from test_forward_domain_gpu import _env, _gbuffer, _oracle, _shade

pytestmark = pytest.mark.gpu

ZENV = None


def zenv():
    global ZENV
    if ZENV is None:
        ZENV = ld.zero_env()
    return ZENV


def term(out):
    return out[..., :3].astype(np.float64).max(-1)


def parity(name, got, ref, skip=None):
    """K1 finite everywhere; oracle NaN only inside `skip` (the deviations); elsewhere the §5 HDR bound: |delta| <= 1e-4 max(1, |ref|)
    and <= 1e-4 where |ref| <= 1. The probes reach values of 1e5 by construction (lights 1e-3 away, brightness 1e30 at 1.8e19),
    so the share of ALL values within an absolute 1e-4 is not asked for."""
    skip = np.zeros(got.shape[:2], bool) if skip is None else skip
    assert np.isfinite(got[~skip]).all(), (name, np.argwhere(~np.isfinite(got).all(-1) & ~skip)[:4])
    fin = np.isfinite(ref).all(-1)
    assert not (~fin & ~skip).any(), (name, np.argwhere(~fin & ~skip)[:4])
    keep = fin & ~skip
    return assert_scaled(name, got[keep], ref[keep], min_frac_strict=0.0)


# ---- range ------------------------------------------------------------------------------------------------------------
def test_range_decisions(ctx, vq, orc):
    """lit (nonzero light term) exactly where sqrt_rn(dot_unfused(L, L)) < range, for every range from the smallest denormal
    to +Inf and 0, -0, -1, NaN, lights and casters; a pixel exactly at a light adds exactly 0"""
    env = zenv()
    n_edge = 0
    for p in ld.range_probes():
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)
        ref = _oracle(orc, p["pf"], p["pv"], p["planes"], env)
        t = term(got)
        at = p["at_light"]
        assert np.array_equal(t[~at] != 0, p["lit"][~at]), (p["name"], np.argwhere((t != 0) != p["lit"])[:4])
        assert (got[at][:, :3] == 0).all(), p["name"]
        assert np.array_equal(~np.isfinite(ref).all(-1), at & p["lit"]), p["name"]
        parity(p["name"], got, ref, at)
        n_edge += int((p["d"].astype(np.float32) == np.float32(p["range"])).sum())
    print(f"range probes: {n_edge} pixels with sqrt_rn(d2) == range")


# ---- spot intensity ---------------------------------------------------------------------------------------------------
def test_spot_intensity(ctx, vq, orc):
    """K1(spot) / K1(point light at the same position, range +Inf) inside the float64 interval on every observable pixel;
    whole-pixel parity with the oracle where the intensity is decided and the oracle's cosine is inside [-1, 1]; K1 finite where
    the oracle's acos is NaN"""
    env = zenv()
    worst = 0.0
    for p in ld.spot_probes():
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)
        pt = _shade(ctx, vq, p["point"][0], p["point"][1], p["planes"], env)
        ref = _oracle(orc, p["pf"], p["pv"], p["planes"], env)
        ts, tp = term(got), term(pt)
        at = p["at_light"]
        assert (got[at][:, :3] == 0).all(), p["name"]
        obs = ~at & (tp > 0)
        ratio = ts[obs] / tp[obs]
        tol = 8 * lr.U24
        lo, hi = p["lo"][obs], p["hi"][obs]
        bad = (ratio < lo - tol) | (ratio > hi + tol)
        assert not bad.any(), (p["name"], ratio[bad][:4], lo[bad][:4], hi[bad][:4], p["theta"][obs][bad][:4])
        nanc = (np.abs(p["cos32"]) > 1) | np.isnan(p["cos32"])
        assert np.array_equal(~np.isfinite(ref).all(-1), nanc | at), p["name"]
        r = parity(p["name"], got, ref, nanc | at | ~lr.decided(p["lo"], p["hi"]))
        worst = max(worst, r["max_scaled"])
    print(f"spot probes: worst scaled parity {worst:.2e}")


# ---- D = 1 escape -----------------------------------------------------------------------------------------------------
def test_escape_decisions(ctx, vq, orc):
    """at N = H bit for bit, K1's light term is the float64 value with D = 1 exactly where the fp32 decision escapes and with
    D = a2 / (PI t^2) elsewhere (the two differ by a factor of 1e5 or more), around the flip at roughness 0.0274"""
    env = zenv()
    for p in ld.mirror_probes():
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)[..., :3].astype(np.float64)
        de = np.abs(got - p["want_escape"]).max(-1) / np.abs(p["want_escape"]).max(-1)
        dg = np.abs(got - p["want_ggx"]).max(-1) / np.abs(p["want_ggx"]).max(-1)
        dg = np.nan_to_num(dg, nan=np.inf)
        k1_escape = de < dg
        assert np.array_equal(k1_escape, p["escape"]), (p["name"], p["planes"][1][..., 3][k1_escape != p["escape"]])
        assert np.minimum(de, dg).max() <= 2e-5, p["name"]
        parity(p["name"], got, _oracle(orc, p["pf"], p["pv"], p["planes"], env)[..., :3])


# ---- the other probe frames ---------------------------------------------------------------------------------------------
def _other_probes():
    return ld.distance_probes() + ld.directional_probe() + [ld.t_sweep_probe(), ld.view_probe()]


def test_probe_parity(ctx, vq, orc):
    """distances from 0 to 2e19, directional N.L at 0, V along and against the light, a zero light direction, GGX t across
    T_EXACT, N.V across NV_EXACT and at 0, the camera at the pixel, |N| cos = 1: whole-pixel parity with the oracle, and the
    documented deviations next to a light"""
    env = zenv()
    for p in _other_probes():
        got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], env)
        ref = _oracle(orc, p["pf"], p["pv"], p["planes"], env)
        skip = None
        if p.get("d2") is not None:
            d2 = p["d2"].astype(np.float64)
            skip = d2 < 1e-26
            assert (got[d2 == 0][:, :3] == 0).all(), p["name"]                         # the light adds exactly 0
            den = (d2 > 0) & (d2 < np.finfo(np.float32).tiny)
            # the oracle overflows; K1 stays finite (the point light lit, the spot dark: its shortened Wi puts theta near pi/2)
            assert not np.isfinite(ref[den][:, :3]).all(-1).any(), p["name"]
            assert (term(got)[den] > 0).all() if p["name"] == "near point" else (term(got)[den] >= 0).all(), p["name"]
            # 1/sqrt(d2 + 1e-30) both attenuates and normalises Wi: K1's light is dimmer than the oracle's, never brighter
            mid = (d2 >= np.finfo(np.float32).tiny) & skip
            assert (term(got)[mid] >= 0).all() and (term(got)[mid] <= term(ref)[mid]).all(), p["name"]
        if "at_cam" in p:
            # the camera exactly at the pixel: V = 0/0. The oracle's saturates drop the NaN and give a finite value; K1's hoisted
            # N.V and G1(V) carry it, so the pixel is NaN (a camera on the surface is behind its own near plane)
            at = p["at_cam"]
            assert at.any() and np.isnan(got[at][:, :3]).all() and np.isfinite(ref[at]).all(), p["name"]
            skip = at
        print(parity(p["name"], got, ref, skip))


# ---- instantiations ---------------------------------------------------------------------------------------------------------
def _all_probes():
    return (ld.range_probes() + ld.spot_probes() + ld.mirror_probes() + _other_probes())


def test_shadowed_instantiation_equals_plain(ctx, vq):
    """every probe frame through vq_forward_lighting_shadowed with point shadow cubes of +Inf (no tap is ever in shadow) and a
    dark point caster where the frame has none: the SHADOWED light loop equals the plain pass bit for bit (the loop is shared and
    scale * 1 is exact)"""
    env = zenv()
    em, keep_env = _env(vq, env)
    n = 0
    for p in _all_probes():
        pf = ld.with_dark_caster(p["pf"])
        plain = _shade(ctx, vq, pf, p["pv"], p["planes"], env)
        h, w = p["planes"][0].shape[:2]
        gb, keep = _gbuffer(vq, p["planes"])
        cubes = dev(np.full((pf.Lights.numPointCasters, 6, 2, 2), np.inf, np.float32))
        out = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
        ctx.forward_lighting_shadowed(pf, p["pv"], gb, em, out, point_cubes=cubes)
        got = host(out)
        assert np.array_equal(got.view(np.uint32), plain.view(np.uint32)), (p["name"], np.argwhere(got != plain)[:4])
        n += 1
    print(f"{n} probe frames: SHADOWED == plain bit for bit")


@pytest.mark.parametrize("kind", ld.MIXED)
def test_mixed_parity(ctx, vq, orc, kind):
    """adversarial G-buffers (random environment) under 0 lights, one of each kind, the ABI maximum, brightness up to 1e4,
    negative and zero brightness, and an HDRI offset (ROT): whole-pixel parity with the oracle"""
    p = ld.mixed_frame(kind, seed=700 + ld.MIXED.index(kind))
    got = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], p["env"])
    ref = _oracle(orc, p["pf"], p["pv"], p["planes"], p["env"])
    # brightness 1e4 puts most values far above 1, where the bound is relative
    print(assert_scaled(p["name"], got, ref, min_frac_strict=0.0 if kind == "bright" else 0.99))


def test_mixed_multi_equals_single(ctx, vq):
    """forward_kernel<MULTI>: the maximum light set stored to two destinations equals the single-destination pass bit for bit"""
    p = ld.mixed_frame("maximum", seed=700 + ld.MIXED.index("maximum"))
    single = _shade(ctx, vq, p["pf"], p["pv"], p["planes"], p["env"])
    h, w = p["planes"][0].shape[:2]
    gb, keep = _gbuffer(vq, p["planes"])
    em, tk = _env(vq, p["env"])
    frames = [torch.zeros((h + 2, w, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
    ctx.forward_lighting_multi(p["pf"], p["pv"], gb, em, [vq.image_of(f) for f in frames], dst_row_offset=2)
    for f in frames:
        got = host(f)
        assert np.array_equal(got[2:].view(np.uint32), single.view(np.uint32)) and (got[:2] == 0).all()
