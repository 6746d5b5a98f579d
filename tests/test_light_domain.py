"""CPU: the light-loop probes of tests/light_domain.py hold on the oracle, so that the GPU tests (test_light_domain_gpu.py)
compare K1 with statements known to be the reference's: the oracle's range decisions are the fp32 rule, its spot intensity
lies inside the float64 interval, its D = 1 escape is the fp32 decision, and the edge search found both sides of every edge."""
import math

import numpy as np
import pytest

import light_domain as ld
import light_ref as lr


@pytest.fixture(scope="module")
def zenv():
    return ld.zero_env()


def _oracle(orc, p, env):
    return orc.forward_lighting(p["pf"], p["pv"], p["planes"], env["diff"], env["diff_res"], env["spec"], env["spec_res"],
                                env["spec_mips"], env["lut"])


def light_term(out):
    """the probe's light sum: the largest rgb channel (the probes' colours are (1, 0.5, 0.25))"""
    return out[..., :3].astype(np.float64).max(-1)


def test_edge_search_straddles_every_range():
    """for every finite positive range below the overflow, the search produced pixels on both sides of the edge and pixels whose
    fp32 distance equals the range; for the ranges beyond sqrt(FLT_MAX), pixels on both sides of the d2 overflow"""
    seen = {}
    for p in ld.range_probes():
        R = p["range"]
        if not (R > 0) or R == ld.DENORM_MIN:
            continue
        s = seen.setdefault(repr(R), [0, 0, 0])
        s[0] += int(p["lit"].sum()); s[1] += int((~p["lit"]).sum())
        s[2] += int((p["d"].astype(np.float32) == np.float32(R)).sum())
    for R, (n_in, n_out, n_eq) in seen.items():
        print(f"range {R}: {n_in} in, {n_out} out, {n_eq} at sqrt_rn(d2) == range")
        assert n_in > 0 and n_out > 0, R
        if float(R) < 1e18:
            assert n_eq > 0, R


def test_oracle_range_decisions_are_the_fp32_rule(orc, zenv):
    """lit (a nonzero light term) exactly where sqrt_rn(dot_unfused(L, L)) < range, lights and casters; a pixel exactly at a light
    in range is NaN in the oracle (Wi = 0/0), the deviation K1 documents"""
    for p in ld.range_probes():
        out = _oracle(orc, p, zenv)
        t = light_term(out)
        nan = np.isnan(out[..., :3]).any(-1)
        assert np.array_equal(nan, p["at_light"] & p["lit"]), p["name"]
        ok = ~nan
        assert np.array_equal(t[ok] != 0, p["lit"][ok]), (p["name"], np.argwhere((t != 0) != p["lit"])[:4])


def test_oracle_spot_intensity_inside_float64_interval(orc, zenv):
    """oracle(spot) / oracle(point light at the same position, range +Inf) inside the float64 interval; NaN exactly where the
    oracle's fp32 cosine rounds outside [-1, 1] (acos NaN: on the axis and directly behind the light) or the pixel is at the
    light"""
    n_nan = 0
    for p in ld.spot_probes():
        s = _oracle(orc, p, zenv)
        q = _oracle(orc, dict(p, pf=p["point"][0], pv=p["point"][1]), zenv)
        nan = np.isnan(s[..., :3]).any(-1)
        assert np.array_equal(nan, (np.abs(p["cos32"]) > 1) | p["at_light"] | np.isnan(p["cos32"])), p["name"]
        n_nan += int(nan.sum())
        ts, tp = light_term(s), light_term(q)
        obs = ~nan & (tp > 0) & np.isfinite(tp)
        ratio = ts[obs] / tp[obs]
        tol = 8 * lr.U24
        bad = (ratio < p["lo"][obs] - tol) | (ratio > p["hi"][obs] + tol)
        assert not bad.any(), (p["name"], ratio[bad][:4], p["lo"][obs][bad][:4], p["hi"][obs][bad][:4], p["theta"][obs][bad][:4])
    print(f"{n_nan} pixels where the oracle's spot cosine rounds outside [-1, 1]")
    assert n_nan > 0


def test_spot_probes_cover_every_edge():
    """every cone has decided pixels on each side and, for the narrow and hard cones, undecided pixels at the edge"""
    for p in ld.spot_probes():
        lo, hi = p["lo"], p["hi"]
        assert (hi >= 1 - 1e-6).any() and (lo <= 1e-6).any() or p["outer"] >= math.pi, p["name"]
        if p["outer"] - p["inner"] <= 1e-3 and p["outer"] >= p["inner"] > 0:
            assert (~lr.decided(lo, hi)).any(), p["name"]


def test_oracle_escape_is_the_fp32_decision(orc, zenv):
    """at N = H bit for bit, the oracle's light term is the float64 value with D = 1 exactly where the fp32 decision says so, and
    with D = a2 / (PI t^2) elsewhere; the roughness list has both, and the flip lies at 0.0274, not 0.024"""
    assert abs(lr.escape_roughness_bound() - 0.0274) < 1e-4
    flips = 0
    for p in ld.mirror_probes():
        out = _oracle(orc, p, zenv)[..., :3].astype(np.float64)
        e = p["escape"]
        want = np.where(e[..., None], p["want_escape"], p["want_ggx"])
        assert np.all(np.abs(out - want) <= 2e-5 * np.abs(want)), p["name"]
        assert e.any() and (~e).any()
        r = p["planes"][1][..., 3]
        assert r[e].max() < 0.0275 and r[~e].min() > 0.0272
        flips += 1
    assert flips == 4


def test_probe_frames_finite_where_expected(orc, zenv):
    """the oracle on the other probe frames: non-finite only where the squared distance to a light is 0 or denormal"""
    for p in ld.distance_probes():
        out = _oracle(orc, p, zenv)
        nan = ~np.isfinite(out[..., :3]).all(-1)
        if p["d2"] is None:
            assert not nan.any(), p["name"]
        else:
            tiny = p["d2"] < np.finfo(np.float32).tiny
            assert np.array_equal(nan, tiny), (p["name"], p["dist"][nan != tiny][:4])
    d, z = ld.directional_probe()
    assert np.isfinite(_oracle(orc, d, zenv)).all()
    # a zero light direction: Wi = 0/0 is NaN, but every use of it goes through saturate() or max(0, .) first, which drop the
    # NaN: N.L = 0 and the light adds exactly 0
    assert (_oracle(orc, z, zenv)[..., :3] == 0).all()
    # the camera at the pixel: V = 0/0, dropped by the same saturates
    v = ld.view_probe()
    assert v["at_cam"].any() and np.isfinite(_oracle(orc, v, zenv)).all()
    assert np.isfinite(_oracle(orc, ld.t_sweep_probe(), zenv)).all()
