"""CPU: the surface producer's oracle (oracle/oracle_surface.cpp) against the float64 restatement of its sampler
(tests/surface_ref.py) over the seeded domain of tests/surface_domain.py, the restatement against known answers, and the
rules for texel coordinates beyond the int range, non-finite coordinates and material indices (the device's conversions,
which the oracle now spells out instead of relying on undefined behaviour)."""
import numpy as np
import pytest

import oracle_lib as orc
import vqengine_b200 as vq
from surface_ref import sample_ref, mip_chain_ref, lod_ref, U
import surface_domain as sd

CASES = sd.sampler_cases()


def _oracle_probe(maps, ru, rv, mat=None, mat_index=0.0):
    planes = sd.planes_from_uv(ru, rv, mat_index)
    return sd.probe_outputs(orc.gbuffer_from_materials(planes, [mat or sd.probe_material()], [maps], 1.0))


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_sampler_within_float64_bound(case):
    name, w, h, levels, kind, seed = case
    level0, ru, rv = sd.build_sampler_case(w, h, levels, kind, seed)
    maps = sd.probe_maps(level0, levels)
    got = _oracle_probe(maps, ru, rv)
    ref = sd.probe_ref(maps, ru, rv)
    worst = 0.0
    for slot, (val, bound) in ref.items():
        g = got[slot].astype(np.float64)
        assert np.array_equal(np.isnan(g), np.isnan(val)), f"{name}/{slot}: NaN where the fp32 coordinate rule does not put it"
        g, val, bound = (np.nan_to_num(a) for a in (g, val, bound))
        err = np.abs(g - val)
        assert (err <= bound).all(), f"{name}/{slot}: {int((err > bound).sum())} samples outside the bound, worst " \
                                     f"{float((err - bound).max()):.3e} at {np.unravel_index(np.argmax(err - bound), err.shape)}"
        worst = max(worst, float((err / bound).max()))
    print(f"{name}: largest error / bound {worst:.3f}")


@pytest.mark.parametrize("scale,offset", [((3e38, 1.0), (0.0, 0.0)), ((1.0, -2e38), (0.0, -2e38)), ((0.0, 0.0), (0.3, 0.7)),
                                          ((-2.5, 1.5), (0.2, -0.3)), ((1e-30, 1e30), (0.5, 0.5))])
def test_oracle_sampler_scale_offset_within_bound(scale, offset):
    """uv scale and offset: zero, negative, tiny, and pairs for which u*s + o overflows"""
    level0, ru, rv = sd.build_sampler_case(37, 19, vq.mip_level_count(37, 19), "random", 7)
    maps = sd.probe_maps(level0, vq.mip_level_count(37, 19))
    got = _oracle_probe(maps, ru, rv, sd.probe_material(scale, offset))
    for slot, (val, bound) in sd.probe_ref(maps, ru, rv, scale, offset).items():
        assert np.array_equal(np.isnan(got[slot]), np.isnan(val)), slot
        assert (np.abs(np.nan_to_num(got[slot] - val)) <= bound).all(), slot


def test_float64_sampler_known_answers():
    """the restatement reproduces the known answers the oracle is pinned to (tests/test_surface_oracle.py)"""
    w, h = 8, 4
    lvl0 = np.zeros((h, w, 4), np.uint8)
    lvl0[..., 0] = np.arange(w)[None, :] * 30
    lvl0[..., 1] = ((np.arange(w)[None, :] + np.arange(h)[:, None]) % 2) * 255
    levels = vq.mip_level_count(w, h)
    ch = mip_chain_ref(lvl0, levels)

    def s(u, v, ddx=(0.0, 0.0), ddy=(0.0, 0.0)):
        val, _ = sample_ref(ch, w, h, levels, [u], [v], (1, 1), (0, 0), ([ddx[0]], [ddx[1]]), ([ddy[0]], [ddy[1]]))
        return val[0]
    assert np.allclose(s(3.5 / w, 2.5 / h)[:2], [90 / 255, 1.0])
    v = s(4.0 / w, 2.5 / h)
    assert abs(v[0] - 105 / 255) < 1e-12 and abs(v[1] - 0.5) < 1e-12
    assert abs(s(0.0, 0.5 / h)[0] - 105 / 255) < 1e-12                     # WRAP: texel w-1 and texel 0
    assert np.allclose(s(0.3, 0.6), s(2.3, -0.4), atol=1e-12)
    assert abs(s(0.5, 0.5, ddx=(2.0 / w, 0))[1] - 127 / 255) < 1e-12       # the checker's level 1 truncates to 127
    v0, v1, vh = s(0.3, 0.3), s(0.3, 0.3, ddx=(2.0 / w, 0)), s(0.3, 0.3, ddx=(np.sqrt(2.0) / w, 0))
    assert np.allclose(vh, 0.5 * (v0 + v1), atol=1e-12)
    lod, _ = lod_ref(64, 64, 7, np.array([1 / 64]), np.array([0.0]), np.array([3 / 64]), np.array([4 / 64]), 0.0)
    assert abs(lod[0] - np.log2(5.0)) < 1e-12
    # and the oracle agrees within the bound at each of them
    for u, v, ddx in ((3.5 / w, 2.5 / h, (0, 0)), (4.0 / w, 2.5 / h, (0, 0)), (0.0, 0.5 / h, (0, 0)), (0.3, 0.3, (np.sqrt(2.0) / w, 0))):
        o, _ = orc.sample_texture8(ch, w, h, levels, u, v, ddx=ddx)
        r, b = sample_ref(ch, w, h, levels, [u], [v], (1, 1), (0, 0), ([ddx[0]], [ddx[1]]), ([0.0], [0.0]))
        assert (np.abs(o - r[0]) <= b[0]).all()


def test_trilinear_is_continuous_across_integer_lods():
    """the LOD bound treats the LOD as continuous: trilinear at k - eps and at k agree to eps times the level step"""
    w = h = 64
    rng = np.random.default_rng(3)
    ch = mip_chain_ref(rng.integers(0, 256, (h, w, 4), dtype=np.uint8), 7)
    u = rng.uniform(-2, 2, 200); v = rng.uniform(-2, 2, 200)
    for k in range(1, 7):
        eps = 2.0 ** -20
        d_at = np.full(200, 2.0 ** k / w)
        d_below = np.full(200, 2.0 ** (k - eps) / w)
        z = np.zeros(200)
        a, _ = sample_ref(ch, w, h, 7, u, v, (1, 1), (0, 0), (d_at, z), (z, z))
        b, _ = sample_ref(ch, w, h, 7, u, v, (1, 1), (0, 0), (d_below, z), (z, z))
        assert np.abs(a - b).max() <= 2 * eps, k


@pytest.mark.parametrize("w,h,levels", [(200, 75, 8), (200, 75, 3), (1000, 3, 10), (129, 257, 9), (97, 41, 7), (1, 300, 9),
                                        (8192, 4, 14)])
def test_mip_chain_restatement_truncated_and_odd(w, h, levels):
    """the box-filter chain of the restatement equals the oracle's, also for truncated chains and odd sizes past 6 levels"""
    lvl0 = np.random.default_rng(w + h).integers(0, 256, (h, w, 4), dtype=np.uint8)
    assert np.array_equal(mip_chain_ref(lvl0, levels), orc.texture_mip_chain(lvl0, levels))


# ---- the rules for coordinates beyond the int range, non-finite coordinates and material indices ----------------------
@pytest.mark.parametrize("w,u", [(w, u) for w in (3, 256, 97) for u in (1e9, 4e9, -1e9, 1e36, -2.0 ** 40)] + [(256, 8.4e6 + 0.25)])
def test_oracle_saturates_coordinates_beyond_int_range(w, u):
    """x = u*W - 0.5 beyond the int range: floor(x) saturates to the int range as on the device (cvt.rzi), then wraps; x is
    integral there, so the sample is one column. (The host conversion was undefined: INT_MIN on x86 for either sign.)"""
    lvl0 = np.zeros((1, w, 4), np.uint8)
    lvl0[0, :, 0] = np.arange(w) % 251
    x = np.float32(np.float32(np.float32(u) * np.float32(w)) - np.float32(0.5))
    assert abs(float(x)) >= 2.0 ** 31
    col = min(max(int(np.floor(float(x))), -2 ** 31), 2 ** 31 - 1) % w
    val, _ = orc.sample_texture8(lvl0.reshape(-1).copy(), w, 1, 1, float(u), 0.5)
    assert val[0] * 255 == pytest.approx(col % 251, abs=1e-4), (w, u, col)


@pytest.mark.parametrize("u,v", [(np.nan, 0.5), (0.5, np.nan), (np.inf, 0.5), (0.5, -np.inf)])
def test_non_finite_coordinate_samples_nan(u, v):
    """a texel coordinate that is not finite blends to NaN, as the device's fx = x - floor(x) does (the oracle returned 0)"""
    lvl0 = np.full((4, 4, 4), 200, np.uint8)
    ch = mip_chain_ref(lvl0, 3)
    val, _ = orc.sample_texture8(ch, 4, 4, 3, u, v)
    assert np.isnan(val).all()
    r, b = sample_ref(ch, 4, 4, 3, [u], [v], (1, 1), (0, 0), ([0.0], [0.0]), ([0.0], [0.0]))
    assert np.isnan(r).all()


def test_coordinate_overflowing_at_one_level_only():
    """u*W overflows fp32 at level 0 but not at level 1: the trilinear blend of the two is NaN"""
    w, h = 2, 2
    lvl0 = np.full((h, w, 4), 200, np.uint8)
    ch = mip_chain_ref(lvl0, 2)
    u = float(np.float32(2.5e38))
    assert not np.isfinite(np.float32(u) * np.float32(2)) and np.isfinite(np.float32(u) * np.float32(1))
    ddx = (np.sqrt(2.0) / w, 0.0)                                           # lod 0.5
    val, lod = orc.sample_texture8(ch, w, h, 2, u, 0.5, ddx=ddx)
    assert abs(lod - 0.5) < 1e-6
    assert np.isnan(val).all()
    r, b = sample_ref(ch, w, h, 2, [u], [0.5], (1, 1), (0, 0), ([ddx[0]], [ddx[1]]), ([0.0], [0.0]))
    assert np.isnan(r).all()
    val, _ = orc.sample_texture8(ch, w, h, 2, u, 0.5, ddx=(2.0 / w, 0.0))  # lod 1 alone: finite
    assert val[0] == pytest.approx(200 / 255, abs=1e-6)


@pytest.mark.parametrize("index,want", [(-3.0, 0), (-0.0, 0), (2.999, 2), (3.0, 3), (4.0, 3), (1e10, 3), (-1e10, 0),
                                        (np.nan, 0), (np.inf, 3), (-np.inf, 0)])
def test_material_index_saturates_then_clamps(index, want):
    """tangent_m.w converts as the device does (NaN -> 0, saturated), then clamps to the table"""
    mats = []
    for i in range(4):
        m = vq.MaterialData()
        m.roughness = 0.1 * (i + 1); m.metalness = 0.5; m.textureConfig = 0.0
        m.uvScaleOffset.x = m.uvScaleOffset.y = 1.0
        mats.append(m)
    ru = np.zeros((2, 2), np.float32)
    planes = sd.planes_from_uv(ru, ru, index)
    out = orc.gbuffer_from_materials(planes, mats, [{} for _ in mats], 1.0)
    assert np.allclose(out[1][..., 3], np.float32(0.1 * (want + 1)))
