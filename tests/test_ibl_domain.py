"""CPU: the oracle's environment-map pieces against the float64 restatement (tests/ibl_ref.py) over the inputs of
tests/ibl_domain.py, the probe identities the GPU probes rely on, the K11 MIN rule on special values, and the scan of
tangent-frame decisions near the 0.999 threshold."""
import ctypes as C
import math

import numpy as np
import pytest

import ibl_domain as dom
import ibl_ref as ref


def _fp(a):
    return np.ascontiguousarray(a, np.float32).ctypes.data_as(C.POINTER(C.c_float))


def _dirs(n, seed=5):
    rng = np.random.default_rng(seed)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    axes = [(sx * a, sy * b, sz * c) for a, b, c in ((1, 0, 0), (0, 1, 0), (0, 0, 1)) for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)]
    seam = [(-1.0, 0.0, 0.0), (-1.0, 0.0, -0.0), (-0.6, 0.8, 0.0), (-0.6, -0.8, -0.0)]
    pole = [(x, y, z) for y in (1.0, -1.0) for x, z in ((1e-3, 0.0), (0.0, 1e-3), (-1e-4, 1e-4), (3e-6, -2e-6))]
    return np.concatenate([d, np.array(axes + seam + pole, np.float64)]).astype(np.float32)


def min_rule(a, b):
    """std::min(a, b) = (b < a) ? b : a"""
    return np.where(b < a, b, a)


def min_pyramid_rule(img, levels):
    """the CPU filter's level chain with the std::min rule, row-major operands (0,0),(1,0),(0,1),(1,1), A = 1"""
    out = [img[..., :3]]
    for _ in range(1, levels):
        s = out[-1]
        h, w = s.shape[0] // 2, s.shape[1] // 2
        s = s[:2 * h, :2 * w]
        s0, s1, s2, s3 = s[0::2, 0::2], s[0::2, 1::2], s[1::2, 0::2], s[1::2, 1::2]
        out.append(min_rule(s0, min_rule(s1, min_rule(s2, s3))))
    return np.concatenate([np.concatenate([l, np.ones(l.shape[:2] + (1,), np.float32)], -1).reshape(-1, 4) for l in out])


@pytest.mark.parametrize("w,h", [(2, 2), (8, 6), (97, 41), (256, 128)])
def test_k11_oracle_follows_std_min_rule(orc, w, h):
    img = dom.special_blocks(w, h)
    levels = orc.lib().orc_mip_level_count(w, h)
    got = orc.hdri_build_mips(img, levels)
    want = min_pyramid_rule(img, levels)
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32))
    # the rule keeps a NaN only in the block's first texel and returns the first operand of a +-0 tie
    lvl1 = got[w * h:w * h + (w // 2) * (h // 2), :3].reshape(h // 2, w // 2, 3)
    first = img[0:2 * (h // 2):2, 0:2 * (w // 2):2, :3]
    assert np.array_equal(np.isnan(lvl1), np.isnan(first))
    if w * h >= 4 * 4 * (4 * len(dom.SPECIALS) + 3):       # large enough to hold every case
        assert (np.signbit(lvl1) & (lvl1 == 0)).any() and (~np.signbit(lvl1) & (lvl1 == 0)).any() and np.isnan(lvl1).any()


def test_direction_to_uv_oracle_within_float64(orc):
    d = _dirs(20000)
    out = np.zeros(2, np.float32)
    got = np.zeros((len(d), 2))
    for i, v in enumerate(d):
        orc.lib().orc_direction_to_equirect_uv(_fp(v), out.ctypes.data_as(C.POINTER(C.c_float)))
        got[i] = out
    u, v = ref.direction_to_uv(d.astype(np.float64))
    du = np.abs(got[:, 0] - u); du = np.minimum(du, np.abs(1 - du))
    # libm atan2f / asinf: <= 2 ulp of the angle, then a division and an addition in fp32
    assert du.max() <= (2 * math.pi * 4 * ref.EPS) / (2 * math.pi) + 2 * ref.EPS, du.max()
    assert np.abs(got[:, 1] - v).max() <= 4 * ref.EPS * (math.pi / 2) / math.pi + 2 * ref.EPS
    # the signed-zero directions: atan2(+-0, -0) = +-pi in libm, so u = 0 or 1 (the same column)
    for dd, uu in (((-1.0, 0.0, 0.0), 0.0), ((-1.0, 0.0, -0.0), 1.0), ((0.0, 1.0, 0.0), 0.5)):
        orc.lib().orc_direction_to_equirect_uv(_fp(dd), out.ctypes.data_as(C.POINTER(C.c_float)))
        assert out[0] == uu


@pytest.mark.parametrize("kind", ["synth", "seam", "noisy_poles", "denormal", "spike65504"])
@pytest.mark.parametrize("w,h,levels", [(97, 41, 3), (256, 128, None), (7, 3, None), (1024, 8, None)])
def test_sample_equirect_oracle_within_float64(orc, kind, w, h, levels):
    img = dom.content(kind, w, h)
    levels = levels or orc.lib().orc_mip_level_count(w, h)
    pyr = orc.hdri_build_mips(img, levels)
    rng = np.random.default_rng(w + h)
    n = 3000
    u = np.concatenate([rng.uniform(0, 1, n), [0.0, 1.0, 0.5 / w, 1 - 0.5 / w, 0.0, 1.0]]).astype(np.float32)
    v = np.concatenate([rng.uniform(0, 1, n), [0.0, 1.0, 0.5 / h, 1 - 0.5 / h, 1.0, 0.0]]).astype(np.float32)
    lod = np.concatenate([rng.uniform(-1, levels + 1, n), [0, levels - 1, 0.5, levels, 100.0, -3.0]]).astype(np.float32)
    got = np.zeros((len(u), 3))
    out = np.zeros(4, np.float32)
    for i in range(len(u)):
        orc.lib().orc_sample_equirect(_fp(pyr), w, h, levels, C.c_float(u[i]), C.c_float(v[i]), C.c_float(lod[i]),
                                      out.ctypes.data_as(C.POINTER(C.c_float)))
        got[i] = out[:3]
    L = ref.pyramid_levels(pyr, w, h, levels)
    want = ref.sample(L, u, v, lod)
    bound = ref.sample_bound(L, u, v, lod, 0.0, 0.0, np.abs(lod.astype(np.float64)) * ref.EPS)
    err = np.abs(got - want)
    assert (err <= bound).all(), (err / np.maximum(bound, 1e-300)).max()


def test_importance_sample_ggx_oracle_within_float64(orc):
    rng = np.random.default_rng(11)
    n_dirs = _dirs(400, seed=12)
    out = np.zeros(3, np.float32)
    worst = 0.0
    for i, N in enumerate(n_dirs):
        N = (N / np.linalg.norm(N.astype(np.float64))).astype(np.float32)
        rough = float(np.float32(rng.choice([1.0, 0.5, 0.1, 1.0 / 9, 1e-3])))
        xi = np.array([rng.uniform(0, 1), rng.uniform(0, 0.999)], np.float32)
        z_frame, undecided = ref.frame_decision(N.astype(np.float64))
        if undecided:
            continue
        orc.lib().orc_importance_sample_ggx(_fp(xi), _fp(N), C.c_float(rough), out.ctypes.data_as(C.POINTER(C.c_float)))
        h = ref.importance_sample_ggx(xi[0], xi[1], N.astype(np.float64), rough)
        worst = max(worst, float(np.abs(out - h).max() / ref.ggx_h_error(xi[1], rough)))
    assert worst <= 1.0, worst


@pytest.mark.parametrize("w,h", [(1, 1), (33, 17), (300, 2), (1, 64)])
def test_integrate_brdf_single_sample_closed_form(orc, w, h):
    got = orc.brdf_integration_lut(w, h, 1)
    want = ref.brdf_lut_single_sample(w, h)
    assert (np.abs(got - want) <= ref.brdf_lut_single_sample_bound(w, h)).all()


def test_ndf_at_full_alignment():
    """D(1) = 1 / (pi r^4): the closed form of the single-sample K3 probe"""
    for r in (1.0, 0.5, 1.0 / 9, 0.25):
        assert math.isclose(float(ref.ndf_ggx(1.0, r)), 1.0 / (math.pi * r ** 4), rel_tol=1e-12)


def test_k3_probe_lod_closed_form():
    """the single-sample lod 0.5*log2(6 W H r^4) - 1 is what the shader's expression gives for pdf = D(1) / 4"""
    for (w, h), r in (((256, 128), 1.0), ((64, 32), 0.5), ((8192, 4096), 1.0 / 9)):
        pdf = ref.ndf_ggx(1.0, r) * 1.0 / 4.0
        omega_p = 4 * math.pi / (6 * w * h)
        lod = max(0.0, 0.5 * math.log2((1.0 / pdf) / omega_p) - 1.0)
        assert math.isclose(lod, ref.k3_single_sample_lod(r, w, h), rel_tol=1e-12, abs_tol=1e-12)


def test_k2_probe_grid():
    """n_phi = 1, n_theta = 2: phi = 0, theta in {0, pi/4}; the theta = 0 sample has weight cos(0) sin(0) = 0 exactly"""
    phis, ths = ref.k2_angles(0.0, 1, 2)
    assert list(phis) == [0.0] and ths[0] == 0.0 and ths[1] == float(np.float32(np.float32(1.5707963268) / np.float32(2)))


def test_k2_step_trip_counts_match_oracle(orc):
    """the float-accumulated loop counts of ibl_ref equal the oracle's (and so the host's) for steps whose last phi / theta
    lands near the loop bound"""
    for step in (0.01, 0.025, 0.05, float(np.float32(6.28318530718) / 7), float(np.float32(1.5707963268) / 3),
                 float(np.nextafter(np.float32(1.5707963268) / np.float32(3), np.float32(1)))):
        p, t = C.c_int(), C.c_int()
        orc.lib().orc_diffuse_angle_counts(C.c_float(step), 0, 0, C.byref(p), C.byref(t))
        phis, ths = ref.k2_angles(step, 0, 0)
        assert (p.value, t.value) == (len(phis), len(ths)), step


def test_frame_decision_scan():
    """near-threshold texels exist (e.g. the +Z face at res = 800), and the fp32 decision the oracle takes (N normalised
    with an unfused dot, correctly rounded sqrt and division) equals the float64 one on every texel the scan lists"""
    texels = dom.near_threshold_texels([800])
    assert len([t for t in texels if t[0] == 4]) >= 1
    for face, px, py, res in texels:
        d = ref.cube_texel_direction(face, px, py, res).astype(np.float32)
        f32 = np.float32
        l2 = f32(f32(d[0] * d[0]) + f32(d[1] * d[1])) + f32(d[2] * d[2])
        nz = f32(d[2] / np.sqrt(f32(l2)))
        decided64, undecided = ref.frame_decision(d.astype(np.float64))
        assert (abs(nz) < f32(0.999)) == bool(decided64) or undecided
