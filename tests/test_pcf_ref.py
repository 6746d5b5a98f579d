"""CPU (-m "not gpu"): the shadowed pass's PCF decisions over their whole domain (tests/shadow_domain.py) against the float64
restatement of Lighting.hlsl's three tests (tests/pcf_ref.py), on the host build of the product's header and on the oracle.

  * every pixel's host count of every slot lies inside the float64 interval, and equals it wherever every tap is decided;
  * the record the device stores decodes to the same counts;
  * the host build equals the oracle bit for bit on the whole shadowed pixel (which carries every observable decision);
  * exact probes (directional taps on texel boundaries, px = +-1, texels equal to pz - bias) equal the exact rule;
  * the degenerate light-space positions (w = 0; x = z = w = 0 gives NaN texel coordinates) run clean under AddressSanitizer and
    UndefinedBehaviorSanitizer (float-cast-overflow included) and index inside their maps."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as orc
import pcf_ref
import shadow_domain as sd
from envmaps import small_env

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST_CHECK = os.path.join(ROOT, "tests", "host_check")


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    out = tmp_path_factory.mktemp("hostcheck") / "libshadowhost.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", str(out),
                           os.path.join(HOST_CHECK, "shadow_math_host.cpp")])
    return C.CDLL(str(out))


@pytest.fixture(scope="module")
def scenes():
    return sd.scenes()


def host_counts(hostlib, s):
    """[11, n] counts of the host build (-1: slot not reported) and its [n] records"""
    import vqengine_b200 as vq
    sm = s.shadow_maps_struct(vq)
    n = s.H * sd.W
    p = [np.ascontiguousarray(a, np.float32) for a in s.planes[:2]]
    cnt = np.zeros((n, 11), np.int32)
    hostlib.hostcheck_pcf_counts(C.byref(s.pf), C.byref(s.pv), C.byref(sm), orc._p(p[0]), orc._p(p[1]), C.c_int(n), orc._p(cnt))
    rec = np.zeros(n, np.uint64)
    hostlib.hostcheck_pcf_records(C.byref(s.pf), C.byref(s.pv), C.byref(sm), orc._p(p[0]), orc._p(p[1]), C.c_int(n),
                                  rec.ctypes.data_as(C.c_void_p))
    return cnt.T.astype(np.int64), rec


@pytest.mark.parametrize("idx", range(len(sd.SIZES)))
def test_host_counts_inside_float64_interval(hostlib, scenes, idx):
    s = scenes[idx]
    cnt, rec = host_counts(hostlib, s)
    lo, hi, in_range = pcf_ref.all_counts(s)
    got = np.where(cnt < 0, 0, cnt)
    assert np.array_equal(pcf_ref.decode(rec), got)                            # the record holds what the sink was handed
    assert ((cnt[:5] >= 0) == in_range).mean() > 0.999 and (cnt[5:] >= 0).all()
    bad = (got < lo) | (got > hi)
    assert not bad.any(), [(int(k), int(j), s.groups[j // 32], int(got[k, j]), int(lo[k, j]), int(hi[k, j])) for k, j in np.argwhere(bad)[:8]]
    # the scenes exercise every slot: most pixels decided, at least 20 of them tested inside range / frustum, with varied counts
    for k in range(11):
        if k == 5 and s.spot_views[0]["near"] == 0:
            continue                                                          # near = 0: pz = 1 everywhere, the probes are the point
        dec = (lo[k] == hi[k])
        tested = dec & (cnt[k] >= 0) & (got[k] < 25)
        assert dec.mean() > 0.8 and tested.sum() >= 20 and len(np.unique(got[k][dec])) >= 2, (k, dec.mean(), tested.sum())
    # the spot probes' degenerate lanes: at the light (w = 0) the frustum test decides or the coordinates are NaN: count 25 or 0
    P = s.planes[0].reshape(-1, 4)[:, :3]
    at_eye = np.nonzero((P == 0).all(-1) & (np.array(s.groups)[np.arange(len(P)) // 32] == "spot_probes"))[0]
    assert len(at_eye) >= 1
    assert (got[5, at_eye] == (0 if s.spot_views[0]["near"] == 0 else 25)).all()


@pytest.mark.parametrize("idx", range(len(sd.SIZES)))
def test_exact_probes_follow_the_exact_rule(hostlib, scenes, idx):
    """directional taps exactly on texel boundaries, px exactly +-1 (inside: the test is `px > 1`), texels exactly equal to
    pz - bias (`>` false): every fp32 operation on the way is exact, so the count is the exact rule's, with no slack"""
    s = scenes[idx]
    if (s.dir_w & (s.dir_w - 1)) or (s.dir_h & (s.dir_h - 1)):
        pytest.skip("1/W is inexact: these probes are checked against the float64 interval instead")
    cnt, _ = host_counts(hostlib, s)
    P = s.planes[0].reshape(-1, 4)[s.exact_idx, :3].astype(np.float64)
    want = pcf_ref.dir_counts(s, P, eps=0)
    assert np.array_equal(cnt[10, s.exact_idx], want["lo"])
    assert not want["outside"][:3].any()                                      # px = 1, -1, 1 are inside the frustum
    assert len(s.eq_lanes) >= 1 and (want["lo"][s.eq_lanes] == 0).all()       # texels == pz - bias: no tap shadowed


@pytest.mark.parametrize("idx", range(len(sd.SIZES)))
def test_host_build_equals_oracle_on_domain_scenes(hostlib, scenes, idx):
    """the whole shadowed pixel (every observable decision) of the host build == the oracle, bit for bit"""
    import vqengine_b200 as vq
    s = scenes[idx]
    env = small_env()
    args = (env["diff"], env["diff_res"], env["spec"], env["spec_res"], env["spec_mips"], env["lut"])
    base_pf = vq.PerFrameData()
    hostlib.hostcheck_per_frame_without_casters(C.byref(s.pf), C.byref(base_pf))
    base = orc.forward_lighting(base_pf, s.pv, s.planes, *args)
    sm = s.shadow_maps_struct(vq)
    out = np.zeros((s.H, sd.W, 4), np.float32)
    p = [np.ascontiguousarray(a, np.float32) for a in s.planes]
    hostlib.hostcheck_shade_casters(C.byref(s.pf), C.byref(s.pv), C.byref(sm), orc._p(p[0]), orc._p(p[1]), orc._p(p[2]), orc._p(base),
                                    C.c_int(s.H * sd.W), orc._p(out))
    want = orc.forward_lighting_shadowed(s.pf, s.pv, s.planes, *args, point_cubes=s.cubes, point_res=s.cube_res, spot_maps=s.spots,
                                         dir_map=s.dmap)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32)), np.argwhere(out.view(np.uint32) != want.view(np.uint32))[:5]


def _scene_blob(s, path):
    with open(path, "wb") as f:
        f.write(bytes(s.pf)); f.write(bytes(s.pv))
        f.write(np.array([s.cube_res, s.spot_w, s.spot_h, s.dir_w, s.dir_h, s.H * sd.W], np.int32).tobytes())
        for a in (s.cubes, s.spots, s.dmap, s.planes[0], s.planes[1]):
            f.write(np.ascontiguousarray(a, np.float32).tobytes())


def test_degenerate_probes_clean_under_sanitizers(hostlib, scenes, tmp_path):
    """w = 0 and NaN texel coordinates: no undefined conversion, no access outside a map, the same counts as the plain build"""
    exe = tmp_path / "pcf_counts_san"
    subprocess.check_call(["g++", "-O1", "-g", "-std=c++17", "-ffp-contract=off", "-fno-fast-math",
                           "-fsanitize=address,undefined,float-cast-overflow", "-fno-sanitize-recover=all", "-o", str(exe),
                           os.path.join(HOST_CHECK, "pcf_counts_main.cpp")])
    for s in scenes:
        blob, out = tmp_path / f"s{s.idx}.bin", tmp_path / f"o{s.idx}.bin"
        _scene_blob(s, blob)
        r = subprocess.run([str(exe), str(blob), str(out)], capture_output=True, text=True,
                           env=dict(os.environ, ASAN_OPTIONS="detect_leaks=0", UBSAN_OPTIONS="print_stacktrace=1"))
        assert r.returncode == 0, r.stderr[-2000:]
        got = np.fromfile(out, np.int32).reshape(-1, 11).T
        assert np.array_equal(got, host_counts(hostlib, s)[0])


def test_nan_light_space_position_counts_nothing():
    """the oracle's 2-D tests at x = y = z = w = 0 (NaN coordinates, texel 0 as D3D converts NaN): no tap shadowed"""
    m = np.full((5, 7), -1.0, np.float32)
    assert orc.shadow_test_pcf((0.0, 0.0, 0.0, 0.0), 0.01, 0.5, m) == 1.0
    assert orc.shadow_test_pcf((0.0, 0.0, 0.0, 0.0), 0.01, 0.5, m, directional=True) == 1.0


@pytest.mark.skipif(orc.hlsl_ref() is None, reason="oracle/_ref/libhlslref.so not built (needs /root/reference at build time)")
def test_oracle_equals_shader_text_with_perspective_spot_views():
    """the oracle's shadowed PSMain against the reference's shader text with PERSPECTIVE spot views (w varies per pixel)"""
    from surface_util import material_set
    from vqengine_b200 import synth
    env = small_env()
    mats, texs, chains = material_set(4, 32, uniform=False)
    planes = synth.surface_inputs(128, 64, 4, seed=6, uv_scale=0.07)
    pf, pv = synth.scene_constants(128, 64, env["spec_mips"], seed=6, n_point=3, n_spot=2, casters=True)
    L = pf.Lights
    L.directional.shadowing = 1
    sc = L.spot_casters[0]
    eye = np.array([sc.position.x, sc.position.y, sc.position.z], np.float64)
    M = sd.look_at_lh(eye, np.array([0.0, -2.0, 0.0]), np.array([0.0, 1.0, 0.0])) @ sd.perspective_fov_lh(1.1, 1.0, 0.5, 60.0)
    sd._set_matrix(L.shadowViews[0], M)
    sd._set_matrix(L.shadowViewDirectional, sd.dir_matrix())
    pf.f2SpotLightShadowMapDimensions.x = pf.f2SpotLightShadowMapDimensions.y = 16.0
    pf.f2DirectionalLightShadowMapDimensions.x = pf.f2DirectionalLightShadowMapDimensions.y = 16.0
    rng = np.random.default_rng(111)
    cubes = rng.uniform(0.0, 1.2, (L.numPointCasters, 6, 8, 8)).astype(np.float32)
    spots = rng.uniform(0.9, 1.0, (L.numSpotCasters, 16, 16)).astype(np.float32)
    dmap = rng.uniform(0.3, 0.7, (16, 16)).astype(np.float32)
    shadow = dict(point_cubes=cubes, point_res=8, spot_maps=spots, dir_map=dmap)
    g = orc.gbuffer_from_materials(planes, mats, chains, pf.fAmbientLightingFactor, emissive=True)
    args = (env["diff"], env["diff_res"], env["spec"], env["spec_res"], env["spec_mips"], env["lut"])
    want = orc.forward_lighting_shadowed_e(pf, pv, g, *args, **shadow)
    got, disc = orc.hlsl_forward_image(pf, pv, planes, mats, chains, env, **shadow)
    assert not disc.any()
    assert np.array_equal(want.view(np.uint32), got.view(np.uint32)), np.argwhere(want.view(np.uint32) != got.view(np.uint32))[:5]
