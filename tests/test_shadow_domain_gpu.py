"""-m gpu: the shadowed pass's PCF decisions over their whole domain (tests/shadow_domain.py) on the device.

tests/device_check/shadow_math_device.cu builds the product's PCF header for sm_90a (the flags of build.sh) and runs its pieces:
  * pcf_record exactly as shadow_pcf_kernel calls it (whole warps, the last pixel duplicated past a row's end): equal to the host
    build of the same header (tests/host_check) bit for bit on every pixel for the point and directional slots — no libm function
    is on their decision path, and sqrt / division are correctly rounded on both builds; the spot slots (tanf(acosf(NdotL)))
    inside the float64 interval of tests/pcf_ref.py;
  * the cube axis path against the general count on every pixel where cube_axis_is_certain holds, without the warp vote, and
    every one of the six faces' axis paths taken by at least one whole warp;
  * sqrt_rn_inrange against __fsqrt_rn on every fp32 of len2_inrange's domain, and fdiv / fdiv2 / fdiv3 against __fdiv_rn on 2^30
    log-uniform pairs of div_fast_ok's domain plus the edges of that domain, texel-boundary quotients and subnormal quotients.
Then the shipped path, vq_forward_lighting_shadowed: each caster's tap counts recovered from the radiance it produces alone equal
the harness records, and the whole pass matches the oracle with no flip budget outside the spot pixels the interval explains."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest
import torch

import oracle_lib as orc
import pcf_ref
import shadow_domain as sd
from envmaps import small_env
from gpu_util import TOL, dev, host

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]


@pytest.fixture(scope="module")
def dclib(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out = tmp_path_factory.mktemp("devicecheck") / "libshadowdevice.so"
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), *FLAGS, "-o", str(out),
                           os.path.join(ROOT, "tests", "device_check", "shadow_math_device.cu")])
    torch.cuda.init()
    lib = C.CDLL(str(out))
    lib.dc_div_sweep.argtypes = [C.c_ulonglong, C.c_ulonglong, C.c_void_p, C.c_void_p, C.c_void_p]
    lib.dc_sqrt_sweep.argtypes = [C.c_uint, C.c_uint, C.c_void_p, C.c_void_p]
    return lib


@pytest.fixture(scope="module")
def hostlib(tmp_path_factory):
    out = tmp_path_factory.mktemp("hostcheck") / "libshadowhost.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", str(out),
                           os.path.join(ROOT, "tests", "host_check", "shadow_math_host.cpp")])
    return C.CDLL(str(out))


@pytest.fixture(scope="module")
def scenes():
    return sd.scenes()


def _ptr(t):
    return C.c_void_p(t.data_ptr())


class Maps:
    """the scene's maps on the device and the VqShadowMaps over them"""
    def __init__(self, vq, s):
        self.t = [dev(s.cubes), dev(s.spots), dev(s.dmap)]
        self.sm = s.shadow_maps_struct(vq, *(t.data_ptr() for t in self.t))


def _crop(s, width, rows=None):
    r0, r1 = rows if rows else (0, s.H)
    return [np.ascontiguousarray(p[r0:r1, :width]) for p in s.planes]


def device_records(dclib, vq, s, planes):
    h, w = planes[0].shape[:2]
    maps = Maps(vq, s)
    pos, nrm = dev(planes[0]), dev(planes[1])
    rec = torch.zeros(h * w, dtype=torch.int64, device="cuda")
    cnt = torch.zeros(h * w * 11, dtype=torch.int32, device="cuda")
    assert dclib.dc_pcf_records(C.byref(s.pf), C.byref(s.pv), C.byref(maps.sm), _ptr(pos), _ptr(nrm), C.c_int(w), C.c_int(h),
                                _ptr(rec), _ptr(cnt)) == 0
    return host(rec).view(np.uint64), host(cnt).reshape(-1, 11).T.astype(np.int64)


def host_records(hostlib, vq, s, planes):
    h, w = planes[0].shape[:2]
    sm = s.shadow_maps_struct(vq)
    p = [np.ascontiguousarray(a, np.float32) for a in planes[:2]]
    rec = np.zeros(h * w, np.uint64)
    hostlib.hostcheck_pcf_records(C.byref(s.pf), C.byref(s.pv), C.byref(sm), orc._p(p[0]), orc._p(p[1]), C.c_int(h * w),
                                  rec.ctypes.data_as(C.c_void_p))
    return rec


def _interval(s, planes):
    """pcf_ref.all_counts on a crop of the scene"""
    class View:
        pass
    v = View()
    v.__dict__.update(s.__dict__)
    v.planes = planes
    return pcf_ref.all_counts(v)


SHAPES = [("full", sd.W, None), ("ragged97", 97, None), ("width1", 1, None), ("odd_rows", sd.W, (3, 7))]


@pytest.mark.parametrize("shape", SHAPES, ids=[x[0] for x in SHAPES])
@pytest.mark.parametrize("idx", range(len(sd.SIZES)))
def test_device_records_equal_host_build(dclib, hostlib, vq, scenes, idx, shape):
    s = scenes[idx]
    _, width, rows = shape
    planes = _crop(s, width, rows)
    rec, cnt = device_records(dclib, vq, s, planes)
    want = host_records(hostlib, vq, s, planes)
    got, exp = pcf_ref.decode(rec), pcf_ref.decode(want)
    assert np.array_equal(got, np.where(cnt < 0, 0, cnt))                    # the record holds what the sink was handed
    exact = [*range(5), 10]
    bad = np.argwhere(got[exact] != exp[exact])
    assert len(bad) == 0, [(exact[k], int(j), int(got[exact[k], j]), int(exp[exact[k], j])) for k, j in bad[:8]]
    lo, hi, _ = _interval(s, planes)
    flips = np.argwhere(got[5:10] != exp[5:10])
    out = [(5 + k, int(j), int(got[5 + k, j]), int(exp[5 + k, j]), int(lo[5 + k, j]), int(hi[5 + k, j])) for k, j in flips]
    print(f"scene {idx} {shape[0]}: observable pixels per slot {[(int((c >= 0).sum())) for c in cnt]}; spot flips "
          f"(slot, pixel, device, host, lo, hi): {out}")
    assert all(l <= g <= h for _, _, g, _, l, h in out), out


@pytest.mark.parametrize("idx", range(len(sd.SIZES)))
def test_axis_path_equals_general_path(dclib, hostlib, vq, scenes, idx):
    s = scenes[idx]
    n = s.H * sd.W
    maps = Maps(vq, s)
    pos = dev(s.planes[0])
    out = torch.zeros(5 * n * 4, dtype=torch.int32, device="cuda")
    assert dclib.dc_point_paths(C.byref(s.pf), C.byref(s.pv), C.byref(maps.sm), _ptr(pos), C.c_int(n), _ptr(out)) == 0
    r = host(out).reshape(5, n, 4).astype(np.int64)
    general, fast, axis, certain = r[..., 0], r[..., 1], r[..., 2], r[..., 3].astype(bool)
    assert certain.any()
    assert np.array_equal(fast[certain], general[certain]), np.argwhere(certain & (fast != general))[:8]
    assert (fast[~certain] == -1).all()
    want = host_records(hostlib, vq, s, s.planes)
    P = s.planes[0].reshape(-1, 4)[:, :3].astype(np.float64)
    for i in range(5):
        in_range = np.linalg.norm(P - s.point_pos[i], axis=-1) < s.point_range[i]
        assert np.array_equal(general[i][in_range], pcf_ref.decode(want)[i][in_range])
    groups = np.array(s.groups)
    # the certainty bound: every lane of a gap_above warp certain, none of gap_below
    for name, flag in (("gap_above", True), ("gap_below", False)):
        w = np.nonzero(groups == name)[0][0]
        assert (certain[0, 32 * w:32 * w + 32] == flag).all(), name
    # which warps the vote sends down an axis path, per face (axis, sign of the major component of the tap direction)
    faces = np.zeros(6, np.int64)
    for i in range(5):
        Lw = s.point_pos[i] - P.astype(np.float32)
        inr = np.linalg.norm(Lw, axis=-1) < s.point_range[i]
        for w in range(n // 32):
            sl = slice(32 * w, 32 * w + 32)
            if not inr[sl].any():
                continue
            a0 = axis[i, sl][inr[sl]][0]
            if (~inr[sl] | (certain[i, sl] & (axis[i, sl] == a0))).all():
                lane = np.nonzero(inr[sl])[0][0]
                faces[2 * a0 + int(-Lw[sl][lane, a0] < 0)] += 1
    print(f"scene {idx}: warps on the axis path per face (+X -X +Y -Y +Z -Z): {faces.tolist()}")
    assert (faces > 0).all(), faces


def test_sqrt_rn_inrange_exhaustive(dclib):
    lo = int(np.float32(1e-30).view(np.uint32)); hi = int(np.float32(1e30).view(np.uint32)) + 1
    cnt = torch.zeros(3, dtype=torch.int64, device="cuda")
    first = torch.full((1,), -1, dtype=torch.int32, device="cuda")          # atomicMin on unsigned: starts at 0xffffffff
    assert dclib.dc_sqrt_sweep(lo, hi, _ptr(cnt), _ptr(first)) == 0
    c = host(cnt)
    print(f"sqrt_rn_inrange: {int(c[2])} inputs in len2_inrange, {int(c[0])} differ from __fsqrt_rn")
    assert c[0] == 0, hex(int(host(first)[0]) & 0xFFFFFFFF)
    assert c[2] == hi - lo - 2                                                 # every fp32 strictly between 1e-30f and 1e30f


def test_division_sampled_and_edges(dclib):
    n = 1 << 30
    cnt = torch.zeros(4, dtype=torch.int64, device="cuda")
    maxsub = torch.zeros(2, dtype=torch.int32, device="cuda")
    firstbad = torch.zeros(3, dtype=torch.float32, device="cuda")
    assert dclib.dc_div_sweep(0x5EED, n, _ptr(cnt), _ptr(maxsub), _ptr(firstbad)) == 0
    c = host(cnt)
    print(f"fdiv/fdiv2/fdiv3: {n} draws, {int(c[1])} inside div_fast_ok, 6 quotients each; {int(c[2])} subnormal results "
          f"(largest difference {int(host(maxsub)[0])} subnormal ulp); {int(c[3])} results with |numerator| < 2^-100 "
          f"(largest difference {int(host(maxsub)[1])} ulp); {int(c[0])} mismatches")
    assert c[0] == 0, host(firstbad)
    assert c[1] > 0.9 * n and c[2] > 0 and int(host(maxsub)[0]) <= 1 and int(host(maxsub)[1]) <= 1
    # the edges of the fast domain, exact texel-boundary quotients, subnormal quotients
    f = np.float32
    inside_b = [np.nextafter(f(1e-15), f(1)), np.nextafter(f(1e15), f(0))]
    a_list, b_list = [], []
    rng = np.random.default_rng(5)
    for b in inside_b + [-x for x in inside_b]:
        for a in [f(0), -f(0), np.nextafter(f(1e15), f(0)), -np.nextafter(f(1e15), f(0)), f(1), f(3.3e-38), f(1e-45), *rng.uniform(-1e3, 1e3, 8).astype(f)]:
            a_list.append(a); b_list.append(b)
    for N in (1, 2, 5, 7, 8, 16, 33, 64):                                      # q = k/N * b / b: a = q*b exact, quotient q
        for k in range(-N, N + 1):
            q = f(2 * k / N - 1) if N & (N - 1) == 0 else f(k) / f(N)
            for b in rng.uniform(0.5, 40, 4).astype(f):
                a = f(q * b)
                if float(a) == float(q) * float(b):
                    a_list.append(a); b_list.append(b)
    for e in range(-30, -20):                                                  # subnormal quotients
        for b in (f(1e14), f(3.7e13), f(9.9e14)):
            a_list.append(f(1.3 * 10.0 ** e)); b_list.append(b)
    a_t, b_t = dev(np.array(a_list, f)), dev(np.array(b_list, f))
    out = torch.zeros(len(a_list) * 4, dtype=torch.float32, device="cuda")
    assert dclib.dc_div_list(_ptr(a_t), _ptr(b_t), C.c_int(len(a_list)), _ptr(out)) == 0
    q = host(out).reshape(-1, 4)
    r = q.view(np.uint32).astype(np.int64)
    sub = (np.abs(q[:, 3]) < np.finfo(np.float32).tiny) | (np.abs(np.array(a_list, f)) < f(2.0 ** -100))
    # a zero numerator: the fast path returns +0 (its correction adds +0 to -0) where __fdiv_rn keeps the sign; no comparison,
    # floor or fma downstream can tell the two apart, so they count as equal here (and are reported)
    zero = (q[:, :3] == 0) & (q[:, 3:4] == 0)
    d = np.where(zero, 0, np.abs(r[:, :3] - r[:, 3:4]))
    print(f"division edge list: zero numerators whose quotient's sign differs from __fdiv_rn: {int((zero & (r[:, :3] != r[:, 3:4])).any(1).sum())}")
    assert (d[~sub] == 0).all(), np.argwhere(d[~sub] != 0)[:5]
    assert (d[sub] <= 1).all()
    print(f"division edge list: {len(a_list)} operand pairs, {int(sub.sum())} subnormal quotients, max subnormal ulp {int(d[sub].max()) if sub.any() else 0}")


# ---- the shipped path: vq_forward_lighting_shadowed -------------------------------------------------------------------------
def _copy(ct):
    return type(ct).from_buffer_copy(ct)


def _shipped(ctx, vq, s, pf, planes, maps, zero_env, rows=None):
    h, w = planes[0].shape[:2]
    dpl = [dev(p) for p in planes[:3]]
    gb = vq.GBuffer(vq.image_of(dpl[0]), vq.image_of(dpl[1]), vq.image_of(dpl[2]), vq.null_image())
    env = small_env()
    tens = [dev(np.zeros_like(env[k]) if zero_env else env[k]) for k in ("diff", "spec", "lut")]
    em = vq.EnvironmentMaps(vq.cubemap_of(tens[0], env["diff_res"], 1), vq.cubemap_of(tens[1], env["spec_res"], env["spec_mips"]),
                            vq.image_of(tens[2], 2))
    out = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
    rb, re = rows if rows else (0, h)
    ctx.forward_lighting_shadowed(pf, s.pv, gb, em, out, point_cubes=maps[0] if maps else None, spot_maps=maps[1] if maps else None,
                                  directional_map=maps[2] if maps else None, row_begin=rb, row_end=re)
    return host(out)


def _isolate(s, slot):
    """every light dark but caster `slot` (all eleven casters stay in the lists), no ambient"""
    pf = _copy(s.pf)
    L = pf.Lights
    L.numPointLights = 0; L.numSpotLights = 0
    pf.fAmbientLightingFactor = 0.0
    for i in range(5):
        if i != slot: L.point_casters[i].brightness = 0.0
        if 5 + i != slot: L.spot_casters[i].brightness = 0.0
    if slot != 10: L.directional.brightness = 0.0
    return pf


SHIPPED = [("full", sd.W, None), ("ragged97", 97, None), ("width1", 1, None), ("odd_rows", sd.W, (3, 7))]


@pytest.mark.parametrize("shape", SHIPPED, ids=[x[0] for x in SHIPPED])
@pytest.mark.parametrize("idx", [0, 2, 4])
def test_shipped_counts_equal_harness_records(ctx, vq, dclib, scenes, idx, shape):
    s = scenes[idx]
    _, width, rows = shape
    planes = _crop(s, width)
    rec, cnt = device_records(dclib, vq, s, planes)
    want = pcf_ref.decode(rec)
    maps = [dev(s.cubes), dev(s.spots), dev(s.dmap)]
    r0, r1 = rows if rows else (0, planes[0].shape[0])
    # what stays lit with every light dark (the G-buffer's own terms): subtracted from both runs
    dark_pf = _isolate(s, 10)
    dark_pf.Lights.directional.brightness = 0.0
    dark = _shipped(ctx, vq, s, dark_pf, planes, None, True, rows)[r0:r1].astype(np.float64)
    seen = []
    for slot in range(11):
        pf = _isolate(s, slot)
        N = 20 if slot < 5 else 25
        out = _shipped(ctx, vq, s, pf, planes, maps, True, rows)[r0:r1].astype(np.float64)
        lit = _shipped(ctx, vq, s, pf, planes, None, True, rows)[r0:r1].astype(np.float64) - dark
        ch = np.nan_to_num(lit[..., :3], nan=-1).argmax(-1)
        lv = np.take_along_axis(lit[..., :3], ch[..., None], -1)[..., 0]
        ov = np.take_along_axis(out[..., :3] - dark[..., :3], ch[..., None], -1)[..., 0]
        obs = np.isfinite(lv) & np.isfinite(ov) & (lv > 1e-3 * np.nanmax(lv, initial=1e-30))
        c = N * (1 - ov[obs] / lv[obs])
        assert (np.abs(c - np.rint(c)) < 1e-3).all(), np.abs(c - np.rint(c)).max()
        exp = want[slot].reshape(planes[0].shape[:2])[r0:r1][obs]
        assert np.array_equal(np.rint(c).astype(np.int64), exp), (slot, np.argwhere(np.rint(c) != exp)[:5])
        seen.append(int(obs.sum()))
    print(f"scene {idx} {shape[0]}: observable pixels per slot {seen}")
    assert sum(seen) > 0


@pytest.mark.parametrize("idx", range(len(sd.SIZES)))
def test_shipped_pass_matches_oracle_without_flip_budget(ctx, vq, orc, dclib, hostlib, scenes, idx):
    s = scenes[idx]
    env = small_env()
    maps = [dev(s.cubes), dev(s.spots), dev(s.dmap)]
    got = _shipped(ctx, vq, s, s.pf, s.planes, maps, False)
    ref = orc.forward_lighting_shadowed(s.pf, s.pv, s.planes, env["diff"], env["diff_res"], env["spec"], env["spec_res"],
                                        env["spec_mips"], env["lut"], point_cubes=s.cubes, point_res=s.cube_res, spot_maps=s.spots,
                                        dir_map=s.dmap)
    # a pixel exactly at a light's position (distance 0: the attenuation 1/d^2 is inf) is not a PCF question: the oracle gives
    # NaN there; its PCF records are still compared above. Every other pixel must be finite on both sides.
    P = s.planes[0].reshape(-1, 4)[:, :3]
    lights = np.concatenate([s.point_pos, [v["eye"] for v in s.spot_views]]).astype(np.float32)
    at_light = (P[:, None, :] == lights[None]).all(-1).any(-1)
    finite = np.isfinite(ref).all(-1).reshape(-1)
    assert np.array_equal(~finite, at_light & ~finite) and np.isfinite(got).all(-1).reshape(-1)[~at_light].all()
    d = np.abs(got.astype(np.float64) - ref.astype(np.float64))
    bad = (d > TOL * np.maximum(1.0, np.abs(ref))).any(-1).reshape(-1) & ~at_light
    rec, _ = device_records(dclib, vq, s, s.planes)
    dv, hv = pcf_ref.decode(rec), pcf_ref.decode(host_records(hostlib, vq, s, s.planes))
    lo, hi, _ = pcf_ref.all_counts(s)
    spot_flip = (dv[5:10] != hv[5:10]) & (dv[5:10] >= lo[5:10]) & (dv[5:10] <= hi[5:10])
    explained = spot_flip.any(0)
    listed = [(int(j), [(5 + k, int(dv[5 + k, j]), int(hv[5 + k, j]), int(lo[5 + k, j]), int(hi[5 + k, j]))
                        for k in np.nonzero(spot_flip[:, j])[0]]) for j in np.nonzero(bad)[0]]
    print(f"scene {idx}: {int(at_light.sum())} pixels at a light's position left out; {int(bad.sum())} pixels outside the HDR "
          f"bound, explained by spot flips: {listed}")
    assert not (bad & ~explained).any(), [j for j in np.nonzero(bad & ~explained)[0][:8]]
    assert (got[..., 3] == ref[..., 3]).all()
