"""-m gpu: the environment-map passes over the whole domain of their inputs (tests/ibl_domain.py), against the float64
restatement (tests/ibl_ref.py) and the oracle.

tests/device_check/equirect_device.cu builds the product's sampling header (vq_equirect.cuh) for sm_90a with the flags of build.sh:
  * atan01 on every fp32 in [0, 1] against double atan (the documented 1.0e-7 must hold);
  * dir_to_equirect on 2^30 pseudo-random directions, the axes with every sign of zero, the seam and the pole neighbourhoods;
  * sample_equirect_level against the oracle's sampler and the float64 one, within the float64 bound;
  * normalize_exact(cube_texel_dir(..)).z on the texels whose tangent-frame decision is within rounding of 0.999.
Then the shipped passes:
  * single-sample probes whose every texel is one environment sample or a closed form: K3 at num_samples = 1 (a trilinear
    sample at N at lod 0.5 log2(6 W H r^4) - 1), K2 at n_phi = 1, n_theta = 2 (one sample 45 degrees from N, every src_mip),
    K4 at num_samples = 1 (((1 - Fc) max(G, 1e-4), Fc max(G, 1e-4))), on every LUT shape, a padded pitch and row ranges;
  * K11 bit-exact against the oracle on every shape and content, special values included, on both paths;
  * whole-domain parity of K2 and K3 at the bounds of DESIGN.md §5;
  * the row-constant identity of K2: faces related by negated components are bit-identical."""
import ctypes as C
import math
import os
import subprocess

import numpy as np
import pytest
import torch

import ibl_domain as dom
import ibl_ref as ref
from gpu_util import TOL, assert_scaled, dev, host, report

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]


@pytest.fixture(scope="module")
def dclib(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out = tmp_path_factory.mktemp("devicecheck") / "libequirectdevice.so"
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), *FLAGS, "-o", str(out),
                           os.path.join(ROOT, "tests", "device_check", "equirect_device.cu")])
    torch.cuda.init()
    lib = C.CDLL(str(out))
    vp = C.c_void_p
    lib.dc_atan01_sweep.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32, vp, vp]
    lib.dc_dir_sweep.argtypes = [C.c_uint64, C.c_uint64, C.c_uint32, vp, vp, vp, vp]
    lib.dc_dir_list.argtypes = [vp, C.c_int, vp]
    lib.dc_sample_list.argtypes = [vp, C.c_int, C.c_int, C.c_int, vp, vp, C.c_int, vp]
    lib.dc_texel_frame.argtypes = [vp, C.c_int, vp]
    return lib


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def _pyramid(ctx, vq, orc, img, levels=None):
    """img [h, w, 4] -> (kernel pyramid tensor, oracle pyramid array, levels) after K11 on both sides"""
    h, w = img.shape[:2]
    levels = levels or vq.mip_level_count(w, h)
    d = torch.zeros((vq.pyramid_texel_count(w, h, levels), 4), dtype=torch.float32, device="cuda")
    d[: w * h] = dev(img).reshape(-1, 4)
    ctx.hdri_build_mips(vq.pyramid_of(d, w, h, levels))
    return d, orc.hdri_build_mips(img, levels), levels


# ---- the sampling header on the device -----------------------------------------------------------------------------
def test_atan01_exhaustive(dclib):
    """every fp32 q in [0, 1] (bit patterns 0 .. 0x3f800000): |atan01(q) - atan(q)| within the documented 1.0e-7"""
    hi, per = 0x3F800001, 64
    blocks = (hi + 256 * per - 1) // (256 * per)
    e = torch.zeros(blocks, dtype=torch.float64, device="cuda"); a = torch.zeros(blocks, dtype=torch.int32, device="cuda")
    assert dclib.dc_atan01_sweep(0, hi, per, _ptr(e), _ptr(a)) == 0
    he, ha = host(e), host(a).view(np.uint32)
    k = int(he.argmax())
    q = float(ha[k:k + 1].view(np.float32)[0])
    print(f"atan01: max |error| {he[k]:.4e} at q = {q!r} over {hi} inputs")
    assert he[k] <= ref.ATAN01_ERR


def test_dir_to_equirect_sweep(dclib):
    """2^30 pseudo-random fp32 directions (uniform in y: every latitude): |du| (wrapped) and |dv| against double atan2 / asin
    of the same fp32 components within the compute error ibl_ref charges the kernels"""
    n, per = 1 << 30, 64
    blocks = (n + 256 * per - 1) // (256 * per)
    bufs = [torch.zeros(blocks, dtype=t, device="cuda") for t in (torch.float64, torch.int32, torch.float64, torch.int32)]
    assert dclib.dc_dir_sweep(0x5EED, n, per, *(_ptr(b) for b in bufs)) == 0
    eu, ev = float(host(bufs[0]).max()), float(host(bufs[2]).max())
    cu, cv = ref.uv_compute_error()
    print(f"dir_to_equirect over 2^30 directions: max |du| {eu:.3e} (bound {cu:.3e}), max |dv| {ev:.3e} (bound {cv:.3e})")
    assert eu <= cu and ev <= cv


def _special_dirs():
    z = (0.0, -0.0)
    axes = [(sx * 1.0, a, b) for sx in (1, -1) for a in z for b in z] + [(a, sy * 1.0, b) for sy in (1, -1) for a in z for b in z] \
        + [(a, b, sz * 1.0) for sz in (1, -1) for a in z for b in z]
    seam = [(-x, y, zz) for x in (1.0, 0.5, 1e-20) for y in (0.0, 0.3, -0.9) for zz in z]
    pole = [(x, sy * math.sqrt(max(0.0, 1 - x * x - zz * zz)), zz) for sy in (1, -1)
            for x, zz in ((1e-3, 0), (0, 1e-3), (-2e-4, 3e-4), (3e-6, -2e-6), (-1e-8, -1e-8), (2.0 ** -12, 0))]
    near = [(float(np.float32(x)), sy * float(np.float32(1 - k * 2.0 ** -24)), 0.0) for sy in (1, -1) for k in (1, 2, 3)
            for x in (2.0 ** -11, 0.0)]
    return np.array(axes + seam + pole + near, np.float32)


def test_dir_to_equirect_special_directions(dclib, orc):
    """axes with every sign of zero, the seam (z = +-0, x < 0) and the pole neighbourhoods: u, v within the compute error of
    float64 (u = 0 and u = 1 are one column); where the direction is exactly on a pole the kernel and libm may disagree on u
    (atan2(+-0, -0)), which only matters if the pole rows are not constant"""
    d = _special_dirs()
    uv = torch.zeros((len(d), 2), device="cuda")
    assert dclib.dc_dir_list(_ptr(dev(d)), len(d), _ptr(uv)) == 0
    got = host(uv).astype(np.float64)
    u, v = ref.direction_to_uv(d.astype(np.float64))
    cu, cv = ref.uv_compute_error()
    du = np.abs(got[:, 0] - u); du = np.minimum(du, np.abs(1 - du))
    pole = (d[:, 0] == 0) & (d[:, 2] == 0)
    assert (du[~pole] <= cu).all(), d[~pole][du[~pole] > cu]
    assert (np.abs(got[:, 1] - v) <= cv).all()
    print("exact-pole u (kernel, float64):", list(zip(got[pole, 0], u[pole])))


@pytest.mark.parametrize("kind", ["synth", "seam", "noisy_poles", "denormal"])
@pytest.mark.parametrize("w,h,levels", [(97, 41, 3), (256, 128, None), (7, 3, None), (8, 1024, None)])
def test_sample_equirect_level_device(dclib, vq, orc, kind, w, h, levels):
    img = dom.content(kind, w, h)
    levels = levels or vq.mip_level_count(w, h)
    pyr = orc.hdri_build_mips(img, levels)
    rng = np.random.default_rng(w * 31 + h)
    n = 20000
    uvl = np.stack([np.concatenate([rng.uniform(0, 1, n), [0, 1, 0.5 / w, 1 - 0.5 / w]]),
                    np.concatenate([rng.uniform(0, 1, n), [1, 0, 0.5 / h, 1 - 0.5 / h]]),
                    np.concatenate([rng.uniform(-1, levels + 1, n), [0, levels - 1, levels + 3, 0.5]])], 1).astype(np.float32)
    off = np.array([vq.pyramid_offset(w, h, l) for l in range(levels)], np.uint32)
    out = torch.zeros((len(uvl), 3), device="cuda")
    assert dclib.dc_sample_list(_ptr(dev(pyr)), w, h, levels, off.ctypes.data_as(C.c_void_p), _ptr(dev(uvl)), len(uvl), _ptr(out)) == 0
    got = host(out).astype(np.float64)
    L = ref.pyramid_levels(pyr, w, h, levels)
    u, v, lod = (uvl[:, k].astype(np.float64) for k in range(3))
    want = ref.sample(L, u, v, lod)
    bound = ref.sample_bound(L, u, v, lod, 0.0, 0.0, np.abs(lod) * ref.EPS)
    assert (np.abs(got - want) <= bound).all(), (np.abs(got - want) / np.maximum(bound, 1e-300)).max()
    o = np.zeros((len(uvl), 3)); t = np.zeros(4, np.float32)
    for i in range(0, len(uvl), 7):
        orc.lib().orc_sample_equirect(orc._p(pyr), w, h, levels, C.c_float(uvl[i, 0]), C.c_float(uvl[i, 1]), C.c_float(uvl[i, 2]), orc._p(t))
        o[i] = t[:3]
    idx = np.arange(0, len(uvl), 7)
    assert (np.abs(got[idx] - o[idx]) <= 2 * bound[idx]).all()


def test_frame_decisions_near_threshold(dclib):
    """the +-Z texels whose |N.z| is within 2 ulp of 0.999f at even res up to 1024 and 800 (legal with <= 5 mips): the device's
    normalize_exact decision equals the float64 one wherever that is decided; undecided ones are counted and reported"""
    sizes = [800] + list(range(2, 1025, 2))
    t = dom.near_threshold_texels(sizes)
    assert len([x for x in t if x[3] == 800 and x[0] == 4]) > 0
    arr = np.array(t, np.int32)
    out = torch.zeros((len(arr), 4), device="cuda")
    assert dclib.dc_texel_frame(_ptr(torch.from_numpy(arr).cuda()), len(arr), _ptr(out)) == 0
    o = host(out)
    d = np.stack([ref.cube_texel_direction(f, x, y, r) for f, x, y, r in t])
    z64, undecided = ref.frame_decision(d)
    dev_z = o[:, 3] == 1.0
    # the oracle's fp32 decision: normalize = v / sqrt(dot) with an unfused dot, correctly rounded sqrt and division
    f32 = np.float32
    d32 = d.astype(f32)
    l2 = (d32[:, 0] * d32[:, 0] + d32[:, 1] * d32[:, 1]).astype(f32) + d32[:, 2] * d32[:, 2]
    orc_z = np.abs(d32[:, 2] / np.sqrt(l2.astype(f32))) < f32(0.999)
    print(f"near-threshold texels: {len(t)}, undecided in float64: {int(undecided.sum())}, "
          f"device == float64 on the decided: {bool((dev_z == z64)[~undecided].all())}, "
          f"device == oracle: {int((dev_z == orc_z).sum())} of {len(t)}, device z-frame: {int(dev_z.sum())}")
    assert (dev_z == z64)[~undecided].all()
    assert (dev_z == orc_z).all()


# ---- single-sample probes -------------------------------------------------------------------------------------------
def _cube_texels(res, mips, faces=range(6), min_mip=0):
    """(mip, face, py, px, flat index) of every texel of the packed cube on the given faces / mips"""
    rows = []
    off = 0
    for m in range(mips):
        n = res >> m
        for f in range(6):
            if m >= min_mip and f in faces:
                py, px = np.mgrid[0:n, 0:n]
                rows.append(np.stack([np.full(n * n, m), np.full(n * n, f), py.ravel(), px.ravel(),
                                      off + f * n * n + py.ravel() * n + px.ravel()], 1))
        off += 6 * n * n
    return np.concatenate(rows)


K3_PROBES = [((2, 2), (256, 128, None), "synth", {}), ((4, 3), (256, 128, None), "noisy_poles", {}),
             ((48, 4), (97, 41, None), "seam", {}), ((48, 4), (256, 128, 3), "synth", {}),       # lod clamp at levels-1
             ((800, 5), (256, 128, None), "synth", dict(faces=(4, 5), min_mip=1)),
             ((512, 10), (1024, 512, None), "synth", dict(min_mip=5)), ((16, 5), (64, 32, 2), "row_constant", {})]


@pytest.mark.parametrize("cube,hdri,kind,sel", K3_PROBES, ids=[f"{c[0]}x{c[1]}-{h[0]}x{h[1]}L{h[2]}-{k}" for c, h, k, _ in K3_PROBES])
def test_k3_single_sample_probe(ctx, vq, orc, cube, hdri, kind, sel):
    res, mips = cube
    w, h, lv = hdri
    d, pyr, levels = _pyramid(ctx, vq, orc, dom.content(kind, w, h), lv)
    out = torch.zeros((vq.cubemap_texel_count(res, mips), 4), device="cuda")
    ctx.specular_prefilter(vq.pyramid_of(d, w, h, levels), vq.cubemap_of(out, res, mips), num_samples=1)
    got = host(out)
    t = _cube_texels(res, mips, **sel)
    o_ref = orc.specular_prefilter_texels(pyr, w, h, levels, res, mips, t[:, 4], num_samples=1)
    L = ref.pyramid_levels(pyr, w, h, levels)
    worst_k = worst_o = 0.0
    pole_needed = 0
    for m in np.unique(t[:, 0]):
        sel_m = t[:, 0] == m
        tm = t[sel_m]
        r = float(np.float32(m) / np.float32(mips - 1))
        N = ref.normalize(ref.cube_texel_direction(tm[:, 1], tm[:, 3], tm[:, 2], res >> m))
        lod = 0.0 if r == 0 else ref.k3_single_sample_lod(r, w, h)
        dlod = 0.0 if r == 0 else ref.k3_single_sample_lod_error(r)
        u, v = ref.direction_to_uv(N)
        want = ref.sample(L, u, v, lod)
        du, dv = ref.uv_delta(N, ref.DIR_DELTA)
        bound = ref.sample_bound(L, u, v, lod, du, dv, dlod) + 4 * ref.EPS * np.abs(want)
        k = got[tm[:, 4], :3].astype(np.float64)
        o = o_ref[sel_m, :3].astype(np.float64)
        assert (got[tm[:, 4], 3] == 1.0).all()
        ek, eo = np.abs(k - want), np.abs(o - want)
        worst_k = max(worst_k, float((ek / np.maximum(bound, 1e-300)).max()))
        worst_o = max(worst_o, float((eo / np.maximum(bound, 1e-300)).max()))
        rho = np.hypot(N[:, 0], N[:, 2])
        pole_needed += int(((ek > 0).any(axis=1) & (rho < 1e-3)).sum())
        assert (ek <= bound).all(), (m, float((ek / np.maximum(bound, 1e-300)).max()))
        assert (eo <= bound).all(), (m, float((eo / np.maximum(bound, 1e-300)).max()))
    print(f"K3 probe {cube} on {hdri} {kind}: kernel / bound {worst_k:.3f}, oracle / bound {worst_o:.3f}, "
          f"texels within 1e-3 rad of a pole with an error: {pole_needed}")


@pytest.mark.parametrize("res", [2, 6, 30])
@pytest.mark.parametrize("w,h,kind", [(256, 128, "synth"), (97, 41, "noisy_poles"), (1024, 8, "seam")])
def test_k2_single_sample_probe(ctx, vq, orc, res, w, h, kind):
    d, pyr, levels = _pyramid(ctx, vq, orc, dom.content(kind, w, h))
    L = ref.pyramid_levels(pyr, w, h, levels)
    t = _cube_texels(res, 1)
    N = ref.normalize(ref.cube_texel_direction(t[:, 1], t[:, 3], t[:, 2], res))
    phis, ths = ref.k2_angles(0.0, 1, 2)
    sd = ref.k2_sample_dirs(N, phis[0], ths[1])
    u, v = ref.direction_to_uv(sd)
    du, dv = ref.uv_delta(sd, ref.DIR_DELTA)
    wgt = math.pi * math.cos(ths[1]) * math.sin(ths[1]) / 2.0
    worst = 0.0
    for src in range(levels):
        out = torch.zeros((6 * res * res, 4), device="cuda")
        ctx.diffuse_irradiance(vq.pyramid_of(d, w, h, levels), vq.cubemap_of(out, res, 1), n_phi=1, n_theta=2, src_mip=src)
        got = host(out)[:, :3].astype(np.float64)
        o = orc.diffuse_irradiance(pyr, w, h, levels, res, n_phi=1, n_theta=2, src_mip=src)[:, :3].astype(np.float64)
        want = wgt * ref.sample(L, u, v, float(src))
        bound = wgt * ref.sample_bound(L, u, v, float(src), du, dv, 0.0) + 32 * ref.EPS * np.abs(want)
        worst = max(worst, float((np.abs(got - want) / np.maximum(bound, 1e-300)).max()))
        assert (np.abs(got - want) <= bound).all(), (src, float((np.abs(got - want) / np.maximum(bound, 1e-300)).max()))
        assert (np.abs(o - want) <= bound).all(), src
    print(f"K2 probe res {res} on {w}x{h} {kind}: kernel / bound {worst:.3f}")


LUTS = [(64, 64, None, None), (300, 5, None, None), (513, 3, None, None), (1, 50, None, None), (50, 1, None, None),
        (1, 1, None, None), (40, 9, 48, None), (257, 12, None, (3, 9))]


@pytest.mark.parametrize("w,h,pitch,rows", LUTS, ids=[f"{a}x{b}-p{c}-r{d}" for a, b, c, d in LUTS])
def test_k4_single_sample_probe(ctx, orc, w, h, pitch, rows):
    """num_samples = 1 on wide ragged LUTs, 1 x N / N x 1, a padded row pitch and a row range (rows outside untouched)"""
    buf = torch.full((h, pitch or w, 2), -7.0, device="cuda")
    view = buf[:, :w]
    r0, r1 = rows or (0, h)
    ctx.brdf_integration_lut(view, 1, r0, r1)
    got = host(buf)
    want = ref.brdf_lut_single_sample(w, h)
    tol = ref.brdf_lut_single_sample_bound(w, h)
    ratio = np.abs(got[r0:r1, :w] - want[r0:r1]) / tol[r0:r1]
    o = orc.brdf_integration_lut(w, h, 1)
    print(f"K4 probe {w}x{h}: kernel / bound {ratio.max():.3f}, oracle / bound {(np.abs(o - want) / tol).max():.3f}")
    assert ratio.max() <= 1.0
    assert (np.abs(o - want) <= tol).all()
    untouched = np.ones(got.shape[:2], bool); untouched[r0:r1, :w] = False
    assert (got[untouched] == -7.0).all()


# ---- K11 bit-exact -------------------------------------------------------------------------------------------------
K11_CASES = [(s, c) for s in dom.K11_SHAPES for c in ("special", "ge1", "synth")
             if c != "synth" or s[0] * s[1] <= 4096 * 64 or s[:2] == (8192, 4096)]


@pytest.mark.parametrize("shape,content", K11_CASES, ids=[f"{s[0]}x{s[1]}L{s[2]}-{c}" for s, c in K11_CASES])
def test_k11_bit_exact(ctx, vq, orc, shape, content):
    w, h, levels = shape
    img = dom.special_blocks(w, h) if content == "special" else dom.content(content, w, h)
    d, want, levels = _pyramid(ctx, vq, orc, img, levels)
    got = host(d)
    bad = np.nonzero(got.view(np.uint32) != want.view(np.uint32))[0]
    assert bad.size == 0, (bad[:8], got[bad[:4]], want[bad[:4]])


@pytest.mark.parametrize("kind", ["constant", "row_constant", "seam", "noisy_poles", "zero", "spike65504", "spike2p20", "denormal"])
def test_k11_contents(ctx, vq, orc, kind):
    for w, h in ((97, 41), (4101, 6)):
        d, want, _ = _pyramid(ctx, vq, orc, dom.content(kind, w, h))
        assert np.array_equal(host(d).view(np.uint32), want.view(np.uint32))


# ---- whole-domain parity --------------------------------------------------------------------------------------------
K2_CASES = ([(kind, (w, h), 6, dict(n_phi=64, n_theta=16)) for kind in ("synth", "row_constant", "seam", "noisy_poles", "zero",
                                                                      "spike65504", "denormal", "ge1")
             for w, h in ((7, 3), (97, 41), (1024, 8), (8, 1024))]
            + [("synth", (256, 128), r, dict(n_phi=64, n_theta=16)) for r in (2, 30, 130)]
            + [("synth", (256, 128), 4, dict(step=s)) for s in (float(np.float32(6.28318530718) / 7),
                                                              float(np.float32(1.5707963268) / 3),
                                                              float(np.nextafter(np.float32(1.5707963268) / np.float32(3), np.float32(1))))]
            + [("synth", (64, 32), 2, dict(n_phi=8192, n_theta=256))])       # 67.5 KB of shared memory: the opt-in path


@pytest.mark.parametrize("kind,shape,res,kw", K2_CASES, ids=[f"{k}-{s[0]}x{s[1]}-r{r}-{'-'.join(f'{a}{b:.4g}' for a, b in kw.items())}"
                                                             for k, s, r, kw in K2_CASES])
def test_k2_parity(ctx, vq, orc, kind, shape, res, kw):
    w, h = shape
    d, pyr, levels = _pyramid(ctx, vq, orc, dom.content(kind, w, h))
    src = min(2, levels - 1)
    out = torch.zeros((6 * res * res, 4), device="cuda")
    ctx.diffuse_irradiance(vq.pyramid_of(d, w, h, levels), vq.cubemap_of(out, res, 1), src_mip=src, **kw)
    want = orc.diffuse_irradiance(pyr, w, h, levels, res, src_mip=src, **kw)
    got = host(out)
    if kw.get("n_phi", 0) * kw.get("n_theta", 0) > 100000:
        # 2 M terms: the reference's sequential fp32 running sum carries its own O(n EPS) error, so (as for the engine's
        # 99 382-term step mode) the kernel is held to the same terms summed in double, no further than the oracle is
        want64 = orc.diffuse_irradiance(pyr, w, h, levels, res, src_mip=src, f64_accum=True, **kw)
        own = float(np.abs(want - want64).max())
        print(report("K2 2M-term grid vs f64 sum", got, want64), "oracle's own", own)
        assert np.abs(got - want64).max() <= own + 2e-5
        return
    print(assert_scaled(f"K2 {kind}", got, want, min_frac_strict=0.0))


K3_CASES = [((2, 2), 1), ((2, 2), 2), ((4, 3), 31), ((4, 3), 33), ((4, 3), 4097), ((2, 2), 8192), ((48, 4), 33), ((16, 5), 2)]


@pytest.mark.parametrize("cube,samples", K3_CASES, ids=[f"{c[0]}x{c[1]}-n{s}" for c, s in K3_CASES])
@pytest.mark.parametrize("levels", [None, 3])
def test_k3_parity(ctx, vq, orc, cube, samples, levels):
    res, mips = cube
    w, h = 128, 64
    d, pyr, levels = _pyramid(ctx, vq, orc, dom.content("synth", w, h), levels)
    out = torch.zeros((vq.cubemap_texel_count(res, mips), 4), device="cuda")
    ctx.specular_prefilter(vq.pyramid_of(d, w, h, levels), vq.cubemap_of(out, res, mips), num_samples=samples)
    want = orc.specular_prefilter(pyr, w, h, levels, res, mips, num_samples=samples)
    o = host(out)
    print(assert_scaled(f"K3 n{samples}", o, want, min_frac_strict=0.0))
    small = np.abs(want) <= 4.0
    assert np.abs(o - want)[small].max() <= TOL


def test_k2_row_constant_faces(ctx, vq, orc):
    """u-independent radiance: faces whose texel directions differ only by negated components (+X / -X, +Z / -Z) give
    bit-identical irradiance on the kernel and the oracle (negation is exact, cross((0,1,0), N) negates with N, a lerp
    between equal texels is exact). A 90-degree rotation (+X / +Z) permutes the components of dot(N, N), whose rounding
    depends on the order: there the faces agree to rounding only."""
    w, h, res = 64, 32, 30
    d, pyr, levels = _pyramid(ctx, vq, orc, dom.content("row_constant", w, h))
    out = torch.zeros((6 * res * res, 4), device="cuda")
    ctx.diffuse_irradiance(vq.pyramid_of(d, w, h, levels), vq.cubemap_of(out, res, 1), n_phi=64, n_theta=16, src_mip=1)
    for faces in (host(out).reshape(6, res, res, 4), orc.diffuse_irradiance(pyr, w, h, levels, res, src_mip=1).reshape(6, res, res, 4)):
        assert np.array_equal(faces[0].view(np.uint32), faces[1].view(np.uint32))
        assert np.array_equal(faces[4].view(np.uint32), faces[5].view(np.uint32))
        assert np.abs(faces[0] - faces[4]).max() <= 1e-5 * np.abs(faces).max()
