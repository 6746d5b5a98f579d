"""CPU (-m "not gpu"): the post chain's float64 restatements (tests/post_ref.py) against the oracle over the domain images of
tests/post_domain.py, and the EASU constant check (vqengine_b200/csrc/vq_easu_check.cuh) built for the host and swept over
every constant FsrEasuCon builds for viewport <= input <= 8192 and output <= 16384, under both up-path tilings: vq_fsr_easu's
(easu_up_kernel) and vq_post_process's (post_fsr_up_kernel)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

import oracle_lib as orc
import post_domain as pd
import post_ref as pr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CURVES = [(0, 1, 0), (0, 0, 0), (1, 0, 0), (1, 0, 1), (2, 0, 0), (7, 0, 0)]     # (curve, gamma, colour space)
NITS = [80.0, 200.0, 1000.0, 10000.0]


def same_nonfinite(a, b):
    """NaN where b is NaN, and the same infinities"""
    return np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.where(np.isinf(a), a, 0), np.where(np.isinf(b), b, 0))


def within(got, ref, bound):
    """|got - ref| <= bound wherever ref and bound are finite; returns the largest |got - ref| / bound"""
    m = np.isfinite(ref) & np.isfinite(bound)
    d = np.abs(got.astype(np.float64)[m] - ref[m])
    assert (d <= bound[m]).all(), f"{int((d > bound[m]).sum())} values outside the bound, worst {np.max(d - bound[m]):.3e}"
    return float(np.max(d / np.maximum(bound[m], 1e-300))) if d.size else 0.0


@pytest.fixture(scope="module")
def easu_host(tmp_path_factory):
    out = tmp_path_factory.mktemp("easucheck") / "libeasucheck.so"
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-fPIC", "-ffp-contract=off", "-fno-fast-math", "-shared", "-o", str(out),
                           os.path.join(ROOT, "tests", "host_check", "easu_check_host.cpp")])
    lib = C.CDLL(str(out))
    lib.hostcheck_easu_check.argtypes = [C.POINTER(C.c_float), C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int)]
    lib.hostcheck_easu_f.argtypes = [C.c_float, C.c_float, C.c_int, C.POINTER(C.c_int)]
    return lib


def easu_check(lib, con0, iw, ih, ow, oh, fused=False):
    """the check vq_fsr_easu makes, or with `fused` the one vq_post_process makes: (verdict, (path, ncx, ncy))"""
    c = (C.c_float * 4)(*[float(v) for v in con0[:4]])
    o = (C.c_int * 3)()
    v = lib.hostcheck_easu_check(c, iw, ih, ow, oh, int(fused), o)
    return v, tuple(o)


def con0_of(con):
    return np.frombuffer(bytes(con), np.float32)[:4]


# ---- tonemapper and blur: oracle within the float64 bound ------------------------------------------------------------
@pytest.mark.parametrize("curve,gamma,cs", CURVES)
@pytest.mark.parametrize("nits", NITS)
def test_oracle_tonemap_within_float64_bound(curve, gamma, cs, nits):
    import vqengine_b200 as vq
    img = pd.hdr_domain(61, 37, seed=3)
    got = orc.tonemap(vq.TonemapperParams(cs, curve, nits, gamma, 1.0), img)
    ref, bound = pr.tonemap_ref(img, curve, gamma, cs, nits)
    assert same_nonfinite(got, ref)
    # the oracle divides exactly where the kernel's __fdividef stops (REINHARD_LIMIT): there it is within 2 u of the exact value
    bound = np.where(np.isnan(bound), 2 * pr.U * np.abs(ref), bound)
    within(got, ref, bound)


def test_tonemap_bound_is_tight_where_pq_amplifies():
    """the PQ exponent 78.84 multiplies MUFU.LG2's 2^-22 absolute error: near q = 1 the bound is ~1e-5, inside 1e-4 but far from
    fp32's 6e-8, so the kernel's pow_sfu is the dominant term and is not hidden by the bound"""
    x = np.zeros((1, 4, 4), np.float32)
    x[0, :, :3] = np.array([1.0, 10.0, 100.0, 1000.0])[:, None]
    ref, bound = pr.tonemap_ref(x, 1, 0, 1, 10000.0)
    assert ref[0, 0, 0] == 1.0 and 1e-6 < bound[0, 0, 0] < 1e-4


@pytest.mark.parametrize("w,h", [(1, 1), (5, 1), (1, 2), (31, 17), (97, 33), (515, 7)])
def test_oracle_blur_within_float64_bound(w, h):
    img = pd.hdr_domain(w, h, seed=w + h)
    for vertical, src in ((False, img), (True, orc.gaussian_blur(img, False))):
        got = orc.gaussian_blur(src, vertical)
        ref, bound = pr.blur_ref(src, vertical)
        assert same_nonfinite(got, ref)
        within(got, ref, bound)


def test_blur_ref_sub_rectangle_equals_oracle_on_the_crop():
    img = pd.hdr_domain(97, 33, seed=2, specials=False)
    ref, bound = pr.blur_ref(img, False, size=(40, 20))
    within(orc.gaussian_blur(np.ascontiguousarray(img[:20, :40]), False), ref, bound)


# ---- EASU zro: the generators reach both sides of the decision -------------------------------------------------------
def test_chroma_edges_put_every_easu_pixel_on_the_zro_path():
    img = pd.chroma_edges(64, 32, seed=1)
    con = orc.fsr_easu_con(64, 32, 64, 32, 128, 64)
    dirR, delta, zro, und = pr.easu_zro(img, con, 128, 64, 0)
    assert (dirR == 0).all() and zro.all() and not und.any()


def test_ramps_straddle_the_zro_threshold():
    img = pd.ramps8(96, 72, seed=2)
    con = orc.fsr_easu_con(96, 72, 96, 72, 192, 144)
    dirR, delta, zro, und = pr.easu_zro(img, con, 192, 144, 0)
    near = np.abs(dirR / pr.ZRO - 1) < 0.01
    assert (near & zro & ~und).any() and (near & ~zro & ~und).any(), "ramps do not reach both sides of 1/32768"
    assert 0 < und.mean() < 0.25


# ---- the EASU constant check, host build -----------------------------------------------------------------------------
def _fsr_pairs():
    """(viewport, input, output) per axis: the engine's presets (PostProcess.h: 0.77 / 0.67 / 0.58 / 0.50 per axis), ratios in
    (0.9, 1], ratio 1, anisotropic and downscale pairs, viewport < input, and seeded random pairs"""
    out = []
    for ow, oh in [(1280, 720), (1920, 1080), (2560, 1440), (3840, 2160), (7680, 4320), (16384, 8640), (16384, 16384)]:
        for s in (0.77, 0.67, 0.58, 0.50):
            iw, ih = max(1, int(ow * s)), max(1, int(oh * s))
            if iw <= 8192 and ih <= 8192:
                out.append(((iw, ih), (iw, ih), (ow, oh)))
    for r in (0.91, 0.95, 0.99, 0.999, 1.0):
        for ow in (64, 100, 1000, 4097, 8192):
            iw = max(1, int(round(ow * r)))
            out.append(((iw, iw), (iw, iw), (ow, ow)))
    out += [((8192, 8192), (8192, 8192), (16384, 16384)), ((8192, 1), (8192, 1), (16384, 2)), ((1, 1), (1, 1), (2, 2)),
            ((2, 1), (2, 1), (4, 2)), ((2, 7), (2, 7), (5, 13)), ((64, 64), (64, 64), (128, 40)), ((100, 30), (100, 30), (60, 90)),
            ((120, 80), (120, 80), (90, 60)), ((8192, 8192), (8192, 8192), (1, 1)), ((3000, 2000), (4096, 4096), (6000, 4000))]
    rng = np.random.default_rng(17)
    for _ in range(400):
        iw, ih = (int(v) for v in rng.integers(1, 8193, 2))
        vw, vh = int(rng.integers(1, iw + 1)), int(rng.integers(1, ih + 1))
        ow, oh = (int(v) for v in rng.integers(1, 16385, 2))
        out.append(((vw, vh), (iw, ih), (ow, oh)))
    return out


# post_fsr_up_kernel's tiling (vq_post.cu): 30 x 14 display tiles, EASU on each widened by RCAS's 1-pixel ring, clipped to the
# display, and 32 x 16 candidate 'f' texels. Written out here from the kernel, so that a FUSED_UP_TILE that stops describing
# the kernel fails the comparisons below.
FUSED_TILE, FUSED_RING, FUSED_CAP = (30, 14), 1, (32, 16)


def sweep_fsr_easu_cons(lib, fused, cap):
    """asserts that no FsrEasuCon upscale is refused and that every up-path footprint fits `cap`; returns the number of up-path
    constants and the largest footprint (ncx, ncy)"""
    import vqengine_b200 as vq
    up = worst_x = worst_y = 0
    for (vw, vh), (iw, ih), (ow, oh) in _fsr_pairs():
        c0 = con0_of(vq.fsr_easu_con(vw, vh, iw, ih, ow, oh))
        v, (path, ncx, ncy) = easu_check(lib, c0, iw, ih, ow, oh, fused)
        assert v == 0, ((vw, vh), (iw, ih), (ow, oh), v)
        if path == 1:
            up += 1
            assert 1 <= ncx <= cap[0] and 1 <= ncy <= cap[1], ((vw, vh), (iw, ih), (ow, oh), ncx, ncy)
            worst_x, worst_y = max(worst_x, ncx), max(worst_y, ncy)
    return up, (worst_x, worst_y)


def test_every_fsr_easu_con_is_accepted(easu_host):
    """vq_fsr_easu's check (easu_up_kernel's 32 x 8 tiles): ratio 1 fills the 32-wide tile exactly"""
    up, worst = sweep_fsr_easu_cons(easu_host, False, (32, 8))
    assert up > 50 and worst == (32, 8)


def test_every_fsr_easu_con_runs_fused(easu_host):
    """vq_post_process's check (post_fsr_up_kernel's 30 x 14 tiles and ring): no refusal, and the footprint reaches the
    32 x 16 candidate capacity on both axes"""
    up, worst = sweep_fsr_easu_cons(easu_host, True, FUSED_CAP)
    assert up > 50 and worst == FUSED_CAP


def brute_force_candidates(f, tile, ring):
    """the largest span of 'f' texels (max - min + 1, what a tile stages) over tiles of `tile` outputs at multiples of `tile`,
    each widened by `ring` outputs on both sides and clipped to [0, n_out): taken from every output's 'f'"""
    n_out = len(f)
    return max(int(np.ptp(f[max(o0 - ring, 0):min(o0 + tile + ring, n_out)])) + 1 for o0 in range(0, n_out, tile))


@pytest.mark.parametrize("scale,bias,n_out", [(0.5, -0.25, 4097), (0.77, -0.115, 3000), (0.99, -0.005, 16384), (1.0, 0.0, 999),
                                              (1.0, -0.5, 8192), (3.0, 1.0, 700), (-0.5, 100.0, 300)])
def test_extent_endpoints_bound_every_pixel(easu_host, scale, bias, n_out):
    """easu_pos is monotone, so its two ends bound every output's 'f'; the footprint the check reports under each kernel's
    tiling equals a brute-force count of that tiling"""
    f = (C.c_int * n_out)()
    easu_host.hostcheck_easu_f(scale, bias, n_out, f)
    f = np.array(f)
    assert f.min() == min(f[0], f[-1]) and f.max() == max(f[0], f[-1])
    assert (np.diff(f) * np.sign(scale) >= 0).all()
    if 0 < scale <= 1:
        iw = int(f.max()) + 3
        v, (path, ncx, ncy) = easu_check(easu_host, [scale, scale, bias, bias], iw, iw, n_out, n_out)
        assert v == 0 and path == 1 and ncx == brute_force_candidates(f, 32, 0) and ncy == brute_force_candidates(f, 8, 0)
        v, (path, ncx, ncy) = easu_check(easu_host, [scale, scale, bias, bias], iw, iw, n_out, n_out, fused=True)
        want = tuple(brute_force_candidates(f, t, FUSED_RING) for t in FUSED_TILE)
        assert path == 1 and (ncx, ncy) == want, ((ncx, ncy), want)
        assert v == (0 if want[0] <= FUSED_CAP[0] and want[1] <= FUSED_CAP[1] else 3)


@pytest.mark.parametrize("case", ["stale_after_resize", "viewport_larger", "nan", "inf", "neg_inf", "huge_bias", "far_negative"])
def test_bad_constants_are_refused(easu_host, case):
    import vqengine_b200 as vq
    iw, ih, ow, oh = 100, 60, 200, 120
    c0 = con0_of(vq.fsr_easu_con(iw, ih, iw, ih, ow, oh)).copy()
    want = 2
    if case == "stale_after_resize":
        c0 = con0_of(vq.fsr_easu_con(4 * iw, 4 * ih, 4 * iw, 4 * ih, ow, oh))
    elif case == "viewport_larger":
        c0 = con0_of(vq.fsr_easu_con(3 * iw, ih, iw, ih, ow, oh))
    elif case in ("nan", "inf", "neg_inf"):
        for slot in range(4):
            bad = c0.copy()
            bad[slot] = {"nan": np.nan, "inf": np.inf, "neg_inf": -np.inf}[case]
            assert easu_check(easu_host, bad, iw, ih, ow, oh)[0] == 1, slot
        return
    elif case == "huge_bias":
        c0[3] = 1e30
    else:
        c0[2] = -float(iw) - 0.5                              # first tap at -w - 2
    assert easu_check(easu_host, c0, iw, ih, ow, oh)[0] == want


def test_wrap_limit_is_exact(easu_host):
    """the last accepted and first refused constants either side of [-w, 2w)"""
    w = 10
    # scale 1, bias b: taps floor(b) - 1 .. floor(b + w - 1) + 2
    assert easu_check(easu_host, [1, 1, -9.0, 0], w, w, w, w)[0] == 0        # first tap -10 = -w
    assert easu_check(easu_host, [1, 1, -9.5, 0], w, w, w, w)[0] == 2        # -11
    assert easu_check(easu_host, [1, 1, 8.0, 0], w, w, w, w)[0] == 0         # last tap 8 + 9 + 2 = 19 = 2w - 1
    assert easu_check(easu_host, [1, 1, 9.0, 0], w, w, w, w)[0] == 2         # 20
    # images under 3 texels: the same rule with size 3 (the % fold takes any tap)
    assert easu_check(easu_host, [1, 1, -2.0, 0], 1, 1, 1, 1)[0] == 0
    assert easu_check(easu_host, [1, 1, -3.0, 0], 1, 1, 1, 1)[0] == 2


def test_path_choice_follows_its_definitions(easu_host):
    """exact 2x: con0 of FsrEasuCon(w, h, w, h, 2w, 2h) AND an output of exactly 2w x 2h; up path: 0 < scale <= 1 on both axes;
    everything else (a scale just above 1 or negative on either axis, or 0) takes the generic kernel"""
    import vqengine_b200 as vq
    path = lambda c0, iw, ih, ow, oh: easu_check(easu_host, c0, iw, ih, ow, oh)[1][0]
    c2x = con0_of(vq.fsr_easu_con(7, 5, 7, 5, 14, 10))
    assert list(c2x) == [0.5, 0.5, -0.25, -0.25]
    assert path(c2x, 7, 5, 14, 10) == 2
    assert path(c2x, 7, 5, 14, 11) == 1 and path(c2x, 7, 5, 15, 10) == 1          # 2x constants, output not 2x
    vp = con0_of(vq.fsr_easu_con(7, 5, 9, 6, 14, 10))                              # viewport < input: same con0, input not half
    assert list(vp) == list(c2x) and path(vp, 9, 6, 14, 10) == 1
    above = float(np.nextafter(np.float32(1), np.float32(2)))
    assert path([1.0, 1.0, 0.0, 0.0], 16, 16, 16, 16) == 1
    assert path([above, 1.0, 0.0, 0.0], 16, 16, 16, 16) == 0
    assert path([1.0, above, 0.0, 0.0], 16, 16, 16, 16) == 0
    assert path([-0.5, 0.5, 7.0, 0.0], 16, 16, 16, 16) == 0
    assert path([0.5, -0.5, 0.0, 7.0], 16, 16, 16, 16) == 0
    assert path([0.0, 0.5, 3.0, 0.0], 16, 16, 16, 16) == 0
