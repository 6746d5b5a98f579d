"""-m gpu: every post kernel (K5-K10) over the domain images of tests/post_domain.py, against the oracle at the parity bounds
(tonemap 1e-4, blur / CAS / RCAS 1e-5, EASU 2e-5) and against the float64 restatements of tests/post_ref.py where they exist.
Non-finite outputs are compared by position (NaN where the oracle has NaN, the same infinities)."""
import ctypes as C

import numpy as np
import pytest
import torch

import post_domain as pd
import post_ref as pr
from gpu_util import dev, host

pytestmark = pytest.mark.gpu

CURVES = [(0, 1, 0), (0, 0, 0), (1, 0, 0), (1, 0, 1), (2, 0, 0), (7, 0, 0)]
HDR_SIZES = [(1, 1), (5, 1), (1, 2), (3, 3), (97, 33), (515, 7)]


def compare(name, got, ref, tol, scaled=False, allowed=None):
    """same non-finite positions, |got - ref| <= tol (* max(1, |ref|) when scaled) elsewhere; pixels in `allowed` [h, w] may
    exceed. Returns (largest |delta| / tol, number of pixels over tol)."""
    assert np.array_equal(np.isnan(got), np.isnan(ref)), f"{name}: NaN positions differ at {np.argwhere(np.isnan(got) != np.isnan(ref))[:5]}"
    inf = np.isinf(ref) | np.isinf(got)
    assert np.array_equal(np.where(inf, got, 0), np.where(inf, ref, 0)), f"{name}: infinities differ"
    m = np.isfinite(ref)
    d = np.where(m, np.abs(got.astype(np.float64) - np.where(m, ref, 0)), 0.0)
    if scaled:
        d = d / np.maximum(1.0, np.abs(np.where(m, ref, 0)))
    over = (d > tol).any(axis=-1)
    if allowed is not None:
        bad = over & ~allowed
    else:
        bad = over
    assert not bad.any(), f"{name}: {int(bad.sum())} pixels over {tol}, first {np.argwhere(bad)[:5].tolist()}, max {d.max():.3e}"
    worst = float(d[~over].max() / tol) if (~over).any() else 0.0
    msg = f"{name}: max |delta|/tol {worst:.3f} on the pixels within tol"
    if over.any():
        where = np.argwhere(over)
        msg += (f"; {len(where)} allowed pixels over tol, largest |delta|/tol {float(d[over].max() / tol):.3f}, "
                f"at (y, x) {where[:10].tolist()}")
    print(msg)
    return worst, int(over.sum())


def within(name, got, ref, bound, skip=None):
    m = np.isfinite(ref) & np.isfinite(bound) & np.isfinite(got)
    if skip is not None:
        m &= ~skip
    d = np.where(m, np.abs(got.astype(np.float64) - np.where(m, ref, 0)), 0.0)
    bad = m & (d > bound)
    assert not bad.any(), f"{name}: {int(bad.sum())} values outside the float64 bound, first {np.argwhere(bad)[:5].tolist()}"
    r = float((d[m] / np.maximum(bound[m], 1e-300)).max()) if m.any() else 0.0
    print(f"{name}: max |delta| / float64 bound {r:.3f}")


# ---- K6 tonemapper ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", HDR_SIZES)
@pytest.mark.parametrize("curve,gamma,cs", CURVES)
@pytest.mark.parametrize("nits", [80.0, 200.0, 1000.0, 10000.0])
def test_tonemap_domain(ctx, vq, orc, w, h, curve, gamma, cs, nits):
    img = pd.hdr_domain(w, h, seed=w * 7 + h)
    p = vq.TonemapperParams(cs, curve, nits, gamma, 1.0)
    out = torch.empty_like(dev(img))
    ctx.tonemap(p, dev(img), out)
    got = host(out)
    ref64, bound = pr.tonemap_ref(img, curve, gamma, cs, nits)
    # vqcuda.h: the sRGB curve's Reinhard divides with __fdividef, which gives 0 for finite denominators above 2^126
    outside = np.isnan(bound) & np.isfinite(ref64)
    if outside.any():
        assert (got[outside] == 0.0).all(), "Reinhard beyond its domain limit no longer returns 0: update vqcuda.h / DESIGN §5"
    want = orc.tonemap(p, img)
    want = np.where(outside, got, want)
    compare(f"tonemap{w}x{h}/{curve}{gamma}{cs}/{nits}", got, want, 1e-4)
    within(f"tonemap{w}x{h}/{curve}{gamma}{cs}/{nits} f64", got, ref64, bound)


def test_tonemap_reinhard_domain_limit_both_sides(ctx, vq, orc):
    lim = np.float32(2.0 ** 126)
    vals = np.array([np.nextafter(lim, np.float32(0)), lim, np.nextafter(lim, np.float32(np.inf)), np.float32(2.0 ** 127),
                     np.float32(pd.F32_MAX), -np.float32(2.0 ** 127), np.float32(65504.0), np.float32(1e30)], np.float32)
    img = np.zeros((1, len(vals), 4), np.float32)
    img[0, :, :3] = vals[:, None]
    for gamma in (0, 1):
        p = vq.TonemapperParams(0, 0, 200.0, gamma, 1.0)
        out = torch.empty_like(dev(img))
        ctx.tonemap(p, dev(img), out)
        got, want = host(out)[0, :, 0], orc.tonemap(p, img)[0, :, 0]
        inside = np.abs(vals.astype(np.float64) + 1) <= 2.0 ** 126
        assert np.abs(got[inside] - want[inside]).max() <= 1e-4 and (want[inside] > 0.99).all()
        assert (got[~inside] == 0.0).all() and (want[~inside] > 0.99).all()


# ---- K5 blur ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", HDR_SIZES + [(1030, 70), (129, 9)])
@pytest.mark.parametrize("full", [False, True])
def test_blur_domain(ctx, orc, w, h, full):
    """the engine's RGBA16F range, then the whole fp32 line with +-Inf and NaN"""
    img = pd.hdr_domain(w, h, seed=w + 3 * h, specials=full, extremes=full)
    d = dev(img)
    tmp, out = torch.empty_like(d), torch.empty_like(d)
    ctx.gaussian_blur(d, tmp, vertical=False)
    ctx.gaussian_blur(tmp, out, vertical=True)
    gx, gy = host(tmp), host(out)
    compare(f"blurX{w}x{h}", gx, orc.gaussian_blur(img, False), 1e-5, scaled=True)
    compare(f"blurY{w}x{h}", gy, orc.gaussian_blur(gx, True), 1e-5, scaled=True)
    for name, src, got, vertical in (("X", img, gx, False), ("Y", gx, gy, True)):
        ref, bound = pr.blur_ref(src, vertical)
        within(f"blur{name}{w}x{h} f64", got, ref, bound)


@pytest.mark.parametrize("sx,sy", [(40, 20), (1, 33), (97, 1), (13, 7)])
def test_blur_sub_rectangle(ctx, vq, orc, sx, sy):
    """iImageSize smaller than the images: the pass filters the top-left rectangle, clamped to it, and writes nothing else"""
    img = pd.hdr_domain(97, 33, seed=sx + sy, specials=False, extremes=False)
    d = dev(img)
    for vertical, fn in ((False, vq.lib.vq_gaussian_blur_x), (True, vq.lib.vq_gaussian_blur_y)):
        out = torch.full_like(d, -7.0)
        p = vq.BlurParams(sx, sy)
        assert fn(ctx._h, C.byref(p), vq.image_of(d), vq.image_of(out), None) == 0
        got = host(out)
        crop = np.ascontiguousarray(img[:sy, :sx])
        compare(f"blur_sub{'XY'[vertical]}{sx}x{sy}", got[:sy, :sx], orc.gaussian_blur(crop, vertical), 1e-5, scaled=True)
        ref, bound = pr.blur_ref(img, vertical, size=(sx, sy))
        within(f"blur_sub{'XY'[vertical]} f64", got[:sy, :sx], ref, bound)
        outside = np.ones(got.shape[:2], bool)
        outside[:sy, :sx] = False
        assert (got[outside] == -7.0).all(), "the blur wrote outside iImageSize"


# ---- K7 CAS, K9 RCAS -------------------------------------------------------------------------------------------------
LDR_SIZES = [(1, 1), (2, 1), (1, 2), (2, 2), (3, 3), (5, 1), (31, 17), (97, 33), (129, 9)]


@pytest.mark.parametrize("gen", ["quantised", "chroma_edges", "ramps8", "denormal"])
@pytest.mark.parametrize("w,h", LDR_SIZES)
def test_cas_domain(ctx, vq, orc, gen, w, h):
    img = pd.LDR_GENERATORS[gen](w, h, seed=w + h)
    for sharp in (0.0, 0.8, 1.0):
        con = vq.cas_setup(sharp, w, h, w, h)
        out = torch.empty_like(dev(img))
        ctx.cas(con, dev(img), out)
        compare(f"cas/{gen}{w}x{h}/{sharp}", host(out), orc.cas(con, img), 1e-5)


@pytest.mark.parametrize("gen", ["quantised", "chroma_edges", "ramps8"])
@pytest.mark.parametrize("w,h", LDR_SIZES)
def test_rcas_domain(ctx, vq, orc, gen, w, h):
    img = pd.LDR_GENERATORS[gen](w, h, seed=w + h)
    for stops in (0.0, 0.2, 2.0):
        con = vq.fsr_rcas_con(stops)
        out = torch.empty_like(dev(img))
        ctx.fsr_rcas(con, dev(img), out)
        compare(f"rcas/{gen}{w}x{h}/{stops}", host(out), orc.fsr_rcas(con, img), 1e-5)


@pytest.mark.parametrize("w,h", [(31, 17), (97, 33), (129, 9)])
def test_rcas_denormal_channels(ctx, vq, orc, w, h):
    """RCAS's hitMin takes rcp.approx.ftz(4*mx4): where 4*mx4 is subnormal (mx4 in (2^-130, 2^-128)) the kernel reads it as 0
    and equals the oracle on the input with denormals flushed; where 4*mx4 is normal or 1/(4*mx4) overflows anyway it equals
    the oracle on the input as it is (DESIGN §5)."""
    con = vq.fsr_rcas_con(0.2)
    ftz = pd.denormal_channels(w, h, seed=w, values=pd.RCAS_FTZ)
    kept = pd.denormal_channels(w, h, seed=w, values=[2.0 ** -149, 2.0 ** -140, 2.0 ** -131, 2.0 ** -127, 2.0 ** -126 * 0.75])
    for name, img, ref in (("ftz", ftz, pd.flush_denormals(ftz)), ("kept", kept, kept)):
        out = torch.empty_like(dev(img))
        ctx.fsr_rcas(con, dev(img), out)
        got = host(out)
        compare(f"rcas_denormal/{name}{w}x{h}", got, orc.fsr_rcas(con, ref), 1e-5)
        if name == "ftz":
            diff = (np.abs(got - orc.fsr_rcas(con, img)) > 1e-5).any(-1)
            print(f"rcas_denormal/ftz{w}x{h}: {int(diff.sum())} pixels differ from the oracle on the unflushed input")


# ---- K8 EASU ---------------------------------------------------------------------------------------------------------
# (viewport, input, output): the exact-2x kernel, the up path (ratios 0.91 / 0.95 / 0.99 / 1 at widths >= 64 stage footprint
# columns 32-35), images under 3 texels (WRAP's % fold), viewport < input, anisotropic and downscale pairs (generic kernel)
EASU_CASES = [((64, 48), (64, 48), (128, 96)), ((1, 1), (1, 1), (2, 2)), ((2, 1), (2, 1), (4, 2)), ((33, 17), (33, 17), (66, 34)),
              ((64, 64), (64, 64), (70, 70)), ((95, 40), (95, 40), (100, 42)), ((99, 20), (99, 20), (100, 21)),
              ((100, 24), (100, 24), (100, 24)), ((2, 7), (2, 7), (5, 13)), ((1, 2), (1, 2), (3, 5)),
              ((48, 30), (64, 40), (96, 60)), ((50, 21), (64, 33), (77, 40)),
              ((64, 40), (64, 40), (96, 30)), ((40, 64), (40, 64), (30, 96)), ((120, 80), (120, 80), (90, 60)), ((5, 1), (5, 1), (3, 1))]


@pytest.mark.parametrize("gen", ["quantised", "chroma_edges", "ramps8", "denormal"])
@pytest.mark.parametrize("case", EASU_CASES, ids=lambda c: "{}x{}in{}x{}to{}x{}".format(*c[0], *c[1], *c[2]))
@pytest.mark.parametrize("mode", [0, 1])
def test_easu_domain(ctx, vq, orc, gen, case, mode):
    (vw, vh), (iw, ih), (ow, oh) = case
    img = pd.LDR_GENERATORS[gen](iw, ih, seed=iw + ih)
    con = vq.fsr_easu_con(vw, vh, iw, ih, ow, oh)
    out = torch.full((oh, ow, 4), float("nan"), dtype=torch.float32, device="cuda")
    ctx.fsr_easu(con, dev(img), out, address_mode=mode)
    _, _, _, undecided = pr.easu_zro(img, con, ow, oh, mode)
    worst, n = compare(f"easu/{gen}/{case}/{mode}", host(out), orc.fsr_easu(con, img, ow, oh, mode), 2e-5, allowed=undecided)
    if n:
        print(f"easu/{gen}/{case}/{mode}: the {n} pixels over 2e-5 are all in the float64 undecided zro set ({int(undecided.sum())} pixels)")


def test_easu_refuses_constants_that_read_outside(ctx, vq):
    """con0 not built for these images (stale after a resize, viewport larger than the image) or not finite: the call fails
    with VQ_ERR_INVALID_ARG before anything is launched"""
    iw, ih, ow, oh = 100, 60, 200, 120
    src = torch.zeros((ih, iw, 4), device="cuda")
    dst = torch.zeros((oh, ow, 4), device="cuda")
    bad = [vq.fsr_easu_con(4 * iw, 4 * ih, 4 * iw, 4 * ih, ow, oh), vq.fsr_easu_con(3 * iw, ih, iw, ih, ow, oh)]
    for slot, v in ((0, np.nan), (1, np.inf), (2, -np.inf), (3, 1e30)):
        c = vq.fsr_easu_con(iw, ih, iw, ih, ow, oh)
        c[slot] = int(np.array([v], np.float32).view(np.uint32)[0])
        bad.append(c)
    torch.cuda.synchronize()
    before = vq.launch_count()
    for i, con in enumerate(bad):
        for mode in (0, 1):
            with pytest.raises(vq.VqError) as e:
                ctx.fsr_easu(con, src, dst, address_mode=mode)
            assert e.value.code == vq.VQ_ERR_INVALID_ARG, i
    assert vq.launch_count() == before
    ctx.fsr_easu(vq.fsr_easu_con(iw, ih, iw, ih, ow, oh), src, dst)
    assert vq.launch_count() == before + 1


# ---- K10 SPD ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,mips", [(1024, 1024, 1), (1024, 1024, 6), (1024, 1024, 7), (1024, 1024, 8), (4096, 64, 1), (4096, 64, 6)])
def test_spd_partial_chains(ctx, vq, orc, w, h, mips):
    img = pd.hdr_domain(w, h, seed=mips, specials=False)
    img[..., :3] = np.clip(img[..., :3], -65504, 65504)      # SPD averages: keep sums of four finite
    (dx, dy), c = vq.spd_setup(w, h)
    c.mips = mips
    dsts = [torch.full((h >> l, w >> l, 4), -7.0, dtype=torch.float32, device="cuda") for l in range(1, mips + 1)]
    ctx.spd_downsample(c, dev(img), dsts)
    ctx.spd_downsample(c, dev(img), dsts)    # twice: a chain past mip 6 must leave the last-block ticket reset for the next call
    ref = orc.spd_downsample(img, mips)
    assert len(ref) == mips
    for l, (g, r) in enumerate(zip(dsts, ref), start=1):
        assert np.array_equal(host(g).view(np.uint32), r.view(np.uint32)), f"spd level {l} of {w}x{h} (mips {mips})"


# ---- the config-4 chain at 4K output ---------------------------------------------------------------------------------
def test_post_chain_config4_4k_quantised(ctx, vq, orc):
    """SPD -> BlurX,Y -> Tonemap -> CAS -> EASU 2x -> RCAS on a quantised HDR image with flat regions, 1920x1080 -> 3840x2160;
    each stage against the oracle applied to the kernel's previous-stage output"""
    from vqengine_b200 import synth
    w, h = 1920, 1080
    img = pd.ldr_quantised(w, h, seed=4)
    img[..., :3] *= 4.0
    d = dev(img)
    (dx, dy), c = vq.spd_setup(w, h)
    c.mips = 6
    dsts = [torch.zeros((h >> l, w >> l, 4), device="cuda") for l in range(1, 7)]
    ctx.spd_downsample(c, d, dsts)
    for l, (g, r) in enumerate(zip(dsts, orc.spd_downsample(img, 6)), start=1):
        assert np.array_equal(host(g), r), l
    a, b, t, s = (torch.empty_like(d) for _ in range(4))
    tm = synth.default_tonemapper()
    e = torch.empty((2 * h, 2 * w, 4), dtype=torch.float32, device="cuda")
    r = torch.empty_like(e)
    ctx.gaussian_blur(d, a, False)
    compare("4k.blur_x", host(a), orc.gaussian_blur(img, False), 1e-5, scaled=True)
    ctx.gaussian_blur(a, b, True)
    compare("4k.blur_y", host(b), orc.gaussian_blur(host(a), True), 1e-5, scaled=True)
    ctx.tonemap(tm, b, t)
    compare("4k.tonemap", host(t), orc.tonemap(tm, host(b)), 1e-4)
    ctx.cas(vq.cas_setup(0.8, w, h, w, h), t, s)
    compare("4k.cas", host(s), orc.cas(orc.cas_setup(0.8, w, h, w, h), host(t)), 1e-5)
    con = vq.fsr_easu_con(w, h, w, h, 2 * w, 2 * h)
    ctx.fsr_easu(con, s, e)
    _, _, _, und = pr.easu_zro(host(s), con, 2 * w, 2 * h, 0)
    compare("4k.easu", host(e), orc.fsr_easu(con, host(s), 2 * w, 2 * h, 0), 2e-5, allowed=und)
    ctx.fsr_rcas(vq.fsr_rcas_con(0.2), e, r)
    compare("4k.rcas", host(r), orc.fsr_rcas(orc.fsr_rcas_con(0.2), host(e)), 1e-5)
