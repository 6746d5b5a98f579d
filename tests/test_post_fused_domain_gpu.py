"""-m gpu: the one-pass post chain (vq_post_process: post_fsr2x_kernel, post_fsr_up_kernel, post_cas_kernel) over the domain
images of tests/post_domain.py, the tonemapper's every branch and brightness, viewports smaller than the input and the tiles
that fill the fused up path's candidate capacity. Every case holds the call to two references on the same input:

  (i)  the fused call makes one launch and equals the separate calls (vq_tonemap -> vq_fsr_easu -> vq_fsr_rcas, or
       vq_tonemap -> vq_cas) bit for bit (`chain` of test_post_fused_gpu.py);
  (ii) each separate stage meets the oracle on the kernel's previous-stage output at the parity bounds of
       test_post_domain_gpu.py: tonemap 1e-4 and the float64 bound of post_ref.tonemap_ref (Reinhard beyond 2^126 gives 0),
       EASU 2e-5 outside post_ref.easu_zro's undecided pixels, RCAS and CAS 1e-5; where a channel's 4 * mx4 is subnormal, RCAS
       meets the oracle on the EASU output with that channel's subnormals flushed (rcp.approx.ftz, DESIGN §5).

(ii) is what makes (i) mean "correct". The stage bounds are absolute on values in [-1, 1]; the linear display curve hands EASU,
RCAS and CAS the engine's HDR range (up to 65504), where fp32 holds a weighted sum only to a few ulps of its largest term, so
there a stage's bound is relative to the largest magnitude of the taps it reads (`footprint_scale`), channel by channel.
Stages after the tonemapper meet the oracle on finite images only: NaN inside EASU's min / max is not compared with the oracle."""
import numpy as np
import pytest

import post_domain as pd
import post_ref as pr
from gpu_util import dev, host
from test_post_domain import FUSED_CAP, easu_check, easu_host  # noqa: F401  (easu_host is a fixture)
from test_post_domain_gpu import CURVES, EASU_CASES, LDR_SIZES, compare, within
from test_post_fused_gpu import assert_same, chain, fused

pytestmark = pytest.mark.gpu

GENS = ["quantised", "chroma_edges", "ramps8", "denormal"]
F32_TINY = np.float32(pd.F32_TINY)


# ---- (ii): the separate chain, stage by stage, against the oracle --------------------------------------------------
def footprint_scale(img, taps):
    """max(1, |value|) over the taps (y, x, inside) a stage reads, per channel: [.., 3]; taps outside read 0"""
    m = np.ones(taps[0][0].shape + (3,), np.float64)
    for ty, tx, inside in taps:
        m = np.maximum(m, np.where(inside[..., None], np.abs(img[ty, tx, :3].astype(np.float64)), 0.0))
    return m


def relative(got, ref, scale):
    """got and ref in units of `scale` (rgb), so that compare's absolute bound becomes relative to it"""
    g, r = got.astype(np.float64).copy(), ref.astype(np.float64).copy()
    g[..., :3] /= scale
    r[..., :3] /= scale
    return g, r


def cross_taps(h, w):
    """the 5-tap cross b, d, e, f, h of every pixel; RCAS and CAS read 0 outside the image"""
    yy, xx = np.mgrid[0:h, 0:w]
    return [(np.clip(yy + dy, 0, h - 1), np.clip(xx + dx, 0, w - 1), (yy + dy >= 0) & (yy + dy < h) & (xx + dx >= 0) & (xx + dx < w))
            for dy, dx in ((-1, 0), (0, -1), (0, 0), (0, 1), (1, 0))]


def easu_taps(con, h, w, oh, ow, mode):
    """the 4 x 4 texels around every output's 'f' (a superset of EASU's 12 taps), folded as load_addr folds them"""
    c = np.frombuffer(bytes(con), np.float32)[:4]
    oy, ox = np.mgrid[0:oh, 0:ow]
    fx = np.floor((ox.astype(np.float32) * c[0]).astype(np.float32) + c[2]).astype(np.int64)
    fy = np.floor((oy.astype(np.float32) * c[1]).astype(np.float32) + c[3]).astype(np.int64)
    fold = (lambda i, n: np.mod(i, n)) if mode == 0 else (lambda i, n: np.clip(i, 0, n - 1))
    return [(fold(fy + dy, h), fold(fx + dx, w), np.ones(fx.shape, bool)) for dy in range(-1, 3) for dx in range(-1, 3)]


def stage_tonemap(ctx, vq, orc, img, tm, name):
    t = dev(np.zeros_like(img))
    ctx.tonemap(tm, dev(img), t)
    got = host(t)
    ref64, bound = pr.tonemap_ref(img, tm.OutputDisplayCurve, tm.ToggleGammaCorrection, tm.ContentColorSpace,
                                  tm.DisplayReferenceBrightnessLevel)
    outside = np.isnan(bound) & np.isfinite(ref64)          # vqcuda.h: Reinhard's __fdividef gives 0 beyond 2^126
    if outside.any():
        assert (got[outside] == 0.0).all(), "Reinhard beyond its domain limit no longer returns 0: update vqcuda.h / DESIGN §5"
    compare(f"tonemap/{name}", got, np.where(outside, got, orc.tonemap(tm, img)), 1e-4)
    within(f"tonemap/{name} f64", got, ref64, bound)
    return got


def stage_easu(ctx, orc, t, easu, oh, ow, mode, name):
    assert np.isfinite(t).all(), name
    e = dev(np.full((oh, ow, 4), np.nan, np.float32))
    ctx.fsr_easu(easu, dev(t), e, address_mode=mode)
    got = host(e)
    _, _, _, undecided = pr.easu_zro(t, easu, ow, oh, mode)
    g, r = relative(got, orc.fsr_easu(easu, t, ow, oh, mode), footprint_scale(t, easu_taps(easu, *t.shape[:2], oh, ow, mode)))
    _, n = compare(f"easu/{name}", g, r, 2e-5, allowed=undecided)
    if n:
        print(f"easu/{name}: the {n} pixels over 2e-5 are all in the float64 undecided zro set ({int(undecided.sum())} pixels)")
    return got


def flush_channels(img, chans):
    """img with the subnormals of channels `chans` read as zeros of their sign, as rcp.approx.ftz reads its argument"""
    out = img.copy()
    for c in chans:
        out[..., c] = np.where(np.abs(out[..., c]) < F32_TINY, np.copysign(np.float32(0), out[..., c]), out[..., c])
    return out


def stage_rcas(ctx, vq, orc, e, stops, name):
    """RCAS's hitMin takes rcp.approx.ftz(4 * mx4) per channel: where a channel's 4 * mx4 is subnormal the kernel equals the
    oracle on the input with that channel's subnormals flushed (test_rcas_denormal_channels's rule, channel by channel: HDR
    neighbourhoods can hold subnormals in one channel whose 4 * mx4 is normal and in another whose 4 * mx4 is not)"""
    con = vq.fsr_rcas_con(stops)
    r = dev(np.zeros_like(e))
    ctx.fsr_rcas(con, dev(e), r)
    got = host(r)
    taps = cross_taps(*e.shape[:2])
    nb = [np.where(inside[..., None], e[ty, tx, :3], np.float32(0)) for ty, tx, inside in taps]
    q = np.abs(np.float32(4.0) * np.maximum(np.maximum(nb[0], nb[1]), np.maximum(nb[3], nb[4])))
    ftz = ((q > 0) & (q < F32_TINY)) @ np.array([1, 2, 4])          # the channels whose 4 * mx4 is subnormal, as bits
    want = orc.fsr_rcas(con, e)
    for m in np.unique(ftz[ftz > 0]):
        chans = [c for c in range(3) if m >> c & 1]
        want[ftz == m] = orc.fsr_rcas(con, flush_channels(e, chans))[ftz == m]
    g, ref = relative(got, want, footprint_scale(e, taps))
    compare(f"rcas/{name}/{stops}" + (f" ({int((ftz > 0).sum())} ftz pixels)" if ftz.any() else ""), g, ref, 1e-5)


def stage_cas(ctx, vq, orc, t, sharp, name):
    h, w = t.shape[:2]
    con = vq.cas_setup(sharp, w, h, w, h)
    c = dev(np.zeros_like(t))
    ctx.cas(con, dev(t), c)
    assert np.isfinite(t).all(), name
    g, r = relative(host(c), orc.cas(con, t), footprint_scale(t, cross_taps(h, w)))
    compare(f"cas/{name}/{sharp}", g, r, 1e-5)


# ---- one case: (i) for every setting, then (ii) -----------------------------------------------------------------------
def check_fsr(ctx, vq, orc, img, tm, easu, oh, ow, mode, stops, name, oracle=True):
    src = dev(img)
    for s in stops:
        rcas = vq.fsr_rcas_con(s)
        assert_same(fused(ctx, src, tm, (oh, ow), easu=easu, rcas=rcas, mode=mode),
                    chain(ctx, src, tm, (oh, ow), easu=easu, rcas=rcas, mode=mode), (name, s))
    if oracle:
        t = stage_tonemap(ctx, vq, orc, img, tm, name)
        e = stage_easu(ctx, orc, t, easu, oh, ow, mode, name)
        for s in stops:
            stage_rcas(ctx, vq, orc, e, s, name)


def check_cas(ctx, vq, orc, img, tm, sharps, name, oracle=True):
    src = dev(img)
    h, w = img.shape[:2]
    for s in sharps:
        con = vq.cas_setup(s, w, h, w, h)
        assert_same(fused(ctx, src, tm, (h, w), cas=con), chain(ctx, src, tm, (h, w), cas=con), (name, s))
    if oracle:
        t = stage_tonemap(ctx, vq, orc, img, tm, name)
        for s in sharps:
            stage_cas(ctx, vq, orc, t, s, name)


def linear(vq):
    """tonemap_px returns the colour unchanged on the kernels and the oracle: EASU and CAS stage the domain image itself"""
    return vq.TonemapperParams(vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_LINEAR, 200.0, 0, 1.0)


# ---- A. the EASU / RCAS / CAS edge images through the fused kernels -------------------------------------------------
SIZES_2X = [(1, 1), (2, 1), (1, 2), (3, 3), (7, 13), (31, 17), (97, 33), (31, 7), (62, 14), (63, 15)]     # input w x h


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("w,h", SIZES_2X)
@pytest.mark.parametrize("gen", GENS)
def test_fsr2x_edge_images(ctx, vq, orc, gen, w, h, mode):
    img = pd.LDR_GENERATORS[gen](w, h, seed=w + h)
    easu = vq.fsr_easu_con(w, h, w, h, 2 * w, 2 * h)
    check_fsr(ctx, vq, orc, img, linear(vq), easu, 2 * h, 2 * w, mode, (0.0, 0.2, 2.0), f"2x/{gen}/{w}x{h}/{mode}")


# (viewport, input, output), w x h: EASU_CASES's upscales (ratios 0.91 .. 1, images under 3 texels, viewport < input; its exact
# 2x rows run post_fsr2x_kernel), FsrEasuCon's 2x constants on inputs that are not half the output (the up path at scale 0.5 on
# both axes), and ratios 0.99 / 0.999 at displays whose tiles fill the fused candidate capacity (FULL_TILES)
FULL_TILES = [((63, 50), (63, 50), (64, 51)), ((1000, 520), (1000, 520), (1001, 521))]
UP_CASES = [c for c in EASU_CASES if c[0][0] <= c[2][0] and c[0][1] <= c[2][1]] + \
           [((7, 5), (9, 6), (14, 10)), ((31, 17), (40, 19), (62, 34))] + FULL_TILES


def case_id(c):
    return "{}x{}in{}x{}to{}x{}".format(*c[0], *c[1], *c[2])


def test_full_tiles_fill_the_fused_capacity(easu_host, vq):
    """FULL_TILES stay on the up path's limit: the host check of vq_post_process reports 32 x 16 candidates"""
    for (vw, vh), (iw, ih), (ow, oh) in FULL_TILES:
        c0 = np.frombuffer(bytes(vq.fsr_easu_con(vw, vh, iw, ih, ow, oh)), np.float32)[:4]
        v, (path, ncx, ncy) = easu_check(easu_host, c0, iw, ih, ow, oh, fused=True)
        assert (v, path, (ncx, ncy)) == (0, 1, FUSED_CAP), ((iw, ih), (ow, oh), v, path, ncx, ncy)


@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("case", UP_CASES, ids=case_id)
@pytest.mark.parametrize("gen", GENS)
def test_fsr_up_edge_images(ctx, vq, orc, gen, case, mode):
    (vw, vh), (iw, ih), (ow, oh) = case
    img = pd.LDR_GENERATORS[gen](iw, ih, seed=iw + ih)
    easu = vq.fsr_easu_con(vw, vh, iw, ih, ow, oh)
    stops = (0.0, 0.2, 2.0) if ow * oh < 10 ** 5 else (0.2,)
    check_fsr(ctx, vq, orc, img, linear(vq), easu, oh, ow, mode, stops, f"up/{gen}/{case_id(case)}/{mode}")


@pytest.mark.parametrize("w,h", LDR_SIZES)
@pytest.mark.parametrize("gen", GENS)
def test_cas_edge_images(ctx, vq, orc, gen, w, h):
    check_cas(ctx, vq, orc, pd.LDR_GENERATORS[gen](w, h, seed=w + h), linear(vq), (0.0, 0.8, 1.0), f"cas/{gen}/{w}x{h}")


def test_fsr2x_1080p_to_4k_quantised(ctx, vq, orc):
    w, h = 1920, 1080
    easu = vq.fsr_easu_con(w, h, w, h, 2 * w, 2 * h)
    check_fsr(ctx, vq, orc, pd.ldr_quantised(w, h, seed=4), linear(vq), easu, 2 * h, 2 * w, 0, (0.2,), "2x/quantised/1920x1080")


# ---- B. the tonemapper inside the fused kernels ---------------------------------------------------------------------
# every CURVES entry (curve, gamma, colour space) including the unknown curve 7; the PQ entries at every brightness
TONEMAPS = [(c, g, cs, nits) for (c, g, cs) in CURVES for nits in ((80.0, 200.0, 1000.0, 10000.0) if c == 1 else (200.0,))]


@pytest.mark.parametrize("engine_range", [True, False], ids=["engine range", "whole fp32 line"])
@pytest.mark.parametrize("w,h", [(31, 17), (97, 33)])
@pytest.mark.parametrize("branch", ["fsr 2x", "fsr preset 0.67", "cas"])
@pytest.mark.parametrize("curve,gamma,cs,nits", TONEMAPS)
def test_tonemapper_in_fused_kernels(ctx, vq, orc, curve, gamma, cs, nits, branch, w, h, engine_range):
    """hdr_domain scene colour: (i) on the whole fp32 line (+-Inf, NaN, 2^126 .. F32_MAX); (i) and (ii) in the engine's range"""
    img = pd.hdr_domain(w, h, seed=w * 7 + h, specials=not engine_range, extremes=not engine_range)
    tm = vq.TonemapperParams(cs, curve, nits, gamma, 1.0)
    name = f"{branch}/{curve}{gamma}{cs}/{nits}/{w}x{h}"
    if branch == "cas":
        check_cas(ctx, vq, orc, img, tm, (0.8,), name, oracle=engine_range)
        return
    ow, oh = (2 * w, 2 * h) if branch == "fsr 2x" else (round(w / 0.67), round(h / 0.67))
    check_fsr(ctx, vq, orc, img, tm, vq.fsr_easu_con(w, h, w, h, ow, oh), oh, ow, 0, (0.2,), name, oracle=engine_range)
