"""Seeded adversarial images for the post chain (K5-K10), numpy only. Each generator names the branch it is meant to reach.

All images are [h, w, 4] float32. LDR generators (CAS / EASU / RCAS inputs) stay in [0, 1] apart from the denormal and -0
channels of `denormal_channels`; `hdr_domain` spans the whole fp32 line (tonemapper, blur, SPD)."""
import numpy as np

# 1x1 ... odd primes, widths off the 32 / 128 / 512 block sizes
SIZES = [(1, 1), (2, 1), (1, 2), (2, 2), (3, 3), (5, 1), (7, 13), (31, 17), (97, 33), (129, 9), (515, 7)]

F32_MAX = float(np.finfo(np.float32).max)
F32_TINY = float(np.finfo(np.float32).tiny)            # 2^-126, smallest normal
DENORMALS = [2.0 ** -149, 2.0 ** -140, 2.0 ** -131, 2.0 ** -129, 2.0 ** -127, 1e-39]
# 2^-130 .. 2^-128: four times these is still subnormal, so rcp.approx.ftz (RCAS's hitMin) sees 0 where 1/x is finite
RCAS_FTZ = [2.0 ** -130 * 1.5, 2.0 ** -129, 2.0 ** -128 * 0.75]


def _rgba(rgb, alpha=1.0):
    h, w = rgb.shape[:2]
    out = np.empty((h, w, 4), np.float32)
    out[..., :3] = rgb
    out[..., 3] = alpha
    return out


def ldr_quantised(w, h, seed):
    """k/255 values with large flat areas, pure 0 and pure 1 regions and 1-pixel lines of 0 and 1.
    Reaches: RCAS's saturated limits ((1 - mx4)*rcp(4*mn4 - 4) = 0*inf on white, mn4*rcp(4*mx4) = 0*inf on black), CAS's
    saturate clamps, EASU's `zro` branch on flat areas and its min/max clamp on hard 0/1 edges."""
    rng = np.random.default_rng(seed)
    k = rng.integers(0, 256, (h, w, 3))
    bw, bh = max(1, w // 4), max(1, h // 4)
    for _ in range(6):                                      # flat blocks of one k/255 colour
        x0, y0 = rng.integers(0, w), rng.integers(0, h)
        k[y0:y0 + bh, x0:x0 + bw] = rng.integers(0, 256, 3)
    k[: h // 3, : w // 3] = 255                             # pure white corner
    k[h - h // 3:, w - w // 3:] = 0                         # pure black corner
    if w > 2:
        k[:, w // 2] = 0                                    # 1-pixel lines
        k[:, (w // 2 + 2) % w] = 255
    if h > 2:
        k[h // 2, :] = 255
        k[(h // 2 + 2) % h, :] = 0
    return _rgba((k / 255.0).astype(np.float32))


def chroma_edges(w, h, seed):
    """stripes and checks of different colours with equal luma2 = 0.5 r + g + 0.5 b (exact in fp32: (2a/255, 0, 0),
    (0, a/255, 0), (0, 0, 2a/255), (a/255, 0, a/255)), so every EASU analysis sees dirR == 0 exactly: the `zro` branch."""
    rng = np.random.default_rng(seed)
    a = np.float32(rng.integers(1, 128) / 255.0)
    two_a = np.float32(2.0) * a
    pal = np.array([[two_a, 0, 0], [0, a, 0], [0, 0, two_a], [a, 0, a]], np.float32)
    yy, xx = np.mgrid[0:h, 0:w]
    idx = np.where(yy < h // 2, (xx // 3) % 4, ((xx // 2) + (yy // 2)) % 4)
    return _rgba(pal[idx])


def ramps8(w, h, seed):
    """red ramps r = t*(x + y): luma2 steps t/2 per pixel on each axis, so dir = (t, t) and dirR = 2t^2, which crosses EASU's
    1/32768 at t = 1/256. Bands of rows use t = k/255 quantised (dirR = 2/255^2 ~ 3.08e-5, 0.8 % above) and t = (1 + j*2^-18)/256
    for j in -4..4 (j = 0 is the threshold itself; the others lie 8e-6*|j| of it away, a few fp32 roundings)."""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float64)
    ts = [1 / 255.0] + [(1 + j * 2.0 ** -18) / 256.0 for j in range(-4, 5)]
    band = (yy.astype(int) * len(ts)) // max(h, 1)
    t = np.array(ts)[band]
    r = (t * (xx + yy)) % 1.0
    r = np.where(band == 0, np.round(r * 255.0) / 255.0, r)
    g = np.full_like(r, rng.integers(0, 64) / 255.0)
    return _rgba(np.stack([r, g, g], -1).astype(np.float32))


def denormal_channels(w, h, seed, values=DENORMALS + RCAS_FTZ):
    """an LDR k/255 image where, in 3x3 neighbourhoods, one channel is drawn from `values` (denormals, by default including
    2^-130..2^-128, where RCAS's rcp.approx.ftz sees 4*mx4 as 0), 0 or -0 while the other two stay ordinary."""
    rng = np.random.default_rng(seed)
    img = ldr_quantised(w, h, seed)
    vals = np.array(list(values) + [0.0, -0.0], np.float32)
    for cy in range(1, h, 3):
        for cx in range(1, w, 3):
            ch = rng.integers(0, 3)
            blk = img[max(cy - 1, 0):cy + 2, max(cx - 1, 0):cx + 2, ch]
            blk[...] = rng.choice(vals, blk.shape)
            if rng.random() < 0.5:
                blk[rng.integers(0, blk.shape[0]), rng.integers(0, blk.shape[1])] = 0.0
    return img


def flush_denormals(img):
    """the image as a device that flushes subnormals to zero (D3D11 allows it) would read it"""
    out = img.copy()
    out[np.abs(out) < F32_TINY] = 0.0
    return out


def hdr_domain(w, h, seed, specials=True, extremes=True):
    """HDR values over the whole fp32 line: 0, -0, denormals, [1e-6, 65504] (the engine's RGBA16F range) on a log scale, a few
    negatives, with `extremes` fp32 extremes (1e30, 2^126, its successor, 2^127; F32_MAX only in red, at isolated pixels away
    from the edges, so that neither a 21-tap blur window nor a Rec.709 -> Rec.2020 row can overflow on it) and, with
    `specials`, +-Inf and NaN. Without `extremes` the finite values stay in the engine's range, where a filter's error is not
    hidden by a 1e38 neighbour.
    Reaches: Reinhard's __fdividef limit (denominators above 2^126), the PQ curve over its whole input range, MUFU.LG2's
    handling of denormals and 0, NaN/Inf propagation."""
    rng = np.random.default_rng(seed)
    n = w * h * 3
    v = 10.0 ** rng.uniform(-6, np.log10(65504.0), n)
    pick = rng.random(n)
    pool = [0.0, -0.0] + DENORMALS + [65504.0, 1.0, -1e-3, -0.5, -2.0]
    if extremes:
        pool += [2.0 ** 126, float(np.nextafter(np.float32(2.0 ** 126), np.float32(np.inf))), 2.0 ** 127, 1e30]
    pool = np.array(pool)
    v = np.where(pick < 0.25, rng.choice(pool, n), v)
    if specials:
        v = np.where(pick > 0.97, rng.choice(np.array([np.inf, -np.inf, np.nan]), n), v)
    rgb = v.reshape(h, w, 3).astype(np.float32)
    if extremes and w >= 32 and h >= 3:
        for x in range(11, w - 11, 23):
            rgb[h // 2, x, 0] = F32_MAX
    out = _rgba(rgb)
    out[..., 3] = rng.uniform(0, 1, (h, w))
    return out


LDR_GENERATORS = {"quantised": ldr_quantised, "chroma_edges": chroma_edges, "ramps8": ramps8, "denormal": denormal_channels}
