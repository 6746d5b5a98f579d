"""Float64 restatements of the post chain's smooth passes, written from the shader text (Tonemapper.hlsl:24-27 and
110-151, HDR.hlsl:76-119, GaussianBlur.hlsl:110-186, ffx_fsr1.h:275-437), not from the oracle, with error bounds derived
from the fp32 operations the kernels perform:

  * tonemap: every fp32 rounding is 2^-24 relative (u). The documented MUFU accuracies are: `__log2f` 2^-22 absolute for
    x in [0.5, 2], else 2 ulp; `exp2f` 2 ulp; `__fdividef` 2 ulp (for divisors up to 2^126). pow_sfu(x, e) = exp2f(e * __log2f(x))
    therefore has relative error <= ln2 * (|e| * dlog + |e log2 x| * u) + 2^-22, and the error of its argument is multiplied by e.
    `__log2f` may flush a subnormal argument to 0, so where the PQ curve's argument is subnormal the bound also admits f(0).
    Where the sRGB branch test `c < 0.0031308` lies within the error of c, the bound admits the other branch.
  * blur: a 21-term fp32 sum of products (fused or not) is within 21 u * sum|w_k x_k| of the exact sum; the fp32 weights are
    within u of the shader's decimal constants: bound 22 u * sum|w_k x_k|.
  * EASU's `zro` test (dirR < 1/32768): dirR from the fp32 lumas and bilinear weights in float64, and the decision is
    "undecided" when dirR lies within a rounding-derived delta of the threshold (as tests/pcf_ref.py does for PCF taps).

For CAS, RCAS and the rest of EASU the reference stays the oracle, which equals the shader text bit for bit."""
import numpy as np

U = 2.0 ** -24
SUB = 2.0 ** -149    # spacing of fp32 subnormals: the absolute part of each rounding below 2^-126
LN2 = np.log(2.0)


def _log2_err(x):
    """documented error of __log2f(x) (absolute, in log2 units)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        L = np.log2(x)
        ulp = 2.0 ** (np.floor(np.log2(np.maximum(np.abs(L), 2.0 ** -126))) - 23)
    return np.where((x >= 0.5) & (x <= 2.0), 2.0 ** -22, 2.0 * ulp)


def _pow_sfu_rel(x, e):
    """relative error bound of pow_sfu(x, e) for an exact argument x > 0"""
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.abs(e * np.log2(x))
    return LN2 * (abs(e) * _log2_err(x) + t * U) + 2.0 ** -22


# ---- tonemapper -----------------------------------------------------------------------------------------------------
M1, M2 = 2610.0 / 4096.0 / 4, 2523.0 / 4096.0 * 128
C1, C2, C3 = 3424.0 / 4096.0, 2413.0 / 4096.0 * 32, 2392.0 / 4096.0 * 32
REC709_TO_2020 = np.array([[0.627402, 0.329292, 0.043306], [0.069095, 0.919544, 0.011360], [0.016394, 0.088028, 0.895578]])
SRGB_CUT = 0.0031308
REINHARD_LIMIT = 2.0 ** 126     # __fdividef(x, y) returns 0 for 2^126 < |y| < 2^128 (CUDA C Programming Guide, intrinsics)


def _st2084(x):
    cp = np.abs(x) ** M1
    return ((C1 + C2 * cp) / (1.0 + C3 * cp)) ** M2


def _st2084_with_bound(x, rel_x):
    """PQ of x >= 0 (float64) given x's relative error; returns (value, absolute bound)"""
    ax = np.abs(x)
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        cp = ax ** M1
        rel_cp = M1 * rel_x + np.where(ax > 0, _pow_sfu_rel(np.where(ax > 0, ax, 1.0), M1), 0.0)
        num, den = C1 + C2 * cp, 1.0 + C3 * cp
        # cp's error reaches q through d(log q)/d(log cp) = cp (C2/num - C3/den); the two fmaf and __fdividef round on top
        rel_q = np.abs(cp * (C2 / num - C3 / den)) * rel_cp + 2 * U + 2.0 ** -22
        q = num / den
        val = q ** M2
        bound = val * (M2 * rel_q + _pow_sfu_rel(q, M2))
    flush = (ax > 0) & (ax < 2.0 ** -126)                   # MUFU.LG2 may see 0 instead of a subnormal argument
    bound = np.where(flush, bound + np.abs(val - C1 ** M2), bound)
    return val, bound


def tonemap_ref(img, curve, gamma, cs, nits):
    """float64 tonemap of the fp32 image [h, w, 4] and a per-value bound on the kernel's error; alpha passes through
    (bound 0). Values whose Reinhard denominator exceeds REINHARD_LIMIT are outside the kernel's domain (vqcuda.h) and come
    back with bound NaN."""
    x = img[..., :3].astype(np.float64)
    out = np.empty(img.shape, np.float64)
    bound = np.zeros(img.shape, np.float64)
    out[..., 3] = img[..., 3]
    with np.errstate(all="ignore"):
        if curve == 0:
            d = x + 1.0
            r = x / d
            rb = np.abs(r) * (U + 2.0 ** -22)
            if gamma:
                e = 1.0 / 2.4
                lin = 12.92 * r
                pw = np.abs(r) ** e
                srgb = 1.055 * pw - 0.055
                rel_p = e * rb / np.maximum(np.abs(r), 1e-300) + np.where(r != 0, _pow_sfu_rel(np.where(r != 0, np.abs(r), 1.0), e), 0.0) \
                    + np.abs(np.log(np.maximum(np.abs(r), 1e-300))) * abs(float(np.float32(e)) - e)
                b_pow = 1.055 * pw * (rel_p + U) + U * np.abs(srgb) + U * 0.055
                b_lin = 12.92 * rb + 2 * U * np.abs(lin)
                val = np.where(r < SRGB_CUT, lin, srgb)
                b = np.where(r < SRGB_CUT, b_lin, b_pow)
                near = np.abs(r - SRGB_CUT) <= rb + U * SRGB_CUT
                b = np.where(near, b + np.abs(lin - srgb), b)
                r, rb = val, b
            out[..., :3] = r
            # __fdividef may flush a subnormal quotient to 0 (and 12.92 * 0 stays 0)
            rb = rb + 4 * SUB + np.where(np.abs(x) < 2.0 ** -126, np.abs(r), 0.0)
            d32 = np.abs(img[..., :3] + np.float32(1.0))
            bound[..., :3] = np.where(np.isfinite(d32) & (d32 > REINHARD_LIMIT), np.nan, rb)
        elif curve == 1:
            scalar = nits / 10000.0
            if cs == 0:
                c = x @ REC709_TO_2020.T
                mag = np.abs(x) @ REC709_TO_2020.T
            else:
                c, mag = x, np.abs(x)
            lx = c * scalar
            rel_x = np.where(lx != 0, 4 * U * mag * scalar / np.abs(np.where(lx != 0, lx, 1.0)), 0.0) + 2 * U
            out[..., :3], bound[..., :3] = _st2084_with_bound(lx, rel_x)
            bound[..., :3] += 4 * SUB
        elif curve == 2:
            out[..., :3] = x
        else:
            out[..., :3] = [1.0, 1.0, 0.0]
    return out, bound


# ---- Gaussian blur --------------------------------------------------------------------------------------------------
GAUSS = np.array([0.224716, 0.191756, 0.119146, 0.053897, 0.017746, 0.004252, 0.000741, 0.000094, 0.000009, 0.000001, 0.0])


def blur_ref(img, vertical, size=None):
    """one pass of GaussianBlur.hlsl over the top-left size = (sx, sy) rectangle (clamp to it); returns (value, bound) of
    the rectangle's [sy, sx, 4] pixels, alpha 1"""
    sx, sy = size or (img.shape[1], img.shape[0])
    src = img[:sy, :sx, :3].astype(np.float64)
    acc = np.zeros_like(src)
    mag = np.zeros_like(src)
    n = sy if vertical else sx
    for k in range(21):
        off = k - 10
        idx = np.clip(np.arange(n) + off, 0, n - 1)
        t = src[idx] if vertical else src[:, idx]
        with np.errstate(invalid="ignore"):
            acc += t * GAUSS[abs(off)]
            mag += np.abs(t) * GAUSS[abs(off)]
    out = np.ones(src.shape[:2] + (4,))
    out[..., :3] = acc
    bound = np.zeros_like(out)
    bound[..., :3] = 22 * U * mag + 22 * SUB
    return out, bound


# ---- EASU zro decision ----------------------------------------------------------------------------------------------
ZRO = 1.0 / 32768.0


def _luma2_f32(rgb):
    rgb = rgb.astype(np.float32)
    return (rgb[..., 2] * np.float32(0.5) + (rgb[..., 0] * np.float32(0.5) + rgb[..., 1])).astype(np.float32)


def _addr(i, n, mode):
    return np.mod(i, n) if mode == 0 else np.clip(i, 0, n - 1)


def easu_zro(img, con, out_w, out_h, mode):
    """per output pixel: float64 dirR, its rounding margin delta, and (zro, undecided) where zro is the float64 decision
    dirR < 1/32768 and undecided marks |dirR - 1/32768| <= delta. The lumas, bilinear weights and pp come from the same fp32
    operations as the kernels; only the four weighted sums and dirR are taken exactly. fp32 evaluates each sum of 4 products
    to within 8 u of the sum of its |terms|, and dirR to within 2 u more."""
    c = np.frombuffer(bytes(con), np.float32)[:4]
    h, w = img.shape[:2]
    oy, ox = np.mgrid[0:out_h, 0:out_w]
    ppx = (ox.astype(np.float32) * c[0]).astype(np.float32) + c[2]
    ppy = (oy.astype(np.float32) * c[1]).astype(np.float32) + c[3]
    fpx, fpy = np.floor(ppx), np.floor(ppy)
    ppx, ppy = (ppx - fpx).astype(np.float32), (ppy - fpy).astype(np.float32)
    fx, fy = fpx.astype(np.int64), fpy.astype(np.int64)
    L = _luma2_f32(img[..., :3])

    def lum(dx, dy):
        return L[_addr(fy + dy, h, mode), _addr(fx + dx, w, mode)]

    b, cc, e, f, g, hh = lum(0, -1), lum(1, -1), lum(-1, 0), lum(0, 0), lum(1, 0), lum(2, 0)
    i, j, k, l, n, o = lum(-1, 1), lum(0, 1), lum(1, 1), lum(2, 1), lum(0, 2), lum(1, 2)
    one = np.float32(1.0)
    ws = [((one - ppx) * (one - ppy)).astype(np.float32), (ppx * (one - ppy)).astype(np.float32),
          ((one - ppx) * ppy).astype(np.float32), (ppx * ppy).astype(np.float32)]
    sets = [(b, e, f, g, j), (cc, f, g, hh, k), (f, i, j, k, n), (g, j, k, l, o)]   # (lA, lB, lC, lD, lE)
    dx = np.zeros(ppx.shape); dy = np.zeros(ppx.shape); mx = np.zeros(ppx.shape); my = np.zeros(ppx.shape)
    for wgt, (lA, lB, lC, lD, lE) in zip(ws, sets):
        ax = (lD - lB).astype(np.float32).astype(np.float64)
        ay = (lE - lA).astype(np.float32).astype(np.float64)
        w64 = wgt.astype(np.float64)
        dx += ax * w64; dy += ay * w64
        mx += np.abs(ax * w64); my += np.abs(ay * w64)
    dirR = dx * dx + dy * dy
    ex, ey = 8 * U * mx, 8 * U * my       # 4 products and 4 sums: fused (kernels) or not (oracle)
    delta = 2 * np.abs(dx) * ex + ex * ex + 2 * np.abs(dy) * ey + ey * ey + 2 * U * (dirR + 2 * (ex + ey) * (np.abs(dx) + np.abs(dy)))
    return dirR, delta, dirR < ZRO, np.abs(dirR - ZRO) <= delta
