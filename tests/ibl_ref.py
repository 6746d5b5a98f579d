"""Float64 restatement of the environment-map sampling and integrals, written from the shader text (ShadingMath.hlsl
DirectionToEquirectUV / Hammersley, BRDF.hlsl ImportanceSampleGGX / NormalDistributionGGX / IntegrateBRDF,
CubemapConvolution.hlsl) and the sampling rules of DESIGN.md §3 — not from the oracle. Every value comes with a bound
derived from documented accuracies:
  * fp32 rounding, EPS = 2^-24 relative per operation;
  * CUDA math appendix: sincosf, sqrtf, rsqrtf <= 2 ulp (full-range, non-fast-math); rcp.approx / sqrt.approx <= 1 ulp;
    lg2.approx absolute error <= 2^-22.6 on [0.5, 2] and relative 2^-22 elsewhere;
  * atan01 (vq_equirect.cuh): ATAN01_ERR, the maximum measured on the device over every fp32 in [0, 1]
    (tests/test_ibl_domain_gpu.py re-measures it and requires it to stay below this constant).
Where a lookup direction is off by delta radians, the sample moves by at most (dx + dy) texels, dx = W*du, dy = H*dv with
du <= delta / (2*pi*rho) and dv <= delta / (pi*rho), rho = sqrt(x^2 + z^2): the bound grows without limit towards the poles
(and the footprint it is measured over widens with it, up to the whole row), instead of being hidden."""
from __future__ import annotations

import math

import numpy as np

EPS = 2.0 ** -24
ATAN01_ERR = 1.0e-7           # vq_equirect.cuh's documented |atan01 - atan| over [0, 1]
PI32 = float(np.float32(3.14159265359))
TWO_PI32 = float(np.float32(6.28318530718))
HALF_PI32 = float(np.float32(1.5707963268))
# direction error of the kernels' lookup vectors, radians: a few fp32 roundings through normalize / reflect / the tangent
# frame (each <= 2 ulp relative) -- the same 2^-19 budget K1's reflection lookup is held to (DESIGN.md §5)
DIR_DELTA = 2.0 ** -19


# ---- packed resources ------------------------------------------------------------------------------------------------
def pyramid_levels(pyr, w, h, levels):
    """packed (n, 4) pyramid -> list of float64 [h_l, w_l, 3] levels"""
    out, o = [], 0
    p = np.asarray(pyr, np.float32).reshape(-1, 4)
    for l in range(levels):
        wl, hl = w >> l, h >> l
        out.append(p[o:o + wl * hl, :3].astype(np.float64).reshape(hl, wl, 3))
        o += wl * hl
    return out


def cube_texel_direction(face, px, py, res):
    """A35 face table (CubemapUtility.cpp:40-48), texel centres; float64 of the fp32 values the kernels form
    (2*(p+0.5)/res - 1 is exact in fp32 for res <= 2^22 when res is a power of two; otherwise rounded, as fp32 does)"""
    f32 = np.float32
    px = np.asarray(px); py = np.asarray(py)
    sx = (f32(2.0) * (px.astype(f32) + f32(0.5)) / f32(res) - f32(1.0)).astype(np.float64)
    sy = (f32(1.0) - f32(2.0) * (py.astype(f32) + f32(0.5)) / f32(res)).astype(np.float64)
    one = np.ones_like(sx)
    table = {0: (one, sy, -sx), 1: (-one, sy, sx), 2: (sx, one, -sy), 3: (sx, -one, sy), 4: (sx, sy, one), 5: (-sx, sy, -one)}
    face = np.broadcast_to(np.asarray(face), sx.shape)
    d = np.zeros(sx.shape + (3,))
    for f, comps in table.items():
        m = face == f
        for k in range(3):
            d[..., k][m] = np.broadcast_to(comps[k], sx.shape)[m]
    return d


def normalize(d):
    d = np.asarray(d, np.float64)
    return d / np.linalg.norm(d, axis=-1, keepdims=True)


# ---- DirectionToEquirectUV and the WRAP trilinear sampler ------------------------------------------------------------
def direction_to_uv(d):
    """ShadingMath.hlsl:70-80: u = atan2(z, x) / (-2 pi) + 0.5, v = asin(-y) / pi + 0.5 (d need not be unit: as the shader)"""
    d = np.asarray(d, np.float64)
    u = np.arctan2(d[..., 2], d[..., 0]) / (-2.0 * math.pi) + 0.5
    v = np.arcsin(np.clip(-d[..., 1], -1.0, 1.0)) / math.pi + 0.5
    return u, v


def uv_compute_error():
    """|du|, |dv| the kernels' dir_to_equirect adds for an exact fp32 input: atan01 plus the rcp.approx quotient (<= 2 ulp of
    q, and d atan/dq <= 1), the octant subtractions (<= pi/2 * EPS each) and the final fmaf. Checked on the device."""
    ang = ATAN01_ERR + 2 * EPS + 2 * math.pi * EPS
    return ang / (2 * math.pi) + EPS, 2 * ang / math.pi + 2 * EPS


def _bilinear(img, u, v):
    H, W = img.shape[:2]
    x = u * W - 0.5
    y = v * H - 0.5
    x0 = np.floor(x); y0 = np.floor(y)
    fx = (x - x0)[..., None]; fy = (y - y0)[..., None]
    ix0 = np.mod(x0.astype(np.int64), W); iy0 = np.mod(y0.astype(np.int64), H)
    ix1 = (ix0 + 1) % W; iy1 = (iy0 + 1) % H
    top = img[iy0, ix0] + fx * (img[iy0, ix1] - img[iy0, ix0])
    bot = img[iy1, ix0] + fx * (img[iy1, ix1] - img[iy1, ix0])
    return top + fy * (bot - top), x0.astype(np.int64), y0.astype(np.int64)


def sample(levels, u, v, lod):
    """trilinear WRAP sample (DESIGN.md §3): lod clamped to [0, levels-1], floor(lod) and floor(lod)+1 blended"""
    u = np.asarray(u, np.float64); v = np.asarray(v, np.float64)
    lod = np.clip(np.broadcast_to(np.asarray(lod, np.float64), u.shape), 0.0, len(levels) - 1)
    l0 = np.floor(lod).astype(np.int64)
    f = (lod - l0)[..., None]
    out = np.zeros(u.shape + (3,))
    for l in np.unique(l0):
        m = l0 == l
        c0 = _bilinear(levels[l], u[m], v[m])[0]
        c1 = _bilinear(levels[l + 1], u[m], v[m])[0] if l + 1 < len(levels) else c0
        out[m] = c0 + f[m] * (c1 - c0)
    return out


def _range_filter(img, rx, ry):
    """per texel: max - min over the (2ry+3) x (2rx+3) WRAP neighbourhood (per channel)"""
    from scipy.ndimage import maximum_filter, minimum_filter
    size = (min(2 * ry + 3, 2 * img.shape[0] + 1), min(2 * rx + 3, 2 * img.shape[1] + 1), 1)
    return maximum_filter(img, size=size, mode="wrap") - minimum_filter(img, size=size, mode="wrap")


def _pow2_ceil(a):
    return np.where(a <= 0, 0, 2 ** np.ceil(np.log2(np.maximum(a, 1e-300)))).astype(np.int64)


def level_bound(img, u, v, du, dv):
    """how far one bilinear WRAP sample of `img` can move when (u, v) moves by at most (du, dv), plus the rounding of the
    three fp32 lerps and of x = u*W - 0.5: (dx + dy) * (max - min over every texel the moving footprint touches), capped
    at that range (a bilinear sample is a convex combination of the footprint)"""
    H, W = img.shape[:2]
    dx = W * du + W * np.abs(u) * EPS + EPS
    dy = H * dv + H * np.abs(v) * EPS + EPS
    _, x0, y0 = _bilinear(img, u, v)
    rx = np.minimum(_pow2_ceil(np.ceil(dx)), W); ry = np.minimum(_pow2_ceil(np.ceil(dy)), H)
    out = np.zeros(np.shape(u) + (3,))
    amax = np.abs(img).max() if img.size else 0.0
    for a, b in set(zip(rx.ravel().tolist(), ry.ravel().tolist())):
        m = (rx == a) & (ry == b)
        rng = _range_filter(img, int(a), int(b))
        # the footprint's cell is anchored at (x0, y0); the filter is centred, so look one texel further right / down
        r = np.maximum(rng[np.mod(y0[m], H), np.mod(x0[m], W)], rng[np.mod(y0[m] + 1, H), np.mod(x0[m] + 1, W)])
        out[m] = np.minimum(1.0, (dx[m] + dy[m]))[..., None] * r
    return out + 8 * EPS * amax + 16 * 2.0 ** -149          # relative rounding, and the absolute rounding of subnormals


def sample_bound(levels, u, v, lod, du, dv, dlod):
    """bound on |sample(u', v', lod') - sample(u, v, lod)| for |u'-u| <= du, |v'-v| <= dv, |lod'-lod| <= dlod"""
    u = np.asarray(u, np.float64); v = np.asarray(v, np.float64)
    lod = np.clip(np.broadcast_to(np.asarray(lod, np.float64), u.shape), 0.0, len(levels) - 1)
    du = np.broadcast_to(du, u.shape); dv = np.broadcast_to(dv, u.shape)
    dlod = np.broadcast_to(np.asarray(dlod, np.float64), u.shape)
    nl = len(levels)
    lo = np.clip(np.floor(lod - dlod), 0, nl - 1).astype(np.int64)
    hi = np.clip(np.floor(lod + dlod) + 1, 0, nl - 1).astype(np.int64)
    out = np.zeros(u.shape + (3,))
    # spatial movement on every level the blend can touch
    for l in range(nl):
        m = (lo <= l) & (l <= hi)
        if m.any():
            out[m] = np.maximum(out[m], level_bound(levels[l], u[m], v[m], du[m], dv[m]))
    # lod movement: the trilinear value moves along the chain of level samples at the float64 (u, v)
    if (dlod > 0).any():
        chain = np.stack([_bilinear(levels[l], u, v)[0] for l in range(nl)], axis=0)
        step = np.abs(np.diff(chain, axis=0)) if nl > 1 else np.zeros((1,) + chain.shape[1:])
        idx = np.arange(step.shape[0])[:, None]
        sel = (idx >= lo.ravel()[None, :] - 1) & (idx <= hi.ravel()[None, :])
        steps = np.where(sel[..., None], step.reshape(step.shape[0], -1, 3), 0.0).max(axis=0).reshape(u.shape + (3,))
        out = out + np.minimum(2.0, 2 * dlod)[..., None] * steps
    return out


def uv_delta(d, delta):
    """(du, dv) for a lookup direction d (any length) off by `delta` radians, plus the kernel's own uv arithmetic"""
    d = np.asarray(d, np.float64)
    n = np.linalg.norm(d, axis=-1)
    rho = np.hypot(d[..., 0], d[..., 2]) / n
    cu, cv = uv_compute_error()
    with np.errstate(divide="ignore"):
        du = np.where(rho > 0, delta / (2 * math.pi * rho), np.inf)
        dv = np.where(rho > 0, delta / (math.pi * np.maximum(rho, 1e-300)), np.inf)
    # |d| = 1 only up to rounding: asin(-y) sees the length error as a y error of |y| * (|d| - 1)
    dv = dv + np.abs(n - 1.0) * 4 / (math.pi * np.maximum(rho, 1e-300))
    return np.minimum(du + cu, 1.0), np.minimum(dv + cv, 1.0)


# ---- Hammersley and ImportanceSampleGGX ------------------------------------------------------------------------------
def radical_inverse(i):
    i = np.asarray(i, np.uint64)
    out = np.zeros(i.shape, np.float64)
    for b in range(32):
        out += ((i >> np.uint64(b)) & np.uint64(1)).astype(np.float64) * 2.0 ** -(b + 1)
    return out


def hammersley(i, n):
    """ShadingMath.hlsl:119-127 (i/n rounded to fp32 as the shader divides in float)"""
    i = np.asarray(i)
    return (i.astype(np.float32) / np.float32(n)).astype(np.float64), radical_inverse(i)


FRAME_THRESHOLD = float(np.float32(0.999))


def frame_decision(n_dir):
    """BRDF.hlsl:231: up = |N.z| < 0.999 ? +Z : +X, on the float64 unit N. 'undecided' where |N.z| is within the rounding an
    fp32 normalisation can add (4 ulp of 1) of the threshold, so fp32 evaluations may take either side."""
    nz = np.abs(normalize(n_dir)[..., 2])
    return nz < FRAME_THRESHOLD, np.abs(nz - FRAME_THRESHOLD) <= 4 * 2.0 ** -24


def importance_sample_ggx(xi_x, xi_y, n_dir, roughness):
    """BRDF.hlsl:217-238 in float64 -> unit H (the frame decided in float64)"""
    a = roughness * roughness
    phi = 2.0 * math.pi * np.asarray(xi_x, np.float64)
    xi_y = np.asarray(xi_y, np.float64)
    cos_t = np.sqrt((1.0 - xi_y) / (1.0 + (a * a - 1.0) * xi_y))
    sin_t = np.sqrt(np.maximum(0.0, 1.0 - cos_t * cos_t))
    N = normalize(n_dir)
    z_frame, _ = frame_decision(N)
    up = np.where(z_frame[..., None], [0.0, 0.0, 1.0], [1.0, 0.0, 0.0])
    T = normalize(np.cross(up, N))
    B = np.cross(N, T)
    h = T * (np.cos(phi) * sin_t)[..., None] + B * (np.sin(phi) * sin_t)[..., None] + N * cos_t[..., None]
    return normalize(h)


def ggx_h_error(xi_y, roughness):
    """per-component bound on |H_fp32 - H| for ImportanceSampleGGX evaluated in fp32: the denominator
    1 + (a^2 - 1) xi_y cancels as xi_y -> 1 at small roughness (its rounding, relative to itself, grows like 1/D), the
    square roots are correctly rounded, sin = sqrt(1 - cos^2) amplifies the cos error by cos/sin, and the frame
    (two normalisations, two cross products, the sum of three terms and the final normalize) adds <= 16 EPS"""
    a2 = float(roughness) ** 4
    xi_y = np.asarray(xi_y, np.float64)
    D = 1.0 + (a2 - 1.0) * xi_y
    e_d = xi_y * (3 * EPS * a2 + 2 * EPS * abs(a2 - 1.0)) + EPS * np.abs(D)
    cos_t = np.sqrt((1.0 - xi_y) / D)
    sin_t = np.sqrt(np.maximum(0.0, 1.0 - cos_t * cos_t))
    d_cos = cos_t * ((3 * EPS + e_d / np.abs(D)) / 2 + 2 * EPS)
    e_sq = 2 * d_cos + 2 * EPS
    with np.errstate(divide="ignore", invalid="ignore"):
        d_sin = np.minimum(np.where(sin_t > 0, e_sq / (2 * sin_t), np.inf), np.sqrt(e_sq)) + EPS
    return d_cos + d_sin + 16 * EPS


def ndf_ggx(nh, roughness):
    """BRDF.hlsl:65-79 (the 1e-12 guard of the denominator included)"""
    a2 = roughness ** 4
    t = nh * nh * (a2 - 1.0) + 1.0
    den = math.pi * t * t
    return np.where(den < 1e-12, 1.0, a2 / np.where(den < 1e-12, 1.0, den))


# ---- single-sample probes --------------------------------------------------------------------------------------------
def k3_single_sample_lod(roughness, hdri_w, hdri_h):
    """K3 with num_samples = 1: Xi = (0, 0) -> H = N, L = N, pdf = D(1)/4 = 1/(4 pi r^4), so
    lod = 0.5 * log2(1 / (pdf * OmegaP)) - 1 = 0.5 * log2(6 W H r^4) - 1 (clamped at 0; OmegaP = 4 pi / (6 W H))"""
    r = float(roughness)
    return max(0.0, 0.5 * math.log2(6.0 * hdri_w * hdri_h * r ** 4) - 1.0)


def k3_single_sample_lod_error(roughness):
    """|lod_fp32 - lod|: N.H = 1 - k*EPS after the fp32 frame and normalisations (k <= 8), so t = nh^2 (a^2 - 1) + 1 is
    a^2 + O(16 EPS): relative 16 EPS / a^2 (the cancellation at small roughness), D ~ 1/t^2 and lod = -0.5 log2(D ...):
    |dlod| <= (16 EPS / a^2 + 16 EPS) / ln 2, plus lg2.approx (2^-22) and the fp32 roughness m/(mips-1)."""
    a2 = float(roughness) ** 4
    return (16 * EPS / a2 + 32 * EPS) / math.log(2.0) + 2.0 ** -21


def k2_angles(step, n_phi, n_theta):
    """the (phi, theta) grid of CubemapConvolution.hlsl:129-135 as fp32 values; step > 0: the float-accumulated loops
    (trip counts from the fp32 comparisons against the fp32 bounds, as the host computes them)"""
    f32 = np.float32
    if step > 0:
        st = f32(step)
        phis, p = [], f32(0)
        while p < f32(6.28318530718):
            phis.append(p); p = f32(p + st)
        ths, t = [], f32(0)
        while t < f32(1.5707963268):
            ths.append(t); t = f32(t + st)
        return np.array(phis, np.float64), np.array(ths, np.float64)
    dphi = f32(f32(6.28318530718) / f32(n_phi)); dth = f32(f32(1.5707963268) / f32(n_theta))
    return ((np.arange(n_phi).astype(f32) * dphi).astype(np.float64), (np.arange(n_theta).astype(f32) * dth).astype(np.float64))


def k2_sample_dirs(n_dir, phi, theta):
    """CubemapConvolution.hlsl:119-140: right = normalize(cross(+Y, N)), up = normalize(cross(N, right)),
    sample = right sin(theta) cos(phi) + up sin(theta) sin(phi) + N cos(theta)"""
    N = normalize(n_dir)
    right = normalize(np.cross([0.0, 1.0, 0.0], N))
    up = normalize(np.cross(N, right))
    st, ct = math.sin(theta), math.cos(theta)
    return normalize(right * st * math.cos(phi) + up * st * math.sin(phi) + N * ct)


def brdf_lut_single_sample(w, h):
    """K4 with num_samples = 1 (Xi = (0, 0): H = +Z, L = reflect(-V, +Z), N.L = N.V, V.H = N.V): the LUT texel is
    ((1 - Fc) G_Vis, Fc G_Vis) with Fc = (1 - NdotV)^5 and G_Vis = max(G * NdotV / (1 * NdotV), 1e-4) = max(G, 1e-4),
    G = g(NdotV)^2, g(x) = x / (x (1 - k) + k + 1e-4), k = r^2 / 2; NdotV = (x+0.5)/w, r = (y+0.5)/h (fp32 rounded)"""
    f32 = np.float32
    nv = ((np.arange(w).astype(f32) + f32(0.5)) / f32(w)).astype(np.float64)[None, :]
    r = ((np.arange(h).astype(f32) + f32(0.5)) / f32(h)).astype(np.float64)[:, None]
    k = r * r / 2.0
    g = nv / (nv * (1.0 - k) + k + 1e-4)
    gv = np.maximum(g * g, 1e-4)
    fc = (1.0 - nv) ** 5
    return np.stack([(1.0 - fc) * gv, fc * gv], axis=-1)


def brdf_lut_single_sample_bound(w, h):
    """|fp32 - float64| of the single-sample LUT texel: <= 32 EPS relative for the products and quotients (the reflected L
    is re-normalised with rsqrtf, the geometry terms divide twice, pow5 multiplies three times), plus the cancellation of
    1 - Fc: fp32 Fc carries 4 EPS * Fc absolute, which 1 - Fc keeps while it shrinks towards 5 NdotV as NdotV -> 0"""
    v = brdf_lut_single_sample(w, h)
    f32 = np.float32
    nv = ((np.arange(w).astype(f32) + f32(0.5)) / f32(w)).astype(np.float64)[None, :]
    fc = (1.0 - nv) ** 5
    gv = v[..., 0] + v[..., 1]
    b = 32 * EPS * np.abs(v)
    b[..., 0] += 8 * EPS * fc * gv
    return b + 1e-30
