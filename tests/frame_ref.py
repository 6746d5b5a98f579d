"""References for the passes either side of the shading path, written from stb (stb_image.h stbi__hdr_load /
stbi__hdr_convert, stb_image_write.h stbiw__linear_to_rgbe, stb_image_resize.h's Mitchell filter) and the shader text
(Skydome.hlsl, ApplyReflections.hlsl, DownsampleDepth.hlsl), not from the oracle:
  * RGBE decode, exact: texel = ldexp(m, e - 136), e == 0 -> black; MaxLuminance in left-to-right float32 arithmetic.
  * RGBE encode, exact: for finite maxcomp, mant * 256 / maxcomp is exactly 2^(8 - e), so c * 2^(8 - e) is one exact float64
    product and the byte is its truncation; the non-finite and negative cases follow the rule stated in vqcuda.h.
  * Downsize: stb's Mitchell coefficients (mitchell_table), gathered in float64 with edge clamp, bounded (resize_ref).
  * Skydome: a float64 ray from the fp32 matrix, atan2 / asin, WRAP bilinear of level 0 (ibl_ref's sampler and its
    pole-widened bound).
  * Reflection composite: numpy float32 operations, which round as __fadd_rn / __fmul_rn do: bit-exact.
  * Depth pyramid: np.fmin over the ceil-halved, zero-padded domain, clipped to D3D mip sizes."""
from __future__ import annotations

import re

import numpy as np

import ibl_ref as ir

f32 = np.float32
EPS = 2.0 ** -24


# ---- Radiance .hdr -----------------------------------------------------------------------------------------------------
def _gettoken(data, i):
    """stbi__hdr_gettoken: one line without its '\\n', cut at 1023 characters (the rest of the line skipped)"""
    n = len(data)
    s = bytearray()
    c = data[i] if i < n else 0; i += 1
    while i <= n and c != 10:
        s.append(c)
        if len(s) == 1023:
            while i < n and data[i] != 10:
                i += 1
            i += 1
            break
        c = data[i] if i < n else 0; i += 1
    return bytes(s), i


def rgbe_to_float(px):
    """[..., 4] uint8 RGBE -> [..., 4] float32: rgb * 2^(e - 136), alpha 1; e == 0 -> (0, 0, 0, 1)"""
    px = np.asarray(px, np.uint8)
    e = px[..., 3].astype(np.int64)
    out = np.ones(px.shape, f32)
    for k in range(3):
        out[..., k] = np.where(e == 0, 0.0, np.ldexp(px[..., k].astype(np.float64), e - 136)).astype(f32)
    return out


def max_luminance(img):
    """Image::CalculateMaxLuminance: 0.2126 r + 0.7152 g + 0.0722 b in float32, left to right; the largest value above 0"""
    lum = (f32(0.2126) * img[..., 0] + f32(0.7152) * img[..., 1]) + f32(0.0722) * img[..., 2]
    return f32(max(0.0, float(lum.max()))) if lum.size else f32(0.0)


def hdr_decode(data: bytes):
    """stbi__hdr_load with req_comp 4 -> (0, [h, w, 4] float32, MaxLuminance) or (failure, None, None). A stream that ends
    inside a run-length encoded scanline is a failure (stb would read zeros forever)."""
    i = 0
    tok, i = _gettoken(data, i)
    if tok not in (b"#?RADIANCE", b"#?RGBE"):
        return 1, None, None
    valid = False
    while True:
        tok, i = _gettoken(data, i)
        if not tok:
            break
        valid |= tok == b"FORMAT=32-bit_rle_rgbe"
    if not valid:
        return 2, None, None
    tok, i = _gettoken(data, i)
    m = re.match(rb"-Y (\d+) +\+X (\d+)", tok)
    if not m:
        return 3, None, None
    h, w = int(m.group(1)), int(m.group(2))
    n = len(data)
    get = lambda p: data[p] if p < n else 0                     # noqa: E731  (stbi__get8: 0 past the end)
    px = np.zeros((h * w, 4), np.uint8)

    def flat_from(texel, p):
        cnt = (h * w - texel) * 4
        raw = np.frombuffer(data[p:p + cnt].ljust(cnt, b"\0"), np.uint8)
        px[texel:] = raw.reshape(-1, 4)

    if w < 8 or w >= 32768:
        flat_from(0, i)
    else:
        for j in range(h):
            c1, c2, ln = get(i), get(i + 1), get(i + 2)
            if c1 != 2 or c2 != 2 or (ln & 0x80):
                px[0] = (c1, c2, ln, get(i + 3))
                flat_from(1, i + 4)
                break
            if ((ln << 8) | get(i + 3)) != w:
                return 4, None, None
            i += 4
            row = np.zeros((w, 4), np.uint8)
            for k in range(4):
                x = 0
                while x < w:
                    if i >= n:
                        return 5, None, None
                    c = data[i]; i += 1
                    if c > 128:
                        c -= 128
                        if c > w - x:
                            return 5, None, None
                        row[x:x + c, k] = get(i); i += 1
                    else:
                        if c > w - x:
                            return 5, None, None
                        seg = data[i:i + c].ljust(c, b"\0")
                        row[x:x + c, k] = np.frombuffer(seg, np.uint8)
                        i += c
                    x += c
            px[j * w:(j + 1) * w] = row
    img = rgbe_to_float(px).reshape(h, w, 4)
    return 0, img, max_luminance(img)


def _trunc_byte(x):
    """the low byte of x truncated toward zero to int32, NaN -> 0, saturated at the int32 range (cvt.rzi.s32.f32)"""
    x = np.asarray(x, np.float64)
    with np.errstate(invalid="ignore"):
        i = np.where(np.isnan(x), 0, np.clip(np.trunc(np.nan_to_num(x, nan=0.0)), -2.0 ** 31, 2.0 ** 31 - 1)).astype(np.int64)
    return (i & 0xFF).astype(np.uint8)


def rgbe_encode(rgba):
    """stbiw__linear_to_rgbe per texel -> [..., 4] uint8:
    maxcomp = stbiw__max(r, stbiw__max(g, b)) with stbiw__max(a, b) = a > b ? a : b (a NaN in r or g is ignored, a NaN in
    b is not); maxcomp < 1e-32 (negative, -0 and -Inf included) -> (0, 0, 0, 0); else e = the frexp exponent (0 for +Inf
    and NaN), byte c = trunc(c * mant * 256 / maxcomp) & 0xff (NaN -> 0), byte e = (e + 128) & 0xff: maxcomp >= 2^127
    wraps to 0 (decoded as black, as stb decodes what stb writes)"""
    a = np.asarray(rgba, f32)
    r, g, b = a[..., 0], a[..., 1], a[..., 2]
    with np.errstate(invalid="ignore"):
        gb = np.where(g > b, g, b)
        mc = np.where(r > gb, r, gb)
        enc = ~(mc < f32(1e-32))
        mant, e = np.frexp(mc.astype(np.float64))
        norm = (mant * 256.0 / mc.astype(np.float64)).astype(f32)        # exact 2^(8 - e) when finite
        out = np.zeros(a.shape[:-1] + (4,), np.uint8)
        for k, c in enumerate((r, g, b)):
            out[..., k] = _trunc_byte((c.astype(np.float64) * norm.astype(np.float64)).astype(f32))
    out[..., 3] = ((e + 128) & 0xFF).astype(np.uint8)
    out[~enc] = 0
    return out


# ---- Mitchell downsize -------------------------------------------------------------------------------------------------
def _gamma(n):
    u = EPS
    return n * u / (1 - n * u)


def _mitchell(x):
    """stbir__filter_mitchell, B = C = 1/3, support 2, in float32 as C evaluates it"""
    x = np.abs(np.asarray(x, f32))
    with np.errstate(all="ignore"):
        a = (f32(16) + x * x * (f32(21) * x - f32(36))) / f32(18)
        b = (f32(32) + x * (f32(-60) + x * (f32(36) - f32(7) * x))) / f32(18)
    return np.where(x < 1, a, np.where(x < 2, b, f32(0))).astype(f32)


def mitchell_table(in_size, out_size):
    """The per-output tap table of one axis of stbir_resize_float's downsize, from stb_image_resize.h's text, in float32 as
    stb computes it -> (start, count, weights [out, max_taps]) in the layout of vq.resize_axis_table.
    stb scatters every input sample j (edge-clamped virtual samples included, `margin` either side) to the outputs
    first_j .. last_j with coefficient mitchell(out_centre - centre_j) * scale (stbir__calculate_coefficients_downsample),
    drops the zero coefficients at both ends of that range, and normalises per output by the float32 sum over j
    (stbir__normalize_downsample_coefficients). Here the same numbers are gathered per output: its samples in increasing j,
    from the first to the last one stb adds to it. Float32 throughout, because stb's sample centre is a float32 product
    (its rounding moves a weight by ~1e-5 at 4096 texels): float64 weights would not be stb's."""
    scale = f32(out_size) / f32(in_size)
    radius = f32(2.0) / scale
    margin = int(np.ceil(np.float64(f32(4.0) / scale))) // 2
    n = in_size + 2 * margin
    c = (np.arange(n) - margin).astype(f32) + f32(0.5)
    centre = (c * scale).astype(f32)
    first = np.floor(((c - radius) * scale).astype(f32).astype(np.float64) + 0.5).astype(np.int64)
    last = np.floor(((c + radius) * scale).astype(f32).astype(np.float64) - 0.5).astype(np.int64)
    v0, v1 = first.copy(), last.copy()                  # the range stb visits: zero coefficients dropped at both ends
    for j in range(n):
        while v1[j] >= v0[j] and _mitchell(f32(v1[j]) + f32(0.5) - centre[j]) * scale == 0:
            v1[j] -= 1
        while v0[j] <= v1[j] and _mitchell(f32(v0[j]) + f32(0.5) - centre[j]) * scale == 0:
            v0[j] += 1
    start = np.zeros(out_size, np.int32); count = np.zeros(out_size, np.int32); rows = []
    jlo = 0
    for i in range(out_size):
        while jlo < n and last[jlo] < i:
            jlo += 1
        jhi = jlo
        while jhi + 1 < n and first[jhi + 1] <= i:
            jhi += 1
        js = np.arange(jlo, jhi + 1)
        inside = (first[js] <= i) & (i <= last[js])
        k = np.where(inside, (_mitchell(f32(i) + f32(0.5) - centre[js]) * scale).astype(f32), f32(0))
        total = np.add.accumulate(k, dtype=f32)[-1]
        k = (k * (f32(1) / total)).astype(f32)
        vis = np.flatnonzero((v0[js] <= i) & (i <= v1[js]))
        lo, hi = (int(vis[0]), int(vis[-1]) + 1) if vis.size else (0, 0)
        start[i] = jlo + lo - margin; count[i] = hi - lo; rows.append(k[lo:hi])
    taps = max(1, max(len(r) for r in rows))
    wt = np.zeros((out_size, taps), f32)
    for i, r in enumerate(rows):
        wt[i, :len(r)] = r
    return start, count, wt


def _gather(x, table, axis, skip_zero=False):
    """float64 sum_t w[i, t] * x[clamp(start[i] + t)] along `axis` (1: columns, 0: rows) and sum_t |w x|; x [h, w, 4] float64"""
    start, count, wt = table
    T = wt.shape[1]
    size = x.shape[axis]
    idx = np.clip(start[:, None] + np.arange(T)[None, :], 0, size - 1)
    live = np.arange(T)[None, :] < count[:, None]
    if skip_zero:
        live &= wt != 0
    w = np.where(live, wt.astype(np.float64), 0.0)
    if axis == 1:
        g = x[:, idx, :]                                  # [h, o, T, 4]
        ww = w[None, :, :, None]; lv = live[None, :, :, None]
        red = 2
    else:
        g = x[idx, :, :]                                  # [o, T, w, 4]
        ww = w[:, :, None, None]; lv = live[:, :, None, None]
        red = 1
    with np.errstate(invalid="ignore"):
        terms = np.where(lv, g * ww, 0.0)
    return terms.sum(axis=red), np.abs(terms).sum(axis=red), np.abs(w).sum(axis=1)


def resize_ref(img, tab_h, tab_v, skip_zero=True):
    """stbir_resize_float as the two gather passes (horizontal into an (out_w x in_h) fp32 intermediate, then vertical)
    in float64 -> (value [oh, ow, 4], bound [oh, ow, 4]).
    Bound. A pass sums n products left to right without FMA: fl(...fl(fl(w1 x1) + fl(w2 x2))...), whose error is at most
    gamma_n * sum |w_i x_i|, gamma_n = n u / (1 - n u), u = 2^-24 (Higham, Accuracy and Stability, 3.1). For n <= 4 that
    is the 2^-22 * sum |w_i x_i| of a short filter; the downsize gathers up to 4 * ratio taps, so gamma_n is used. The
    vertical pass reads the fp32 horizontal result H~ with |H~ - H| <= E_h: its error is sum |w| E_h + gamma_m sum |w| (|H| +
    E_h). The tables are mitchell_table's, computed from stb's text; tests/test_frame_domain.py checks that the kernels'
    host tables (vq.resize_axis_table) are the same bits.
    stb never adds a zero coefficient (it drops them from both ends of every input sample's range, and a Mitchell zero, at
    |x| = 8/7 or >= 2, can only sit at an end); skip_zero=True follows it. The gather tables keep the zero weight that a
    sample in the middle of an output's taps can have at |x| = 8/7 (7:5 and similar ratios): skip_zero=False is what the
    kernels compute, and differs from stb only where that tap meets a non-finite input (0 * Inf = NaN; vqcuda.h)."""
    x = np.asarray(img, f32).astype(np.float64)
    H, absH, _ = _gather(x, tab_h, 1, skip_zero)
    E_h = _gamma(tab_h[1].max()) * absH[:, :]            # per (row, output column)
    # vertical: E_v = sum |w| E_h + gamma_m sum |w| (|H| + E_h)
    start, count, wt = tab_v
    V, _, _ = _gather(H, tab_v, 0, skip_zero)
    sumE, _, _ = _gather(E_h, (start, count, np.abs(wt)), 0)
    absHE = np.where(np.isfinite(H), np.abs(H), 0.0) + np.where(np.isfinite(E_h), E_h, 0.0)
    sumHE, _, _ = _gather(absHE, (start, count, np.abs(wt)), 0)
    bound = sumE + _gamma(count.max()) * sumHE
    return V, bound


# ---- skydome -----------------------------------------------------------------------------------------------------------
def sky_ref(m, w, h, hdri, rows=None, mask=None, base=None):
    """Skydome PSMain per pixel in float64 -> (value [h, w, 4], bound [h, w, 3], written [h, w] bool).
    The ray is ((nx m0 + ny m4) + m8) + m12 per component in float64 from the fp32 matrix and the fp32 pixel centre (the
    kernel's nx, ny are correctly rounded, as numpy's). The kernel forms it in fp32: each component is off by at most
    4 u sum |terms| (three additions, two products), which moves the direction by at most |e_xyz| / |r_xyz|; the divide by w
    only scales it (unless |w| is within its own error of 0), the divide and the two normalisations round each component
    once more (8 u). A pixel whose fp32 ray has x = z = 0 exactly is a pole in both: there u depends only on the signs of
    the zeros and the only error is the uv arithmetic. Non-finite directions (w = 0) sample black, as the oracle decides;
    so do rays whose fp32 quotient overflows the normalisation (|ray / w|^2 > FLT_MAX: w within ~1e-19 of 0)."""
    import frame_domain as fd
    m = np.asarray(m, f32).reshape(16)
    hh, hw = hdri.shape[:2]
    xs = np.arange(w, dtype=f32); ys = np.arange(h, dtype=f32)
    nx = (((xs + f32(0.5)) / f32(w)) * f32(2.0) - f32(1.0)).astype(np.float64)[None, :]
    ny = (f32(1.0) - ((ys + f32(0.5)) / f32(h)) * f32(2.0)).astype(np.float64)[:, None]
    m64 = m.astype(np.float64)
    ray = [((nx * m64[c] + ny * m64[4 + c]) + m64[8 + c]) + m64[12 + c] for c in range(4)]
    S = [np.abs(nx * m64[c]) + np.abs(ny * m64[4 + c]) + np.abs(m64[8 + c]) + np.abs(m64[12 + c]) for c in range(4)]
    r32 = fd.sky_ray(m, w, h)
    with np.errstate(all="ignore"):
        d = np.stack([ray[c] / ray[3] for c in range(3)], axis=-1)
        n = np.linalg.norm(d, axis=-1)
        q32 = (r32[:3] / r32[3]).astype(f32)                          # the fp32 quotients and the first normalisation's dot
        dot32 = ((q32[0] * q32[0] + q32[1] * q32[1]) + q32[2] * q32[2]).astype(f32)
        ok = np.isfinite(n) & (n > 0) & np.isfinite(dot32) & (dot32 >= np.finfo(f32).tiny)
        du_ = np.where(ok[..., None], d, 1.0) / np.where(ok, n, 1.0)[..., None]
        rxyz = np.sqrt(sum(ray[c] ** 2 for c in range(3)))
        exyz = 4 * EPS * np.sqrt(sum(S[c] ** 2 for c in range(3)))
        delta = np.where(rxyz > 0, exyz / np.where(rxyz > 0, rxyz, 1.0), np.inf) + 8 * EPS
        delta = np.where(np.abs(ray[3]) > 4 * EPS * S[3], delta, np.inf)
    u, v = ir.direction_to_uv(du_)
    du, dv = ir.uv_delta(du_ * (1 + 8 * EPS), np.minimum(delta, 10.0))
    pole = (r32[0] == 0) & (r32[2] == 0) & ok
    cu, cv = ir.uv_compute_error()
    du = np.where(pole, cu, du); dv = np.where(pole, cv, dv)
    levels = [np.asarray(hdri, f32)[..., :3].astype(np.float64)]
    col = ir.sample(levels, u, v, 0.0)
    bound = ir.sample_bound(levels, u, v, 0.0, du, dv, 0.0)
    col = np.where(ok[..., None], col, 0.0)
    bound = np.where(ok[..., None], bound, 0.0)
    written = np.zeros((h, w), bool)
    rb, re_ = rows if rows else (0, h)
    written[rb:re_] = True
    if mask is not None:
        written &= (mask[..., 0] == 0) & (mask[..., 1] == 0) & (mask[..., 2] == 0)
    out = np.array(base, np.float64) if base is not None else np.zeros((h, w, 4))
    out[written, :3] = col[written]
    out[written, 3] = 1.0
    return out, np.where(written[..., None], bound, 0.0), written, pole


# ---- reflection composite ----------------------------------------------------------------------------------------------
def composite_ref(scene, refl, bv=None):
    """ApplyReflections CSMain in float32: scene.rgb + refl.rgb, alpha = scene.a; with the bounding-volume layer
    b.rgb * b.a + sum * (1 - b.a), alpha = b.a. Every operation rounded on its own (no FMA)."""
    s = np.asarray(scene, f32); r = np.asarray(refl, f32)
    with np.errstate(all="ignore"):
        o = (s[..., :3] + r[..., :3]).astype(f32)
        a = s[..., 3].copy()
        if bv is not None:
            b = np.asarray(bv, f32)
            oma = (f32(1.0) - b[..., 3]).astype(f32)
            o = (b[..., :3] * b[..., 3:4]).astype(f32) + (o * oma[..., None]).astype(f32)
            a = b[..., 3].copy()
    return np.concatenate([o, a[..., None]], axis=-1).astype(f32)


# ---- MIN depth pyramid -------------------------------------------------------------------------------------------------
def depth_ref(depth, n_levels):
    """-> (levels, ties): level l = MIN of the zero-padded 2x2 block of level l-1 in the ceil-halved domain, NaN ignored
    unless all four are NaN, stored clipped to max(1, w >> l) x max(1, h >> l). ties[l] marks results whose sign is not
    decided: the smallest value of the block is a zero and zeros of both signs (or an undecided zero) reach it. There
    D3D's min, and fminf, may return either zero."""
    d = np.asarray(depth, f32)
    h, w = d.shape
    levels = [d.copy()]; ties = [np.zeros_like(d, bool)]
    cur, tie = d, np.zeros_like(d, bool)
    for l in range(1, n_levels):
        ph, pw = (cur.shape[0] + 1) // 2, (cur.shape[1] + 1) // 2
        P = np.zeros((2 * ph, 2 * pw), f32); P[:cur.shape[0], :cur.shape[1]] = cur
        T = np.zeros((2 * ph, 2 * pw), bool); T[:cur.shape[0], :cur.shape[1]] = tie
        q = [P[0::2, 0::2], P[0::2, 1::2], P[1::2, 0::2], P[1::2, 1::2]]
        t = [T[0::2, 0::2], T[0::2, 1::2], T[1::2, 0::2], T[1::2, 1::2]]
        with np.errstate(invalid="ignore"):
            mn = np.fmin(np.fmin(q[0], q[1]), np.fmin(q[2], q[3]))
        zero = mn == 0
        pos = sum(((x == 0) & ~np.signbit(x)).astype(int) for x in q)
        neg = sum(((x == 0) & np.signbit(x)).astype(int) for x in q)
        und = sum(((x == 0) & tt).astype(int) for x, tt in zip(q, t))
        nt = zero & (((pos > 0) & (neg > 0)) | (und > 0))
        # a decided zero result takes the sign all its zeros share
        mn = np.where(zero & ~nt & (neg > 0), f32(-0.0), np.where(zero & ~nt, f32(0.0), mn)).astype(f32)
        lw, lh = max(1, w >> l), max(1, h >> l)
        levels.append(mn[:lh, :lw].copy()); ties.append(nt[:lh, :lw].copy())
        cur, tie = mn, nt
    return levels, ties


def depth_equal(got, want, tie):
    """bit for bit, NaN by position, either zero where `tie`"""
    g = np.asarray(got, f32); wv = np.asarray(want, f32)
    nan = np.isnan(wv)
    same = (g.view(np.uint32) == wv.view(np.uint32)) | (nan & np.isnan(g)) | (tie & (g == 0) & (wv == 0))
    return same & (np.isnan(g) == nan)
