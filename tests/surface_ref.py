"""Float64 restatement of the surface producer's texture sampler (ForwardLighting.hlsl:226-235 with the sampler decisions in
the header of vq_surface.cu / oracle_surface.cpp: fine quad derivatives, isotropic LOD, floor-halved packed levels, WRAP
bilinear at x = u*W - 0.5, trilinear with the last level taken alone), written from those rules and not from the oracle,
with a per-value bound on the error of an fp32 implementation:

  * coordinate: the fp32 sequence x = fl(fl(fl(ru*s) + o) * W) - 0.5 differs from the exact x by |dx|; the blend moves by at
    most |dx| times the largest byte step of the 4x4 texels around the footprint, over 255. Where |dx| reaches a texel the
    bound is the level's whole byte range.
  * LOD: the fp32 LOD (lg2.approx: 2^-22 absolute near 1, else 2 ulp) differs from the exact one by dlod; trilinear is
    continuous in the LOD across integers (the last level of a pair at k - eps equals the first at k), so the value moves by
    at most dlod times the largest difference between the blends of adjacent levels around l0.
  * the blend itself: bytes are exact, three fp32 lerps and a scale by 1/255: 8 u.
  * decisions: a level whose fp32 texel coordinate is not finite blends to NaN (vqcuda.h: fx = x - floor(x) is NaN there);
    that is a rule of the fp32 coordinate, so it is taken from the fp32 sequence. Beyond 2^31 the fp32 coordinate is far from
    the exact one (its spacing is >= 256 texels) and the conversion saturates, so the bound there is the level's whole
    range whichever texel is read; tests/test_surface_domain*.py pin the saturated texel itself.
    alpha < 0.01 is undecided where |alpha - 0.01| <= its bound.
"""
import numpy as np

U = 2.0 ** -24
F32MAX = float(np.finfo(np.float32).max)


def level_dims(w, h, l):
    return w >> l, h >> l


def level_offset(w, h, l):
    return sum((w >> k) * (h >> k) for k in range(l))


def mip_chain_ref(level0, levels):
    """packed RGBA8 chain by the box filter (a+b+c+d)/4 truncating over complete 2x2 blocks (DXGIUtils.cpp:263-287)"""
    out, cur = [level0.reshape(-1)], level0.astype(np.uint32)
    for _ in range(1, levels):
        hh, ww = cur.shape[0] // 2 * 2, cur.shape[1] // 2 * 2
        s = cur[:hh, :ww]
        cur = (s[0::2, 0::2] + s[0::2, 1::2] + s[1::2, 0::2] + s[1::2, 1::2]) // 4
        out.append(cur.astype(np.uint8).reshape(-1))
    return np.concatenate(out)


def _f32(a):
    return np.asarray(a, np.float32)


def _level_blend(chain, w, h, l, x, y):
    """float64 bilinear WRAP of level l at texel-space (x, y) (finite float64 arrays) -> (value [n,4] in [0,1], 4x4 byte range
    [n,4], level byte range [4])"""
    W, H = level_dims(w, h, l)
    lv = chain[4 * level_offset(w, h, l): 4 * (level_offset(w, h, l) + W * H)].reshape(H, W, 4)
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    ix = [np.mod(x0 + k, W).astype(np.int64) for k in (-1, 0, 1, 2)]
    iy = [np.mod(y0 + k, H).astype(np.int64) for k in (-1, 0, 1, 2)]
    t = lambda i, j: lv[iy[j], ix[i]].astype(np.float64)
    val = ((1 - fy) * ((1 - fx) * t(1, 1) + fx * t(2, 1)) + fy * ((1 - fx) * t(1, 2) + fx * t(2, 2))) / 255.0
    nb = np.stack([t(i, j) for i in range(4) for j in range(4)])
    flat = lv.reshape(-1, 4)
    return val, (nb.max(0) - nb.min(0)) / 255.0, (flat.max(0).astype(np.float64) - flat.min(0)) / 255.0


def lod_ref(w, h, levels, dudx, dvdx, dudy, dvdy, bias):
    """exact LOD of float64 derivatives, its fp32 emulation's distance from it plus the documented lg2.approx error -> (lod, dlod)"""
    W, H = float(w), float(h)
    with np.errstate(all="ignore"):
        m = np.maximum(dudx ** 2 * W * W + dvdx ** 2 * H * H, dudy ** 2 * W * W + dvdy ** 2 * H * H)
        lod = np.where(m > 0, 0.5 * np.log2(np.where(m > 0, m, 1.0)), -126.0) + bias
        a = [(_f32(d) * np.float32(s)).astype(np.float32) for d, s in ((dudx, W), (dvdx, H), (dudy, W), (dvdy, H))]
        m32 = np.maximum(a[0] * a[0] + a[1] * a[1], a[2] * a[2] + a[3] * a[3]).astype(np.float32)
        l32 = np.where(m32 > 0, 0.5 * np.log2(np.where(m32 > 0, m32, 1).astype(np.float64)), -126.0) + bias
        approx = 0.5 * np.where((m32 >= 0.5) & (m32 <= 2), 2.0 ** -22, 2 * 2.0 ** -23 * np.maximum(1, np.abs(np.log2(np.where(m32 > 0, m32, 1)))))
        hi = levels - 1.0
        c = lambda v: np.clip(np.nan_to_num(v, nan=0.0, posinf=hi, neginf=0.0), 0.0, hi)
        dl = np.abs(c(l32) - c(lod)) + approx + 4 * U * (np.abs(l32) + abs(bias)) + 8 * U
    return c(lod), np.where(np.isfinite(dl), dl, hi)


def sample_ref(chain, w, h, levels, ru, rv, s, o, ddx, ddy, bias=0.0):
    """Sample()/SampleBias() of one RGBA8 map at n pixels. ru, rv: raw uv (fp32); s, o: uvScale and uvOffset (fp32 pairs);
    ddx, ddy: the raw quad differences (fp32 pairs of arrays, exact inputs). Returns (value [n,4], bound [n,4])."""
    ru, rv = _f32(ru).ravel(), _f32(rv).ravel()
    n = ru.size
    su, sv, ou, ov = (float(np.float32(v)) for v in (s[0], s[1], o[0], o[1]))
    if chain is None:
        return np.zeros((n, 4)), np.zeros((n, 4))
    with np.errstate(all="ignore"):
        u64, v64 = ru.astype(np.float64) * su + ou, rv.astype(np.float64) * sv + ov
        u32 = (ru * np.float32(su)).astype(np.float32) + np.float32(ou)
        v32 = (rv * np.float32(sv)).astype(np.float32) + np.float32(ov)
    dd = [_f32(a).ravel().astype(np.float64) for a in (ddx[0], ddx[1], ddy[0], ddy[1])]
    lod, dlod = lod_ref(w, h, levels, dd[0] * su, dd[1] * sv, dd[2] * su, dd[3] * sv, bias)
    l0 = np.floor(lod).astype(np.int64)
    f = lod - l0
    val = np.zeros((n, 4))
    bound = np.full((n, 4), 8 * U)
    blends = {}
    for l in range(levels):
        sel_any = (l0 >= l - 2) & (l0 <= l + 1)
        if not sel_any.any():
            continue
        W, H = level_dims(w, h, l)
        with np.errstate(all="ignore"):
            x32 = (u32 * np.float32(W)).astype(np.float32) - np.float32(0.5)
            y32 = (v32 * np.float32(H)).astype(np.float32) - np.float32(0.5)
            x64, y64 = u64 * W - 0.5, v64 * H - 0.5
        zero = ~(np.isfinite(x32) & np.isfinite(y32))            # the rule: this level blends to NaN
        fin = np.isfinite(x64) & np.isfinite(y64) & ~zero
        xs, ys = np.where(fin, x64, 0.0), np.where(fin, y64, 0.0)
        v_l, nb, full = _level_blend(chain, w, h, l, xs, ys)
        with np.errstate(all="ignore"):
            d = np.abs(x32.astype(np.float64) - x64) + np.abs(y32.astype(np.float64) - y64)
            # |x| >= 2^31: the conversion saturates (vqcuda.h), a domain limit tested on its own; any texel of the level
            wide = (np.abs(x32) >= 2.0 ** 31) | (np.abs(y32) >= 2.0 ** 31)
            far = (~(d < 1.0) | wide) & ~zero
            cb = np.where(far[:, None], full[None, :], np.where(fin[:, None], d[:, None] * nb, 0.0))
        v_l = np.where(zero[:, None], np.nan, v_l)
        blends[l] = (v_l, cb)
    lv = lambda l: blends[min(max(l, 0), levels - 1)]
    for l in np.unique(l0):
        sel = l0 == l
        a, ba = (x[sel] for x in lv(l))
        fs = f[sel][:, None]
        if l + 1 < levels:
            b, bb = (x[sel] for x in lv(l + 1))
            with np.errstate(invalid="ignore"):
                val[sel] = np.where(fs > 0, (1 - fs) * a + fs * b, a)         # f = 0 reads the lower level alone
            bound[sel] += ba + bb
        else:
            val[sel] = a
            bound[sel] += ba
        steps = [np.abs(lv(k + 1)[0][sel] - lv(k)[0][sel]) for k in range(l - 1, l + 2) if 0 <= k and k + 1 < levels]
        if steps:
            bound[sel] += dlod[sel][:, None] * np.nan_to_num(np.max(steps, axis=0))
    return val, bound


def alpha_decision(alpha, bound, thr=0.01):
    """(discard, undecided) of the alpha mask: alpha < 0.01, undecided within the bound of the threshold"""
    return alpha < thr, np.abs(alpha - thr) <= bound + U
