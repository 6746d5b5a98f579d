"""The three PCF tests of the shadowed pass in float64, vectorised over pixels x taps, written from the shader text
(Lighting.hlsl:113-263) and the decisions listed at the top of oracle/oracle_shadow.cpp — not from the oracle's code:

  * cube taps: the face of the largest |component| (ties X > Y > Z), face-plane coordinates (-z,y)/(z,y)/(x,-z)/(x,z)/(x,y)/(-x,y)
    over |major|, texel min(floor(s*N), N-1) with s = 0.5 + sx/2, t = 0.5 - sy/2; a tap is shadowed when
    |Lw| > closest*far + bias + 0.001;
  * 2-D taps: p = ls.xyz / ls.w; outside the frustum (any of px, py outside [-1, 1], pz outside [0, 1]) the count is 25;
    otherwise texel (floor(u*W) mod W, floor(v*H) mod H) for u = 0.5 + px/2 + k*tsx, v = 0.5 - py/2 + k*tsy (WRAP, POINT), and a
    tap is shadowed when pz - BIAS > closest (BIAS = depthBias for the directional light, depthBias*tan(acos(NdotL)) for a spot).

Every tap comes with a `decided` flag: its depth margin, texel-coordinate margins, face-tie margin and frustum margins all exceed
EPS (2^-18) times a bound on the magnitudes the fp32 computation rounds (sums of |term|). fp32 rounds each of its ~10 operations
on the way to a decision to 2^-24 of those magnitudes, so a decided tap cannot flip. The per-pixel result is an interval
[lo, hi]: lo counts the decided shadowed taps, hi adds the undecided ones (and, for a spot caster, the taps whose comparison
changes while BIAS ranges over its interval: acos to 4 fp32 ulp, tan to 2^-18). The fp32 count must lie inside it, and equal
lo where lo == hi. With eps=0 every comparison is taken as exact (for inputs whose fp32 evaluation is exact: `exact` probes)."""
import numpy as np

EPS = 2.0 ** -18
A, B = float(np.float32(0.5773502691896258)), float(np.float32(0.7071067811865475))
OFFSETS = np.array([[A, A, A], [A, -A, A], [-A, -A, A], [-A, A, A], [A, A, -A], [A, -A, -A], [-A, -A, -A], [-A, A, -A],
                    [B, B, 0], [B, -B, 0], [-B, -B, 0], [-B, B, 0], [B, 0, B], [-B, 0, B], [B, 0, -B], [-B, 0, -B],
                    [0, B, B], [0, -B, B], [0, -B, -B], [0, B, -B]])


def _f3(v):
    return np.array([v.x, v.y, v.z], np.float64)


def _margin_ok(margin, scale, eps):
    return np.ones(np.shape(margin), bool) if eps == 0 else (np.abs(margin) > eps * scale)


def cube_faces(v):
    """face index (0..5 = +X -X +Y -Y +Z -Z), nu, nv, |major|, second-largest |component| for directions v [..., 3]"""
    ax, ay, az = np.abs(v[..., 0]), np.abs(v[..., 1]), np.abs(v[..., 2])
    isX = (ax >= ay) & (ax >= az)
    isY = ~isX & (ay >= az)
    ma = np.where(isX, ax, np.where(isY, ay, az))
    second = np.where(isX, np.maximum(ay, az), np.where(isY, np.maximum(ax, az), np.maximum(ax, ay)))
    comp = np.where(isX, v[..., 0], np.where(isY, v[..., 1], v[..., 2]))
    pos = comp > 0
    nu = np.where(isX, np.where(pos, -v[..., 2], v[..., 2]), np.where(isY, v[..., 0], np.where(pos, v[..., 0], -v[..., 0])))
    nv = np.where(isY, np.where(pos, -v[..., 2], v[..., 2]), v[..., 1])
    face = np.where(isX, 0, np.where(isY, 2, 4)) + np.where(pos, 0, 1)
    return face, nu, nv, ma, second


def _texel(sc, n):
    """cube texel index of face coordinate sc in [-1, 1] and its distance (in sc units) to the nearest interior texel boundary"""
    x = np.clip(np.floor((0.5 + 0.5 * sc) * n), 0, n - 1).astype(np.int64)
    if n == 1:
        return x, np.full(np.shape(sc), np.inf)
    k = np.clip(np.rint((0.5 + 0.5 * sc) * n), 1, n - 1)
    return x, np.abs(sc - (2.0 * k / n - 1.0))


def point_counts(scene, P, i, eps=EPS):
    """point caster i at pixels P [n, 3] (fp32 values): dict(lo, hi, in_range, axis, gap, r) — counts over the 20 taps"""
    L = scene.pf.Lights.point_casters[i]
    pos, far, bias = _f3(L.position), float(L.range), float(L.depthBias)
    R, cube = scene.cube_res, scene.cubes[i].astype(np.float64)
    Lw = pos - P
    lenLw = np.linalg.norm(Lw, axis=-1)
    vd = np.linalg.norm(P - scene.cam.astype(np.float32).astype(np.float64), axis=-1)
    dr = (1.0 + vd / far) * 0.125
    v = -(Lw[:, None, :] + OFFSETS[None] * dr[:, None, None])                          # [n, 20, 3]
    face, nu, nv, ma, second = cube_faces(v)
    S = (np.abs(pos).sum() + np.abs(P).sum(-1) + dr)[:, None]                           # magnitudes fp32 rounds on the way
    with np.errstate(all="ignore"):
        sx, sy = nu / ma, nv / ma
    x, mx = _texel(sx, R)
    y, my = _texel(-sy, R)                                                              # t = 0.5 - sy/2: the same rule on -sy
    closest = cube[face, y, x] * far
    thr = closest + bias + 0.001
    shadowed = lenLw[:, None] > thr
    decided = (_margin_ok(ma - second, S, eps) & _margin_ok(mx, 2 * S / ma, eps) & _margin_ok(my, 2 * S / ma, eps)
               & _margin_ok(lenLw[:, None] - thr, lenLw[:, None] + thr + S, eps))
    lo = (shadowed & decided).sum(-1)
    hi = lo + (~decided).sum(-1)
    # the major axis of Lw itself and its gap (for the axis path)
    fL, _, _, maL, secL = cube_faces(-Lw)
    in_range = lenLw < far
    lo = np.where(_margin_ok(lenLw - far, lenLw + far + S[:, 0], eps), lo, 0)             # the range test itself undecided:
    hi = np.where(_margin_ok(lenLw - far, lenLw + far + S[:, 0], eps), hi, 20)            # the slot may be unwritten (0)
    return dict(lo=lo, hi=hi, in_range=in_range, axis=fL // 2, gap=maL - secL, r=B * dr, face=face)


def _ls(P, M):
    """light-space position (f64) of row vector (P, 1) times the row-major M, and the sums of |term| per component"""
    h = np.concatenate([P, np.ones((len(P), 1))], 1)
    return h @ M, np.abs(h) @ np.abs(M)


def pcf2d(ls, S, bias_lo, bias_hi, dmap, ts, eps=EPS):
    """the 5x5 test for light-space positions ls [n, 4] with magnitude sums S [n, 4] and BIAS in [bias_lo, bias_hi]:
    dict(lo, hi, outside, tx [n, 5], ty [n, 5], pz)"""
    Hh, Ww = dmap.shape
    n = len(ls)
    w = ls[:, 3]
    with np.errstate(all="ignore"):
        p = ls[:, :3] / w[:, None]
        E = (S[:, :3] + np.abs(p) * S[:, 3:4]) / np.abs(w)[:, None]                     # what fp32 rounds, in units of p
    exact_w0 = (w == 0)                                                                 # x/0: +-inf or NaN, decided by IEEE rules
    px, py, pz = p[:, 0], p[:, 1], p[:, 2]
    outside = (px < -1) | (px > 1) | (py < -1) | (py > 1) | (pz < 0) | (pz > 1)
    fr_dec = exact_w0 | (_margin_ok(px + 1, E[:, 0], eps) & _margin_ok(px - 1, E[:, 0], eps) & _margin_ok(py + 1, E[:, 1], eps)
                         & _margin_ok(py - 1, E[:, 1], eps) & _margin_ok(pz, E[:, 2], eps) & _margin_ok(pz - 1, E[:, 2], eps))
    k = np.arange(-2, 3, dtype=np.float64)
    with np.errstate(all="ignore"):
        U = (0.5 + 0.5 * px)[:, None] + k[None] * ts[0]
        V = (0.5 - 0.5 * py)[:, None] + k[None] * ts[1]
        fu, fv = U * Ww, V * Hh
        tx = np.where(np.isfinite(fu), np.floor(np.nan_to_num(fu)), 0).astype(np.int64) % Ww   # NaN -> 0 (D3D / cvt.rmi)
        ty = np.where(np.isfinite(fv), np.floor(np.nan_to_num(fv)), 0).astype(np.int64) % Hh
        du = np.abs(fu - np.rint(fu)) / Ww; dv = np.abs(fv - np.rint(fv)) / Hh               # distance to a boundary, in u units
    tex_dec = ((Ww == 1) | _margin_ok(du, (E[:, 0:1] + 3), eps)) & ((Hh == 1) | _margin_ok(dv, (E[:, 1:2] + 3), eps))   # [n, 5]
    closest = dmap.astype(np.float64)[ty[:, None, :], tx[:, :, None]]                         # [n, x 5, y 5]
    with np.errstate(all="ignore"):
        zb_hi, zb_lo = pz - bias_lo, pz - bias_hi                                           # pz - BIAS over the BIAS interval
        surely = zb_lo[:, None, None] > closest
        maybe = zb_hi[:, None, None] > closest
        scale = (E[:, 2] + np.abs(bias_hi) + np.abs(bias_lo) + 1)[:, None, None]
        dec = (_margin_ok(zb_lo[:, None, None] - closest, scale, eps) & _margin_ok(zb_hi[:, None, None] - closest, scale, eps)
               & tex_dec[:, :, None] & tex_dec[:, None, :])
    nanz = ~np.isfinite(pz - bias_lo)
    dec = dec | nanz[:, None, None]                                                         # NaN: every comparison is false
    lo_in = (surely & dec).reshape(n, -1).sum(-1)
    hi_in = (maybe | ~dec).reshape(n, -1).sum(-1)
    # an undecided frustum test: either 25 (outside) or the count inside
    lo = np.where(fr_dec, np.where(outside, 25, lo_in), lo_in)
    hi = np.where(fr_dec, np.where(outside, 25, hi_in), 25)
    return dict(lo=lo, hi=hi, outside=outside, tx=tx, ty=ty, pz=pz, frustum_decided=fr_dec)


def dir_counts(scene, P, eps=EPS):
    L = scene.pf.Lights
    M = np.array(L.shadowViewDirectional.m, np.float64).reshape(4, 4)
    ls, S = _ls(P, M)
    b = float(L.directional.depthBias)
    ts = (float(np.float32(1.0) / np.float32(scene.dir_w)), float(np.float32(1.0) / np.float32(scene.dir_h)))
    return pcf2d(ls, S, b, b, scene.dmap, ts, eps)


def dir_taps(scene, P):
    """texel indices of the directional taps and the fp32 value of pz - bias (for pixels whose fp32 evaluation is exact)"""
    r = dir_counts(scene, P, eps=0)
    pzb32 = (r["pz"].astype(np.float32) - np.float32(scene.pf.Lights.directional.depthBias)).astype(np.float32)
    return dict(tx=r["tx"], ty=r["ty"], pzb32=pzb32)


def spot_ndotl32(scene, P, Nraw, i):
    """saturate(dot(Nraw, normalize(light - P))) in fp32, every operation rounded as the kernel rounds it (all correctly rounded)"""
    f = np.float32
    l = _f3(scene.pf.Lights.spot_casters[i].position).astype(f)
    P32, N32 = P.astype(f), Nraw.astype(f)
    Lv = (l[None] - P32).astype(f)
    d = ((Lv[:, 0] * Lv[:, 0] + Lv[:, 1] * Lv[:, 1]).astype(f) + (Lv[:, 2] * Lv[:, 2]).astype(f)).astype(f)
    ln = np.sqrt(d).astype(f)
    with np.errstate(all="ignore"):
        Ln = (Lv / ln[:, None]).astype(f)
    dot = ((N32[:, 0] * Ln[:, 0] + N32[:, 1] * Ln[:, 1]).astype(f) + (N32[:, 2] * Ln[:, 2]).astype(f)).astype(f)
    return np.minimum(np.maximum(dot, f(0)), f(1))


def spot_bias_interval(depth_bias, ndotl32):
    """depthBias * tan(acos(NdotL)) over acos to 4 fp32 ulp and tan to 2^-18 (libm on either build); acos(0) is taken as the fp32
    nearest pi/2 (both builds return it), so a saturated NdotL gets the large NEGATIVE tan of that angle, as fp32 does"""
    x = ndotl32.astype(np.float64)
    th = np.arccos(x)
    th32 = np.arccos(ndotl32.astype(np.float32)).astype(np.float32).astype(np.float64)
    u = 4 * np.spacing(th.astype(np.float32)).astype(np.float64)
    t_lo, t_hi = np.tan(th - u), np.tan(th + u)
    at0 = ndotl32 == 0
    t_lo = np.where(at0, np.tan(th32), t_lo); t_hi = np.where(at0, np.tan(th32), t_hi)
    cross = ~at0 & (th - u < np.pi / 2) & (th + u > np.pi / 2)                          # tan changes sign inside: anything goes
    lo = np.minimum(t_lo, t_hi) * (1 - EPS); hi = np.maximum(t_lo, t_hi) * (1 + EPS)
    lo = np.where(lo < 0, np.minimum(t_lo, t_hi) * (1 + EPS), lo); hi = np.where(hi < 0, np.maximum(t_lo, t_hi) * (1 - EPS), hi)
    lo = np.where(cross, -np.inf, lo); hi = np.where(cross, np.inf, hi)
    return depth_bias * lo, depth_bias * hi


def spot_counts(scene, P, Nraw, i, eps=EPS):
    L = scene.pf.Lights
    M = np.array(L.shadowViews[i].m, np.float64).reshape(4, 4)
    ls, S = _ls(P, M)
    b_lo, b_hi = spot_bias_interval(float(L.spot_casters[i].depthBias), spot_ndotl32(scene, P, Nraw, i))
    ts = (float(np.float32(1.0) / np.float32(scene.spot_w)), float(np.float32(1.0) / np.float32(scene.spot_h)))
    return pcf2d(ls, S, b_lo, b_hi, scene.spots[i], ts, eps)


def all_counts(scene, eps=EPS):
    """[11, n] lo / hi per record slot (point casters, spot casters, directional) and the point casters' range flags [5, n]"""
    P = scene.planes[0].reshape(-1, 4)[:, :3].astype(np.float64)
    N = scene.planes[1].reshape(-1, 4)[:, :3].astype(np.float64)
    lo, hi, rng = [], [], []
    for i in range(5):
        r = point_counts(scene, P, i, eps)
        lo.append(np.where(r["in_range"], r["lo"], np.minimum(r["lo"], 0)))
        hi.append(np.where(r["in_range"], r["hi"], np.where(r["hi"] == 20, 20, 0)))
        rng.append(r["in_range"])
    for i in range(5):
        r = spot_counts(scene, P, N, i, eps)
        lo.append(r["lo"]); hi.append(r["hi"])
    r = dir_counts(scene, P, eps)
    lo.append(r["lo"]); hi.append(r["hi"])
    return np.array(lo), np.array(hi), np.array(rng)


def decode(rec):
    """[n] uint64 records -> [11, n] counts"""
    rec = np.asarray(rec, np.uint64)
    return np.array([(rec >> np.uint64(5 * s)) & np.uint64(31) for s in range(11)]).astype(np.int64)
