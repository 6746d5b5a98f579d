"""Seeded scenes and G-buffers for K1's light loop over the whole domain of its inputs (test input generation, no GPU).

Every pixel is one configuration, in 256-pixel rows (one K1 tile), so that a tile and each warp hold configurations that
are alike or deliberately mixed. A PROBE frame isolates the light sum the way test_forward_mirror_kat does: ao = 0, no
emissive plane and all-zero environment maps, so the output is sum(BRDF * radiance * N.L) over the frame's lights.

  range_probes      point lights and point casters at ranges from the smallest denormal to +Inf (and 0, -0, -1, NaN), with
                    pixels found by an fp32 search where sqrt_rn(d2) equals the range, and their +-1..4 ulp neighbours
  distance_probes   pixels exactly at a light, 1e-3 .. 1e-16 away, at a denormal squared distance, lights 1e18..2e19 away
  spot_probes       cones with inner = 0, narrow and hard ramps, inner > outer, outer >= pi; pixels on the axis, near it,
                    around both edges and behind the light; each with the companion frame of a point light at the same
                    position (range +Inf), so that K1(spot) / K1(point) is the spot intensity
  directional_probe N.L exactly 0 and a denormal away, V parallel and antiparallel to the light, a zero direction
  mirror_probes     N = H bit for bit (the mirror KAT's geometry) at roughness around the D = 1 escape
  t_sweep_probe     GGX t across T_EXACT = 0.02 from both sides, one pixel per warp on the exact path
  view_probe        |N.V| across NV_EXACT = 1e-3, N.V exactly 0, the camera at the pixel, raw normals with |N| cos = 1
  mixed_frames      adversarial G-buffers (forward_domain) under 0, 1 of each kind and the ABI maximum of lights
"""
import ctypes as C
import math

import numpy as np

import forward_domain as fd
import light_ref as lr

F32 = np.float32
FLT_MAX = float(np.finfo(F32).max)
SQRT_MAX = float(F32(math.sqrt(FLT_MAX)))
DENORM_MIN = float(np.nextafter(F32(0), F32(1)))

# finite positive ranges searched for their edge; the rest have no edge
EDGE_RANGES = [1e-3, 0.3, 1.0, 1.1, 7.3, 14.0, 50.0, 1000.0, 1024.0, 123456.7,
               float(F32(SQRT_MAX * (1 - 2 ** -23))), SQRT_MAX, float(F32(SQRT_MAX * (1 + 2 ** -23))), FLT_MAX, math.inf]
NO_EDGE_RANGES = [0.0, -0.0, -1.0, math.nan, DENORM_MIN]


def zero_env():
    """all-zero environment maps: the environment terms vanish and the output is the light sum"""
    return fd.make_env(2, 2, (2, 2), seed=0, diff=np.zeros((30, 4), F32), spec=np.zeros((30, 4), F32),
                       lut=np.zeros((2, 2, 2), F32))


def _set3(v, x):
    v.x, v.y, v.z = (float(c) for c in x)


def scene(cam, points=(), spots=(), pcasters=(), scasters=(), directional=None, offset=0.0, max_lod=1):
    """PerFrameData / PerViewLightingData with the given lights (dicts: pos, range / dir, inner, outer, color, brightness)"""
    pf, pv = fd.constants(cam, max_lod, offset)
    L = pf.Lights
    for arr, lst, cnt in ((L.point_lights, points, "numPointLights"), (L.point_casters, pcasters, "numPointCasters")):
        setattr(L, cnt, len(lst))
        for i, p in enumerate(lst):
            _set3(arr[i].position, p["pos"]); _set3(arr[i].color, p.get("color", (1.0, 0.5, 0.25)))
            arr[i].range, arr[i].brightness = p.get("range", math.inf), p.get("brightness", 1.0)
    for arr, lst, cnt in ((L.spot_lights, spots, "numSpotLights"), (L.spot_casters, scasters, "numSpotCasters")):
        setattr(L, cnt, len(lst))
        for i, s in enumerate(lst):
            _set3(arr[i].position, s["pos"]); _set3(arr[i].color, s.get("color", (1.0, 0.5, 0.25)))
            _set3(arr[i].spotDir, s["dir"])
            arr[i].innerConeAngle, arr[i].outerConeAngle = s["inner"], s["outer"]
            arr[i].brightness, arr[i].range = s.get("brightness", 1.0), 100.0
    if directional is not None:
        d = L.directional
        d.enabled = 1
        _set3(d.lightDirection, directional["dir"]); _set3(d.color, directional.get("color", (1.0, 0.5, 0.25)))
        d.brightness = directional.get("brightness", 1.0)
    return pf, pv


def frame(P, N, rough, albedo=(0.5, 0.4, 0.3), metal=0.0):
    """per-pixel columns -> [H, 256, 4] planes (ao = 0) and the index of the configuration each pixel holds"""
    n = len(P)
    pos = np.concatenate([np.asarray(P, F32), np.zeros((n, 1), F32)], 1)
    nrm = np.concatenate([np.asarray(N, F32), np.broadcast_to(np.asarray(rough, F32), (n,))[:, None]], 1)
    alb = np.concatenate([np.broadcast_to(np.asarray(albedo, F32), (n, 3)), np.broadcast_to(np.asarray(metal, F32), (n,))[:, None]], 1)
    planes, idx = fd._frame([pos, nrm, alb])
    return planes, idx


def _facing(P, Lpos):
    """unit normals from the pixel towards the light (N.L = 1), float64 -> fp32; +Y where the pixel is at the light"""
    d = np.asarray(Lpos, np.float64)[None] - np.asarray(P, np.float64)
    n = np.linalg.norm(d, axis=1, keepdims=True)
    out = np.where(n > 0, d / np.where(n > 0, n, 1.0), np.array([[0.0, 1.0, 0.0]]))
    return out.astype(F32)


def _ulp_steps(x, k):
    """x moved by k ulp (k may be negative), elementwise, fp32"""
    x = np.asarray(x, F32).copy()
    k = np.broadcast_to(np.asarray(k), x.shape)
    for s in range(1, int(np.abs(k).max(initial=0)) + 1):
        m = np.abs(k) >= s
        x[m] = np.nextafter(x[m], np.where(k[m] > 0, F32(np.inf), F32(-np.inf)))
    return x


def octant_dirs(n, rng):
    """the 8 octant diagonals, then random directions"""
    s = np.array([[sx, sy, sz] for sx in (1, -1) for sy in (1, -1) for sz in (1, -1)], np.float64)
    d = s * np.array([0.577, 0.5, 0.648])
    d = np.concatenate([d, rng.normal(size=(max(0, n - 8), 3))])[:n]
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def edge_search(Lpos, R, dirs):
    """for each direction: scan the pixel's major coordinate over +-96 ulp around distance R (or sqrt(FLT_MAX) for ranges
    beyond it) and centre on where the fp32 rule flips (a pixel with sqrt_rn(d2) == R if there is one), then take the
    +-1..4 ulp neighbours of that centre on each axis. Returns the fp32 pixels."""
    T = min(R, SQRT_MAX * (1 - 2 ** -22)) if math.isfinite(R) else SQRT_MAX * (1 - 2 ** -22)
    Lp = np.asarray(Lpos, np.float64)
    out = []
    for u in dirs:
        P0 = (Lp - T * u).astype(F32)
        ax = int(np.argmax(np.abs(u)))
        k = np.arange(-96, 97)
        cand = np.repeat(P0[None], len(k), 0)
        cand[:, ax] = _ulp_steps(np.full(len(k), P0[ax]), k)
        with np.errstate(all="ignore"):
            d = np.sqrt(lr.light_d2(cand, Lpos))
        eq = np.nonzero(d == F32(R))[0] if math.isfinite(R) else np.zeros(0, int)
        lit = lr.in_range(cand, Lpos, R)
        flips = np.nonzero(lit[1:] != lit[:-1])[0]
        c = eq[len(eq) // 2] if len(eq) else (flips[0] if len(flips) else len(k) // 2)
        centre = cand[c]
        pts = [centre]
        for a in range(3):
            for s in (-4, -3, -2, -1, 1, 2, 3, 4):
                p = centre.copy()
                p[a] = _ulp_steps(p[a:a + 1], s)[0]
                pts.append(p)
        out.append(np.array(pts, F32))
    return np.concatenate(out)


def range_probes(seed=1):
    """one probe per (range, light or caster[, direction group for ranges beyond 1e18]); meta: the fp32 rule per pixel"""
    rng = np.random.default_rng(seed)
    probes = []
    for R in EDGE_RANGES + NO_EDGE_RANGES:
        big = not math.isfinite(R) or R > 1e18
        if R in NO_EDGE_RANGES or (isinstance(R, float) and math.isnan(R)):
            Lpos = np.array([0.5, -0.25, 0.125], F32)
            dist = np.concatenate([[0.0], 10.0 ** rng.uniform(-3, 2, 63)])
            P = (Lpos[None].astype(np.float64) - dist[:, None] * octant_dirs(64, rng)).astype(F32)
            P[0] = Lpos
            groups = [(P, Lpos + np.array([0, 3, -4], F32))]
        else:
            Lpos = (np.array([0.75, -0.5, 0.25]) * (R if not big else 1.0)).astype(F32)
            dirs = octant_dirs(8 if big else 16, rng)
            if big:      # the camera half way to the pixels of one direction: V stays finite next to an overflowing d2
                groups = []
                for u in dirs:
                    P = edge_search(Lpos, R, u[None])
                    groups.append((P, (Lpos.astype(np.float64) - 0.5 * SQRT_MAX * u).astype(F32)))
            else:
                groups = [(edge_search(Lpos, R, dirs), Lpos)]
        bright = 1e30 if big else 1.0
        for gi, (P, cam) in enumerate(groups):
            N = _facing(P, Lpos)
            planes, idx = frame(P, N, 0.5)
            Pf = planes[0][..., :3].reshape(-1, 3)
            light = dict(pos=Lpos, range=R, brightness=bright)
            for caster in (False, True):
                pf, pv = scene(cam, points=[] if caster else [light], pcasters=[light] if caster else [])
                probes.append(dict(name=f"range {R!r} {'caster' if caster else 'light'} group {gi}", planes=planes, pf=pf, pv=pv,
                                   range=R, lit=lr.in_range(Pf, Lpos, R).reshape(planes[0].shape[:2]),
                                   at_light=(lr.light_d2(Pf, Lpos) == 0).reshape(planes[0].shape[:2]),
                                   d=np.sqrt(lr.light_d2(Pf, Lpos).astype(np.float64)).reshape(planes[0].shape[:2])))
    return probes


# ---- distances ---------------------------------------------------------------------------------------------------------
NEAR_DISTANCES = [0.0, 1e-3, 1e-8, 1e-12, 1e-16, 1e-20, 5e-22]     # 1e-20 and 5e-22: the fp32 d2 is denormal
FAR_DISTANCES = [1e18, 3e18, 1e19, 1.5e19, 1.8e19, 2e19]


def distance_probes(seed=2):
    """a point light (range +Inf) and, separately, a spot (cone 1.5 rad around -Y) at the origin, pixels at NEAR_DISTANCES in
    every octant; then a frame lit by point lights and spots FAR_DISTANCES away"""
    rng = np.random.default_rng(seed)
    dirs = octant_dirs(16, rng)
    dirs[:, 1] = -np.abs(dirs[:, 1])                  # below the spot
    P, dist = [], []
    for d in NEAR_DISTANCES:
        for u in dirs:
            P.append(u * d); dist.append(d)
    P = np.array(P).astype(F32)
    N = _facing(P, np.zeros(3))
    planes, idx = frame(P, N, 0.5)
    cam = (0.0, 3.0, -4.0)
    Pf = planes[0][..., :3].reshape(-1, 3)
    d2 = lr.light_d2(Pf, np.zeros(3, F32)).reshape(planes[0].shape[:2])
    out = []
    for kind in ("point", "spot"):
        if kind == "point":
            pf, pv = scene(cam, points=[dict(pos=(0, 0, 0), range=math.inf, brightness=1.0)])
        else:
            pf, pv = scene(cam, spots=[dict(pos=(0, 0, 0), dir=(0, -2, 0), inner=0.0, outer=1.5, brightness=1.0)])
        out.append(dict(name=f"near {kind}", planes=planes, pf=pf, pv=pv, d2=d2,
                        dist=np.asarray(dist)[idx].reshape(planes[0].shape[:2])))
    # far lights: pixels near the origin, lights 1e18..2e19 away (d2 overflows from about 1.8e19 on)
    Pn = rng.uniform(-2, 2, (256, 3)).astype(F32)
    Nn = fd._unit(rng.normal(size=(256, 3))).astype(F32)
    planes, _ = frame(Pn, Nn, 0.5)
    pts, sps = [], []
    for i, d in enumerate(FAR_DISTANCES):
        u = dirs[i]
        pts.append(dict(pos=(u * d).astype(F32), range=math.inf, brightness=1e30))
        pts.append(dict(pos=(u * d).astype(F32), range=FLT_MAX, brightness=1e30))
        sps.append(dict(pos=(u * d).astype(F32), dir=-u * 3.0, inner=0.0, outer=0.5, brightness=1e30))
    pf, pv = scene(cam, points=pts, spots=sps)
    out.append(dict(name="far lights", planes=planes, pf=pf, pv=pv, d2=None, dist=None))
    return out


# ---- spot cones --------------------------------------------------------------------------------------------------------
CONES = [(0.0, 0.05), (0.0, 0.1), (0.0, 0.5), (0.0, 1.5),                  # inner = 0
         (0.4, 0.4 + 1e-6), (0.4, 0.401), (0.4, 0.7),                       # ramps 1e-6, 1e-3, 0.3 wide
         (0.3, 0.3), (0.0, 0.0),                                            # hard edges: inner == outer
         (0.6, 0.2),                                                        # inner > outer
         (0.2, float(F32(math.pi))), (0.0, 4.0)]                            # outer >= pi


def _spot_pixels(Lpos, u, inner, outer, rng, axis_aligned):
    """pixels around a spot at Lpos pointing along unit u: on the axis, at theta 1e-5..1e-2, a few ulp of theta around inner and
    outer, uniform over the cone and behind the light; distances 0.5..5"""
    p = fd._unit(np.cross(u, rng.normal(size=3)))
    q = np.cross(u, p)
    th = [0.0] * (32 if not axis_aligned else 8)
    for t in (1e-5, 1e-4, 1e-3, 1e-2):
        th += [t] * 8
    for e in (inner, outer):
        th += list(e + np.arange(-4, 5) * 2.0 ** -24 * max(e, 2 ** -10) * 4)
        th += list(e + np.linspace(-3e-3, 3e-3, 13))
    th += list(rng.uniform(0, min(outer + 0.2, math.pi), 48))
    th += list(rng.uniform(math.pi / 2, math.pi, 16)) + [math.pi]
    th = np.clip(np.array(th), 0.0, math.pi)
    phi = rng.uniform(0, 2 * math.pi, len(th))
    dist = rng.uniform(0.5, 5.0, len(th))
    if axis_aligned:
        dist[:8] = [0.5, 1.0, 2.0, 3.0, 4.0, 0.75, 1.5, 2.5]       # exactly on the axis: cosine exactly 1
    d = (np.cos(th)[:, None] * u + np.sin(th)[:, None] * (np.cos(phi)[:, None] * p + np.sin(phi)[:, None] * q))
    return (np.asarray(Lpos, np.float64)[None] + dist[:, None] * d).astype(F32)


def spot_probes(seed=3):
    """per cone, an axis-aligned and an oblique spot (direction not unit length), as a spot light and as a spot caster;
    each with its companion point-light frame. meta: the float64 intensity interval, theta and the oracle's fp32 cosine"""
    rng = np.random.default_rng(seed)
    out = []
    for ci, (inner, outer) in enumerate(CONES):
        for axis_aligned in (True, False):
            if axis_aligned:
                Lpos = np.array([1.0, 4.0, -2.0], F32)
                sdir = np.array([0.0, -2.0, 0.0], F32)
            else:
                Lpos = rng.uniform(-3, 3, 3).astype(F32)
                sdir = (fd._unit(rng.normal(size=3)) * rng.uniform(0.3, 3.0)).astype(F32)
            u = sdir.astype(np.float64) / np.linalg.norm(sdir.astype(np.float64))
            P = _spot_pixels(Lpos, u, inner, outer, rng, axis_aligned)
            N = _facing(P, Lpos)
            planes, _ = frame(P, N, 0.5)
            Pf = planes[0][..., :3].reshape(-1, 3)
            lo, hi, th = lr.spot_interval(Pf, Lpos, sdir, inner, outer)
            sh = planes[0].shape[:2]
            cam = (Lpos.astype(np.float64) + np.array([0.3, 1.7, -0.9])).astype(F32)
            spot = dict(pos=Lpos, dir=sdir, inner=inner, outer=outer)
            pf_pt, pv_pt = scene(cam, points=[dict(pos=Lpos, range=math.inf)])
            for caster in (False, True):
                pf, pv = scene(cam, spots=[] if caster else [spot], scasters=[spot] if caster else [])
                out.append(dict(name=f"cone {inner}-{outer} {'axis' if axis_aligned else 'oblique'} {'caster' if caster else 'light'}",
                                planes=planes, pf=pf, pv=pv, point=(pf_pt, pv_pt), lo=lo.reshape(sh), hi=hi.reshape(sh),
                                theta=th.reshape(sh), cos32=lr.oracle_spot_cos(Pf, Lpos, sdir).reshape(sh),
                                at_light=(lr.light_d2(Pf, Lpos) == 0).reshape(sh), inner=inner, outer=outer))
    return out


# ---- directional ----------------------------------------------------------------------------------------------------------
def directional_probe(seed=4):
    """light along +X (direction -X): normals (delta, 1, 0) * len with N.L = delta from exactly 0 to a denormal and a few ulp
    either side; pixels whose V is parallel (V = Wi) and antiparallel (V = -Wi: 2 + 2c = 0) to the light; and a second frame
    with a zero light direction (Wi = 0/0: every use of it is saturated, so the light adds 0)"""
    rng = np.random.default_rng(seed)
    cam = np.array([2.0, 1.0, -3.0], F32)
    deltas = np.array([0.0, -0.0, DENORM_MIN, -DENORM_MIN, 2.0 ** -126, -2.0 ** -126, 2.0 ** -30, -2.0 ** -30, 2.0 ** -24,
                       -2.0 ** -24, 1e-7, -1e-7, 1e-3, -1e-3, 0.3, -0.3])
    lens = np.array([1.0, 0.5, 2.0, 1.3])
    N = np.array([[d, 1.0, 0.0] for d in deltas for _ in lens]) * np.tile(lens, len(deltas))[:, None]
    P = rng.uniform(-2, 2, (len(N), 3))
    # V parallel / antiparallel to Wi = +X: the pixel on the camera's x line
    par = np.array([[float(cam[0]) - t, cam[1], cam[2]] for t in (0.5, 1.0, 2.0, 4.0)] +
                   [[float(cam[0]) + t, cam[1], cam[2]] for t in (0.5, 1.0, 2.0, 4.0)])
    Npar = np.array([[0.0, 1.0, 0.0], [0.6, 0.8, 0.0], [-0.6, 0.8, 0.0], [1.0, 0.0, 0.0]] * 2)
    P = np.concatenate([P, par]).astype(F32)
    N = np.concatenate([N, Npar]).astype(F32)
    rough = np.resize(np.array([0.5, 0.2, 0.9, 0.05], F32), len(P))
    planes, _ = frame(P, N, rough)
    out = []
    for name, d in (("directional", (-1.0, 0.0, 0.0)), ("directional zero", (0.0, 0.0, 0.0))):
        pf, pv = scene(cam, directional=dict(dir=d, brightness=2.0))
        out.append(dict(name=name, planes=planes, pf=pf, pv=pv))
    return out


# ---- highlights -------------------------------------------------------------------------------------------------------------
ESCAPE_ROUGHNESS = [0.0, 0.01, 0.02, 0.024, 0.026, 0.0273, 0.0274, 0.0275, 0.03]


def escape_roughness():
    """ESCAPE_ROUGHNESS and every fp32 roughness between 0.0272 and 0.0276 where the fp32 t (= a2 at N.H = 1) changes, with
    its neighbours: the D = 1 escape flips between t = 9 * 2^-24 (PI t^2 = 9.0e-13) and 10 * 2^-24 (1.12e-12), so PI t^2 is
    never nearer to 1e-12 than that at N.H = 1"""
    r = np.arange(np.float32(0.0272), np.float32(0.0276), np.float32(2e-7), dtype=F32)
    t = lr.ggx_t(np.ones_like(r), r)
    ch = np.nonzero(t[1:] != t[:-1])[0]
    pick = np.unique(np.concatenate([ch, ch + 1]))
    return np.unique(np.concatenate([np.array(ESCAPE_ROUGHNESS, F32), r[pick]]))


def mirror_probes():
    """N = H bit for bit (test_forward_mirror_kat's construction): P = 0, N along an axis, camera and light at mirror
    positions whose normalised components are bit-identical up to sign (they differ by a power of 2), so N.H = 1 exactly and
    t = 1 * (a2 - 1) + 1. meta: the fp32 escape decision per pixel, the float64 light term with D = 1 and with D = a2 / (PI t^2)"""
    rs = escape_roughness()
    out = []
    for (u, v), axis in (((1.0, 1.0), 1), ((1.0, 3.0), 1), ((3.0, 1.0), 2), ((1.0, 2.0), 0)):
        e = np.eye(3)[axis]
        side = np.eye(3)[(axis + 1) % 3]
        cam = (-4.0 * u * side + 4.0 * v * e).astype(F32)
        lpos = (2.0 * u * side + 2.0 * v * e).astype(F32)
        n = len(rs)
        planes, idx = frame(np.zeros((n, 3)), np.repeat(e[None], n, 0), rs, albedo=(0.5, 0.25, 0.75))
        r = planes[1][..., 3].astype(np.float64)
        pf, pv = scene(cam, points=[dict(pos=lpos, range=100.0, brightness=50.0)])
        c = v / math.hypot(u, v)                        # N.V = N.L = H.V (float64)
        col = np.array([1.0, 0.5, 0.25])
        alb = np.array([0.5, 0.25, 0.75])
        F = 0.04 + 0.96 * (1.0 - c) ** 5
        k = (r + 1.0) ** 2 / 8.0
        G = (c / (c * (1 - k) + k + 1e-4)) ** 2
        a = (planes[1][..., 3] * planes[1][..., 3])
        a2 = (a * a).astype(np.float64)
        t = lr.ggx_t(np.ones_like(a), planes[1][..., 3]).astype(np.float64)     # (a2 - 1) + 1: a multiple of 2^-24
        D = np.where(t > 0, a2 / (math.pi * np.where(t > 0, t, 1.0) ** 2), np.inf)
        att = 50.0 / (4.0 * (u * u + v * v))
        def term(Dv):
            return (((1.0 - F) * alb / math.pi)[None, None] + (F * Dv * G / max(4 * c * c, 1e-4))[..., None]) * col * att * c
        out.append(dict(name=f"mirror {u},{v} axis {axis}", planes=planes, pf=pf, pv=pv,
                        escape=lr.d_escape(np.ones_like(r, F32), planes[1][..., 3]), want_escape=term(np.ones_like(r)),
                        want_ggx=term(D)))
    return out


def t_sweep_probe(seed=5):
    """one directional light, V fixed: normals at the angle from H where the float64 t = nh^2 (a2 - 1) + 1 is 0.02 * (1 + k 1e-3),
    k in -16..15, at roughness 0.03..0.2; in each warp's 32 pixels exactly one has t below T_EXACT, the others above"""
    rng = np.random.default_rng(seed)
    cam = np.array([0.0, 3.0, -4.0])
    wi = fd._unit(np.array([0.4, 1.0, 0.3]))
    P = rng.uniform(-0.5, 0.5, (512, 3))
    rough = np.repeat(rng.uniform(0.03, 0.2, 16), 32)
    k = np.tile(np.concatenate([[-1], np.arange(1, 32)]), 16).astype(np.float64)
    t = 0.02 * (1.0 + k * 1e-3)
    V = fd._unit(cam[None] - P)
    H = fd._unit(V + wi[None])
    a2 = rough.astype(np.float64) ** 4
    nh = np.sqrt((1.0 - t) / (1.0 - a2))
    ang = np.arccos(np.clip(nh, -1, 1))
    ax = fd._perp(H, rng)
    N = np.cos(ang)[:, None] * H + np.sin(ang)[:, None] * ax
    planes, _ = frame(P.astype(F32), N.astype(F32), rough.astype(F32))
    pf, pv = scene(cam.astype(F32), directional=dict(dir=-wi, brightness=3.0))
    return dict(name="t sweep", planes=planes, pf=pf, pv=pv)


def view_probe(seed=6):
    """N.V across NV_EXACT from both sides and exactly 0, the camera at the pixel (NaN on both sides), raw normal lengths
    0.5..2 with |N| cos(N, L) around 1 (the saturate of Lighting.hlsl:316); one point light and the directional light"""
    rng = np.random.default_rng(seed)
    cam = np.array([1.0, 2.0, -3.0], F32)
    lpos = np.array([-2.0, 5.0, 1.0], F32)
    P = rng.uniform(-2, 2, (192, 3)).astype(F32)
    V = fd._unit(cam.astype(np.float64)[None] - P.astype(np.float64))
    s = np.concatenate([1e-3 * (1 + np.arange(-8, 8) * 1e-4), -1e-3 * (1 + np.arange(-8, 8) * 1e-4),
                        rng.choice([0.0, 5e-4, -5e-4, 2e-3, -2e-3, 1e-6], 32)])
    s = np.resize(s, 128)
    perp = fd._perp(V[:128], rng)
    N1 = s[:, None] * V[:128] + np.sqrt(1 - s * s)[:, None] * perp
    # N.V exactly 0: cam - P along x only, N in the y-z plane
    P2 = np.stack([cam[0] - rng.uniform(0.5, 3, 32), np.full(32, cam[1]), np.full(32, cam[2])], 1).astype(F32)
    N2 = np.stack([np.zeros(32), rng.normal(size=32), rng.normal(size=32)], 1)
    # the camera at the pixel
    P3 = np.repeat(cam[None], 8, 0)
    N3 = fd._unit(rng.normal(size=(8, 3)))
    # |N| cos(N, L) around 1: N = len * (cos a Wi + sin a perp) with len cos a = 1 +- small
    P4 = P[128:152]
    wi = fd._unit(lpos.astype(np.float64)[None] - P4.astype(np.float64))
    ln = rng.uniform(0.5, 2.0, 24)
    cs = np.clip((1.0 + np.resize(np.array([-1e-6, 0.0, 1e-6, -1e-3, 1e-3, 2e-7]), 24)) / ln, -1, 1)
    N4 = ln[:, None] * (cs[:, None] * wi + np.sqrt(1 - cs * cs)[:, None] * fd._perp(wi, rng))
    lens = np.concatenate([rng.uniform(0.5, 2.0, 128), np.ones(32), np.ones(8), np.ones(24)])
    Pall = np.concatenate([P[:128], P2, P3, P4]).astype(F32)
    Nall = (np.concatenate([N1, fd._unit(N2), N3, N4 / ln[:, None]]) * lens[:, None])
    Nall[-24:] = N4
    rough = np.resize(np.array([0.5, 0.05, 0.9, 0.2, 0.03], F32), len(Pall))
    planes, _ = frame(Pall, Nall.astype(F32), rough, metal=0.5)
    pf, pv = scene(cam, points=[dict(pos=lpos, range=50.0, brightness=20.0)],
                   directional=dict(dir=(0.3, -1.0, 0.2), brightness=1.5))
    at_cam = (planes[0][..., :3] == cam).all(-1)
    return dict(name="view", planes=planes, pf=pf, pv=pv, at_cam=at_cam)


# ---- mixed frames -----------------------------------------------------------------------------------------------------------
CAM = (0.0, 5.0, -17.0)


def _rand_lights(rng, n_pt, n_sp, bright):
    pts = [dict(pos=rng.uniform(-25, 25, 3) * (1, 0.4, 1) + (0, 8, 0), range=float(rng.choice([14.0, 50.0, 1000.0, math.inf])),
                brightness=float(bright(rng)), color=rng.choice([0.0, 0.3, 1.0], 3)) for _ in range(n_pt)]
    sps = []
    for _ in range(n_sp):
        inner = float(rng.choice([0.0, 0.3, 0.6]))
        sps.append(dict(pos=rng.uniform(-25, 25, 3) * (1, 0.4, 1) + (0, 15, 0), dir=(rng.normal(size=3) - (0, 3, 0)) * rng.uniform(0.3, 3),
                        inner=inner, outer=inner + float(rng.choice([0.1, 0.3, 0.8])), brightness=float(bright(rng)),
                        color=rng.choice([0.0, 0.5, 1.0], 3)))
    return pts, sps


MIXED = ["none", "one of each", "maximum", "bright", "negative and zero", "rotated"]


def mixed_frame(kind, seed):
    """forward_domain.adversarial_gbuffer (random environment) under a light set: 'none'; 'one of each' (point light, point caster,
    spot light, spot caster, directional); 'maximum' (100 + 5 point, 20 + 5 spot and the directional light); 'bright' (point and
    directional brightness up to 1e4, spot radiance kept below 1 at the pixels: its ramp is checked by the intensity bound);
    'negative and zero' brightness; 'rotated' (an HDRI offset: the ROT instantiation). Colours with a zero channel throughout."""
    rng = np.random.default_rng(seed)
    w, h = 515, 21
    planes, _ = fd.adversarial_gbuffer(w, h, seed, CAM, emissive=(kind == "one of each"))
    env = fd.make_env(8, 16, (20, 48), seed=seed)
    dirl = dict(dir=(0.3, -1.0, 0.4), brightness=1.5, color=(1.0, 0.0, 0.7))
    if kind == "none":
        pts, sps, pcs, scs, d = [], [], [], [], None
    elif kind in ("one of each", "rotated"):
        pts, sps = _rand_lights(rng, 2, 2, lambda g: g.uniform(50, 500))
        pcs, scs, d = pts[1:], sps[1:], dirl
        pts, sps = pts[:1], sps[:1]
    elif kind == "maximum":
        pts, sps = _rand_lights(rng, 105, 25, lambda g: g.uniform(10, 800))
        pcs, scs, d = pts[100:], sps[20:], dirl
        pts, sps = pts[:100], sps[:20]
    elif kind == "bright":
        pts, sps = _rand_lights(rng, 8, 3, lambda g: g.choice([1e3, 1e4]))
        for s in sps:
            s["brightness"] = 0.5
        pcs, scs, d = [], [], dict(dirl, brightness=1e4)
    else:
        pts, sps = _rand_lights(rng, 8, 4, lambda g: g.choice([0.0, -0.0, -300.0, 400.0]))
        pcs, scs, d = pts[6:], sps[3:], dict(dirl, brightness=-2.0)
        pts, sps = pts[:6], sps[:3]
    pf, pv = scene(CAM, points=pts, spots=sps, pcasters=pcs, scasters=scs, directional=d,
                   offset=0.7 if kind == "rotated" else 0.0, max_lod=env["spec_mips"])
    return dict(name=f"mixed {kind}", planes=planes, pf=pf, pv=pv, env=env)


def copy_pf(pf):
    return type(pf).from_buffer_copy(pf)


def with_dark_caster(pf):
    """the frame with a point caster of brightness 0 appended when it has none, so that the shadowed pass with point shadow cubes
    runs its SHADOWED instantiation (a dark caster adds exactly 0)"""
    q = copy_pf(pf)
    L = q.Lights
    if L.numPointCasters == 0:
        c = L.point_casters[0]
        C.memset(C.byref(c), 0, C.sizeof(c))
        _set3(c.position, (1e3, 1e3, 1e3))
        c.range, c.brightness = 1.0, 0.0
        L.numPointCasters = 1
    return q
