"""Seeded K1 inputs over the whole domain the kernel accepts (test input generation, no GPU):
  * sampler probes: G-buffers whose output is ONE environment sample (specular cube, diffuse cube, one LUT channel), with
    the float64 value it must have and a per-pixel bound derived from how far the kernel's lookup coordinate can be off;
  * adversarial G-buffers for whole-pixel parity: normals of length 0.5..2 over the whole sphere, back-facing and grazing
    pixels, roughness down to 0 (the TINY light loop) and exactly 1 (the mip clamp), pixels without a surface.
"""
import math

import numpy as np

import sampling_ref as sr

U24 = 2.0 ** -24
PROBE_W = 256


def _unit(v):
    v = np.asarray(v, np.float64)
    return v / np.linalg.norm(v, axis=-1, keepdims=True)


def _perp(v, rng):
    """unit vectors perpendicular to the rows of v"""
    return _unit(np.cross(v, rng.normal(size=v.shape)))


def make_env(diff_res, spec_res, lut_wh, seed, diff=None, spec=None, lut=None):
    """environment maps with FULL mip chains (the diffuse cube too: K1 must read its mip 0); None -> uniform [0,1] texels"""
    w, h = lut_wh
    return dict(diff=sr.random_cube(diff_res, seed) if diff is None else diff, diff_res=diff_res, diff_mips=sr.mip_count(diff_res),
                spec=sr.random_cube(spec_res, seed + 1) if spec is None else spec, spec_res=spec_res,
                spec_mips=sr.mip_count(spec_res), lut=sr.random_lut(w, h, seed + 2) if lut is None else lut)


def constants(cam, max_lod, offset=0.0, lights=None, diffuse_only=False):
    """PerFrameData / PerViewLightingData: no lights unless `lights` = (pf from synth.scene_constants) is given"""
    import ctypes as C
    import vqengine_b200 as vq
    if lights is None:
        pf = vq.PerFrameData()
        C.memset(C.byref(pf), 0, C.sizeof(pf))
    else:
        pf = lights
    pf.fHDRIOffsetInRadians = offset
    pv = vq.PerViewLightingData()
    C.memset(C.byref(pv), 0, C.sizeof(pv))
    pv.CameraPosition.x, pv.CameraPosition.y, pv.CameraPosition.z = (float(c) for c in cam)
    pv.MaxEnvMapLODLevels = float(max_lod)
    pv.EnvironmentMapDiffuseOnlyIllumination = int(diffuse_only)
    return pf, pv


def _frame(cols):
    """per-pixel columns (n, 4) x planes -> [H, PROBE_W, 4] planes; the tail of the last row repeats the first pixels"""
    n = cols[0].shape[0]
    h = -(-n // PROBE_W)
    idx = np.arange(h * PROBE_W) % n
    return [np.ascontiguousarray(c[idx].reshape(h, PROBE_W, 4).astype(np.float32)) for c in cols], idx


def _views(n, rng, cam):
    """view directions uniform over the sphere, positions at distance 0.5..20 from the camera (float32)"""
    V = sr.uniform_directions(n, rng).astype(np.float64)
    P = (np.asarray(cam)[None] - V * rng.uniform(0.5, 20.0, (n, 1))).astype(np.float32)
    return P


def _v64(P, cam):
    return _unit(np.asarray(cam, np.float64)[None] - P.astype(np.float64))


def _normals_for_nv(V, rng, lengths):
    """normals whose N.V covers [−1, 1], with exact-zero (perpendicular), near-zero, and exactly-one groups"""
    n = len(V)
    c = rng.uniform(-1, 1, n)
    k = np.arange(n) % 16
    c[k == 0] = 0.0
    c[k == 1] = rng.choice([1e-6, -1e-6, 1e-4, 5e-4, 1e-3, 2e-3, -1e-3], size=(k == 1).sum())
    c[k == 2] = 1.0
    c[k == 3] = rng.uniform(0.98, 1.0, (k == 3).sum())
    t = _perp(V, rng)
    nh = c[:, None] * V + np.sqrt(np.maximum(0.0, 1.0 - c * c))[:, None] * t
    return nh * lengths[:, None]


def _roughness_for_mips(n, rng, max_lod, mips):
    """roughness values that land on every mip int(r * int(max_lod)) can reach, the exact mip boundaries, 0 and 1"""
    L = int(max_lod)
    vals = [0.0, 1.0]
    if L > 0:
        vals += [(m + 0.5) / L for m in range(L)] + [m / L for m in range(1, L)]
    vals = np.array([v for v in vals if 0.0 <= v <= 1.0])
    r = rng.uniform(0, 1, n)
    k = np.arange(n) % 3
    r[k == 0] = vals[rng.integers(0, len(vals), (k == 0).sum())]
    return r.astype(np.float32)


def spec_mip(r, max_lod, mips):
    """the specular mip rule: int(roughness * int(MaxEnvMapLODLevels)) in fp32, clamped to the chain"""
    return np.clip(np.trunc(np.float32(r) * np.float32(int(max_lod))).astype(np.int64), 0, mips - 1)


def _cube_tol(N, rel_dir, span):
    """a lookup direction off by `rel_dir` (relative) moves each face coordinate by at most 2*sqrt(3)*rel_dir (the major
    component is at least |d|/sqrt(3)), i.e. each texel coordinate by sqrt(3)*N*rel_dir; the seamless bilinear sample moves
    by at most the sum of the two times the largest texel difference; the lerps add a few ulp"""
    return 2 * math.sqrt(3) * N * rel_dir * span + 16 * U24


# ---- probes ------------------------------------------------------------------------------------------------------
def specular_probe(env, max_lod, n_uniform, seed, offset=0.0):
    """metalness 1, albedo 1, ao 0, no lights, LUT = (1, 0): output rgb = specular sample at reflect(-V, N) (raw N) and mip
    int(roughness * MAX_LOD), times Ks = F0 + ..., which is within 2 ulp of 1"""
    rng = np.random.default_rng(seed)
    cam = (0.25, -0.5, 1.5)
    res, mips = env["spec_res"], env["spec_mips"]
    special = sr.special_directions(res, rng)
    n = n_uniform + len(special)
    P = _views(n, rng, cam)
    V = _v64(P, cam)
    target = np.concatenate([sr.uniform_directions(n_uniform, rng), special]).astype(np.float64)
    s = np.where(np.arange(n) < n_uniform // 2, rng.uniform(0.5, 2.0, n), 1.0)
    h = V + target
    bad = np.linalg.norm(h, axis=1) < 1e-3
    h[bad] = _perp(V[bad], rng)
    N = _unit(h) * s[:, None]
    m = n_uniform // 4                                   # a quarter of the pixels: N.V over [-1, 1] incl. 0, ~0 and 1
    N[:m] = _normals_for_nv(V[:m], rng, rng.uniform(0.5, 2.0, m))
    r = _roughness_for_mips(n, rng, max_lod, mips)
    N = N.astype(np.float32)
    pos = np.concatenate([P, np.zeros((n, 1), np.float32)], 1)
    nrm = np.concatenate([N, r[:, None]], 1)
    alb = np.ones((n, 4), np.float32)
    planes, idx = _frame([pos, nrm, alb])
    V = _v64(planes[0][..., :3].reshape(-1, 3), cam)
    Nf = planes[1][..., :3].reshape(-1, 3).astype(np.float64)
    rf = planes[1][..., 3].ravel()
    R = -V + 2.0 * (Nf * V).sum(1, keepdims=True) * Nf
    Rr = sr.rotate_hdri(R, offset) if offset else R
    mip = spec_mip(rf, max_lod, mips)
    want = sr.sample_cube(env["spec"], res, mips, Rr, mip)[:, :3]
    # R = -V + 2 (N.V) N in fp32 from V (rsqrt), N = normalize(N) * |N|: component errors <= 2^-19 * (1 + 2|N|^2)
    rel = 2.0 ** -19 * (1.0 + 2.0 * (Nf * Nf).sum(1)) / np.linalg.norm(R, axis=1)
    span = float(env["spec"].max() - env["spec"].min())
    tol = _cube_tol((res >> mip).astype(np.float64), rel, span) + 4 * U24 * np.abs(want).max(1)
    pf, pv = constants(cam, max_lod, offset)
    return dict(planes=planes, pf=pf, pv=pv, want=want.reshape(planes[0].shape[:2] + (3,)),
                tol=tol.reshape(planes[0].shape[:2]))


def diffuse_probe(env, n_uniform, seed, offset=0.0, max_lod=5):
    """specular cube = 0, LUT = 0, metalness 0, albedo 1, roughness 1, ao 0, no lights: output rgb =
    (1 - 0.04f) * diffuse sample at N (raw N, rotated by the HDRI offset), mip 0 of the diffuse cube"""
    rng = np.random.default_rng(seed)
    cam = (-1.0, 0.75, -0.5)
    res = env["diff_res"]
    special = sr.special_directions(res, rng)
    n = n_uniform + len(special)
    P = _views(n, rng, cam)
    d = np.concatenate([sr.uniform_directions(n_uniform, rng), special]).astype(np.float64)
    s = np.where(np.arange(n) < n_uniform // 2, rng.uniform(0.5, 2.0, n), np.where(np.arange(n) % 2 == 0, 1.0, 2.0))
    N = (d * s[:, None]).astype(np.float32)
    pos = np.concatenate([P, np.zeros((n, 1), np.float32)], 1)
    nrm = np.concatenate([N, np.ones((n, 1), np.float32)], 1)
    alb = np.concatenate([np.ones((n, 3), np.float32), np.zeros((n, 1), np.float32)], 1)
    planes, _ = _frame([pos, nrm, alb])
    Nf = planes[1][..., :3].reshape(-1, 3).astype(np.float64)
    Nr = sr.rotate_hdri(Nf, offset) if offset else Nf
    kd = float(np.float32(1.0) - np.float32(0.04))
    want = kd * sr.sample_cube(env["diff"], res, env["diff_mips"], Nr, 0)[:, :3]
    span = float(env["diff"].max() - env["diff"].min())
    tol = _cube_tol(float(res), 2.0 ** -19, span) + 4 * U24 * np.abs(want).max(1)
    pf, pv = constants(cam, max_lod, offset)
    return dict(planes=planes, pf=pf, pv=pv, want=want.reshape(planes[0].shape[:2] + (3,)),
                tol=tol.reshape(planes[0].shape[:2]))


def lut_probe(env, channel, n, seed, max_lod=5):
    """specular cube = 1, metalness 1, albedo 1, ao 0, no lights; the other LUT channel = 0: output rgb = LUT[channel] at
    (saturate(dot(N, V)) of the raw N, roughness) (channel 0 times Ks, within 2 ulp of 1)"""
    rng = np.random.default_rng(seed)
    cam = (0.5, 1.0, -2.0)
    lut = env["lut"]
    H, W = lut.shape[:2]
    P = _views(n, rng, cam)
    V = _v64(P, cam)
    N = _normals_for_nv(V, rng, np.where(np.arange(n) % 2 == 0, 1.0, rng.uniform(0.5, 2.0, n))).astype(np.float32)
    r = rng.uniform(0, 1, n)
    k = np.arange(n) % 5
    edges = np.concatenate([[0.0, 1.0], (np.arange(H) + 0.5) / H, np.arange(H + 1) / H])
    r[k == 0] = edges[rng.integers(0, len(edges), (k == 0).sum())]
    r = r.astype(np.float32)
    pos = np.concatenate([P, np.zeros((n, 1), np.float32)], 1)
    nrm = np.concatenate([N, r[:, None]], 1)
    alb = np.ones((n, 4), np.float32)
    planes, _ = _frame([pos, nrm, alb])
    V = _v64(planes[0][..., :3].reshape(-1, 3), cam)
    Nf = planes[1][..., :3].reshape(-1, 3).astype(np.float64)
    u = np.clip((Nf * V).sum(1), 0.0, 1.0)
    want = sr.sample_lut(lut, u, planes[1][..., 3].ravel())[:, channel]
    # u = saturate(|N| * dot(normalize(N), V)) with approximate rsqrt: off by <= 2^-20 * max(1, |N|); x = u*W - 0.5 and
    # y = v*H - 0.5 round (or fuse) differently: W * 2^-23, H * 2^-23
    du = 2.0 ** -20 * np.maximum(1.0, np.linalg.norm(Nf, axis=1))
    span = float(lut[..., channel].max() - lut[..., channel].min())
    tol = (W * (du + 2.0 ** -23) + H * 2.0 ** -23) * span + 16 * U24
    pf, pv = constants(cam, max_lod)
    return dict(planes=planes, pf=pf, pv=pv, want=np.repeat(want[:, None], 3, 1).reshape(planes[0].shape[:2] + (3,)),
                tol=tol.reshape(planes[0].shape[:2]))


def probe_env(kind, base, channel=0):
    """the probe's environment: `base` (make_env) with the maps the probe identity needs replaced by constants"""
    e = dict(base)
    if kind == "spec":
        e["lut"] = np.stack([np.ones_like(base["lut"][..., 0]), np.zeros_like(base["lut"][..., 0])], -1)
    elif kind == "diff":
        e["spec"] = np.zeros_like(base["spec"])
        e["lut"] = np.zeros_like(base["lut"])
    else:
        e["spec"] = np.ones_like(base["spec"])
        lut = base["lut"].copy()
        lut[..., 1 - channel] = 0.0
        e["lut"] = lut
    return e


# ---- adversarial G-buffers -------------------------------------------------------------------------------------------
ROUGH_MIX = (0.0, 1e-3, 0.0239, 0.0241, None, 1.0)      # None: U(0.04, 1)


def adversarial_gbuffer(w, h, seed, cam, emissive=False, sky_frac=0.0):
    """normals uniform over the sphere with lengths in [0.5, 2] (half the pixels back-facing), 1/16 grazing (N.V = 0) and
    1/16 nearly grazing, roughness mixed from ROUGH_MIX, metalness in {0, 1, U(0,1)}; every 4th row is rough (U(0.04, 1))
    except ONE pixel of roughness 1e-3, so that one warp of each tile runs the TINY light loop for a single pixel.
    sky_frac: that fraction of pixels is an all-zero texel (no surface, as the engine clears the G-buffer).
    Returns planes and the sky mask."""
    rng = np.random.default_rng(seed)
    n = w * h
    P = np.stack([rng.uniform(-20, 20, n), rng.uniform(-5, 5, n), rng.uniform(-20, 20, n)], 1).astype(np.float32)
    V = _v64(P, cam)
    lengths = rng.uniform(0.5, 2.0, n)
    N = sr.uniform_directions(n, rng).astype(np.float64) * lengths[:, None]
    k = np.arange(n) % 16
    g = (k == 5) | (k == 11)
    N[g] = _normals_for_nv(V[g], rng, lengths[g])
    pick = rng.integers(0, len(ROUGH_MIX), n)
    r = np.array([ROUGH_MIX[i] if ROUGH_MIX[i] is not None else rng.uniform(0.04, 1.0) for i in pick], np.float32)
    r2 = r.reshape(h, w)
    r2[3::4] = rng.uniform(0.04, 1.0, r2[3::4].shape)
    r2[3::4, 37::256] = 1e-3
    sel = rng.integers(0, 3, n)
    metal = np.where(sel == 0, 0.0, np.where(sel == 1, 1.0, rng.uniform(0, 1, n)))
    pos = np.concatenate([P, rng.uniform(0, 0.3, (n, 1))], 1)
    nrm = np.concatenate([N, r.reshape(-1, 1)], 1)
    alb = np.concatenate([rng.uniform(0.02, 1.0, (n, 3)), metal[:, None]], 1)
    planes = [pos, nrm, alb]
    if emissive:
        em = np.concatenate([rng.uniform(0, 1, (n, 3)), np.where(rng.uniform(0, 1, n) < 0.3, rng.uniform(0, 4, n), 0.0)[:, None]], 1)
        planes.append(em)
    planes = [np.ascontiguousarray(p.reshape(h, w, 4).astype(np.float32)) for p in planes]
    sky = np.zeros((h, w), bool)
    if sky_frac:
        sky = rng.uniform(0, 1, (h, w)) < sky_frac
        for p in planes:
            p[sky] = 0.0
    return planes, sky


def lights(w, h, seed, offset):
    """4 point + 3 spot lights, a point and a spot caster (unshadowed) and the directional light of synth.scene_constants"""
    from vqengine_b200 import synth
    pf, _ = synth.scene_constants(w, h, 1, seed=seed, n_point=4, n_spot=3, directional=True, hdri_offset=offset, casters=True)
    return pf
