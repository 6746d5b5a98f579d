"""Seeded inputs of the surface producer over the whole domain its sampler and decisions see: texture shapes (1x1, strips,
non-square and odd sizes, square powers of two for the closed-form level offset), truncated chains, maximum-contrast and
random texels, uv at texel centres and boundaries of every level, WRAP seams, the edges of fp32 and int ranges, NaN and
Inf, per-quad derivatives from flat to overflowing, and the materials / interpolants / planes the decisions branch on.

PROBES: a material with roughness = metalness = 1, ambient 1, no SSAO and textureConfig = AO | ROUGHNESS | METALLIC writes
one Sample() channel into each of normal_roughness.w (roughness map .r), albedo_metalness.w (metalness map .r) and
position_ao.w (AO map .r). The three maps are the same texture with its channels rotated, so the probes read R, G and B of
one texture; on the record path they read three of the four record words byte by byte."""
import numpy as np

import vqengine_b200 as vq
from surface_ref import sample_ref
from vqengine_b200.shader_data import TEXCFG_AO, TEXCFG_ROUGHNESS, TEXCFG_METALLIC


PROBE_CFG = TEXCFG_AO | TEXCFG_ROUGHNESS | TEXCFG_METALLIC
PROBE_SLOTS = (("roughness", 0), ("metalness", 1), ("local_ao", 2))     # slot, channel rotation
# (plane, channel) of each probe's output
PROBE_OUT = {"roughness": (1, 3), "metalness": (2, 3), "local_ao": (0, 3)}

SHAPES = [(1, 1), (1, 16), (16, 1), (2, 2), (64, 4), (4, 64), (7, 3), (97, 41), (37, 19), (64, 64), (256, 256),
          (4096, 4096), (8192, 1024), (16384, 2)]


def texels(kind, w, h, rng):
    if kind == "const":
        return np.full((h, w, 4), 173, np.uint8)
    if kind == "checker":
        c = (((np.arange(w)[None, :] + np.arange(h)[:, None]) % 2) * 255).astype(np.uint8)
        return np.stack([c, 255 - c, c, 255 - c], -1)
    if kind == "ramp":
        x = (np.arange(w)[None, :] * 255 // max(w - 1, 1)) * np.ones((h, 1), np.int64)
        y = (np.arange(h)[:, None] * 255 // max(h - 1, 1)) * np.ones((1, w), np.int64)
        return np.stack([x, y, (x + y) // 2, 255 - x], -1).astype(np.uint8)
    return rng.integers(0, 256, (h, w, 4), dtype=np.uint8)


def level_counts(w, h):
    full = vq.mip_level_count(w, h)
    return sorted({full, 1, min(2, full), max(1, full - 3)})


def chain(level0, levels):
    import oracle_lib
    return oracle_lib.texture_mip_chain(level0, levels)


def probe_maps(level0, levels):
    """slot -> (packed chain, w, h, levels) of the three probe maps (channels rotated by 0, 1, 2)"""
    h, w = level0.shape[:2]
    return {slot: (chain(np.roll(level0, -r, axis=2).copy(), levels), w, h, levels) for slot, r in PROBE_SLOTS}


def _uv_bases(w, h, levels, rng, n):
    """n (u, v) quad bases aimed at the sampler's edges for a w x h texture"""
    out = []
    for l in range(levels):
        W, H = max(w >> l, 1), max(h >> l, 1)
        i, j = rng.integers(-3, W + 3), rng.integers(-3, H + 3)
        out += [((i + 0.5) / W, (j + 0.5) / H), (i / W, j / H), ((i + 1e-3) / W, (j - 1e-3) / H)]
    out += [(0.0, 0.0), (-0.0, -0.0), (1.0, 1.0), (-1.0, 2.0), (-0.25, -3.75), (5.0, -7.0)]
    for p in (23, 24, 31):                                    # |u * W| near 2^23, 2^24 and 2^31, both sides of each
        for d in (-1.0, 0.0, 1.0, 300.0):
            u = (2.0 ** p + d) / w
            out += [(u, 0.5), (-u, 0.25), (0.5, (2.0 ** p + d) / h)]
    for big in (1e9, 4e9, -1e9, 8.4e6, 3e38, -3e38):
        out += [(big, 0.3), (0.3, big)]
    out += [(float(np.float32(3.4e38)) / 1.5, 0.5)]           # u * W overflows at level 0 for W >= 2, not at level 1 of W = 2
    out += [(np.nan, 0.5), (0.5, np.nan), (np.inf, 0.5), (-np.inf, -0.5), (0.5, np.inf)]
    while len(out) < n:
        out.append(tuple(rng.uniform(-4, 4, 2)))
    return out[:n] if len(out) > n else out


def _derivs(w, h, levels, rng, n):
    """n (ddx, ddy) pairs in uv units"""
    out = [((0.0, 0.0), (0.0, 0.0))]
    for k in range(levels + 2):                               # exactly 2^k texels per pixel: integral LOD, up to and past levels-1
        out += [((2.0 ** k / w, 0.0), (0.0, 0.0)), ((0.0, 0.0), (0.0, -(2.0 ** k) / h))]
    out += [((3.0 / w, 0.0), (0.0, 1.0 / h)), ((0.5 / w, 0.0), (0.0, 6.0 / h)), ((-2.0 / w, -1.0 / h), (1.0 / w, -2.0 / h)),
            ((1e-42, 0.0), (0.0, 1e-42)), ((1e30, 0.0), (0.0, 0.0)), ((0.0, 3e38), (0.0, 0.0)), ((2.0 ** 0.5 / w, 0.0), (0.0, 0.0))]
    while len(out) < n:
        out.append(((rng.uniform(-3, 3) / w, rng.uniform(-3, 3) / h), (rng.uniform(-3, 3) / w, rng.uniform(-3, 3) / h)))
    return out


def quad_planes(bases, derivs, pw, ph):
    """raw uv planes [ph, pw] whose aligned 2x2 quads start at bases[k] and step by derivs[k] (fp32 sums). Quads cut by an odd
    edge keep their in-image pixels."""
    ru = np.zeros((ph, pw), np.float32)
    rv = np.zeros((ph, pw), np.float32)
    k = 0
    for qy in range(0, ph, 2):
        for qx in range(0, pw, 2):
            (bu, bv), ((xu, xv), (yu, yv)) = bases[k % len(bases)], derivs[(k * 7) % len(derivs)]
            k += 1
            for dy in (0, 1):
                for dx in (0, 1):
                    if qy + dy < ph and qx + dx < pw:
                        with np.errstate(all="ignore"):
                            ru[qy + dy, qx + dx] = np.float32(bu) + np.float32(dx * xu) + np.float32(dy * yu)
                            rv[qy + dy, qx + dx] = np.float32(bv) + np.float32(dx * xv) + np.float32(dy * yv)
    return ru, rv


def planes_from_uv(ru, rv, mat_index=0.0, rng=None):
    ph, pw = ru.shape
    rng = rng or np.random.default_rng(5)
    pos = np.zeros((ph, pw, 4), np.float32); nrm = np.zeros((ph, pw, 4), np.float32); tan = np.zeros((ph, pw, 4), np.float32)
    pos[..., :3] = rng.uniform(-5, 5, (ph, pw, 3))
    nrm[..., 2] = 1.0; tan[..., 0] = 1.0
    pos[..., 3], nrm[..., 3] = ru, rv
    tan[..., 3] = mat_index
    return [pos, nrm, tan]


def sampler_cases(seed=20261016):
    """(name, level0, levels, planes-size) probe cases: every shape, every level count kind, every texel kind"""
    rng = np.random.default_rng(seed)
    kinds = ("const", "checker", "random", "ramp")
    cases = []
    for si, (w, h) in enumerate(SHAPES):
        big = w * h > 1 << 20
        for li, levels in enumerate(level_counts(w, h)):
            if big and li not in (0, len(level_counts(w, h)) - 1):
                continue
            kind = kinds[(si + li) % 4]
            cases.append((f"{w}x{h}/L{levels}/{kind}", w, h, levels, kind, int(rng.integers(1 << 30))))
    return cases


def build_sampler_case(w, h, levels, kind, seed, pw=34, ph=17):
    rng = np.random.default_rng(seed)
    level0 = texels(kind, w, h, rng)
    nq = ((pw + 1) // 2) * ((ph + 1) // 2)
    ru, rv = quad_planes(_uv_bases(w, h, levels, rng, nq), _derivs(w, h, levels, rng, nq), pw, ph)
    return level0, ru, rv


def probe_material(scale=(1.0, 1.0), offset=(0.0, 0.0)):
    m = vq.MaterialData()
    m.diffuse.x = m.diffuse.y = m.diffuse.z = 0.5
    m.alpha = 1.0
    m.roughness, m.metalness = 1.0, 1.0
    m.uvScaleOffset.x, m.uvScaleOffset.y, m.uvScaleOffset.z, m.uvScaleOffset.w = scale[0], scale[1], offset[0], offset[1]
    m.textureConfig = float(PROBE_CFG)
    return m


def quad_derivs(ru, rv):
    """fine quad differences of the raw uv planes (aligned 2x2 quads, partner clamped to the image): fp32, exact inputs"""
    ph, pw = ru.shape
    xs, ys = np.arange(pw), np.arange(ph)
    qx, qy = xs & ~1, ys & ~1
    qx1, qy1 = np.minimum(qx + 1, pw - 1), np.minimum(qy + 1, ph - 1)
    with np.errstate(all="ignore"):
        ddx = (ru[:, qx1] - ru[:, qx], rv[:, qx1] - rv[:, qx])
        ddy = (ru[qy1, :] - ru[qy, :], rv[qy1, :] - rv[qy, :])
    return ddx, ddy


def probe_ref(maps, ru, rv, scale=(1.0, 1.0), offset=(0.0, 0.0)):
    """slot -> (value [ph, pw], bound [ph, pw]) of the probe channel of each map (channel 0 of the rotated map)"""
    ddx, ddy = quad_derivs(ru, rv)
    out = {}
    for slot, _ in PROBE_SLOTS:
        ch, w, h, levels = maps[slot]
        v, b = sample_ref(ch, w, h, levels, ru, rv, scale, offset, ddx, ddy)
        out[slot] = (v[:, 0].reshape(ru.shape), b[:, 0].reshape(ru.shape))
    return out


def probe_outputs(gbuf):
    return {slot: gbuf[p][..., c] for slot, (p, c) in PROBE_OUT.items()}
