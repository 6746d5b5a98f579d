"""K1's domain inputs (tests/forward_domain.py, tests/light_domain.py) in the form the one-pass PSMain kernel takes them (test input
generation, no GPU).

adapt()  turns a G-buffer scene into interpolants and map-less materials that the surface producer turns back into the same
         G-buffer: position_u = (P, 0), normal_v = (N, 0), tangent_m = (+X, material index), the SSAO plane = the scene's ao and
         fAmbientLightingFactor = 1 (so the producer's ao = 1 * ssao is exact), one material per distinct (albedo.rgb, metalness,
         roughness, emissive rgb, intensity) with textureConfig = 0 and alpha 1. The producer writes the normal as N * rsqrtf(N.N):
         K1's raw normals of length 0.5..2 reach the shading code at unit length (within a few ulp). That is the fused path's
         domain, so every expectation is re-evaluated on the G-buffer the producer makes, not taken from the scene.

fold()   puts K1 pixel (row y, column c) of a 256-wide tile into (row 2y + (c >= 128), column c mod 128) of a 128-wide tile.
         K1's thread t shades (y, x0+t) and (y, x0+t+128); psmain's thread t shades (y0, x0+t) and (y0+1, x0+t). After the fold,
         K1's warps and pixel pairs are exactly psmain's, so a construction aimed at one warp layout keeps its property (the t
         sweep's one exact-path pixel per warp, the TINY and escape votes). The unfolded frame puts the same pixels into other
         warps.
"""
import numpy as np

import vqengine_b200 as vq

F32 = np.float32
TILE = 256                       # K1's tile: 256 consecutive pixels of one row; psmain's: 2 rows x 128 columns
MAX_MATERIALS = 1 << 20          # the material table's limit


def _zeros1(h, w):
    return np.zeros((h, w, 1), F32)


def material(albedo, metal, rough, emissive, intensity):
    m = vq.MaterialData()
    m.diffuse.x, m.diffuse.y, m.diffuse.z = (float(c) for c in albedo)
    m.alpha = 1.0
    m.emissiveColor.x, m.emissiveColor.y, m.emissiveColor.z = (float(c) for c in emissive)
    m.emissiveIntensity = float(intensity)
    m.uvScaleOffset.x, m.uvScaleOffset.y = 1.0, 1.0
    m.roughness, m.metalness = float(rough), float(metal)
    m.textureConfig = 0.0
    return m


def adapt(planes):
    """G-buffer planes [position_ao, normal_roughness, albedo_metalness(, emissive)] -> (surface planes [position_u, normal_v,
    tangent_m, ssao [H, W, 1]], materials). The producer reads the SSAO texel (x+1, y+1) with WRAP, so the plane is the ao
    plane rolled by one pixel in both axes."""
    pos, nrm, alb = planes[:3]
    h, w = pos.shape[:2]
    em = planes[3] if len(planes) > 3 else np.zeros((h, w, 4), F32)
    key = np.ascontiguousarray(np.concatenate([alb, nrm[..., 3:4], em], -1).reshape(-1, 9).astype(F32))
    uniq, inv = np.unique(key.view(np.uint32), axis=0, return_inverse=True)
    assert len(uniq) <= MAX_MATERIALS
    u = uniq.view(F32)
    mats = [material(r[0:3], r[3], r[4], r[5:8], r[8]) for r in u]
    pu = np.concatenate([pos[..., :3], _zeros1(h, w)], -1)
    nv = np.concatenate([nrm[..., :3], _zeros1(h, w)], -1)
    tm = np.zeros((h, w, 4), F32)
    tm[..., 0] = 1.0
    tm[..., 3] = inv.reshape(h, w).astype(F32)
    ssao = np.roll(pos[..., 3], (1, 1), axis=(0, 1)).astype(F32).reshape(h, w, 1)
    return [np.ascontiguousarray(p, dtype=F32) for p in (pu, nv, tm, ssao)], mats


def renormalised(planes):
    """the scene's G-buffer as the producer hands it to the shading code, in float64: N / |N| (up to the producer's few ulp)"""
    n = planes[1][..., :3].astype(np.float64)
    return n / np.linalg.norm(n, axis=-1, keepdims=True)


# ---- fold ------------------------------------------------------------------------------------------------------------
def fold(a):
    """[H, W, ...] with W a multiple of 256 -> [2H, W/2, ...]: K1 tile j's half k of row y -> psmain tile j's row 2y + k"""
    h, w = a.shape[:2]
    assert w % TILE == 0, w
    rest = a.shape[2:]
    t = a.reshape((h, w // TILE, 2, TILE // 2) + rest)
    t = np.swapaxes(t, 1, 2)
    return np.ascontiguousarray(t.reshape((2 * h, w // 2) + rest))


def unfold(a):
    """the inverse of fold"""
    h2, w2 = a.shape[:2]
    assert h2 % 2 == 0 and w2 % (TILE // 2) == 0
    rest = a.shape[2:]
    t = a.reshape((h2 // 2, 2, w2 // (TILE // 2), TILE // 2) + rest)
    t = np.swapaxes(t, 1, 2)
    return np.ascontiguousarray(t.reshape((h2 // 2, 2 * w2) + rest))


def k1_warps(shape):
    """[H, W] warp id of each pixel under K1 (tile = 256 pixels of a row; warp k holds columns 32k.. of both halves)"""
    h, w = shape
    y, x = np.mgrid[0:h, 0:w]
    tile, c = x // TILE, x % TILE
    return (y * (-(-w // TILE)) + tile) * 4 + (c % (TILE // 2)) // 32


def ps_warps(shape):
    """[H, W] warp id of each pixel under psmain (tiles of 2 rows x 128 columns from an even row; warp k: columns 32k.. of both
    rows)"""
    h, w = shape
    y, x = np.mgrid[0:h, 0:w]
    return ((y // 2) * (-(-w // (TILE // 2))) + x // (TILE // 2)) * 4 + (x % (TILE // 2)) // 32


def ps_ctas_per_column(w, sm_count):
    """psmain's persistent grid: CTAs per 128-column tile column (4 per SM over the row's tiles, vq_forward.cu). A range of more
    row pairs than this makes some CTA shade a second tile, from a stage that still holds its first tile's texels."""
    return max(1, sm_count * 4 // (-(-w // (TILE // 2))))


def fold_probe(p):
    """the probe with its planes and every per-pixel array folded"""
    sh = p["planes"][0].shape[:2]
    q = dict(p)
    q["planes"] = [fold(x) for x in p["planes"]]
    for k, v in p.items():
        if k != "planes" and isinstance(v, np.ndarray) and v.shape[:2] == sh:
            q[k] = fold(v)
    q["name"] = p.get("name", "probe") + " folded"
    return q


def crop(p, w):
    """the probe's first w columns (so that a frame of any width folds)"""
    sh = p["planes"][0].shape[:2]
    q = dict(p)
    q["planes"] = [np.ascontiguousarray(x[:, :w]) for x in p["planes"]]
    for k, v in p.items():
        if k != "planes" and isinstance(v, np.ndarray) and v.shape[:2] == sh:
            q[k] = np.ascontiguousarray(v[:, :w])
    return q


# ---- the votes a frame's pixels cast -----------------------------------------------------------------------------------
def tiny_pixels(planes):
    """pixels whose roughness lets the `denom < EPSILON` escape happen (the per-warp TINY vote: PI (1 + min(a2-1, 0))^2 < 2e-12
    in fp32)"""
    r = planes[1][..., 3].astype(F32)
    a = r * r
    a2m1 = (a * a) - F32(1.0)
    tmin = F32(1.0) + np.minimum(a2m1, F32(0.0))
    return F32(np.pi) * (tmin * tmin) < F32(2e-12)


def ggx_t(planes, cam, wi):
    """float64 GGX t = (N.H)^2 (a2 - 1) + 1 of a directional light from direction wi (unit, towards the light) on the planes"""
    P = planes[0][..., :3].astype(np.float64)
    N = renormalised(planes)
    V = np.asarray(cam, np.float64) - P
    V /= np.linalg.norm(V, axis=-1, keepdims=True)
    H = V + np.asarray(wi, np.float64)
    H /= np.linalg.norm(H, axis=-1, keepdims=True)
    nh = (N * H).sum(-1)
    r = planes[1][..., 3].astype(np.float64)
    return nh * nh * (r ** 4 - 1.0) + 1.0


def per_warp(mask, warps):
    """count of mask pixels in each warp, over the warps that occur"""
    ids, inv = np.unique(warps.ravel(), return_inverse=True)
    return np.bincount(inv, weights=mask.ravel().astype(np.float64), minlength=len(ids)).astype(int)
