"""Float64 restatement of the texture-sampling rules of DESIGN.md §3 (cubemap and BRDF LUT), vectorised with numpy.

Written from the rules as DESIGN.md §3 states them, not from oracle/oracle_shading.cpp, so that the oracle's sampler and K1's
bordered sampling copies are checked against an independent statement of the seamless cube rule:
  * face selection: the largest |component|, ties X > Y > Z, face coordinates (sx, sy) in [-1, 1] (D3D cube orientation);
  * texel-space coordinate x = (sx*0.5+0.5)*N - 0.5, y = (0.5-sy*0.5)*N - 0.5;
  * bilinear, lerp(a, b, t) = a + t*(b-a);
  * a tap one texel outside the face is the neighbouring face's texel: the direction of the virtual texel centre, in units
    of 1/N, has one component of magnitude N+1 (the neighbour's axis), and the texel is floor((c+N+1)*N/(2N+2)) for each
    of the neighbour's coordinates c in those units (rightward and downward);
  * the one tap that can be outside in both directions (a cube corner) is the mean of the other three;
  * LUT: bilinear CLAMP.
Inputs are float32 values; everything after them is float64.
"""
import numpy as np

# per face: major axis M, right U, up V (unit vectors); the direction of face coordinates (sx, sy) is M + sx*U + sy*V
_FACES = np.array([
    [(1, 0, 0), (0, 0, -1), (0, 1, 0)],      # +X
    [(-1, 0, 0), (0, 0, 1), (0, 1, 0)],      # -X
    [(0, 1, 0), (1, 0, 0), (0, 0, -1)],      # +Y
    [(0, -1, 0), (1, 0, 0), (0, 0, 1)],      # -Y
    [(0, 0, 1), (1, 0, 0), (0, 1, 0)],       # +Z
    [(0, 0, -1), (-1, 0, 0), (0, 1, 0)],     # -Z
], dtype=np.int64)


def mip_count(res: int) -> int:
    return int(res).bit_length()


def cube_texel_count(res: int, mips: int) -> int:
    return sum(6 * (res >> m) ** 2 for m in range(mips))


def face_of(d):
    """(n,3) directions -> face (n,), sx, sy (float64)"""
    d = np.asarray(d, np.float64)
    a = np.abs(d)
    isx = (a[:, 0] >= a[:, 1]) & (a[:, 0] >= a[:, 2])
    isy = ~isx & (a[:, 1] >= a[:, 2])
    axis = np.where(isx, 0, np.where(isy, 1, 2))
    major = d[np.arange(len(d)), axis]
    face = 2 * axis + (major <= 0.0)
    U, V = _FACES[face, 1].astype(np.float64), _FACES[face, 2].astype(np.float64)
    ma = np.abs(major)
    return face, (d * U).sum(1) / ma, (d * V).sum(1) / ma


def neighbour_texel(N, face, i, j):
    """integer edge rule: texel (i, j) of `face` with exactly one coordinate in {-1, N} -> (face', i', j') (arrays)"""
    N = np.asarray(N, np.int64)
    A, B = 2 * i + 1 - N, N - 1 - 2 * j
    v = A[:, None] * _FACES[face, 1] + B[:, None] * _FACES[face, 2] + N[:, None] * _FACES[face, 0]
    M = N + 1
    axis = np.argmax(np.abs(v), axis=1)
    comp = v[np.arange(len(v)), axis]
    assert (np.abs(comp) == M).all()
    nf = 2 * axis + (comp < 0)
    nsx, nsy = (v * _FACES[nf, 1]).sum(1), (v * _FACES[nf, 2]).sum(1)
    # texel = floor((c+M)*N/(2M)) for the rightward (sx) and downward (-sy) coordinate: rows run down from sy = +1
    ni = np.clip(((nsx + M) * N) // (2 * M), 0, N - 1)
    nj = np.clip(((M - nsy) * N) // (2 * M), 0, N - 1)
    return nf, ni, nj


def sample_cube(cube, res, mips, dirs, mip):
    """SampleCubeLevel in float64: cube (texels, 4) packed mip-major / face-minor, dirs (n,3), mip int or (n,) -> (n,4)"""
    t = np.asarray(cube, np.float64).reshape(-1, 4)
    d = np.asarray(dirs, np.float64).reshape(-1, 3)
    n = len(d)
    m = np.clip(np.broadcast_to(np.asarray(mip, np.int64), (n,)), 0, mips - 1)
    N = np.int64(res) >> m
    base = np.array([cube_texel_count(res, k) for k in range(mips)], np.int64)[m]
    face, sx, sy = face_of(d)
    x = (sx * 0.5 + 0.5) * N - 0.5
    y = (0.5 - sy * 0.5) * N - 0.5
    i0 = np.clip(np.floor(x), -1, N - 1).astype(np.int64)
    j0 = np.clip(np.floor(y), -1, N - 1).astype(np.int64)
    fx, fy = (x - i0)[:, None], (y - j0)[:, None]
    taps, corner = [], []
    for k in range(4):
        i, j = i0 + (k & 1), j0 + (k >> 1)
        oi, oj = (i < 0) | (i >= N), (j < 0) | (j >= N)
        f2, i2, j2 = face.copy(), i.copy(), j.copy()
        e = oi ^ oj
        if e.any():
            f2[e], i2[e], j2[e] = neighbour_texel(N[e], face[e], i[e], j[e])
        c = oi & oj
        i2[c] = 0; j2[c] = 0
        taps.append(t[base + (f2 * N + j2) * N + i2])
        corner.append(c)
    taps = np.stack(taps)                     # (4, n, 4)
    corner = np.stack(corner)                 # (4, n)
    if corner.any():
        assert (corner.sum(0) <= 1).all()
        mean = (taps.sum(0) - (taps * corner[..., None]).sum(0)) / 3.0
        taps = np.where(corner[..., None], mean[None], taps)
    lerp = lambda a, b, w: a + w * (b - a)
    return lerp(lerp(taps[0], taps[1], fx), lerp(taps[2], taps[3], fx), fy)


def sample_lut(lut, u, v):
    """SampleLUT in float64: lut [H, W, 2], u, v (n,) -> (n, 2), bilinear CLAMP"""
    l = np.asarray(lut, np.float64)
    H, W = l.shape[:2]
    u = np.asarray(u, np.float32).astype(np.float64).ravel()
    v = np.asarray(v, np.float32).astype(np.float64).ravel()
    x, y = u * W - 0.5, v * H - 0.5
    x0, y0 = np.floor(x), np.floor(y)
    fx, fy = (x - x0)[:, None], (y - y0)[:, None]
    ix0, ix1 = np.clip(x0, 0, W - 1).astype(int), np.clip(x0 + 1, 0, W - 1).astype(int)
    iy0, iy1 = np.clip(y0, 0, H - 1).astype(int), np.clip(y0 + 1, 0, H - 1).astype(int)
    lerp = lambda a, b, w: a + w * (b - a)
    return lerp(lerp(l[iy0, ix0], l[iy0, ix1], fx), lerp(l[iy1, ix0], l[iy1, ix1], fx), fy)


def rotate_hdri(d, offset):
    """GetHDRIRotationMatrix (Lighting.hlsl:348-358), mul(v, m), with the fp32 cos/sin of -offset the host computes"""
    c, s = float(np.cos(np.float32(-offset))), float(np.sin(np.float32(-offset)))
    d = np.asarray(d, np.float64)
    return np.stack([d[:, 0] * c - d[:, 2] * s, d[:, 1], d[:, 0] * s + d[:, 2] * c], axis=1)


# ---- inputs ---------------------------------------------------------------------------------------------------
CUBE_RES = (1, 2, 5, 16, 33)                  # every mip of each, down to 1x1 (33: 6 mips)
LUT_SIZES = ((1, 1), (48, 20), (20, 48))      # (W, H)


def random_cube(res, seed):
    """a full mip chain of uniform [0, 1] texels: a wrong texel, face or half-record shows up at once"""
    rng = np.random.default_rng(seed)
    return rng.uniform(0, 1, (cube_texel_count(res, mip_count(res)), 4)).astype(np.float32)


def random_lut(w, h, seed):
    return np.random.default_rng(seed).uniform(0, 1, (h, w, 2)).astype(np.float32)


def uniform_directions(n, rng):
    d = rng.normal(size=(n, 3))
    return (d / np.linalg.norm(d, axis=1, keepdims=True)).astype(np.float32)


def special_directions(N, rng, n_edge=8):
    """axes, exact edges (|a| = |b| > |c|), exact corners, and the texel-centre and texel-boundary directions of every face
    of an N x N mip (float32)"""
    out = [np.concatenate([np.eye(3), -np.eye(3)])]
    s = np.array([-1.0, 1.0])
    for a, b in ((0, 1), (0, 2), (1, 2)):
        c = 3 - a - b
        for sa in s:
            for sb in s:
                e = np.zeros((n_edge + 1, 3))
                e[:, a], e[:, b] = sa, sb
                e[:-1, c] = rng.uniform(-0.999, 0.999, n_edge)
                out.append(e)
    out.append(np.array([(x, y, z) for x in s for y in s for z in s]))
    centre = (2 * np.arange(N) + 1) / N - 1
    bound = 2 * np.arange(N + 1) / N - 1
    for grid in (centre, bound):
        sx, sy = np.meshgrid(grid, grid)
        sx, sy = sx.ravel(), sy.ravel()
        for f in range(6):
            M, U, V = _FACES[f].astype(np.float64)
            out.append(M[None] + sx[:, None] * U[None] + sy[:, None] * V[None])
    return np.concatenate(out).astype(np.float32)
