"""Seeded inputs for the environment-map passes (K11, K2, K3, K4 and the shared equirect sampler): HDRI contents aimed at
each rule of the sampler and the MIN pyramid, HDRI shapes aimed at both K11 paths and their edges, and the cube texels
whose tangent-frame decision (BRDF.hlsl:231, |N.z| < 0.999) sits within rounding of the threshold."""
from __future__ import annotations

import numpy as np

from vqengine_b200 import synth

SEED = 0x1B1


def _rgba(rgb):
    h, w = rgb.shape[:2]
    out = np.ones((h, w, 4), np.float32)
    out[..., :3] = rgb
    return out


def content(kind, w, h, seed=SEED):
    """[h, w, 4] float32 HDRI of one kind (alpha 1)"""
    rng = np.random.default_rng(seed + 7919 * w + h)
    if kind == "synth":
        return synth.hdri(w, h, seed=seed) if w >= 2 and h >= 1 else _rgba(rng.uniform(0.05, 16.0, (h, w, 3)))
    if kind == "constant":
        return _rgba(np.broadcast_to(np.array([2.0, 0.5, 1.25], np.float32), (h, w, 3)))
    if kind == "row_constant":          # independent of u: every column is the same
        col = rng.uniform(0.0, 8.0, (h, 1, 3)).astype(np.float32)
        return _rgba(np.broadcast_to(col, (h, w, 3)))
    if kind == "seam":                  # columns 0 and W-1 differ strongly
        img = rng.uniform(0.5, 1.0, (h, w, 3)).astype(np.float32)
        img[:, 0] = 64.0; img[:, -1] = 0.0
        return _rgba(img)
    if kind == "noisy_poles":           # high-contrast noise in the pole rows
        img = rng.uniform(0.2, 1.0, (h, w, 3)).astype(np.float32)
        rows = sorted({0, h - 1} | ({1, h - 2} if h > 3 else set()))
        img[rows] = rng.choice(np.array([0.0, 1000.0], np.float32), size=(len(rows), w, 3))
        return _rgba(img)
    if kind == "zero":
        return _rgba(np.zeros((h, w, 3), np.float32))
    if kind in ("spike65504", "spike2p20"):
        img = np.full((h, w, 3), 0.25, np.float32)
        img[rng.integers(h), rng.integers(w)] = 65504.0 if kind == "spike65504" else 2.0 ** 20
        return _rgba(img)
    if kind == "denormal":
        bits = rng.integers(1, 0x007FFFFF, size=(h, w, 3), dtype=np.uint32)
        return _rgba(bits.view(np.float32))
    if kind == "ge1":                   # every value >= 1: a zero read from padding would be the block's MIN
        return _rgba(rng.uniform(1.0, 4.0, (h, w, 3)).astype(np.float32))
    raise ValueError(kind)


CONTENTS = ["synth", "constant", "row_constant", "seam", "noisy_poles", "zero", "spike65504", "spike2p20", "denormal", "ge1"]
SPECIALS = [np.nan, np.inf, -np.inf, -0.0, 0.0, -1.5, 2.0 ** -140]


def special_blocks(w, h, seed=SEED):
    """K11 only: values >= 1 with one special value (NaN, +-Inf, -0, +0, a negative, a denormal) at each of the four
    positions of the 2x2 blocks in turn, in every channel, plus blocks that hold both zeros in each order and 2x2 blocks
    of NaN; the specials sit at every level's block corners because the pattern repeats with period 2 in x and y"""
    rng = np.random.default_rng(seed + 3 * w + h)
    img = rng.uniform(1.0, 4.0, (h, w, 3)).astype(np.float32)
    ys, xs = np.mgrid[0:h, 0:w]
    blk = (ys // 2) * ((w + 1) // 2) + xs // 2
    pos = (ys % 2) * 2 + (xs % 2)                       # 0:(0,0) 1:(1,0) 2:(0,1) 3:(1,1)
    case = blk % (4 * len(SPECIALS) + 3)
    for c in range(3):
        cc = (case + 5 * c) % (4 * len(SPECIALS) + 3)
        for k, s in enumerate(SPECIALS):
            for p in range(4):
                m = (cc == 4 * k + p) & (pos == p)
                img[..., c][m] = s
        zero_pm = cc == 4 * len(SPECIALS)               # +0 then -0 (row-major), and the reverse
        img[..., c][zero_pm & (pos == 0)] = 0.0; img[..., c][zero_pm & (pos == 1)] = -0.0
        img[..., c][zero_pm & (pos >= 2)] = 0.0
        zero_mp = cc == 4 * len(SPECIALS) + 1
        img[..., c][zero_mp & (pos == 0)] = -0.0; img[..., c][zero_mp & (pos >= 1)] = 0.0
        img[..., c][zero_mp & (pos == 2)] = -0.0
        img[..., c][cc == 4 * len(SPECIALS) + 2] = np.nan
    return _rgba(img)


# (w, h, levels) for K11: None = the full pyramid. Both paths: SPD (w, h <= 4096) and per level (w or h > 4096).
K11_SHAPES = [
    (1, 1, None), (2, 1, None), (7, 3, None), (97, 41, None), (1024, 8, None), (8, 1024, None), (256, 128, None),
    (256, 128, 1), (256, 128, 3), (97, 41, 3),
    (128, 128, 2), (4096, 64, 7), (4096, 128, 8),        # SPD mips 1, 6 (no tail), 7 (tail of one level)
    (64, 64, None), (65, 65, None),                      # one SPD tile, and one texel past it
    (4095, 3, None), (65, 4096, None),                   # ragged SPD tiles, 1-row and 1-column levels
    (4101, 6, None), (8193, 5, None), (8192, 4096, None),  # per-level path (odd widths above 4096, the engine's 8K HDRIs)
]


def near_threshold_texels(sizes, ulps=2):
    """(face, px, py, res) of the +-Z face texels whose float64 |N.z| lies within `ulps` fp32 ulps of 0.999f, for each res:
    the texels where the tangent frame of K3 (BRDF.hlsl:231) hangs on the last bits of the normalisation"""
    thr = float(np.float32(0.999))
    ulp = float(np.spacing(np.float32(0.999)))
    out = []
    for res in sizes:
        sx = np.float32(2.0) * (np.arange(res).astype(np.float32) + np.float32(0.5)) / np.float32(res) - np.float32(1.0)
        sy = np.float32(1.0) - np.float32(2.0) * (np.arange(res).astype(np.float32) + np.float32(0.5)) / np.float32(res)
        X, Y = np.meshgrid(sx.astype(np.float64), sy.astype(np.float64))
        nz = 1.0 / np.sqrt(X * X + Y * Y + 1.0)
        py, px = np.nonzero(np.abs(nz - thr) <= ulps * ulp)
        for face in (4, 5):
            # face 5 is (-sx, sy, -1): the same |N.z| at the same (px, py)
            out += [(face, int(a), int(b), res) for a, b in zip(px, py)]
    return out
