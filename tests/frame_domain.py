"""Seeded inputs over the whole domain of the passes either side of the shading path (SURVEY §8(f).2-(f).4): the Radiance
.hdr codec, the Mitchell downsize, the skydome, the reflection composite and the MIN depth pyramid. numpy only; each
generator names the branch of vq_frame.cu / vq_shadow.cu it aims at (tests/test_frame_domain.py checks that it lands there)."""
from __future__ import annotations

import itertools
import math

import numpy as np

f32 = np.float32
F32_MAX = float(np.finfo(np.float32).max)
DENORM = float(np.float32(1.0e-40))
HEADER = b"#?RADIANCE\nFORMAT=32-bit_rle_rgbe\n\n"
CUTOFF = f32(1e-32)                      # stbiw__linear_to_rgbe: maxcomp < 1e-32 -> (0, 0, 0, 0)


# ---- RGBE encode -----------------------------------------------------------------------------------------------------
def rgbe_exponent_walk(seed=1):
    """[rows, 32, 4]: per row one binary exponent e of maxcomp, from the 1e-32 cut-off to FLT_MAX (frexp exponents -105 ..
    128; 128 wraps the exponent byte to 0). Columns: the max in r, g or b, mantissas at 0.5, just below 1 and random, the
    other channels random fractions of it (some negative)."""
    rng = np.random.default_rng(seed)
    es = np.arange(-106, 128)
    out = np.zeros((len(es), 32, 4), f32)
    for r, e in enumerate(es):
        m = np.concatenate([[0.5, np.nextafter(f32(1.0), f32(0.0)), 0.75], rng.uniform(0.5, 1.0, 29)]).astype(f32)
        mx = np.ldexp(m.astype(np.float64), int(e))
        mx = np.minimum(mx, F32_MAX).astype(f32)
        oth = rng.uniform(-0.2, 1.0, (32, 3)) * mx[:, None]
        for c in range(32):
            k = c % 3
            oth[c, k] = mx[c]
        out[r, :, :3] = oth.astype(f32)
        out[r, :, 3] = 1.0
    out[-1, 0, :3] = (F32_MAX, F32_MAX, F32_MAX)
    out[-1, 1, :3] = (F32_MAX, 0.0, 1.0)
    return out


def rgbe_cutoff():
    """[1, 25, 4]: maxcomp at 1e-32 and its +-1, +-2 ulp neighbours, in each channel position, and with equal channels"""
    c = [np.nextafter(np.nextafter(CUTOFF, f32(0)), f32(0)), np.nextafter(CUTOFF, f32(0)), CUTOFF,
         np.nextafter(CUTOFF, f32(1)), np.nextafter(np.nextafter(CUTOFF, f32(1)), f32(1))]
    px = []
    for v in c:
        px += [(v, 0, 0), (0, v, 0), (0, 0, v), (v, v, v), (v, v * f32(0.5), -v)]
    a = np.ones((1, len(px), 4), f32)
    a[0, :, :3] = np.array(px, f32)
    return a


SPECIALS = [-0.0, 0.0, -1.0, 1.0, 0.5, -math.inf, math.inf, math.nan, 2.0 ** 127, F32_MAX, 3e-33, 0.75 * 2.0 ** 127]


def rgbe_specials():
    """[12, 144, 4]: every (r, g, b) over SPECIALS: -0, negatives, +-Inf, NaN in each position (the nesting of stbiw__max
    decides which NaN is ignored), maxcomp >= 2^127 (exponent byte wraps to 0)"""
    px = np.array(list(itertools.product(SPECIALS, repeat=3)), f32)
    a = np.ones((len(SPECIALS), len(SPECIALS) ** 2, 4), f32)
    a[..., :3] = px.reshape(len(SPECIALS), len(SPECIALS) ** 2, 3)
    return a


def encode_images():
    return {"exponent_walk": rgbe_exponent_walk(), "cutoff": rgbe_cutoff(), "specials": rgbe_specials()}


# ---- RGBE decode streams ----------------------------------------------------------------------------------------------
RLE_WIDTHS = [8, 63, 64, 65, 127, 128, 129, 2047, 2048, 2049, 32767]


def _channel_records(rng, vals, zero_at=(), literal_only=False):
    """run list of one channel for the byte plane `vals`: random mix of repeat and literal records, zero-length literal
    records inserted before every texel index in `zero_at` (each a no-op byte)"""
    out = bytearray()
    w = len(vals)
    zero_at = sorted(zero_at)
    zi = 0
    i = 0
    while i < w:
        while zi < len(zero_at) and zero_at[zi] <= i:
            out.append(0); zi += 1
        nxt = zero_at[zi] if zi < len(zero_at) else w
        n = int(min(nxt - i, w - i, 128 if literal_only else rng.integers(1, 129)))
        if not literal_only and rng.random() < 0.4:
            n = min(n, 127)
            vals[i:i + n] = vals[i]
            out += bytes([128 + n, int(vals[i])])
        else:
            out += bytes([n]) + bytes(vals[i:i + n].tobytes())
        i += n
    while zi < len(zero_at):
        out.append(0); zi += 1
    return bytes(out)


def rle_file(width, height, seed=0, zero_blocks=False, literal_only=False):
    """a run-length encoded file: random records (or literals only) with zero-length records on every 64-texel block
    boundary when zero_blocks; -> (file bytes, [h, w, 4] uint8 RGBE texels)"""
    rng = np.random.default_rng(seed)
    body = bytearray(); px = np.zeros((height, width, 4), np.uint8)
    for j in range(height):
        body += bytes([2, 2, width >> 8, width & 255])
        for k in range(4):
            vals = rng.integers(0, 256, width, dtype=np.uint8) if k < 3 else rng.integers(100, 160, width, dtype=np.uint8)
            zs = list(range(64, width, 64)) if zero_blocks else []
            body += _channel_records(rng, vals, zs, literal_only)
            px[j, :, k] = vals
    return HEADER + f"-Y {height} +X {width}\n".encode() + bytes(body), px


def staging_capacity(width):
    """hdr_decode_launch's `tight`: the most bytes of one scanline's window (its 16-byte-aligned start to the next scanline's
    first run list) that the STAGED kernel copies to shared memory"""
    return (16 + 4 + 4 * (width + width // 64 + 2) + 15) & ~15


def staging_file(width, height, excess, seed=0):
    """every scanline's window exactly staging_capacity + excess bytes (excess 0: staged; 16: read from global memory),
    filled up with zero-length records on 64-texel block boundaries; -> (file, texels, [window bytes per scanline])"""
    rng = np.random.default_rng(seed)
    head = HEADER + f"-Y {height} +X {width}\n".encode()
    body = bytearray(); px = np.zeros((height, width, 4), np.uint8); windows = []
    cap = staging_capacity(width) + excess
    for j in range(height):
        begin = len(head) + len(body) + 4
        tail = 0 if j == height - 1 else 4
        blocks = list(range(0, width, 64))                          # one zero-length record on every block start ...
        planes = [rng.integers(0, 256, width, dtype=np.uint8) for _ in range(4)]
        base = sum(len(_channel_records(rng, v, blocks, literal_only=True)) for v in planes)
        pad = cap - (begin - (begin & ~15)) - tail - base
        if pad < 0:
            blocks = []
            pad = cap - (begin - (begin & ~15)) - tail - sum(len(_channel_records(rng, v, (), literal_only=True)) for v in planes)
        assert pad >= 0, "scanline too long for the target window"
        body += bytes([2, 2, width >> 8, width & 255])
        for k, vals in enumerate(planes):                          # ... and the rest at texel 0
            px[j, :, k] = vals
            body += _channel_records(rng, vals, blocks + [0] * (pad // 4 + (1 if k < pad % 4 else 0)), literal_only=True)
        windows.append(len(head) + len(body) + tail - (begin & ~15))
    return head + bytes(body), px, windows


def non_rle_marker_file(width, height, j, seed=0, truncate=0):
    """RLE scanlines 0..j-1, then a scanline that does not start with {2, 2, hi<128}: stb decodes those 4 bytes as texel 0 and
    the rest of the image flat from there, restarting at row 0 (vq_hdr_parse). `truncate` bytes are cut off the end."""
    rng = np.random.default_rng(seed)
    body = bytearray()
    for _ in range(j):
        body += bytes([2, 2, width >> 8, width & 255])
        for k in range(4):
            body += _channel_records(rng, rng.integers(0, 256, width, dtype=np.uint8))
    flat = rng.integers(0, 256, (height * width, 4), dtype=np.uint8)
    flat[:, 3] = rng.integers(110, 150, height * width)
    flat[0, :2] = (1, 2)                                          # not the {2, 2} marker
    out = HEADER + f"-Y {height} +X {width}\n".encode() + bytes(body) + flat.tobytes()
    return out[:len(out) - truncate] if truncate else out


def flat_file(width, height, seed=0, truncate=0):
    """width < 8 or >= 32768: texels stored flat; truncated: missing bytes read as 0"""
    rng = np.random.default_rng(seed)
    px = rng.integers(0, 256, (height, width, 4), dtype=np.uint8)
    out = HEADER + f"-Y {height} +X {width}\n".encode() + px.tobytes()
    return out[:len(out) - truncate] if truncate else out


def decode_files():
    """name -> file bytes that decode (vq_hdr_parse accepts them)"""
    files = {}
    for w in RLE_WIDTHS:
        h = 2 if w > 4096 else 3
        files[f"rle-w{w}"] = rle_file(w, h, seed=w)[0]
    files["rle-w700-zero-blocks"] = rle_file(700, 3, seed=5, zero_blocks=True)[0]
    files["rle-w129-zero-blocks"] = rle_file(129, 2, seed=6, zero_blocks=True)[0]
    for w in (64, 700, 2049):
        for ex in (0, 16):
            files[f"staging-w{w}+{ex}"] = staging_file(w, 3, ex, seed=w + ex)[0]
    for j, h in ((0, 4), (1, 4), (3, 4)):
        files[f"marker-row{j}-of{h}"] = non_rle_marker_file(40, h, j, seed=j)
    files["marker-row1-truncated"] = non_rle_marker_file(40, 4, 1, seed=9, truncate=301)
    files["flat-w7-truncated"] = flat_file(7, 5, seed=3, truncate=37)
    files["flat-w32768"] = flat_file(32768, 1, seed=4)
    return files


def corrupt_files():
    """name -> file bytes that stb refuses: a stream that ends inside a scanline, a record longer than the scanline"""
    good, _ = rle_file(200, 3, seed=11)
    head = HEADER + b"-Y 1 +X 16\n"
    return {"rle-truncated-mid-scanline": good[:len(good) - 150],
            "rle-record-overruns-width": head + bytes([2, 2, 0, 16, 128 + 17, 5]) + bytes(64)}


# ---- Mitchell downsize -------------------------------------------------------------------------------------------------
RESIZE_SPAN = 576                         # vq_frame.cu: resize_h_kernel stages a 64-output block's span up to this many texels


def block_span(table):
    """largest number of input texels one 64-output block of resize_h_kernel touches, from vq.resize_axis_table"""
    start, count, _ = table
    o = len(start)
    return max(int(start[min(x0 + 63, o - 1)] + count[min(x0 + 63, o - 1)] - start[x0]) for x0 in range(0, o, 64))


# (name, in_w, in_h, out_w, out_h, what it aims at). The four span cases put the widest block's span at 575 / 576 (staged)
# and 577 / 1190 (direct path); they were found with block_span(vq.resize_axis_table(in_w, out_w)), and
# tests/test_frame_domain.py re-derives them.
RESIZE_CASES = [
    ("span575", 1098, 9, 128, 9, "staged, widest span 575"),
    ("span576", 1100, 9, 128, 9, "staged, widest span = RESIZE_SPAN"),
    ("span577", 1102, 9, 128, 9, "direct path, widest span 577"),
    ("span1190", 2272, 7, 128, 5, "direct path, span about 1200"),
    ("span577-o65", 560, 6, 65, 3, "direct path, 65 outputs: a full block and a 1-output block"),
    ("span576-o64", 550, 5, 64, 5, "staged, exactly one block"),
    ("span577-o64", 551, 5, 64, 5, "direct path, exactly one block"),
    ("w1to1-h300to1", 37, 600, 37, 2, "1:1 horizontally, 300:1 vertically"),
    ("w300to1-h1to1", 900, 5, 3, 5, "300:1 horizontally (direct path), 1:1 vertically"),
    ("w300to1-o1", 300, 3, 1, 1, "direct path, one output of 1200 taps per axis"),
    ("w97to1-h3to1", 6305, 6, 65, 2, "direct path at 97:1"),
    ("o63", 200, 11, 63, 7, "63 outputs"),
    ("o64", 256, 13, 64, 6, "64 outputs"),
    ("o65", 130, 10, 65, 10, "65 outputs at 2:1"),
    ("o1x1", 9, 9, 1, 1, "1 x 1 output"),
    ("h-not-mult4", 70, 7, 30, 5, "in and out heights not multiples of 4"),
    ("w1-column", 1, 17, 1, 3, "single-column image"),
]


def resize_input(in_w, in_h, seed, specials=False):
    """[in_h, in_w, 4] radiance in [-0.5, 8) (negative lobes meet negative data); with `specials` a sprinkling of +-Inf and NaN
    (the Mitchell lobes are negative, so a lone Inf comes out NaN where it meets both signs)"""
    rng = np.random.default_rng(seed)
    a = (rng.random((in_h, in_w, 4)) * 8.5 - 0.5).astype(f32)
    if specials:
        n = max(1, a.size // 400)
        idx = rng.integers(0, a.size, (3, n))
        flat = a.reshape(-1)
        flat[idx[0]] = np.inf; flat[idx[1]] = -np.inf; flat[idx[2]] = np.nan
    return a


# ---- skydome ---------------------------------------------------------------------------------------------------------
def view_proj(world3, fov_y, aspect, near=0.1, far=1000.0):
    """inverse of view * proj (row vectors) for a camera at the origin with orientation world3 (3x3, rows = right, up,
    forward), XMMatrixPerspectiveFovLH; inverse written out (inv(proj) @ world) so exact 0 / +-1 rotations stay exact"""
    h = 1.0 / math.tan(0.5 * fov_y)
    w = h / aspect
    q = far / (far - near)
    inv_proj = np.array([[1 / w, 0, 0, 0], [0, 1 / h, 0, 0], [0, 0, 0, -1 / (near * q)], [0, 0, 1, 1 / near]], np.float64)
    world = np.eye(4); world[:3, :3] = world3
    return (inv_proj @ world).astype(f32).reshape(16)


def yaw_pitch(yaw, pitch):
    cy, sy, cp, sp = math.cos(yaw), math.sin(yaw), math.cos(pitch), math.sin(pitch)
    rot_y = np.array([[cy, 0, -sy], [0, 1, 0], [sy, 0, cy]])
    rot_x = np.array([[1, 0, 0], [0, cp, sp], [0, -sp, cp]])
    return rot_x @ rot_y


def axis_rotations():
    """the 24 rotations of the cube: signed permutation matrices with determinant +1, entries exactly 0 / +-1"""
    out = []
    for perm in itertools.permutations(range(3)):
        for signs in itertools.product((1.0, -1.0), repeat=3):
            m = np.zeros((3, 3))
            for r, c in enumerate(perm):
                m[r, c] = signs[r]
            if round(np.linalg.det(m)) == 1:
                out.append(m)
    return out


def negative_zeros(m):
    """the same matrix with every zero entry as -0 (an inverse computed by a caller can carry them)"""
    m = np.array(m, f32)
    m[m == 0] = f32(-0.0)
    return m


def sky_ray(m, w, h, rows=None):
    """the fp32 ray of skydome_pair_kernel for every pixel: ((nx*m0 + ny*m4) + m8) + m12 per component, no contraction;
    -> [4, h, w] float32 (x, y, z, w)"""
    m = np.asarray(m, f32).reshape(16)
    xs = np.arange(w, dtype=f32); ys = np.arange(h, dtype=f32)
    nx = ((xs + f32(0.5)) / f32(w)) * f32(2.0) - f32(1.0)
    ny = f32(1.0) - ((ys + f32(0.5)) / f32(h)) * f32(2.0)
    nx = nx[None, :]; ny = ny[:, None]
    with np.errstate(all="ignore"):
        return np.stack([((nx * m[c] + ny * m[4 + c]) + m[8 + c]) + m[12 + c] for c in range(4)]).astype(f32)


def sky_fallback(ray):
    """pixels whose pair takes the __fdiv_rn branch: |w| <= 1e-15, >= 1e15 or a ray component >= 1e15 (either pixel of the
    pair: rows y, y+1 of the launch; approximated per pixel)"""
    aw = np.abs(ray[3]); big = np.abs(ray[:3]).max(axis=0)
    return ~((aw > f32(1e-15)) & (aw < f32(1e15)) & (big < f32(1e15)))


def sky_hdri(w, h, seed=0):
    """band-limited radiance with one bright lobe near each pole and distinct edge columns (so that a wrong seam or a
    clamped v shows), alpha 1"""
    rng = np.random.default_rng(seed)
    v, u = np.meshgrid((np.arange(h) + 0.5) / h, (np.arange(w) + 0.5) / w, indexing="ij")
    img = np.ones((h, w, 4), np.float64)
    for c in range(3):
        a = rng.uniform(0.2, 1.0, 3)
        img[..., c] = (1.0 + a[0] * np.sin(2 * np.pi * u + a[1]) * np.sin(np.pi * v) + 0.5 * a[2] * np.cos(4 * np.pi * u + c)
                       + 2.0 * (1 - v) ** 6 * (c + 1) + 0.5 * v ** 8)
    return img.astype(f32)


def sky_cases():
    """(name, inv_view_proj[16] fp32, frame w, h, hdri w, h, rows, mask kind). Mask kinds: None, "holes" (random surface
    pixels), "signed" (normals of -0 and NaN: -0 == 0 is no surface, NaN != 0 is a surface)"""
    cases = []
    cases.append(("pitch+90", view_proj(yaw_pitch(0.4, math.pi / 2), 1.2, 1.0), 65, 33, 256, 128, None, None))
    cases.append(("pitch-90", view_proj(yaw_pitch(-1.1, -math.pi / 2), 1.2, 1.0), 33, 65, 256, 128, None, None))
    cases.append(("pitch+90-1e-3", view_proj(yaw_pitch(0.0, math.pi / 2 - 1e-3), 0.6, 1.5), 97, 41, 512, 256, None, None))
    cases.append(("pitch-90+1e-3", view_proj(yaw_pitch(2.0, -math.pi / 2 + 1e-3), 0.6, 1.5), 97, 41, 512, 256, None, None))
    # the u = 0 / 1 seam (direction -X: atan2(+-0, -1) = +-pi) through the middle of the frame
    cases.append(("seam-minus-x", view_proj(yaw_pitch(-math.pi / 2, 0.0), 1.0, 16 / 9), 161, 91, 300, 150, (0, 91), "holes"))
    cases.append(("seam-tilted", view_proj(yaw_pitch(-math.pi / 2 + 0.2, 0.3), 1.4, 1.0), 64, 64, 64, 32, None, None))
    for k, yaw in enumerate((math.pi / 4, 3 * math.pi / 4, -math.pi / 4, -3 * math.pi / 4)):
        cases.append((f"diagonal{k}", view_proj(yaw_pitch(yaw, 0.1 * k), 1.1, 4 / 3), 81, 61, 128, 64, None, None))
    for i, rot in enumerate(axis_rotations()):
        m = view_proj(rot, math.pi / 2, 1.0)
        if i % 2:
            m = negative_zeros(m)
        cases.append((f"axis{i:02d}{'-negzero' if i % 2 else ''}", m, 7 if i % 3 else 5, 5 if i % 3 else 7, 64, 32, None, None))
    cases.append(("far1e7", view_proj(yaw_pitch(0.3, 0.2), 1.1, 16 / 9, far=1e7), 48, 27, 128, 64, None, None))
    cases.append(("far1e16", view_proj(yaw_pitch(-0.6, -0.4), 1.1, 16 / 9, far=1e16), 48, 27, 128, 64, None, None))
    wcol = np.arange(16) % 4 == 3                                   # the w column of the row-major matrix
    cases.append(("tiny-w", (view_proj(yaw_pitch(0.9, 0.1), 1.1, 1.0) * np.where(wcol, 1e-14, 1.0)).astype(f32), 33, 21, 128, 64,
                  None, None))
    cases.append(("huge-ray", (view_proj(yaw_pitch(-2.2, 0.5), 1.1, 1.0) * np.where(wcol, 1.0, 1e16)).astype(f32), 33, 21, 128, 64,
                  None, None))
    for hw, hh in ((1, 1), (2, 1), (1, 2), (3, 5)):
        cases.append((f"hdri{hw}x{hh}", view_proj(yaw_pitch(0.7, 0.6), 1.6, 1.0), 31, 17, hw, hh, None, None))
    cases.append(("hdri4096x2048", view_proj(yaw_pitch(2.9, -0.2), 1.0, 16 / 9), 160, 90, 4096, 2048, None, "signed"))
    cases.append(("rows-empty", view_proj(yaw_pitch(0.2, 0.0), 1.0, 1.0), 40, 30, 64, 32, (13, 13), None))
    cases.append(("rows-odd", view_proj(yaw_pitch(0.2, 0.3), 1.0, 1.0), 40, 31, 64, 32, (3, 30), "signed"))
    cases.append(("rows-last", view_proj(yaw_pitch(0.2, -0.3), 1.0, 1.0), 40, 31, 64, 32, (30, 31), None))
    return cases


def sky_mask(kind, w, h, seed=0):
    """normal plane: None, or rows where normal.xyz is a surface (!= 0) or not (== 0, -0 included; NaN is a surface)"""
    if kind is None:
        return None
    rng = np.random.default_rng(seed)
    m = (rng.random((h, w, 4)) + 0.1).astype(f32)
    hole = rng.random((h, w)) < 0.6
    m[hole, :3] = 0.0
    if kind == "signed":
        sel = hole & (rng.random((h, w)) < 0.5)
        m[sel, :3] = f32(-0.0)
        m[sel & (rng.random((h, w)) < 0.3), 1] = np.nan
        m[~hole & (rng.random((h, w)) < 0.2), 0] = np.nan
    return m


# ---- reflection composite ----------------------------------------------------------------------------------------------
COMPOSITE_VALUES = [0.0, -0.0, 1.0, -2.5, 3e38, -3e38, math.inf, -math.inf, math.nan, DENORM, 0.3]
ALPHAS = [-1.0, 0.0, 1.0, 2.0, math.nan, 0.25]


def composite_planes(w, h, seed=0):
    """scene, reflection and bounding-volume planes [h, w, 4]: random radiance with blocks of COMPOSITE_VALUES (Inf + -Inf,
    NaN, overflow of the sum, denormals) and bounding-volume alphas from ALPHAS"""
    rng = np.random.default_rng(seed)
    s = (rng.random((h, w, 4)) * 8).astype(f32)
    r = rng.random((h, w, 4)).astype(f32)
    b = rng.random((h, w, 4)).astype(f32)
    vals = np.array(COMPOSITE_VALUES, f32)
    for p in (s, r, b):
        sel = rng.random((h, w, 4)) < 0.3
        p[sel] = vals[rng.integers(0, len(vals), int(sel.sum()))]
    # every (scene, reflection) value pair once, in the first rows
    pairs = np.array(list(itertools.product(COMPOSITE_VALUES, repeat=2)), f32)
    n = min(len(pairs), w * h)
    s.reshape(-1, 4)[:n, 0] = pairs[:n, 0]; r.reshape(-1, 4)[:n, 0] = pairs[:n, 1]
    b[..., 3] = np.array(ALPHAS, f32)[rng.integers(0, len(ALPHAS), (h, w))]
    return s, r, b


COMPOSITE_SIZES = [(1, 1), (11, 11), (64, 5), (257, 3), (3840, 2160)]


# ---- MIN depth pyramid -------------------------------------------------------------------------------------------------
DEPTH_DIMS = [1, 2, 3, 4, 5, 63, 64, 65, 127, 128, 129, 4095, 4096, 4097]
DEPTH_VALUES = [0.0, -0.0, 1.0, math.inf, -math.inf, math.nan, DENORM, -DENORM, -0.5, 0.25]


def depth_sizes():
    """widths x heights from DEPTH_DIMS; the 4K-class edges only against small ones (keeps the sweep's texel count low)"""
    big = {4095, 4096, 4097}
    return [(w, h) for w in DEPTH_DIMS for h in DEPTH_DIMS if not (w in big and h > 5) and not (h in big and w > 5)] + \
        [(4097, 65), (129, 4095), (4096, 4096)]


def depth_plane(w, h, seed=0):
    """uniform depths with 2x2-aligned blocks of DEPTH_VALUES (one value, one texel of it, or a mix), +-0 tie blocks (+0 and
    -0 in one 2x2 block, in every order) and single special texels on the ragged last row / column"""
    rng = np.random.default_rng(seed)
    d = rng.uniform(0.05, 1.0, (h, w)).astype(f32)
    vals = np.array(DEPTH_VALUES, f32)
    bh, bw = (h + 1) // 2, (w + 1) // 2
    n = min(bh * bw, max(1, bh * bw // 4), 40000)
    pick = rng.choice(bh * bw, n, replace=False)
    kinds = rng.integers(0, 4, n)
    for b, kind in zip(pick.tolist(), kinds.tolist()):
        by, bx = 2 * (b // bw), 2 * (b % bw)
        blk = d[by:by + 2, bx:bx + 2]
        if kind == 0:
            blk[...] = vals[rng.integers(0, len(vals))]
        elif kind == 1:
            z = np.array([0.0, -0.0, 0.0 if rng.random() < 0.5 else -0.0, -0.0 if rng.random() < 0.5 else 0.0], f32)[rng.permutation(4)]
            blk[...] = z[:blk.size].reshape(blk.shape)
        elif kind == 2:
            blk.reshape(-1)[rng.integers(0, blk.size)] = vals[rng.integers(0, len(vals))]
        else:
            blk[...] = vals[rng.integers(0, len(vals), blk.shape)]
    d[-1, rng.integers(0, w, min(w, 8))] = vals[rng.integers(0, len(vals), min(w, 8))]
    d[rng.integers(0, h, min(h, 8)), -1] = vals[rng.integers(0, len(vals), min(h, 8))]
    return d


RAGGED13 = (4097, 2049)          # 13 levels (4097 -> 1 in 12 halvings), odd at every level


def depth_n_levels():
    """(w, h, n_levels): the sweep 1..13 on the ragged 13-level shape (the second launch starts at n = 8)"""
    return [(RAGGED13[0], RAGGED13[1], n) for n in range(1, 14)]
