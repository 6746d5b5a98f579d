"""-m gpu: the surface producer over the seeded domain of tests/surface_domain.py. The kernel matches the oracle at the parity
bound (1e-4) with NaN at the oracle's positions, stays within the float64 bound of tests/surface_ref.py on both sampling
paths, and the record path equals the map-by-map path bit for bit; the alpha discard, row ranges, padded planes, the
material-index and textureConfig rules, and tex_mip6_kernel's launches and vector path."""
import numpy as np
import pytest
import torch

import oracle_lib as orc
import vqengine_b200 as vq
from vqengine_b200.shader_data import (TEXCFG_DIFFUSE, TEXCFG_NORMAL, TEXCFG_AO, TEXCFG_ROUGHNESS, TEXCFG_METALLIC,
                                       TEXCFG_EMISSIVE, TEXCFG_ORM)
from gpu_util import TOL
from surface_ref import sample_ref, mip_chain_ref, alpha_decision
import surface_domain as sd

pytestmark = pytest.mark.gpu

NAMES = ("position_ao", "normal_roughness", "albedo_metalness", "emissive")
INIT = -7.0
WORST = {}


@pytest.fixture(scope="module", autouse=True)
def _report_worst():
    yield
    for k, v in sorted(WORST.items()):
        print(f"surface domain: largest error / float64 bound, {k}: {v:.3f}")


def _padded(a, pad=3):
    """a device copy of a [h, w, c] plane inside a wider tensor: the row pitch is not w * c"""
    h, w, c = a.shape
    big = torch.full((h, w + pad, c), 123.0, dtype=torch.float32, device="cuda")
    big[:, :w] = torch.from_numpy(np.ascontiguousarray(a, np.float32)).cuda()
    return big, big[:, :w]


def _image(t, c=4):
    return vq.Image(t.data_ptr(), t.shape[1], t.shape[0], t.stride(0) * 4) if t is not None else vq.null_image()


def run_kernel(ctx, planes, mats, chains, *, ssao=None, emissive=True, alpha_mask=False, ambient=1.0, rows=None, records=True,
               monkeypatch=None):
    """the kernel on padded planes (every input and output plane, and SSAO); returns the G-buffer planes and whether the
    padding stayed untouched"""
    h, w = planes[0].shape[:2]
    if monkeypatch is not None:
        monkeypatch.setenv("VQ_SURFACE_RECORDS", "1" if records else "0")
    keep, tex = [], []
    for d in chains:
        mt = vq.MaterialTextures()
        for slot in vq.MATERIAL_TEXTURE_SLOTS:
            e = d.get(slot)
            if e is not None:
                buf, tw, th, tl = e
                t = torch.from_numpy(buf).cuda()
                keep.append(t)
                setattr(mt, slot, vq.texture_of(t, tw, th, tl))
        tex.append(mt)
    table = ctx.material_table(mats, tex)
    ins = [_padded(p) for p in planes[:3]]
    ss = _padded(ssao[..., None]) if ssao is not None else (None, None)
    outs = [_padded(np.full((h, w, 4), INIT, np.float32)) for _ in range(4 if emissive else 3)]
    si = vq.SurfaceInputs(_image(ins[0][1]), _image(ins[1][1]), _image(ins[2][1]), _image(ss[1], 1) if ssao is not None else vq.null_image())
    gb = vq.GBuffer(*(_image(o[1]) for o in outs), *(() if emissive else (vq.null_image(),)))
    rb, re = rows or (0, h)
    ctx.gbuffer_from_materials(si, table, ambient, gb, alpha_mask=alpha_mask, row_begin=rb, row_end=re)
    torch.cuda.synchronize()
    got = [o[1].cpu().numpy() for o in outs]
    pad_ok = all(bool((o[0][:, w:] == 123.0).all()) for o in outs)
    table.close()
    return got, pad_ok


# unit N and T0 come from rsqrtf (2 ulp) on the device and 1/sqrt on the host: relative error <= EPS each, dot included
EPS = 2.0 ** -21


def check_parity(tag, got, ref, loose=None, residual=None):
    """|delta| <= 1e-4 with NaN (and Inf) exactly at the oracle's positions; the same pixels written.

    `loose` marks pixels whose Gram-Schmidt residual T0 - N (N.T0) is 0 up to rounding in float64 (a tangent parallel or
    antiparallel to N, a zero tangent or normal): the output normal is 0/0 there, so each side only has to stay bounded or be
    NaN (check_degenerate_normals); every other channel is held to the bar.

    `residual` = r = |T0 - N (N.T0)| of the unit interpolants in float64, per pixel. The residual's absolute error is at most
    4 EPS (T0 once, N twice and the dot); normalising it divides that by r, and B = cross(T, N) inherits it, so each side's
    T sx + B sy + N sz moves by at most sqrt(2) 4 EPS / r per component: the normal channels are held to 1e-4 + 12 EPS / r
    (a tangent 1e-3 rad from N: r ~ 1e-3, about 6e-3)."""
    if loose is not None:
        got, ref = [g.copy() for g in got], [r.copy() for r in ref]
        check_degenerate_normals(tag, got[1], ref[1], loose)
        for a in (got[1], ref[1]):
            a[loose & (a[..., 3] != INIT), :3] = 0.0
    for k, (name, g, r) in enumerate(zip(NAMES, got, ref)):
        tol = np.full(g.shape, TOL)
        if residual is not None and k == 1:
            with np.errstate(divide="ignore"):
                tol[..., :3] += (12 * EPS / residual)[..., None]
        assert np.array_equal(g == INIT, r == INIT), f"{tag}/{name}: different pixels written"
        gn, rn = ~np.isfinite(g), ~np.isfinite(r)
        assert np.array_equal(np.isnan(g), np.isnan(r)), f"{tag}/{name}: NaN at {np.argwhere(np.isnan(g) != np.isnan(r))[:5]}"
        assert np.array_equal(np.isinf(g) & (g > 0), np.isinf(r) & (r > 0)) and np.array_equal(np.isinf(g) & (g < 0), np.isinf(r) & (r < 0)), \
            f"{tag}/{name}: Inf positions"
        fin = ~(gn | rn)
        d = np.abs(g[fin].astype(np.float64) - r[fin])
        assert d.size == 0 or (d <= tol[fin]).all(), \
            f"{tag}/{name}: |delta| {d.max():.3e} over the bound at {np.argwhere(fin)[np.argmax(d - tol[fin])]}"


def check_degenerate_normals(tag, g, r, loose):
    """the domain limit of degenerate interpolants, on each side: NaN, or T*s.x + B*s.y + N*s.z with unit T, B, N and a unit s
    whose T is rounding noise not orthogonal to N, so |N| <= |s.x| + |s.y| + |s.z| <= sqrt(3)"""
    for side, a in (("kernel", g), ("oracle", r)):
        n = a[loose & (a[..., 3] != INIT)][:, :3].astype(np.float64)
        ln = np.sqrt((n ** 2).sum(-1))
        ok = np.isnan(ln) | (ln <= np.sqrt(3.0) * (1 + 1e-5))
        assert ok.all(), f"{tag}/{side}: degenerate tangent frame gave |N| = {ln[~ok][:4]}"


# ---- the sampler, through the probes -----------------------------------------------------------------------------------
CASES = sd.sampler_cases()


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_sampler_probes_domain(ctx, case, monkeypatch):
    name, w, h, levels, kind, seed = case
    level0, ru, rv = sd.build_sampler_case(w, h, levels, kind, seed)
    maps = sd.probe_maps(level0, levels)
    planes = sd.planes_from_uv(ru, rv)
    mats = [sd.probe_material()]
    ref = orc.gbuffer_from_materials(planes, mats, [maps], 1.0)
    f64 = sd.probe_ref(maps, ru, rv)
    res = {}
    for records in (True, False):
        got, pad_ok = run_kernel(ctx, planes, mats, [maps], records=records, monkeypatch=monkeypatch)
        assert pad_ok, f"{name}: wrote outside the image"
        check_parity(f"{name}/records={records}", got, ref)
        probes = sd.probe_outputs(got)
        for slot, (val, bound) in f64.items():
            g = probes[slot].astype(np.float64)
            assert np.array_equal(np.isnan(g), np.isnan(val)), f"{name}/{slot}: NaN where the fp32 coordinate rule does not put it"
            g, val, bound = (np.nan_to_num(a) for a in (g, val, bound))
            err = np.abs(g - val)
            assert (err <= bound).all(), f"{name}/{slot}/records={records}: {int((err > bound).sum())} outside the float64 bound"
            key = f"probe {slot} {'records' if records else 'map-by-map'}"
            WORST[key] = max(WORST.get(key, 0.0), float((err / bound).max()))
        res[records] = got
    for name_, a, b in zip(NAMES, res[True], res[False]):
        assert np.array_equal(a, b, equal_nan=True), f"{name}/{name_}: record path differs from the map-by-map path"


@pytest.mark.parametrize("w,u", [(3, 1e9), (3, 4e9), (3, -1e9), (256, 8.4e6), (97, 3e7), (256, -2.0 ** 40)])
def test_coordinates_beyond_int_range_saturate(ctx, w, u, monkeypatch):
    """|u*W - 0.5| >= 2^31: floor(x) saturates to the int range and then wraps, on the device and in the oracle"""
    lvl0 = np.zeros((1, w, 4), np.uint8)
    lvl0[0, :, :3] = (np.arange(w) % 251)[:, None]
    maps = sd.probe_maps(lvl0, 1)
    ru = np.full((2, 2), u, np.float32); rv = np.full((2, 2), 0.5, np.float32)
    x = np.float32(np.float32(np.float32(u) * np.float32(w)) - np.float32(0.5))
    want = (min(max(int(np.floor(float(x))), -2 ** 31), 2 ** 31 - 1) % w) % 251 / 255.0
    planes = sd.planes_from_uv(ru, rv)
    for records in (True, False):
        got, _ = run_kernel(ctx, planes, [sd.probe_material()], [maps], records=records, monkeypatch=monkeypatch)
        for slot, v in sd.probe_outputs(got).items():
            assert np.allclose(v, want, atol=1e-6), (slot, records, v.ravel(), want)


@pytest.mark.parametrize("u,v", [(np.nan, 0.5), (np.inf, 0.5), (0.5, -np.inf), (-np.inf, np.nan)])
def test_non_finite_coordinates_sample_nan(ctx, u, v, monkeypatch):
    """a texel coordinate that is not finite blends to NaN on both paths, and in the oracle (which returned 0 before)"""
    maps = sd.probe_maps(np.full((2, 2, 4), 200, np.uint8), 2)
    planes = sd.planes_from_uv(np.full((2, 2), u, np.float32), np.full((2, 2), v, np.float32))
    mats = [sd.probe_material()]
    ref = orc.gbuffer_from_materials(planes, mats, [maps], 1.0)
    for records in (True, False):
        got, _ = run_kernel(ctx, planes, mats, [maps], records=records, monkeypatch=monkeypatch)
        check_parity(f"nonfinite({u},{v})/records={records}", got, ref)
        for g in sd.probe_outputs(got).values():
            assert np.isnan(g).all()


def test_level_zero_overflow_only(ctx, monkeypatch):
    """u*W overflows fp32 at level 0 but not at level 1 of a 2x2 texture (uv offset 2.5e38, lod 0.5 from the quad): the
    trilinear blend is NaN on both sides"""
    maps = sd.probe_maps(np.full((2, 2, 4), 200, np.uint8), 2)
    d = np.float32(np.sqrt(2.0) / 2)
    ru = np.array([[0.0, d], [0.0, d]], np.float32)
    planes = sd.planes_from_uv(ru, np.full((2, 2), 0.5, np.float32))
    mats = [sd.probe_material(offset=(float(np.float32(2.5e38)), 0.0))]
    ref = orc.gbuffer_from_materials(planes, mats, [maps], 1.0)
    for records in (True, False):
        got, _ = run_kernel(ctx, planes, mats, [maps], records=records, monkeypatch=monkeypatch)
        check_parity(f"overflow-one-level/records={records}", got, ref)
        for g in sd.probe_outputs(got).values():
            assert np.isnan(g).all(), g


@pytest.mark.parametrize("bias", [0.0, 0.75])
@pytest.mark.parametrize("u,v,offset", [(np.nan, 0.5, 0.0), (np.inf, 0.5, 0.0), (0.5, -np.inf, 0.0), (0.0, 0.5, 2.5e38)])
def test_normal_map_at_non_finite_coordinates(ctx, u, v, offset, bias, monkeypatch):
    """a normal-mapped material whose texel coordinate is not finite, or overflows at level 0 only (uv offset 2.5e38 on a
    2x2 map at lod 0.5): the NaN sample fails `length(Normal) < 0.01` and unpacks (ForwardLighting.hlsl:267), so the output
    normal is NaN on both paths and in the oracle"""
    maps = {slot: (orc.texture_mip_chain(np.full((2, 2, 4), c, np.uint8), 2), 2, 2, 2)
            for slot, c in (("normals", 200), ("roughness", 90), ("diffuse", 160))}
    m = _textured_materials(1, 3)[0]
    m.textureConfig = float(TEXCFG_DIFFUSE | TEXCFG_NORMAL | TEXCFG_ROUGHNESS)
    m.normalMapMipBias = bias
    m.uvScaleOffset.z = float(np.float32(offset))
    d = np.float32(np.sqrt(2.0) / 2) if offset else np.float32(0.0)
    ru = np.array([[u, u + d], [u, u + d]], np.float32)
    planes = sd.planes_from_uv(ru, np.full((2, 2), v, np.float32))
    ref = orc.gbuffer_from_materials(planes, [m], [maps], 0.5)
    if not (offset and bias):                                   # with the bias the normal map reads level 1 alone: finite
        assert np.isnan(ref[1][..., :3]).all()
    res = {}
    for records in (True, False):
        got, _ = run_kernel(ctx, planes, [m], [maps], ambient=0.5, records=records, monkeypatch=monkeypatch)
        check_parity(f"normal map at u={u}, v={v}, offset={offset}, bias={bias}/records={records}", got, ref)
        res[records] = got
    for name, a, b in zip(NAMES, res[True], res[False]):
        assert np.array_equal(a, b, equal_nan=True), name


# ---- materials, interpolants, decisions ---------------------------------------------------------------------------------
def _full_map_set(w, h, seed, grey_normals=False):
    rng = np.random.default_rng(seed)
    levels = vq.mip_level_count(w, h)
    d = {}
    for slot in vq.MATERIAL_TEXTURE_SLOTS:
        lvl0 = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        if slot == "diffuse":
            lvl0[..., 3] = rng.integers(0, 6, (h, w))                   # alpha bytes around the 0.01 threshold
            lvl0[: h // 2, :, 3] = rng.integers(0, 256, (h // 2, w))
        if slot == "normals":
            k = rng.integers(0, 4, (h, w))
            lvl0[k == 0, :3] = rng.integers(127, 129, ((k == 0).sum(), 3))   # 2s - 1 ~ 0, exactly 0 at some blends
            lvl0[k == 1, :3] = 0
            lvl0[k == 2, :3] = (128, 128, 255)
            if grey_normals:
                lvl0[..., :3] = rng.integers(127, 129, (h, w, 3))
        d[slot] = (orc.texture_mip_chain(lvl0, levels), w, h, levels)
    return d


def _surface_planes(pw, ph, n_mats, seed, indices=None, smooth=False):
    rng = np.random.default_rng(seed)
    ru = rng.uniform(-3, 3, (ph, pw)).astype(np.float32)
    rv = rng.uniform(-3, 3, (ph, pw)).astype(np.float32)
    if smooth:                                                  # 0.8 texels per pixel of a 16 x 8 map: lod near 0
        ru = (np.arange(pw, dtype=np.float32)[None, :] * np.float32(0.05) - np.float32(1.3)) * np.ones((ph, 1), np.float32)
        rv = (np.arange(ph, dtype=np.float32)[:, None] * np.float32(0.1) - np.float32(0.7)) * np.ones((1, pw), np.float32)
    ru[:, 1::2] += np.float32(0.01); rv[1::2, :] += np.float32(0.02)
    planes = sd.planes_from_uv(ru, rv, 0.0, rng)
    nrm, tan = planes[1], planes[2]
    nrm[..., :3] = rng.normal(size=(ph, pw, 3)) * rng.choice([1.0, 1e-3, 40.0], (ph, pw, 1))
    kind = rng.integers(0, 8, (ph, pw))
    tan[..., :3] = rng.normal(size=(ph, pw, 3))
    tan[kind == 0, :3] = nrm[kind == 0, :3]                                     # parallel
    tan[kind == 1, :3] = -2.0 * nrm[kind == 1, :3]                              # antiparallel
    near = nrm[kind == 2, :3] + 1e-3 * np.linalg.norm(nrm[kind == 2, :3], axis=-1, keepdims=True) * rng.normal(size=((kind == 2).sum(), 3))
    tan[kind == 2, :3] = near                                                    # within ~1e-3 rad of N
    tan[kind == 3, :3] = 0.0                                                     # zero tangent
    nrm[kind == 4, :3] = 0.0                                                     # zero normal
    idx = rng.integers(0, n_mats, (ph, pw)).astype(np.float32) if indices is None else indices
    tan[..., 3] = idx
    n64 = nrm[..., :3].astype(np.float64); t64 = tan[..., :3].astype(np.float64)
    with np.errstate(all="ignore"):
        n64 /= np.linalg.norm(n64, axis=-1, keepdims=True); t64 /= np.linalg.norm(t64, axis=-1, keepdims=True)
        res = np.linalg.norm(t64 - n64 * (n64 * t64).sum(-1, keepdims=True), axis=-1)
    degenerate = (kind == 0) | (kind == 1) | (kind == 3) | (kind == 4)
    return planes, degenerate, np.where(degenerate, np.inf, res)


def _textured_materials(n, seed):
    rng = np.random.default_rng(seed)
    mats = []
    for i in range(n):
        m = vq.MaterialData()
        m.diffuse.x, m.diffuse.y, m.diffuse.z = rng.uniform(0.2, 1, 3)
        m.alpha = 1.0
        m.emissiveColor.x, m.emissiveColor.y, m.emissiveColor.z = rng.uniform(0, 2, 3)
        m.emissiveIntensity = 1.5
        m.roughness, m.metalness = rng.uniform(0.1, 1, 2)
        m.normalMapMipBias = (-20.0, -0.5, 0.0, 0.75, 40.0)[i % 5]
        m.uvScaleOffset.x, m.uvScaleOffset.y, m.uvScaleOffset.z, m.uvScaleOffset.w = 1.0, 1.0, 0.0, 0.0
        m.textureConfig = float(i % 512)
        mats.append(m)
    return mats


@pytest.mark.parametrize("alpha_mask", [False, True])
def test_every_texture_config_both_paths(ctx, alpha_mask, monkeypatch):
    """all 512 textureConfig values over one map set (biases -20 .. 40, grey, zero and flat normals, degenerate interpolants):
    oracle parity, records == map by map, and the alpha discard decided as in float64 outside the undecided set"""
    pw, ph = 128, 64
    maps = _full_map_set(16, 8, 41)
    mats = _textured_materials(512, 42)
    chains = [maps] * 512
    idx = (np.arange(pw * ph) % 512).reshape(ph, pw).astype(np.float32)
    planes, loose, residual = _surface_planes(pw, ph, 512, 43, idx, smooth=True)
    ssao = np.random.default_rng(44).uniform(0, 1, (ph, pw)).astype(np.float32)
    init = [np.full((ph, pw, 4), INIT, np.float32) for _ in range(4)]
    ref = orc.gbuffer_from_materials(planes + [ssao], mats, chains, 0.3, alpha_mask=alpha_mask, init=init)
    res = {}
    for records in (True, False):
        got, pad_ok = run_kernel(ctx, planes, mats, chains, ssao=ssao, alpha_mask=alpha_mask, ambient=0.3, records=records,
                                 monkeypatch=monkeypatch)
        assert pad_ok
        check_parity(f"cfg512/mask={alpha_mask}/records={records}", got, ref, loose, residual)
        res[records] = got
    for name, a, b in zip(NAMES, res[True], res[False]):
        assert np.array_equal(a, b, equal_nan=True), f"{name}: record path differs from the map-by-map path"
    if alpha_mask:
        ch, w, h, levels = maps["diffuse"]
        ddx, ddy = sd.quad_derivs(planes[0][..., 3], planes[1][..., 3])
        a, b = sample_ref(ch, w, h, levels, planes[0][..., 3], planes[1][..., 3], (1, 1), (0, 0), ddx, ddy)
        discard, undecided = alpha_decision(a[:, 3].reshape(ph, pw), b[:, 3].reshape(ph, pw))
        has = (idx.astype(int) & TEXCFG_DIFFUSE) != 0
        gone = (res[True][2] == INIT).all(-1)
        want = discard & has
        bad = (gone != want) & ~undecided
        print(f"alpha discard: {int(want.sum())} discarded, {int((undecided & has).sum())} undecided")
        assert want.sum() > 100
        assert not bad.any(), f"{int(bad.sum())} pixels decided against the float64 alpha"


@pytest.mark.parametrize("index", [-3.0, -0.0, 2.999, 3.0, 1e10, -1e10, np.nan, np.inf])
def test_material_index_domain(ctx, index, monkeypatch):
    """material indices outside the table: saturated conversion, then clamped, on both sides"""
    maps = _full_map_set(8, 8, 5)
    mats = _textured_materials(3, 6)
    for m in mats:
        m.textureConfig = float(TEXCFG_DIFFUSE | TEXCFG_ROUGHNESS | TEXCFG_NORMAL)
        m.normalMapMipBias = 0.0
    mats[1].roughness, mats[2].roughness = 0.25, 0.75
    idx = np.full((6, 10), index, np.float32)
    planes, loose, residual = _surface_planes(10, 6, 3, 7, idx)
    ref = orc.gbuffer_from_materials(planes, mats, [maps] * 3, 0.5)
    got, _ = run_kernel(ctx, planes, mats, [maps] * 3, ambient=0.5, monkeypatch=monkeypatch)
    check_parity(f"material index {index}", got, ref, loose, residual)


def test_partners_with_other_materials_and_null_maps(ctx, monkeypatch):
    """quad partners of a different material, a null SRV in each slot with its flag set, odd image sizes"""
    mats = _textured_materials(8, 8)
    chains = []
    for k in range(7):
        d = _full_map_set(32, 16, 50 + k)
        d[vq.MATERIAL_TEXTURE_SLOTS[k]] = None
        chains.append(d)
    chains.append(_full_map_set(64, 8, 60))
    for m in mats:
        m.textureConfig = float(TEXCFG_DIFFUSE | TEXCFG_NORMAL | TEXCFG_AO | TEXCFG_ROUGHNESS | TEXCFG_METALLIC | TEXCFG_EMISSIVE | TEXCFG_ORM)
    mats[3].uvScaleOffset.x, mats[3].uvScaleOffset.y = -2.0, 0.0
    for pw, ph in ((1, 1), (1, 2), (2, 1), (33, 17), (515, 7)):
        planes, loose, residual = _surface_planes(pw, ph, 8, pw * 100 + ph)
        init = [np.full((ph, pw, 4), INIT, np.float32) for _ in range(4)]
        ref = orc.gbuffer_from_materials(planes, mats, chains, 0.4, init=init)
        for records in (True, False):
            got, pad_ok = run_kernel(ctx, planes, mats, chains, ambient=0.4, records=records, monkeypatch=monkeypatch)
            assert pad_ok
            check_parity(f"partners {pw}x{ph}/records={records}", got, ref, loose, residual)


@pytest.mark.parametrize("rows", [(1, 6), (3, 4), (6, 7), (0, 1), (5, 7)])
def test_row_ranges_and_ssao_wrap(ctx, rows, monkeypatch):
    """row ranges from odd rows, of length 1, at the last row; SSAO read at (x+1, y+1) wrapping at the last row and column;
    pixels outside the range untouched"""
    mats = _textured_materials(2, 9)
    for m in mats:
        m.textureConfig = float(TEXCFG_DIFFUSE | TEXCFG_AO | TEXCFG_ROUGHNESS)
    chains = [_full_map_set(16, 16, 70), _full_map_set(16, 16, 71)]
    pw, ph = 33, 7
    planes, loose, residual = _surface_planes(pw, ph, 2, 72)
    ssao = np.random.default_rng(73).uniform(0, 1, (ph, pw)).astype(np.float32)
    init = [np.full((ph, pw, 4), INIT, np.float32) for _ in range(3)]
    ref = orc.gbuffer_from_materials(planes + [ssao], mats, chains, 0.6, init=init, emissive=False, row_begin=rows[0], row_end=rows[1])
    got, pad_ok = run_kernel(ctx, planes, mats, chains, ssao=ssao, emissive=False, ambient=0.6, rows=rows, monkeypatch=monkeypatch)
    assert pad_ok
    check_parity(f"rows {rows}", got, ref, loose, residual)
    for g in got:
        assert (g[: rows[0]] == INIT).all() and (g[rows[1]:] == INIT).all()


@pytest.mark.parametrize("cfg", [np.nan, np.inf, -1.0, 2.0 ** 31, -np.inf])
def test_texture_config_outside_int_range_is_refused(ctx, cfg):
    mats = _textured_materials(2, 1)
    mats[1].textureConfig = cfg
    with pytest.raises(vq.VqError):
        ctx.material_table(mats, [vq.MaterialTextures(), vq.MaterialTextures()])
    mats[1].textureConfig = 2.0 ** 31 - 128                      # the largest float below 2^31 is accepted
    ctx.material_table(mats, [vq.MaterialTextures(), vq.MaterialTextures()]).close()


# ---- tex_mip6_kernel -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h,levels,fill,misalign", [
    (64, 64, 7, "random", 0), (128, 128, 8, "random", 0), (4096, 4096, 13, "random", 0), (8192, 8192, 14, "255", 0),
    (200, 75, 7, "random", 0), (1000, 3, 2, "random", 0), (129, 257, 8, "random", 0), (97, 41, 4, "random", 0),
    (64, 64, 3, "random", 0), (256, 256, 1, "random", 0), (256, 128, 8, "255", 0), (4288, 200, 8, "random", 0),
    (4288, 200, 8, "255", 0), (128, 64, 7, "random", 4), (260, 36, 6, "random", 4), (8192, 4, 3, "255", 4)])
def test_mip6_bit_exact(ctx, w, h, levels, fill, misalign):
    """one, two and three six-level launches, truncated chains, odd sizes whose later launches take the scalar path (4288 >> 6 =
    67), a source
    4-byte but not 16-byte aligned, and all-255 texels (the carry of box4's 16-bit lanes)"""
    lvl0 = np.full((h, w, 4), 255, np.uint8) if fill == "255" else \
        np.random.default_rng(w * 31 + h).integers(0, 256, (h, w, 4), dtype=np.uint8)
    ref = orc.texture_mip_chain(lvl0, levels)
    assert np.array_equal(ref, mip_chain_ref(lvl0, levels))
    store = torch.zeros(ref.size + 32, dtype=torch.uint8, device="cuda")     # base <= 15 + 4: in bounds for any alignment
    base = (-store.data_ptr()) % 16 + misalign
    t = store[base: base + ref.size]
    assert t.data_ptr() % 16 == misalign % 16
    t[: w * h * 4] = torch.from_numpy(lvl0.reshape(-1).copy()).cuda()
    ctx.texture_build_mips(vq.texture_of(t, w, h, levels))
    torch.cuda.synchronize()
    assert np.array_equal(t.cpu().numpy(), ref)
