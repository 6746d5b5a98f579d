"""CPU: the references of tests/frame_ref.py against the oracle on every generator of tests/frame_domain.py, and the
generators' own properties (each lands on the branch it names). The kernels meet both in tests/test_frame_domain_gpu.py."""
import numpy as np
import pytest

import frame_domain as fd
import frame_ref as fr


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same_bits(got, want):
    """bit for bit, NaN by position (a NaN's payload is not part of the contract)"""
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(w)
    return np.array_equal(np.isnan(g), nan) and np.array_equal(_bits(g)[~nan], _bits(w)[~nan])


# ---- RGBE encode -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(fd.encode_images()))
def test_rgbe_encode_ref_matches_oracle(orc, name):
    a = fd.encode_images()[name]
    assert np.array_equal(fr.rgbe_encode(a), orc.linear_to_rgbe(a))


def test_rgbe_generators_reach_their_branches(orc):
    walk = fd.rgbe_exponent_walk()
    mc = np.nanmax(walk[..., :3], axis=-1).astype(np.float64)
    e = np.frexp(mc)[1]
    assert e.min() <= -105 and e.max() == 128                 # from the cut-off to the wrapping exponent
    assert set(range(-105, 129)) <= set(e.ravel().tolist())   # every binary exponent in between
    enc = fr.rgbe_encode(walk)
    assert (enc[..., 3][e == 128] == 0).all() and (enc[..., :3][e == 128] != 0).any()   # wrapped: rgb bytes, exponent 0
    cut = fr.rgbe_encode(fd.rgbe_cutoff())[0]
    assert (cut[:10] == 0).all() and (cut[10:, 3] != 0).all()                     # below 1e-32: black; at and above: encoded
    sp = fd.rgbe_specials().reshape(-1, 4)
    for k in range(3):
        assert np.isnan(sp[:, k]).any() and np.isneginf(sp[:, k]).any() and (np.signbit(sp[:, k]) & (sp[:, k] == 0)).any()
    # the nesting of stbiw__max: a NaN in r or g is ignored, in b it is not (maxcomp NaN -> (0, 0, 0, 128)); maxcomp +Inf
    # gives (0, 0, 0, 128) too, -Inf is below the cut-off
    t = fr.rgbe_encode(np.array([[np.nan, 1.0, 0.5, 1], [1.0, np.nan, 0.5, 1], [1.0, 0.5, np.nan, 1],
                                 [np.inf, 1.0, 0.5, 1], [-np.inf, -1.0, -np.inf, 1]], np.float32))
    assert t.tolist() == [[0, 128, 64, 129], [128, 0, 64, 129], [0, 0, 0, 128], [0, 0, 0, 128], [0, 0, 0, 0]]
    # every position of NaN and +-Inf in the special-value image, against the oracle (the bytes vqcuda.h states)
    sp = fd.rgbe_specials()
    assert np.array_equal(fr.rgbe_encode(sp), orc.linear_to_rgbe(sp))


def test_rgbe_encode_decodes_back_within_rgbe_precision():
    """the reference encoder against the reference decoder on finite non-negative inputs: decode(encode(x)) <= x and within
    1/128 of maxcomp, black for maxcomp < 1e-32 and for maxcomp >= 2^127"""
    a = fd.rgbe_exponent_walk()
    a[..., :3] = np.abs(a[..., :3])
    d = fr.rgbe_to_float(fr.rgbe_encode(a))
    mc = a[..., :3].max(axis=-1, keepdims=True).astype(np.float64)
    small = ((mc >= np.float32(1e-32)) & (mc < 2.0 ** 127))[..., 0]
    x = a[..., :3].astype(np.float64)
    assert (d[..., :3][small] <= x[small]).all()
    assert (x[small] - d[..., :3][small] <= mc[small] / 128).all()
    assert (d[..., :3][~small] == 0).all() and (~small).sum() >= 24


# ---- RGBE decode -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(fd.decode_files()))
def test_hdr_decode_ref_matches_oracle(orc, name):
    data = fd.decode_files()[name]
    rc, img, lum = fr.hdr_decode(data)
    orc_rc, orc_img, orc_lum = orc.hdr_decode(data)
    assert rc == 0 and orc_rc == 0
    assert np.array_equal(_bits(img), _bits(orc_img))
    assert _bits(lum) == _bits(np.float32(orc_lum))


@pytest.mark.parametrize("name", sorted(fd.corrupt_files()))
def test_hdr_corrupt_files_refused_everywhere(orc, vq, name):
    data = fd.corrupt_files()[name]
    assert fr.hdr_decode(data)[0] == 5 and orc.hdr_decode(data)[0] == 5
    with pytest.raises(vq.VqError):
        vq.hdr_parse(data)


def test_hdr_decode_generators_reach_their_branches(vq):
    files = fd.decode_files()
    for w in (64, 700, 2049):
        for ex in (0, 16):
            data, px, windows = fd.staging_file(w, 3, ex, seed=w + ex)
            assert data == files[f"staging-w{w}+{ex}"]
            assert windows == [fd.staging_capacity(w) + ex] * 3
            info, offs = vq.hdr_parse(data)
            got = [int(offs[4 * j + 4]) - (int(offs[4 * j]) & ~15) for j in range(3)]
            assert got == windows                                       # the kernel's window, from the host index
            rc, img, _ = fr.hdr_decode(data)
            assert np.array_equal(img, fr.rgbe_to_float(px))
    for name, flat in [("marker-row0-of4", 1), ("marker-row1-of4", 1), ("marker-row3-of4", 1), ("flat-w32768", 1),
                       ("rle-w32767", 0), ("rle-w8", 0)]:
        assert vq.hdr_parse(files[name])[0].flat == flat, name
    data, px = fd.rle_file(129, 2, seed=6, zero_blocks=True)
    assert data == files["rle-w129-zero-blocks"] and np.array_equal(fr.hdr_decode(data)[1], fr.rgbe_to_float(px))


# ---- Mitchell downsize -------------------------------------------------------------------------------------------------
def _tables(vq, c):
    _, iw, ih, ow, oh, _ = c
    return vq.resize_axis_table(iw, ow), vq.resize_axis_table(ih, oh)


TABLE_PAIRS = sorted({(c[1], c[3]) for c in fd.RESIZE_CASES} | {(c[2], c[4]) for c in fd.RESIZE_CASES} |
                     {(i, o) for i in range(1, 25) for o in range(1, i + 1)} | {(7, 5), (14, 10), (4096, 2048), (4096, 1024)})


def test_host_tables_are_stbs_coefficients(vq):
    """the kernels' gather tables (host code) against the coefficients computed from stb's text: same taps, same weight bits"""
    for i, o in TABLE_PAIRS:
        a, b = fr.mitchell_table(i, o), vq.resize_axis_table(i, o)
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]), (i, o)
        assert a[2].shape == b[2].shape and np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32)), (i, o)


def test_resize_cases_land_on_their_side_of_the_span(vq):
    spans = {}
    for c in fd.RESIZE_CASES:
        th, _ = _tables(vq, c)
        spans[c[0]] = fd.block_span(th)
        assert (spans[c[0]] > fd.RESIZE_SPAN) == ("direct" in c[5]), (c, spans[c[0]])
    assert spans["span575"] == 575 and spans["span576"] == 576 and spans["span577"] == 577
    assert 1150 <= spans["span1190"] <= 1250
    assert spans["span577-o65"] == 577 and spans["span576-o64"] == 576 and spans["span577-o64"] == 577
    ratios = {c[1] / c[3] for c in fd.RESIZE_CASES} | {c[2] / c[4] for c in fd.RESIZE_CASES}
    assert min(ratios) == 1 and max(ratios) >= 300
    assert {1, 63, 64, 65} <= {c[3] for c in fd.RESIZE_CASES}
    assert any(c[2] % 4 and c[4] % 4 for c in fd.RESIZE_CASES)


@pytest.mark.parametrize("specials", [False, True], ids=["finite", "inf-nan"])
@pytest.mark.parametrize("case", fd.RESIZE_CASES, ids=[c[0] for c in fd.RESIZE_CASES])
def test_resize_ref_bounds_the_oracle(orc, vq, case, specials):
    name, iw, ih, ow, oh, _ = case
    a = fd.resize_input(iw, ih, seed=iw + 7 * ih, specials=specials)
    th, tv = fr.mitchell_table(iw, ow), fr.mitchell_table(ih, oh)
    ref, bound = fr.resize_ref(a, th, tv)
    got = orc.resize_downsample(a, ow, oh)
    assert np.array_equal(np.isnan(got), np.isnan(ref)) and np.array_equal(np.isposinf(got), np.isposinf(ref))
    assert np.array_equal(np.isneginf(got), np.isneginf(ref))
    fin = np.isfinite(ref)
    assert (np.abs(got[fin] - ref[fin]) <= bound[fin]).all()
    if specials:
        assert np.isnan(ref).any()                                      # Inf meets both lobe signs somewhere


# ---- skydome -----------------------------------------------------------------------------------------------------------
def _sky_hdri(case):
    return fd.sky_hdri(case[4], case[5], seed=case[4] + case[5])


def test_sky_generators_reach_their_branches():
    cases = {c[0]: c for c in fd.sky_cases()}
    negzero_pole = 0
    for name, c in cases.items():
        r = fd.sky_ray(c[1], c[2], c[3])
        if name.startswith("axis"):
            assert c[2] % 2 and c[3] % 2                                  # odd: a pixel centre on the axis
            pole = (r[0] == 0) & (r[2] == 0)
            negzero_pole += int((pole & np.signbit(r[0]) & (r[1] != 0)).any())
        if name.startswith("far"):
            assert fd.sky_fallback(r).all() and (r[3] == 0).all()        # w rounds to 0 in fp32: no direction at all
        if name in ("tiny-w", "huge-ray"):
            assert fd.sky_fallback(r).all()
            d = r[:3].astype(np.float64) / r[3]
            assert np.isfinite(d).all()
    assert negzero_pole >= 2                                              # x = -0, z = +-0 at a pole pixel
    r = fd.sky_ray(cases["seam-minus-x"][1], 161, 91)
    assert ((r[0] < 0) & (r[2] > 0)).any() and ((r[0] < 0) & (r[2] < 0)).any()   # the u = 0 / 1 seam crosses the frame
    assert len([n for n in cases if n.startswith("axis")]) == 24
    assert {(c[4], c[5]) for c in cases.values()} >= {(1, 1), (2, 1), (1, 2), (3, 5), (4096, 2048)}


@pytest.mark.parametrize("case", fd.sky_cases(), ids=[c[0] for c in fd.sky_cases()])
def test_sky_ref_bounds_the_oracle(orc, case):
    name, m, w, h, hw, hh, rows, mk = case
    hdri = _sky_hdri(case)
    mask = fd.sky_mask(mk, w, h, seed=w)
    base = np.full((h, w, 4), -7.0, np.float32)
    ref, bound, written, _ = fr.sky_ref(m, w, h, hdri, rows, mask, base)
    got = orc.skydome(hdri, hw, hh, 1, m, base.copy(), normal_mask=mask, rows=rows)
    assert np.array_equal(got[~written], base[~written])
    d = np.abs(got[..., :3].astype(np.float64) - ref[..., :3])
    assert np.isfinite(got).all() and (d <= bound).all(), (name, float((d - bound).max()))


# ---- reflection composite ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bv", [False, True])
@pytest.mark.parametrize("w,h", fd.COMPOSITE_SIZES[:4])
def test_composite_ref_matches_oracle(orc, w, h, bv):
    s, r, b = fd.composite_planes(w, h, seed=w * 3 + h)
    ref = fr.composite_ref(s, r, b if bv else None)
    got = orc.apply_reflections(s.copy(), r, b if bv else None)
    assert same_bits(got, ref)


def test_composite_planes_cover_the_specials():
    s, r, b = fd.composite_planes(64, 5)
    assert (np.isposinf(s[..., 0]) & np.isneginf(r[..., 0])).any()
    assert set(np.unique(np.nan_to_num(b[..., 3], nan=9.0)).tolist()) == {-1.0, 0.0, 0.25, 1.0, 2.0, 9.0}


# ---- MIN depth pyramid -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("w,h", fd.depth_sizes(), ids=[f"{w}x{h}" for w, h in fd.depth_sizes()])
def test_depth_ref_matches_oracle(orc, vq, w, h):
    d = fd.depth_plane(w, h, seed=w * 7 + h)
    n = vq.depth_pyramid_level_count(w, h)
    want, ties = fr.depth_ref(d, n)
    got = orc.depth_min_pyramid(d)
    assert len(got) == n
    for l in range(n):
        assert fr.depth_equal(got[l], want[l], ties[l]).all(), l


def test_depth_planes_cover_the_specials():
    d = fd.depth_plane(65, 64, seed=3)
    _, ties = fr.depth_ref(d, 7)
    assert ties[1].any()
    assert np.isnan(d).any() and np.isposinf(d).any() and ((d == 0) & np.signbit(d)).any()
    assert ((d != 0) & (np.abs(d) < np.finfo(np.float32).tiny)).any()
    assert fd.RAGGED13 and all(n in range(1, 14) for _, _, n in fd.depth_n_levels())
