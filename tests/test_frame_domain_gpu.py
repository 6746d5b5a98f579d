"""-m gpu: the .hdr codec, the Mitchell downsize, the skydome, the reflection composite and the MIN depth pyramid over the
inputs of tests/frame_domain.py, against the oracle and against the references of tests/frame_ref.py. The codec, the
downsize, the composite and the pyramid bit for bit (NaN by position); the skydome inside its float64 bound."""
import numpy as np
import pytest
import torch

import frame_domain as fd
import frame_ref as fr
from gpu_util import dev, host

pytestmark = pytest.mark.gpu


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same_bits(name, got, want, allowed=None):
    """bit for bit, NaN by position; where `allowed`, `got` must be NaN"""
    g, w = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(w)
    if allowed is not None:
        assert np.isnan(g[allowed]).all(), f"{name}: not NaN where allowed"
        nan = nan | allowed
    bad = (np.isnan(g) != nan) | (~nan & (_bits(g) != _bits(w)))
    assert not bad.any(), f"{name}: {int(bad.sum())} values differ, first at {np.argwhere(bad)[:5].tolist()}: " \
                          f"{g[bad][:5].tolist()} vs {w[bad][:5].tolist()}"


# ---- RGBE --------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", sorted(fd.encode_images()))
def test_rgbe_encode_domain(ctx, orc, name):
    a = fd.encode_images()[name]
    got = host(ctx.hdr_encode_rgbe(dev(a)))
    assert np.array_equal(got, fr.rgbe_encode(a))
    assert np.array_equal(got, orc.linear_to_rgbe(a))


@pytest.mark.parametrize("name", sorted(fd.decode_files()))
def test_hdr_decode_domain(ctx, orc, name):
    data = fd.decode_files()[name]
    rc, ref, lum = fr.hdr_decode(data)
    assert rc == 0
    out, dlum = ctx.hdr_decode(data)
    got = host(out)
    assert np.array_equal(_bits(got), _bits(ref))
    assert _bits(host(dlum))[0] == _bits(lum)
    o_rc, o_img, o_lum = orc.hdr_decode(data)
    assert o_rc == 0 and np.array_equal(_bits(got), _bits(o_img)) and _bits(host(dlum))[0] == _bits(np.float32(o_lum))
    if name.startswith("rle-w2"):                      # the blocking host call: same bytes
        o2 = torch.zeros_like(out)
        assert np.float32(ctx.hdr_load_host(data, o2)) == lum and torch.equal(o2, out)


@pytest.mark.parametrize("name", sorted(fd.corrupt_files()))
def test_hdr_decode_refuses_corrupt_streams(ctx, vq, name):
    with pytest.raises(vq.VqError):
        ctx.hdr_decode(fd.corrupt_files()[name])


def test_hdr_save_round_trip_of_specials(ctx, orc):
    """the whole file of the special-value image, byte for byte, and what decoding it gives back"""
    a = fd.rgbe_specials()
    data = ctx.hdr_save_host(dev(a))
    assert data == orc.hdr_encode(a)
    rc, ref, _ = fr.hdr_decode(data)
    assert rc == 0 and np.array_equal(_bits(ref), _bits(fr.rgbe_to_float(fr.rgbe_encode(a))))


# ---- Mitchell downsize -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("specials", [False, True], ids=["finite", "inf-nan"])
@pytest.mark.parametrize("case", fd.RESIZE_CASES, ids=[c[0] for c in fd.RESIZE_CASES])
def test_resize_domain(ctx, vq, orc, case, specials):
    name, iw, ih, ow, oh, _ = case
    a = fd.resize_input(iw, ih, seed=iw + 7 * ih, specials=specials)
    th, tv = fr.mitchell_table(iw, ow), fr.mitchell_table(ih, oh)
    out = torch.full((oh, ow, 4), -5.0, dtype=torch.float32, device="cuda")
    ctx.image_resize(dev(a), out)
    got = host(out)
    ref, bound = fr.resize_ref(a, th, tv)
    kern, _ = fr.resize_ref(a, th, tv, skip_zero=False)
    # where a zero weight inside an output's taps meets a non-finite input, the kernels add 0 * Inf = NaN (vqcuda.h)
    allowed = np.isnan(kern) & ~np.isnan(ref)
    same_bits(name, got, orc.resize_downsample(a, ow, oh), allowed)
    assert np.array_equal(np.isnan(got), np.isnan(kern)) and np.array_equal(np.where(np.isinf(kern), kern, 0), np.where(np.isinf(got), got, 0))
    fin = np.isfinite(ref) & ~allowed
    d = np.abs(got[fin].astype(np.float64) - ref[fin])
    assert (d <= bound[fin]).all()
    direct = fd.block_span(vq.resize_axis_table(iw, ow)) > fd.RESIZE_SPAN
    print(f"{name}: {'direct' if direct else 'staged'} path, max |delta| / bound {float((d / np.maximum(bound[fin], 1e-300)).max()) if d.size else 0.0:.3f}")


# ---- skydome -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", fd.sky_cases(), ids=[c[0] for c in fd.sky_cases()])
def test_skydome_domain(ctx, vq, orc, case):
    name, m, w, h, hw, hh, rows, mk = case
    hdri = fd.sky_hdri(hw, hh, seed=hw + hh)
    mask = fd.sky_mask(mk, w, h, seed=w)
    base = np.full((h, w, 4), -7.0, np.float32)
    ref, bound, written, pole = fr.sky_ref(m, w, h, hdri, rows, mask, base)
    out = dev(base)
    kw = {"normal_mask": dev(mask)} if mask is not None else {}
    if rows:
        kw.update(row_begin=rows[0], row_end=rows[1])
    ctx.skydome(m, vq.pyramid_of(dev(hdri), hw, hh, 1), out, **kw)
    got = host(out)
    assert np.array_equal(_bits(got[~written]), _bits(base[~written])), "pixels outside the rows or under a surface changed"
    assert np.isfinite(got).all() and (got[written, 3] == 1.0).all()
    d = np.abs(got[..., :3].astype(np.float64) - ref[..., :3])
    over = d > bound
    assert not over.any(), f"{name}: {int(over.sum())} values outside the bound at {np.argwhere(over)[:5].tolist()}, max excess {float((d - bound).max()):.3e}"
    o = orc.skydome(hdri, hw, hh, 1, m, base.copy(), normal_mask=mask, rows=rows)
    assert (np.abs(got[..., :3].astype(np.float64) - o[..., :3]) <= 2 * bound).all()
    frac = float((d[written] / np.maximum(bound[written], 1e-300)).max()) if written.any() else 0.0
    print(f"{name}: max |delta| / bound {frac:.3f}; {int(pole.sum())} exact pole pixels")


# ---- reflection composite ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bv", [False, True], ids=["plain", "bounding-volumes"])
@pytest.mark.parametrize("w,h", fd.COMPOSITE_SIZES, ids=[f"{w}x{h}" for w, h in fd.COMPOSITE_SIZES])
def test_apply_reflections_domain(ctx, orc, w, h, bv):
    """special values in every plane, alphas outside [0, 1] and NaN; 3840 x 2160 runs the grid-stride loop (gy is capped)"""
    s, r, b = fd.composite_planes(w, h, seed=w * 3 + h)
    ref = fr.composite_ref(s, r, b if bv else None)
    ds = dev(s)
    ctx.apply_reflections(ds, dev(r), dev(b) if bv else None)
    got = host(ds)
    same_bits(f"composite{w}x{h}", got, ref)
    if w * h <= 1 << 16:
        same_bits(f"composite{w}x{h} vs oracle", got, orc.apply_reflections(s.copy(), r, b if bv else None))


# ---- MIN depth pyramid -------------------------------------------------------------------------------------------------
def _pyramid(ctx, vq, depth_t, w, h, n):
    total = vq.depth_pyramid_texel_count(w, h, n)
    levels = torch.full((total + 1,), -3.0, dtype=torch.float32, device="cuda")
    ctx.depth_min_pyramid(depth_t, levels, n_levels=n)
    got = host(levels)
    assert got[total] == -3.0, "wrote past the last level"
    return got


def _check_levels(name, got, want, ties, n):
    o = 0
    for l in range(n):
        g = got[o:o + want[l].size].reshape(want[l].shape)
        o += want[l].size
        ok = fr.depth_equal(g, want[l], ties[l])
        assert ok.all(), f"{name} level {l}: {int((~ok).sum())} texels differ, first {np.argwhere(~ok)[:3].tolist()}"


@pytest.mark.parametrize("w,h", fd.depth_sizes(), ids=[f"{w}x{h}" for w, h in fd.depth_sizes()])
def test_depth_min_pyramid_domain(ctx, vq, orc, w, h):
    d = fd.depth_plane(w, h, seed=w * 7 + h)
    n = vq.depth_pyramid_level_count(w, h)
    want, ties = fr.depth_ref(d, n)
    got = _pyramid(ctx, vq, torch.from_numpy(d).cuda(), w, h, n)
    _check_levels(f"{w}x{h}", got, want, ties, n)
    o = 0
    for l, lv in enumerate(orc.depth_min_pyramid(d)):                 # the oracle, under the same rule
        assert fr.depth_equal(got[o:o + lv.size].reshape(lv.shape), lv, ties[l]).all(), l
        o += lv.size


@pytest.mark.parametrize("w,h,n", fd.depth_n_levels(), ids=[f"n{n}" for _, _, n in fd.depth_n_levels()])
def test_depth_min_pyramid_level_counts(ctx, vq, w, h, n):
    """every n_levels on one 13-level shape: one launch up to n = 7, two from n = 8; nothing past level n-1 is written"""
    d = fd.depth_plane(w, h, seed=77)
    want, ties = fr.depth_ref(d, n)
    got = _pyramid(ctx, vq, torch.from_numpy(d).cuda(), w, h, n)
    _check_levels(f"n{n}", got, want, ties, n)


@pytest.mark.parametrize("w,h", [(63, 5), (129, 66), (4097, 3)])
def test_depth_min_pyramid_unaligned_source(ctx, vq, w, h):
    """a source view that starts one column into its allocation: not 16-byte aligned, so the scalar load path"""
    d = fd.depth_plane(w, h, seed=5 + w)
    big = torch.full((h, w + 3), 0.125, dtype=torch.float32, device="cuda")
    big[:, 1:w + 1] = torch.from_numpy(d).cuda()
    view = big[:, 1:w + 1]
    assert view.data_ptr() % 16 != 0
    n = vq.depth_pyramid_level_count(w, h)
    want, ties = fr.depth_ref(d, n)
    _check_levels(f"unaligned{w}x{h}", _pyramid(ctx, vq, view, w, h, n), want, ties, n)
