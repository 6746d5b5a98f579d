"""No GPU needed: vq_gaussian_blur and vq_gaussian_blur_multi_signal check every argument before they touch the device, so each
refusal below comes back as VQ_ERR_INVALID_ARG with a message naming the cause, even without a context. Also the row plan of a
blur band in front of the post chain (distributed.blur_rows)."""
import ctypes as C
import os
import re

import pytest

import vqengine_b200 as vq
from vqengine_b200.distributed import blur_rows, equal_tiles, post_chain_rows

W, H = 40, 24
FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks


def _img(k, w=W, h=H):
    """a descriptor at a distinct, aligned, never-dereferenced address"""
    return vq.Image((k + 1) << 24, w, h, w * 16)


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(n_ranks):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _frames(n, w=W, h=H):
    return [_img(8 + k, w, h) for k in range(n)]


def _msg():
    return (vq.lib.vq_last_error() or b"").decode()


def _single(src=None, dst=None, size=(W, H), params="ok"):
    p = C.byref(vq.BlurParams(*size)) if params == "ok" else None
    rc = vq.lib.vq_gaussian_blur(None, p, src if src is not None else _img(0), dst if dst is not None else _img(1), None)
    return rc, _msg()


def _multi(outs, rows=None, sig=None, src=None, size=(W, H), params="ok"):
    p = C.byref(vq.BlurParams(*size)) if params == "ok" else None
    arr = (vq.Image * max(len(outs), 1))(*outs)
    rb, re = rows if rows is not None else (0, size[1])
    rc = vq.lib.vq_gaussian_blur_multi_signal(None, p, src if src is not None else _img(0), arr if outs else None, len(outs),
                                              rb, re, C.byref(sig) if sig is not None else None, None)
    return rc, _msg()


def _refused(rc, msg, reason):
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


COMMON = [   # the checks of vq_gaussian_blur_x, with its messages: (name, keyword arguments of both calls, reason)
    ("null params", dict(params=None), "params is null"),
    ("null source", dict(src=vq.Image(None, W, H, W * 16)), "bad image descriptor"),
    ("short source pitch", dict(src=vq.Image(1 << 24, W, H, W * 16 - 16)), "bad image descriptor"),
    ("misaligned source", dict(src=vq.Image((1 << 24) + 8, W, H, W * 16)), "bad image descriptor"),
    ("zero width", dict(size=(0, H)), "blur: image size must be positive"),
    ("negative height", dict(size=(W, -1)), "blur: image size must be positive"),
    ("iImageSizeX beyond the images", dict(size=(W + 1, H)), "blur: iImageSize exceeds the images"),
    ("iImageSizeY beyond the images", dict(size=(W, H + 1)), "blur: iImageSize exceeds the images"),
    ("iImageSize beyond the source", dict(src=_img(0, W - 1, H)), "blur: iImageSize exceeds the images"),
]


@pytest.mark.parametrize("case,kw,reason", COMMON, ids=[c[0] for c in COMMON])
def test_single_refusals(case, kw, reason):
    _refused(*_single(**kw), reason)


def test_single_destination_refusals():
    _refused(*_single(dst=vq.Image(None, W, H, W * 16)), "bad image descriptor")
    _refused(*_single(dst=_img(1, W, H - 1)), "blur: iImageSize exceeds the images")
    _refused(*_single(src=_img(3), dst=_img(3)), "blur: in-place is not supported")


def test_single_valid_arguments_reach_the_context():
    """iImageSize smaller than either image, pitched images: the only refusal is the missing context"""
    for kw in (dict(), dict(size=(1, 1)), dict(src=_img(0, W + 7, H + 3), dst=vq.Image(2 << 24, W, H, W * 16 + 256)),
               dict(size=(W - 5, H - 9))):
        _refused(*_single(**kw), "null context")


@pytest.mark.parametrize("case,kw,reason", COMMON, ids=[c[0] for c in COMMON])
def test_multi_shares_the_single_refusals(case, kw, reason):
    _refused(*_multi(_frames(2), **kw), reason)


MULTI = [
    ("no destination", dict(outs=[]), "null destination list"),
    ("nine destinations", dict(outs=_frames(9)), "1..8 destinations"),
    ("rows past iImageSizeY", dict(outs=_frames(2, W, H + 8), rows=(0, H + 1)), "row range out of bounds"),
    ("rows past a smaller iImageSizeY", dict(outs=_frames(2), size=(W, H - 4), rows=(0, H - 3)), "row range out of bounds"),
    ("negative first row", dict(outs=_frames(2), rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", dict(outs=_frames(2), rows=(9, 8)), "row range out of bounds"),
    ("signal with one destination", dict(outs=_frames(1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", dict(outs=_frames(2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal", dict(outs=_frames(2), sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
    ("bad destination descriptor", dict(outs=_frames(1) + [vq.Image(None, W, H, W * 16)]), "bad image descriptor"),
    ("destination smaller than iImageSize", dict(outs=_frames(2) + [_img(12, W, H - 1)]), "blur: iImageSize exceeds the images"),
    ("destination of another size", dict(outs=_frames(2) + [_img(12, W + 4, H)]), "every destination must have the size of the first"),
]


@pytest.mark.parametrize("case,kw,reason", MULTI, ids=[c[0] for c in MULTI])
def test_multi_refusals(case, kw, reason):
    _refused(*_multi(**kw), reason)


def test_multi_zero_destination_count():
    """a non-null list with n_outs = 0 or negative"""
    for n in (0, -1):
        arr = (vq.Image * 2)(*_frames(2))
        rc = vq.lib.vq_gaussian_blur_multi_signal(None, C.byref(vq.BlurParams(W, H)), _img(0), arr, n, 0, H, None, None)
        _refused(rc, _msg(), "1..8 destinations")


@pytest.mark.parametrize("slot", [0, 2, 7])
def test_source_aliasing_a_destination(slot):
    outs = _frames(8)
    _refused(*_multi(outs, src=outs[slot]), "blur: in-place is not supported")


def test_signal_without_a_peer_flag_array():
    sig = _signal(2)
    sig.flags[1] = None
    _refused(*_multi(_frames(2), sig=sig), "null flag array in the peer signal")


def test_multi_valid_arguments_reach_the_context():
    """with every argument valid (empty ranges, one-rank signals, rows up to a smaller iImageSizeY, destinations larger than
    iImageSize), the only refusal is the missing context"""
    for kw in (dict(outs=_frames(1)), dict(outs=_frames(8), rows=(3, 11)), dict(outs=_frames(3), rows=(7, 7)),
               dict(outs=_frames(1), sig=_signal(1)), dict(outs=_frames(2), rows=(0, 1), sig=_signal(2, 1)),
               dict(outs=_frames(2, W + 3, H + 5), size=(W - 2, H - 6), rows=(H - 7, H - 6))):
        _refused(*_multi(**kw), "null context")


def test_exported_and_bound():
    """every symbol vqcuda_blur.h declares is listed, exported and bound, and vqcuda.h includes the header"""
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    hdr = re.sub(r"/\*.*?\*/", " ", open(os.path.join(root, "include", "vqcuda_blur.h")).read(), flags=re.S)
    declared = sorted(re.findall(r"VQ_API\s+[\w\s\*]*?\b(vq_\w+)\s*\(", hdr))
    assert declared == sorted(vq.BLUR_SYMBOLS) == ["vq_gaussian_blur", "vq_gaussian_blur_multi_signal"]
    assert '#include "vqcuda_blur.h"' in open(os.path.join(root, "include", "vqcuda.h")).read()
    for name in vq.BLUR_SYMBOLS:
        assert getattr(vq.lib, name).argtypes
    for m in ("gaussian_blur2d", "gaussian_blur_multi"):
        assert hasattr(vq.Context, m)


# ---- the row plan: blur band -> post chain band ------------------------------------------------------------------------------
def test_blur_rows_without_sharpening():
    """the tonemapper reads only its own rows: the blur produces exactly the band"""
    for band in [(0, 270), (540, 810), (810, 1080), (0, 1), (1079, 1080), (3, 9)]:
        plan = blur_rows(1080, 1080, band)
        assert plan == {"gaussian_blur": [band], "tonemap": [band]}


def test_blur_rows_with_cas_halo():
    """CAS reads one row each side: the blur's rows are the band plus that halo, clipped at the top and bottom of the frame"""
    assert blur_rows(1080, 1080, (0, 270), cas=True)["gaussian_blur"] == [(0, 271)]            # top
    assert blur_rows(1080, 1080, (540, 810), cas=True)["gaussian_blur"] == [(539, 811)]        # middle
    assert blur_rows(1080, 1080, (810, 1080), cas=True)["gaussian_blur"] == [(809, 1080)]      # bottom
    assert blur_rows(1080, 1080, (5, 6), cas=True)["gaussian_blur"] == [(4, 7)]


@pytest.mark.parametrize("mode", [vq.VQ_ADDRESS_WRAP, vq.VQ_ADDRESS_CLAMP])
def test_blur_rows_with_fsr(mode):
    """with FSR the blur's rows are EASU's source rows of the RCAS halo: two ranges under WRAP at the top and bottom edge"""
    ih, oh = 540, 1080
    con = vq.fsr_easu_con(960, ih, 960, ih, 1920, oh)
    for band in equal_tiles(oh, 4) + [(0, 1), (oh - 1, oh), (500, 501)]:
        plan = blur_rows(ih, oh, band, fsr_con=con, address_mode=mode)
        assert plan["gaussian_blur"] == plan["tonemap"]
        assert list(plan)[0] == "gaussian_blur"
        a, b = band
        src = vq.fsr_easu_source_rows(con, ih, oh, max(a - 1, 0), min(b + 1, oh), address_mode=mode)
        assert plan["gaussian_blur"] == src
        for r0, r1 in plan["gaussian_blur"]:
            assert 0 <= r0 < r1 <= ih
    top = blur_rows(ih, oh, (0, oh // 4), fsr_con=con, address_mode=mode)["gaussian_blur"]
    if mode == vq.VQ_ADDRESS_WRAP:
        assert len(top) == 2 and top[-1][1] == ih       # the wrapped taps above row 0 read the last rows
    else:
        assert top[0][0] == 0 and len(top) == 1


def test_blur_rows_keeps_the_post_chain_plan():
    """the post chain's stages are post_chain_rows's, unchanged, after the blur"""
    con = vq.fsr_easu_con(960, 540, 960, 540, 1920, 1080)
    for args, kw in [((1080, 1080, (100, 300)), {}), ((1080, 1080, (100, 300)), dict(cas=True)),
                     ((540, 1080, (100, 300)), dict(fsr_con=con))]:
        plan = blur_rows(*args, **kw)
        rest = dict(plan)
        del rest["gaussian_blur"]
        assert rest == post_chain_rows(*args, **kw)


def test_blur_rows_of_an_empty_band():
    assert blur_rows(1080, 1080, (7, 7), cas=True) == {"gaussian_blur": [], "tonemap": [], "cas": []}


def test_blur_rows_cover_the_frame():
    """the union of every rank's blur rows covers the frame, and each rank's range is its band plus at most the halo"""
    for n in (1, 2, 3, 4, 8):
        covered = set()
        for a, b in equal_tiles(1080, n):
            (r0, r1), = blur_rows(1080, 1080, (a, b), cas=True)["gaussian_blur"]
            assert r0 == max(a - 1, 0) and r1 == min(b + 1, 1080)
            covered.update(range(r0, r1))
        assert covered == set(range(1080))
