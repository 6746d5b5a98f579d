"""No GPU needed: the band forms of the skydome and the reflection composite (vq_skydome_multi_signal,
vq_apply_reflections_multi_signal) check every argument before they touch the device, so each refusal below comes back as
VQ_ERR_INVALID_ARG with a message naming the cause, even without a context."""
import ctypes as C

import pytest

import vqengine_b200 as vq

W, H = 40, 24                                    # the frame
FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks
CALLS = ("skydome", "composite")


def _img(k, w=W, h=H):
    """a descriptor at a distinct, aligned, never-dereferenced address"""
    return vq.Image((k + 1) << 24, w, h, w * 16)


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(min(n_ranks, 8)):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _frames(n, w=W, h=H):
    return [_img(8 + k, w, h) for k in range(n)]


def _call(which, outs, rows=None, off=0, sig=None, plane="ok", bv=None, matrix="ok", pyr="ok"):
    """plane: the mask (skydome) or the reflection image (composite); "ok" = a whole-frame plane, None = no mask"""
    arr = (vq.Image * max(len(outs), 1))(*outs) if outs is not None else None
    n = len(outs) if outs is not None else 2
    rb, re = rows if rows is not None else (0, H)
    sp = C.byref(sig) if sig is not None else None
    p = _img(1) if plane == "ok" else plane
    if which == "skydome":
        m = C.byref(vq.Matrix()) if matrix == "ok" else None
        hd = vq.Pyramid(1 << 30, 64, 32, 1) if pyr == "ok" else pyr
        rc = vq.lib.vq_skydome_multi_signal(None, m, hd, C.byref(p) if p is not None else None, arr, n, off, rb, re, sp, None)
    else:
        p = p if p is not None else vq.null_image()
        rc = vq.lib.vq_apply_reflections_multi_signal(None, p, C.byref(bv) if bv is not None else None, arr, n, off, rb, re,
                                                      sp, None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


def _refused(rc, msg, reason):
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


PLANE = {"skydome": "the mask plane must be as wide as the frame and hold row_end rows",
         "composite": "the reflection image must be as wide as the frame and hold row_end rows"}
CASES = [
    ("no destination list", lambda: dict(outs=None), "null destination list"),
    ("no destination", lambda: dict(outs=[]), "1..8 destinations"),
    ("nine destinations", lambda: dict(outs=_frames(9)), "1..8 destinations"),
    ("bad destination descriptor", lambda: dict(outs=_frames(1) + [vq.Image(None, W, H, W * 16)]), "bad image descriptor"),
    ("misaligned destination", lambda: dict(outs=_frames(1) + [vq.Image((3 << 24) + 8, W, H, W * 16)]), "bad image descriptor"),
    ("short pitch", lambda: dict(outs=_frames(1) + [vq.Image(3 << 24, W, H, W * 16 - 16)]), "bad image descriptor"),
    ("wider peer", lambda: dict(outs=_frames(2) + [_img(12, W + 1, H)]), "every destination must have the size of the first"),
    ("narrower peer", lambda: dict(outs=_frames(2) + [_img(12, W - 1, H)]), "every destination must have the size of the first"),
    ("taller peer", lambda: dict(outs=_frames(1) + [_img(12, W, H + 1)]), "every destination must have the size of the first"),
    ("shorter peer", lambda: dict(outs=_frames(1) + [_img(12, W, H - 1)]), "every destination must have the size of the first"),
    ("peer is the local frame", lambda: dict(outs=_frames(2) + _frames(1)), "a peer destination must not be the local frame"),
    ("negative offset", lambda: dict(outs=_frames(2), off=-2, rows=(2, 8)), "negative destination row offset"),
    ("rows past the frame", lambda: dict(outs=_frames(2), rows=(0, H + 1), plane=_img(1, W, H + 1)), "row range out of bounds"),
    ("offset rows past the frame", lambda: dict(outs=_frames(2), off=5, rows=(0, H - 4), plane=_img(1, W, H)), "row range out of bounds"),
    ("offset past the frame", lambda: dict(outs=_frames(2), off=H + 1, rows=(0, 0), plane=_img(1, W, 1)), "row range out of bounds"),
    ("negative first row", lambda: dict(outs=_frames(2), rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", lambda: dict(outs=_frames(2), rows=(9, 8)), "row range out of bounds"),
    ("signal with one destination", lambda: dict(outs=_frames(1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", lambda: dict(outs=_frames(2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal index", lambda: dict(outs=_frames(2), sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
    ("nine ranks", lambda: dict(outs=_frames(2), sig=_signal(9)), "bad peer signal descriptor"),
]


@pytest.mark.parametrize("which", CALLS)
@pytest.mark.parametrize("case,kw,reason", CASES, ids=[c[0] for c in CASES])
def test_destination_refusals(which, case, kw, reason):
    _refused(*_call(which, **kw()), reason)


@pytest.mark.parametrize("which", CALLS)
def test_signal_without_a_peer_flag_array(which):
    sig = _signal(3)
    sig.flags[2] = None
    _refused(*_call(which, _frames(3), sig=sig), "null flag array in the peer signal")


@pytest.mark.parametrize("which", CALLS)
@pytest.mark.parametrize("case,plane,rows", [
    ("narrower", _img(1, W - 1, H), (0, H)), ("wider", _img(1, W + 1, H), (0, H)),
    ("fewer rows than row_end", _img(1, W, 7), (2, 8)), ("band one row short", _img(1, W, 5), (0, 6)),
    ("misaligned", vq.Image((1 << 24) + 4, W, H, W * 16), (0, H)), ("short pitch", vq.Image(1 << 24, W, H, W * 16 - 16), (0, H))],
    ids=lambda v: v if isinstance(v, str) else None)
def test_plane_refusals(which, case, plane, rows):
    """the mask / reflection plane: as wide as the frame, rows [0, row_end) present (a band plane may be shorter than the frame)"""
    _refused(*_call(which, _frames(2), rows=rows, plane=plane), PLANE[which])


def test_composite_needs_a_reflection_image():
    _refused(*_call("composite", _frames(2), plane=None), PLANE["composite"])


@pytest.mark.parametrize("bv", [_img(2, W - 1, H), _img(2, W, H - 1), vq.Image((2 << 24) + 4, W, H, W * 16)],
                         ids=["narrower", "fewer rows", "misaligned"])
def test_bounding_volume_refusals(bv):
    _refused(*_call("composite", _frames(2), bv=bv), "the bounding-volume layer must be as wide as the frame and hold row_end rows")


@pytest.mark.parametrize("case,kw", [("no matrix", dict(matrix=None)), ("no HDRI", dict(pyr=vq.Pyramid(None, 64, 32, 1))),
                                     ("empty HDRI", dict(pyr=vq.Pyramid(1 << 30, 0, 32, 1))),
                                     ("too many levels", dict(pyr=vq.Pyramid(1 << 30, 64, 32, 8)))])
def test_skydome_single_call_refusals(case, kw):
    """what vq_skydome refuses (its message)"""
    _refused(*_call("skydome", _frames(2), **kw), "bad arguments")


@pytest.mark.parametrize("which", CALLS)
def test_valid_arguments_reach_the_context(which):
    """with every argument valid (band planes at an offset, empty ranges, one-rank signals, no mask) the only refusal is the
    missing context"""
    for kw in (dict(outs=_frames(1)), dict(outs=_frames(8), rows=(3, 11)), dict(outs=_frames(3), rows=(7, 7)),
               dict(outs=_frames(1), sig=_signal(1)), dict(outs=_frames(2), rows=(0, 1), sig=_signal(2, 1)),
               dict(outs=_frames(3), off=9, rows=(0, 15), plane=_img(1, W, 15)), dict(outs=_frames(2), off=H - 1, rows=(0, 1),
                                                                                     plane=_img(1, W, 1)),
               dict(outs=_frames(2), off=4, rows=(2, 20), plane=_img(1, W, 20)), dict(outs=_frames(2), bv=_img(2, W, H))):
        if which == "composite" or "bv" not in kw:
            _refused(*_call(which, **kw), "null context")
    _refused(*_call("skydome", _frames(2), off=3, rows=(0, H - 3), plane=None), "null context")


def test_exported_and_bound():
    for name in ("vq_skydome_multi_signal", "vq_apply_reflections_multi_signal"):
        assert name in vq.ABI_SYMBOLS and hasattr(vq.lib, name)
    for m in ("skydome_multi", "apply_reflections_multi"):
        assert hasattr(vq.Context, m)
