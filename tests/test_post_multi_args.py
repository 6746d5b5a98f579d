"""No GPU needed: the multi-destination post calls (vq_tonemap_multi_signal, vq_cas_multi_signal, vq_fsr_easu_multi_signal,
vq_fsr_rcas_multi_signal) check every argument before they touch the device, so each refusal below comes back as
VQ_ERR_INVALID_ARG with a message naming the cause, even without a context."""
import ctypes as C

import numpy as np
import pytest

import vqengine_b200 as vq

W, H = 40, 24                                    # source of the same-size passes; EASU upscales it 2x
FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks
CALLS = ("tonemap", "cas", "fsr_easu", "fsr_rcas")


def _img(k, w=W, h=H):
    """a descriptor at a distinct, aligned, never-dereferenced address"""
    return vq.Image((k + 1) << 24, w, h, w * 16)


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(n_ranks):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _out_size(which):
    return (2 * W, 2 * H) if which == "fsr_easu" else (W, H)


def _frames(which, n, size=None):
    w, h = size or _out_size(which)
    return [_img(8 + k, w, h) for k in range(n)]


def _call(which, outs, rows=None, sig=None, src=None, con="ok", mode=vq.VQ_ADDRESS_WRAP, params="ok"):
    src = src if src is not None else _img(0)
    arr = (vq.Image * max(len(outs), 1))(*outs)
    rb, re = rows if rows is not None else (0, _out_size(which)[1])
    sp = C.byref(sig) if sig is not None else None
    if which == "tonemap":
        p = C.byref(vq.TonemapperParams()) if params == "ok" else None
        rc = vq.lib.vq_tonemap_multi_signal(None, p, src, arr, len(outs), rb, re, sp, None)
    elif which == "cas":
        c = vq.cas_setup(0.5, W, H, W, H) if con == "ok" else con
        rc = vq.lib.vq_cas_multi_signal(None, c, src, arr, len(outs), rb, re, sp, None)
    elif which == "fsr_rcas":
        c = vq.fsr_rcas_con(0.2) if con == "ok" else con
        rc = vq.lib.vq_fsr_rcas_multi_signal(None, c, src, arr, len(outs), rb, re, sp, None)
    else:
        c = vq.fsr_easu_con(W, H, W, H, 2 * W, 2 * H) if con == "ok" else con
        rc = vq.lib.vq_fsr_easu_multi_signal(None, c, mode, src, arr, len(outs), rb, re, sp, None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


def _refused(rc, msg, reason):
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


SIZE_MSG = {"tonemap": "tonemap: in/out size mismatch", "cas": "cas: sharpen-only path needs equal sizes",
            "fsr_rcas": "rcas: in/out size mismatch", "fsr_easu": "every destination must have the size of the first"}
CASES = [
    ("no destination", lambda w: dict(outs=[]), "1..8 destinations"),
    ("nine destinations", lambda w: dict(outs=_frames(w, 9)), "1..8 destinations"),
    ("rows past the output", lambda w: dict(outs=_frames(w, 2), rows=(0, _out_size(w)[1] + 1)), "row range out of bounds"),
    ("negative first row", lambda w: dict(outs=_frames(w, 2), rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", lambda w: dict(outs=_frames(w, 2), rows=(9, 8)), "row range out of bounds"),
    ("signal with one destination", lambda w: dict(outs=_frames(w, 1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", lambda w: dict(outs=_frames(w, 2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal", lambda w: dict(outs=_frames(w, 2), sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
    ("bad destination descriptor", lambda w: dict(outs=_frames(w, 1) + [vq.Image(None, *_out_size(w), _out_size(w)[0] * 16)]),
     "bad image descriptor"),
]


@pytest.mark.parametrize("which", CALLS)
@pytest.mark.parametrize("case,kw,reason", CASES, ids=[c[0] for c in CASES])
def test_destination_refusals(which, case, kw, reason):
    _refused(*_call(which, **kw(which)), reason)


@pytest.mark.parametrize("which", CALLS)
@pytest.mark.parametrize("dw,dh", [(1, 0), (-1, 0), (0, 1), (0, -1)])
def test_destination_of_the_wrong_size(which, dw, dh):
    """every destination has the output's size: not narrower, wider, shorter or taller, in any slot"""
    w, h = _out_size(which)
    outs = _frames(which, 2) + [_img(12, w + dw, h + dh)]
    if which == "fsr_easu":
        outs = outs[1:] + outs[:1]           # EASU's output size is the first destination's: put the odd one later
    _refused(*_call(which, outs), SIZE_MSG[which])


@pytest.mark.parametrize("which", CALLS)
def test_signal_without_a_peer_flag_array(which):
    sig = _signal(2)
    sig.flags[1] = None
    _refused(*_call(which, _frames(which, 2), sig=sig), "null flag array in the peer signal")


@pytest.mark.parametrize("which,reason", [("cas", "cas: in-place is not supported"), ("fsr_easu", "easu: in-place is not supported"),
                                          ("fsr_rcas", "rcas: in-place is not supported")])
@pytest.mark.parametrize("slot", [0, 2])
def test_source_aliasing_a_destination(which, reason, slot):
    outs = _frames(which, 3)
    src = vq.Image(outs[slot].ptr, W, H, W * 16) if which == "fsr_easu" else outs[slot]
    _refused(*_call(which, outs, src=src), reason)


def test_tonemap_may_run_in_place():
    """the tonemapper has no in-place rule: an aliased destination gets past every argument check (refused for want of a context)"""
    outs = _frames("tonemap", 2)
    rc, msg = _call("tonemap", outs, src=outs[1])
    _refused(rc, msg, "null context")


@pytest.mark.parametrize("which,reason", [("tonemap", "params is null"), ("cas", "cas_const is null"),
                                          ("fsr_easu", "easu_const is null"), ("fsr_rcas", "rcas_const is null")])
def test_null_constants(which, reason):
    _refused(*_call(which, _frames(which, 2), con=None, params=None), reason)


def test_bad_source_descriptor():
    for which in CALLS:
        _refused(*_call(which, _frames(which, 2), src=vq.Image(None, W, H, W * 16)), "bad image descriptor")


@pytest.mark.parametrize("mode", [-1, 2, 7])
def test_easu_unknown_address_mode(mode):
    _refused(*_call("fsr_easu", _frames("fsr_easu", 2), mode=mode), "easu: unknown address mode")


def _con(c0):
    con = vq.fsr_easu_con(W, H, W, H, 2 * W, 2 * H)
    for i, v in enumerate(c0):
        con[i] = int(np.float32(v).view(np.uint32))
    return con


@pytest.mark.parametrize("c0,reason", [
    ((float("nan"), 0.5, -0.25, -0.25), "easu: con0 is not finite"),
    ((0.5, 0.5, -0.25, float("inf")), "easu: con0 is not finite"),
    ((0.5, 0.5, -0.25, 30.0), "easu: con0 puts taps outside"),
    ((0.5, 0.5, -60.0, -0.25), "easu: con0 puts taps outside"),
])
def test_easu_verdicts(c0, reason):
    """vqeasu::check's verdicts, with the single call's messages"""
    _refused(*_call("fsr_easu", _frames("fsr_easu", 2), con=_con(c0)), reason)


def test_easu_tile_footprint_verdict():
    """the up path's footprint rule: at 1:1 beyond 2^24 columns, (float)x rounds to even, so a 32-wide tile spans 33 candidate
    texels (descriptors only: nothing is dereferenced)"""
    wide = 1 << 25
    src = vq.Image(1 << 24, wide, H, wide * 16)
    outs = [vq.Image((9 + k) << 24, wide, 2 * H, wide * 16) for k in range(2)]
    _refused(*_call("fsr_easu", outs, src=src, con=_con((1.0, 0.5, 0.0, -0.25))),
             "easu: con0 needs more than 32x8 input texels per 32x8 output tile")


@pytest.mark.parametrize("which", CALLS)
def test_valid_arguments_reach_the_context(which):
    """with every argument valid (empty ranges and one-rank signals included), the only refusal is the missing context"""
    for kw in (dict(outs=_frames(which, 1)), dict(outs=_frames(which, 8), rows=(3, 11)), dict(outs=_frames(which, 3), rows=(7, 7)),
               dict(outs=_frames(which, 1), sig=_signal(1)), dict(outs=_frames(which, 2), rows=(0, 1), sig=_signal(2, 1))):
        _refused(*_call(which, **kw), "null context")


def test_exported_and_bound():
    for name in ("vq_tonemap_multi_signal", "vq_cas_multi_signal", "vq_fsr_easu_multi_signal", "vq_fsr_rcas_multi_signal",
                 "vq_fsr_easu_source_rows"):
        assert name in vq.ABI_SYMBOLS and hasattr(vq.lib, name)
    for m in ("tonemap_multi", "cas_multi", "fsr_easu_multi", "fsr_rcas_multi"):
        assert hasattr(vq.Context, m)
