"""No GPU needed: vq_post_process and vq_post_process_multi_signal check every argument before they touch the device, so each
refusal below comes back as VQ_ERR_INVALID_ARG with a message naming the cause, even without a context."""
import ctypes as C

import numpy as np
import pytest

import vqengine_b200 as vq

W, H = 40, 24                                    # scene colour; FSR upscales it 2x
FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks
BRANCHES = ("fsr", "cas", "tonemap")


def _img(k, w=W, h=H):
    """a descriptor at a distinct, aligned, never-dereferenced address"""
    return vq.Image((k + 1) << 24, w, h, w * 16)


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(n_ranks):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _display(branch):
    return (2 * W, 2 * H) if branch == "fsr" else (W, H)


def _consts(branch):
    """(cas, easu, rcas) of a branch"""
    if branch == "fsr":
        return None, vq.fsr_easu_con(W, H, W, H, 2 * W, 2 * H), vq.fsr_rcas_con(0.2)
    if branch == "cas":
        return vq.cas_setup(0.5, W, H, W, H), None, None
    return None, None, None


def _single(branch, dst=None, src=None, tm="ok", consts=None, mode=vq.VQ_ADDRESS_WRAP):
    cas, easu, rcas = consts if consts is not None else _consts(branch)
    p = C.byref(vq.TonemapperParams()) if tm == "ok" else None
    rc = vq.lib.vq_post_process(None, p, cas, easu, mode, rcas, src if src is not None else _img(0),
                                dst if dst is not None else _img(1, *_display(branch)), None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


def _multi(branch, outs, rows=None, sig=None, src=None, consts=None, mode=vq.VQ_ADDRESS_WRAP):
    cas, easu, rcas = consts if consts is not None else _consts(branch)
    arr = (vq.Image * max(len(outs), 1))(*outs)
    rb, re = rows if rows is not None else (0, _display(branch)[1])
    rc = vq.lib.vq_post_process_multi_signal(None, C.byref(vq.TonemapperParams()), cas, easu, mode, rcas,
                                             src if src is not None else _img(0), arr, len(outs), rb, re,
                                             C.byref(sig) if sig is not None else None, None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


def _frames(branch, n, size=None):
    w, h = size or _display(branch)
    return [_img(8 + k, w, h) for k in range(n)]


def _refused(rc, msg, reason):
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


def _con(c0, w=W, h=H, ow=2 * W, oh=2 * H):
    con = vq.fsr_easu_con(w, h, w, h, ow, oh)
    for i, v in enumerate(c0):
        con[i] = int(np.float32(v).view(np.uint32))
    return con


# ---- the single-destination call ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("branch", BRANCHES)
def test_null_params_and_descriptors(branch):
    _refused(*_single(branch, tm=None), "params is null")
    _refused(*_single(branch, src=vq.Image(None, W, H, W * 16)), "bad image descriptor")
    _refused(*_single(branch, dst=vq.Image(None, *_display(branch), _display(branch)[0] * 16)), "bad image descriptor")
    _refused(*_single(branch, src=vq.Image(1 << 24, W, H, W * 16 - 16)), "bad image descriptor")     # pitch below a row


@pytest.mark.parametrize("branch,reason", [("cas", "cas: sharpen-only path needs equal sizes"), ("tonemap", "tonemap: in/out size mismatch")])
@pytest.mark.parametrize("dw,dh", [(1, 0), (-1, 0), (0, 1), (0, -1), (W, H)])
def test_size_rules_without_fsr(branch, reason, dw, dh):
    _refused(*_single(branch, dst=_img(1, W + dw, H + dh)), reason)


@pytest.mark.parametrize("branch", ["fsr", "cas"])
def test_in_place_with_a_stencil(branch):
    w, h = _display(branch)
    src = _img(3, W, H)
    _refused(*_single(branch, src=src, dst=vq.Image(src.ptr, w, h, w * 16)), "post_process: in-place is not supported")


def test_tonemapper_alone_may_run_in_place():
    """as vq_tonemap: an aliased output gets past every argument check (refused for want of a context)"""
    _refused(*_single("tonemap", src=_img(3), dst=_img(3)), "null context")


@pytest.mark.parametrize("which", ["easu only", "rcas only"])
def test_easu_and_rcas_go_together(which):
    easu, rcas = vq.fsr_easu_con(W, H, W, H, 2 * W, 2 * H), vq.fsr_rcas_con(0.2)
    consts = (None, easu, None) if which == "easu only" else (None, None, rcas)
    _refused(*_single("fsr", consts=consts), "post_process: easu_const and rcas_const are given together or not at all")


def test_cas_constants_are_ignored_with_fsr():
    """FSR on: CAS's output is never read, so its constants do not matter (refused only for want of a context)"""
    _, easu, rcas = _consts("fsr")
    _refused(*_single("fsr", consts=(vq.cas_setup(0.5, W, H, W, H), easu, rcas)), "null context")


@pytest.mark.parametrize("mode", [-1, 2, 7])
def test_unknown_address_mode(mode):
    _refused(*_single("fsr", mode=mode), "easu: unknown address mode")


@pytest.mark.parametrize("c0,reason", [
    ((float("nan"), 0.5, -0.25, -0.25), "easu: con0 is not finite"),
    ((0.5, 0.5, -0.25, float("inf")), "easu: con0 is not finite"),
    ((0.5, 0.5, -0.25, 30.0), "easu: con0 puts taps outside"),
    ((0.5, 0.5, -60.0, -0.25), "easu: con0 puts taps outside"),
])
def test_easu_verdicts(c0, reason):
    _, _, rcas = _consts("fsr")
    _refused(*_single("fsr", consts=(None, _con(c0), rcas)), reason)


def test_downscaling_path_is_refused():
    """con0 that FsrEasuCon builds for a downscale (scale > 1): the fused kernels have no generic path"""
    ow, oh = 25, 15
    con = vq.fsr_easu_con(W, H, W, H, ow, oh)
    _refused(*_single("fsr", dst=_img(1, ow, oh), consts=(None, con, vq.fsr_rcas_con(0.2))),
             "post_process: con0 is on EASU's downscaling path")


def test_fused_tile_footprint():
    """the up path's footprint rule for the fused tile: at 1:1 beyond 2^24 columns, (float)x rounds to even, so a display tile
    and its ring (32 outputs) span 33 candidate texels (descriptors only: nothing is dereferenced)"""
    wide = 1 << 25
    src = vq.Image(1 << 24, wide, H, wide * 16)
    dst = vq.Image(9 << 24, wide, 2 * H, wide * 16)
    _refused(*_single("fsr", src=src, dst=dst, consts=(None, _con((1.0, 0.5, 0.0, -0.25), wide, H, wide, 2 * H), vq.fsr_rcas_con(0.2))),
             "post_process: con0 needs more than 32x16 input texels per 30x14 display tile and its ring")


@pytest.mark.parametrize("ratio", [1.0, 1 / 1.3, 0.67, 0.58, 0.5])
def test_every_fsr_preset_passes(ratio):
    """FsrEasuCon's constants for the presets at 4K output reach the context"""
    ow, oh = 3840, 2160
    iw, ih = round(ow * ratio), round(oh * ratio)
    con = vq.fsr_easu_con(iw, ih, iw, ih, ow, oh)
    _refused(*_single("fsr", src=_img(0, iw, ih), dst=_img(1, ow, oh), consts=(None, con, vq.fsr_rcas_con(0.2))), "null context")


@pytest.mark.parametrize("branch", BRANCHES)
def test_valid_arguments_reach_the_context(branch):
    _refused(*_single(branch), "null context")


# ---- the multi-destination call -----------------------------------------------------------------------------------------------
CASES = [
    ("null list", lambda b: dict(outs=None), "null destination list"),
    ("no destination", lambda b: dict(outs=[]), "1..8 destinations"),
    ("nine destinations", lambda b: dict(outs=_frames(b, 9)), "1..8 destinations"),
    ("rows past the output", lambda b: dict(outs=_frames(b, 2), rows=(0, _display(b)[1] + 1)), "row range out of bounds"),
    ("negative first row", lambda b: dict(outs=_frames(b, 2), rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", lambda b: dict(outs=_frames(b, 2), rows=(9, 8)), "row range out of bounds"),
    ("signal with one destination", lambda b: dict(outs=_frames(b, 1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", lambda b: dict(outs=_frames(b, 2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal", lambda b: dict(outs=_frames(b, 2), sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
    ("bad destination descriptor", lambda b: dict(outs=_frames(b, 1) + [vq.Image(None, *_display(b), _display(b)[0] * 16)]),
     "bad image descriptor"),
]


@pytest.mark.parametrize("branch", BRANCHES)
@pytest.mark.parametrize("case,kw,reason", CASES, ids=[c[0] for c in CASES])
def test_multi_destination_refusals(branch, case, kw, reason):
    kw = kw(branch)
    if kw["outs"] is None:
        rc = vq.lib.vq_post_process_multi_signal(None, C.byref(vq.TonemapperParams()), *[None] * 2, vq.VQ_ADDRESS_WRAP, None, _img(0),
                                                 None, 1, 0, H, None, None)
        _refused(rc, (vq.lib.vq_last_error() or b"").decode(), reason)
        return
    _refused(*_multi(branch, **kw), reason)


@pytest.mark.parametrize("branch", BRANCHES)
def test_multi_destination_of_another_size(branch):
    w, h = _display(branch)
    reason = {"fsr": "every destination must have the size of the first", "cas": "cas: sharpen-only path needs equal sizes",
              "tonemap": "tonemap: in/out size mismatch"}[branch]
    if branch == "fsr":      # the display size is the first destination's: the odd one comes later
        reason = "every destination must have the size of the first"
        _refused(*_multi(branch, _frames(branch, 2) + [_img(12, w + 1, h)]), reason)
    else:
        _refused(*_multi(branch, [_img(12, w, h + 1)] + _frames(branch, 2)), reason)
        _refused(*_multi(branch, _frames(branch, 2) + [_img(12, w - 1, h)]), "every destination must have the size of the first")


@pytest.mark.parametrize("branch", ["fsr", "cas"])
@pytest.mark.parametrize("slot", [0, 2])
def test_multi_source_aliasing_a_destination(branch, slot):
    outs = _frames(branch, 3)
    _refused(*_multi(branch, outs, src=vq.Image(outs[slot].ptr, W, H, W * 16)), "post_process: in-place is not supported")


def test_multi_constant_checks():
    easu, rcas = vq.fsr_easu_con(W, H, W, H, 2 * W, 2 * H), vq.fsr_rcas_con(0.2)
    _refused(*_multi("fsr", _frames("fsr", 2), consts=(None, easu, None)), "easu_const and rcas_const are given together")
    _refused(*_multi("fsr", _frames("fsr", 2), mode=5), "easu: unknown address mode")
    _refused(*_multi("fsr", _frames("fsr", 2), consts=(None, _con((0.5, 0.5, -0.25, 30.0)), rcas)), "easu: con0 puts taps outside")


@pytest.mark.parametrize("branch", BRANCHES)
def test_multi_valid_arguments_reach_the_context(branch):
    """with every argument valid (empty ranges and one-rank signals included), the only refusal is the missing context"""
    for kw in (dict(outs=_frames(branch, 1)), dict(outs=_frames(branch, 8), rows=(3, 11)), dict(outs=_frames(branch, 3), rows=(7, 7)),
               dict(outs=_frames(branch, 1), sig=_signal(1)), dict(outs=_frames(branch, 2), rows=(0, 1), sig=_signal(2, 1))):
        _refused(*_multi(branch, **kw), "null context")


def test_refusals_launch_nothing():
    n0 = vq.launch_count()
    _single("fsr", tm=None)
    _multi("cas", [])
    assert vq.launch_count() == n0


def test_exported_and_bound():
    for name in ("vq_post_process", "vq_post_process_multi_signal"):
        assert name in vq.ABI_SYMBOLS and hasattr(vq.lib, name)
    for m in ("post_process", "post_process_multi"):
        assert hasattr(vq.Context, m)
