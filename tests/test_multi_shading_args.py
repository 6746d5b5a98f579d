"""No GPU needed: the multi-destination shadowed and from-materials calls (vq_forward_lighting_shadowed_multi_signal,
vq_forward_lighting_from_materials_multi_signal) check their destinations, row range, signal and shadow maps before they touch the
device, so every refusal below comes back as VQ_ERR_INVALID_ARG with a message naming the cause, even without a context."""
import ctypes as C

import pytest

import vqengine_b200 as vq
from test_psmain_args import DUMMY_TABLE, H, W, _img
from test_psmain_shadowed_args import _maps

FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(n_ranks):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _call(which, outs, offset=0, rows=(0, H), sig=None, sm="bound", pf=None, src_h=H):
    pf = pf or vq.PerFrameData()
    pv, env = vq.PerViewLightingData(), vq.EnvironmentMaps()
    arr = (vq.Image * max(len(outs), 1))(*outs)
    maps = _maps() if sm == "bound" else sm
    smp = C.byref(maps) if maps is not None else None
    sp = C.byref(sig) if sig is not None else None
    if which == "shadowed":
        gb = vq.GBuffer(_img(0, h=src_h), _img(1, h=src_h), _img(2, h=src_h), vq.null_image())
        rc = vq.lib.vq_forward_lighting_shadowed_multi_signal(None, C.byref(pf), C.byref(pv), C.byref(gb), C.byref(env), smp, arr,
                                                              len(outs), offset, rows[0], rows[1], sp, None)
    else:
        ins = vq.SurfaceInputs(_img(0, h=src_h), _img(1, h=src_h), _img(2, h=src_h), vq.null_image())
        rc = vq.lib.vq_forward_lighting_from_materials_multi_signal(None, C.byref(pf), C.byref(pv), C.byref(ins),
                                                                    C.cast(DUMMY_TABLE, C.c_void_p), 0, C.byref(env), smp, arr,
                                                                    len(outs), offset, rows[0], rows[1], sp, None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


def _frames(n, h=H, w=W):
    return [_img(8 + k, w=w, h=h) for k in range(n)]


CASES = [
    ("no destination", dict(outs=[]), "1..8 destinations"),
    ("nine destinations", dict(outs=_frames(9)), "1..8 destinations"),
    ("negative offset", dict(outs=_frames(2), offset=-2), "negative destination row offset"),
    ("narrow destination", dict(outs=_frames(1) + [_img(12, w=W - 1)]), "every destination must be as wide"),
    ("wide destination", dict(outs=[_img(12, w=W + 1)] + _frames(1)), "every destination must be as wide"),
    ("short destination", dict(outs=_frames(2, h=H + 3), offset=4), "hold dst_row_offset + height rows"),
    ("rows past the source", dict(outs=_frames(2), rows=(0, H + 1)), "row range out of bounds"),
    ("signal with one destination", dict(outs=_frames(1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", dict(outs=_frames(2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal", dict(outs=_frames(2), sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
]


@pytest.mark.parametrize("which", ["shadowed", "from_materials"])
@pytest.mark.parametrize("case,kw,reason", CASES, ids=[c[0] for c in CASES])
def test_destination_refusals(which, case, kw, reason):
    rc, msg = _call(which, **kw)
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


@pytest.mark.parametrize("which", ["shadowed", "from_materials"])
def test_signal_without_a_peer_flag_array(which):
    sig = _signal(2)
    sig.flags[1] = None
    rc, msg = _call(which, _frames(2), sig=sig)
    assert rc == vq.VQ_ERR_INVALID_ARG and "null flag array in the peer signal" in msg, (rc, msg)


@pytest.mark.parametrize("which", ["shadowed", "from_materials"])
@pytest.mark.parametrize("case,reason", [
    ("point_res 0", "point shadow cubes need a resolution in 1..16384"),
    ("spot 2^31 texels", "spot shadow maps need positive dimensions (< 2^31 texels)"),
    ("directional height 0", "directional shadow map needs positive dimensions (< 2^31 texels)"),
    ("point casters beyond the array", "caster counts exceed the cbuffer arrays"),
])
def test_shadow_map_refusals(which, case, reason):
    pf = vq.PerFrameData()
    sm = _maps()
    if case == "point_res 0":
        sm.point_res = 0
    elif case == "spot 2^31 texels":
        sm.spot_width, sm.spot_height = 1 << 16, 1 << 15
    elif case == "directional height 0":
        sm.directional_height = 0
    else:
        pf.Lights.numPointCasters = 6
    rc, msg = _call(which, _frames(2), sm=sm, pf=pf)
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


def test_shadowed_call_needs_shadow_maps():
    rc, msg = _call("shadowed", _frames(2), sm=None)
    assert rc == vq.VQ_ERR_INVALID_ARG and "null parameter block" in msg, (rc, msg)


@pytest.mark.parametrize("offset", [1, 3, 7])
def test_odd_offset_refused_from_materials(offset):
    """a band at an odd frame row would pair the frame's rows into quads differently, and so change the texture LOD"""
    rc, msg = _call("from_materials", _frames(2, h=H + 8), offset=offset)
    assert rc == vq.VQ_ERR_INVALID_ARG and "dst_row_offset must be even" in msg, (rc, msg)


def test_odd_offset_accepted_for_the_gbuffer_call():
    """the G-buffer call has no quads: an odd offset passes its checks (and is refused only for want of a context)"""
    rc, msg = _call("shadowed", _frames(2, h=H + 8), offset=3)
    assert rc != vq.VQ_OK and "offset" not in msg and "destination" not in msg, (rc, msg)


def test_unshadowed_from_materials_checks_no_maps():
    """NULL shadow maps is the unshadowed call: it gets past every destination and map check to the stand-in material table"""
    rc, msg = _call("from_materials", _frames(3, h=H + 2), offset=2, sm=None)
    assert rc == vq.VQ_ERR_INVALID_ARG and "empty material table" in msg, (rc, msg)


def test_exported_and_bound():
    for name in ("vq_forward_lighting_shadowed_multi_signal", "vq_forward_lighting_from_materials_multi_signal"):
        assert name in vq.ABI_SYMBOLS and hasattr(vq.lib, name)
    assert hasattr(vq.Context, "forward_lighting_shadowed_multi")
    assert hasattr(vq.Context, "forward_lighting_from_materials_multi")
