"""No GPU needed: the rules every band call (a *_multi_signal entry point: one rank's rows stored into 1..8 frames, optionally ending
in the in-kernel rendezvous) shares, run over every band call the public headers declare. Each refusal comes back as
VQ_ERR_INVALID_ARG with the same message from every call (a NULL list: the forward calls' own null-argument message), before the
device is touched, so even without a context. The band calls are read from the headers: a new one fails here until it has a row in
CALLS."""
import ctypes as C
import os
import re

import pytest

import vqengine_b200 as vq
from test_psmain_args import DUMMY_TABLE
from test_psmain_shadowed_args import _maps

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADERS = ("vqcuda.h", "vqcuda_prefilter_multi.h", "vqcuda_blur.h")
W, H = 40, 24                                    # the source of every call; EASU upscales it 2x
RES = 8                                          # the diffuse cube
FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks
HDRI = vq.Pyramid(1 << 30, 64, 32, 4)


def _img(k, w=W, h=H, texel=16):
    """a descriptor at a distinct, aligned, never-dereferenced address"""
    return vq.Image((k + 1) << 24, w, h, w * texel)


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(min(n_ranks, 8)):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _frames(n, w=W, h=H, texel=16):
    return [_img(8 + k, w, h, texel) for k in range(n)]


def _cubes(n):
    return [vq.Cubemap((k + 8) << 24, RES, 1) for k in range(n)]


class Band:
    """a band call with valid arguments apart from the destinations, rows, offset and signal under test"""

    def __init__(self, call, dests, rows, offset=False, null_list="null destination list", needs_device=False, past="null context"):
        self.call, self.dests, self.rows, self.offset = call, dests, rows, offset
        self.null_list, self.needs_device, self.past = null_list, needs_device, past

    def __call__(self, ctx=None, outs="ok", n=2, rows=None, off=0, sig=None):
        outs = self.dests(n) if outs == "ok" else outs
        typ = vq.Cubemap if self.dests is _cubes else vq.Image
        arr = (typ * max(len(outs), 1))(*outs) if outs is not None else None
        n = len(outs) if outs is not None else n
        rb, re = rows if rows is not None else (0, self.rows)
        args = [arr, n] + ([off] if self.offset else []) + [rb, re, C.byref(sig) if sig is not None else None, None]
        rc = self.call(ctx, *args)
        return rc, (vq.lib.vq_last_error() or b"").decode()


def _forward(fn, pf, pv, gb, env, *sm):
    return lambda ctx, *a: fn(ctx, C.byref(pf), C.byref(pv), C.byref(gb), C.byref(env), *sm, *a)


_PF, _PV, _ENV = vq.PerFrameData(), vq.PerViewLightingData(), vq.EnvironmentMaps()
_GB = vq.GBuffer(_img(0), _img(1), _img(2), vq.null_image())
_INS = vq.SurfaceInputs(_img(0), _img(1), _img(2), vq.null_image())
_MAPS = _maps()
_TM, _BLUR = vq.TonemapperParams(), vq.BlurParams(W, H)
_DIFFUSE = vq.DiffuseIrradianceParams(0.0, 16, 4, 2)
lib = vq.lib

CALLS = {
    "vq_forward_lighting_multi_signal":
        Band(_forward(lib.vq_forward_lighting_multi_signal, _PF, _PV, _GB, _ENV), _frames, H, offset=True,
             null_list="null parameter block", needs_device=True),
    "vq_forward_lighting_shadowed_multi_signal":
        Band(_forward(lib.vq_forward_lighting_shadowed_multi_signal, _PF, _PV, _GB, _ENV, C.byref(_MAPS)), _frames, H, offset=True,
             null_list="null parameter block"),
    "vq_forward_lighting_from_materials_multi_signal":
        Band(lambda ctx, *a: lib.vq_forward_lighting_from_materials_multi_signal(
                 ctx, C.byref(_PF), C.byref(_PV), C.byref(_INS), C.cast(DUMMY_TABLE, C.c_void_p), 0, C.byref(_ENV), C.byref(_MAPS), *a),
             _frames, H, offset=True, null_list="null argument", past="empty material table"),
    "vq_tonemap_multi_signal":
        Band(lambda ctx, *a: lib.vq_tonemap_multi_signal(ctx, C.byref(_TM), _img(0), *a), _frames, H),
    "vq_cas_multi_signal":
        Band(lambda ctx, *a: lib.vq_cas_multi_signal(ctx, vq.cas_setup(0.5, W, H, W, H), _img(0), *a), _frames, H),
    "vq_fsr_rcas_multi_signal":
        Band(lambda ctx, *a: lib.vq_fsr_rcas_multi_signal(ctx, vq.fsr_rcas_con(0.2), _img(0), *a), _frames, H),
    "vq_fsr_easu_multi_signal":
        Band(lambda ctx, *a: lib.vq_fsr_easu_multi_signal(ctx, vq.fsr_easu_con(W, H, W, H, 2 * W, 2 * H), vq.VQ_ADDRESS_WRAP,
                                                          _img(0), *a),
             lambda n: _frames(n, 2 * W, 2 * H), 2 * H),
    "vq_post_process_multi_signal":
        Band(lambda ctx, *a: lib.vq_post_process_multi_signal(ctx, C.byref(_TM), None, None, vq.VQ_ADDRESS_WRAP, None, _img(0), *a),
             _frames, H),
    "vq_gaussian_blur_multi_signal":
        Band(lambda ctx, *a: lib.vq_gaussian_blur_multi_signal(ctx, C.byref(_BLUR), _img(0), *a), _frames, H),
    "vq_skydome_multi_signal":
        Band(lambda ctx, *a: lib.vq_skydome_multi_signal(ctx, C.byref(vq.Matrix()), vq.Pyramid(1 << 30, 64, 32, 1), None, *a),
             _frames, H, offset=True),
    "vq_apply_reflections_multi_signal":
        Band(lambda ctx, *a: lib.vq_apply_reflections_multi_signal(ctx, _img(1), None, *a), _frames, H, offset=True),
    "vq_diffuse_irradiance_multi_signal":
        Band(lambda ctx, *a: lib.vq_diffuse_irradiance_multi_signal(ctx, C.byref(_DIFFUSE), HDRI, *a), _cubes, 6 * RES),
    "vq_brdf_integration_lut_multi_signal":
        Band(lambda ctx, *a: lib.vq_brdf_integration_lut_multi_signal(ctx, *a[:2], 64, *a[2:]), lambda n: _frames(n, texel=8), H),
}


def _null_flag_array():
    s = _signal(3)
    s.flags[2] = None
    return s


# (rule, keyword arguments of Band.__call__ given the call, reason); reason None: the call's null_list message
RULES = [
    ("null list", lambda b: dict(outs=None), None),
    ("no destination", lambda b: dict(n=0), "1..8 destinations"),
    ("nine destinations", lambda b: dict(n=9), "1..8 destinations"),
    ("bad signal index", lambda b: dict(sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
    ("negative signal index", lambda b: dict(sig=_signal(2, my_index=-1)), "bad peer signal descriptor"),
    ("nine ranks", lambda b: dict(sig=_signal(9)), "bad peer signal descriptor"),
    ("null flag array", lambda b: dict(n=3, sig=_null_flag_array()), "null flag array in the peer signal"),
    ("signal with one destination", lambda b: dict(n=1, sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", lambda b: dict(rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("rows past the source", lambda b: dict(rows=(0, b.rows + 1)), "row range out of bounds"),
    ("negative first row", lambda b: dict(rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", lambda b: dict(rows=(9, 8)), "row range out of bounds"),
]
OFFSET_RULES = [("negative offset", lambda b: dict(off=-2), "negative destination row offset")]


def _cases(device):
    return [(name, rule, kw, reason) for name, b in CALLS.items() if b.needs_device == device
            for rule, kw, reason in RULES + (OFFSET_RULES if b.offset else [])]


def _check(ctx, name, kw, reason):
    b = CALLS[name]
    rc, msg = b(ctx, **kw(b))
    reason = reason or b.null_list
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (name, rc, msg)


def test_every_band_call_has_a_row():
    """every *_multi_signal entry point of the public headers is in CALLS (and so runs every rule below)"""
    declared = set()
    for h in HEADERS:
        text = re.sub(r"/\*.*?\*/", " ", open(os.path.join(ROOT, "include", h)).read(), flags=re.S)
        declared |= set(re.findall(r"VQ_API\s+int\s+(vq_\w+_multi_signal)\s*\(", text))
    assert declared == set(CALLS), set(declared) ^ set(CALLS)


@pytest.mark.parametrize("name,rule,kw,reason", _cases(False), ids=[f"{c[0]}-{c[1]}" for c in _cases(False)])
def test_shared_refusals(name, rule, kw, reason):
    _check(None, name, kw, reason)


@pytest.mark.parametrize("name", [n for n, b in CALLS.items() if not b.needs_device])
def test_valid_arguments_reach_the_context(name):
    """the same arguments without the fault get past every band rule: the only refusal is the missing context (the stand-in
    material table of the from-materials call)"""
    b = CALLS[name]
    for kw in (dict(n=1), dict(n=8), dict(n=2, rows=(3, 5)), dict(n=3, rows=(7, 7)), dict(n=1, sig=_signal(1)),
               dict(n=2, rows=(0, 1), sig=_signal(2, 1))):
        rc, msg = b(None, **kw)
        assert rc == vq.VQ_ERR_INVALID_ARG and b.past in msg, (name, kw, rc, msg)


@pytest.mark.gpu
@pytest.mark.parametrize("name,rule,kw,reason", _cases(True), ids=[f"{c[0]}-{c[1]}" for c in _cases(True)])
def test_shared_refusals_after_the_device(ctx, name, rule, kw, reason):
    """the G-buffer band call activates its context's device before it checks: the same rules with a context (nothing launches)"""
    n0 = vq.launch_count()
    _check(ctx._h, name, kw, reason)
    assert vq.launch_count() == n0
