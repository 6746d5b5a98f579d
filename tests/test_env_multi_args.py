"""No GPU needed: the band forms of K2 and K4 (vq_diffuse_irradiance_multi_signal, vq_brdf_integration_lut_multi_signal) and the
one-launch cube blur (vq_gaussian_blur_cube) check every argument before they touch the device, so each refusal below comes back
as VQ_ERR_INVALID_ARG with a message naming the cause, even without a context."""
import ctypes as C
import os
import re

import pytest

import vqengine_b200 as vq
from vqengine_b200 import distributed as vd

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RES = 8                                          # the diffuse cube
LW, LH = 40, 24                                  # the LUT
FLAGS = 1 << 26                                  # flag-array addresses: never dereferenced by the argument checks
HDRI = vq.Pyramid(1 << 30, 64, 32, 4)


def _signal(n_ranks=2, my_index=0):
    s = vq.PeerSignal()
    for k in range(min(n_ranks, 8)):
        s.flags[k] = FLAGS * (k + 1)
    s.n_ranks, s.my_index, s.epoch = n_ranks, my_index, 1
    return s


def _cubes(n, res=RES, mips=1):
    return [vq.Cubemap((k + 8) << 24, res, mips) for k in range(n)]


def _luts(n, w=LW, h=LH):
    return [vq.Image((k + 8) << 24, w, h, w * 8) for k in range(n)]


def _msg():
    return (vq.lib.vq_last_error() or b"").decode()


def _diffuse(outs, rows=(0, 6 * RES), sig=None, params="ok", hdri=HDRI, n=None):
    p = vq.DiffuseIrradianceParams(0.0, 16, 4, 2) if params == "ok" else params
    arr = (vq.Cubemap * max(len(outs), 1))(*outs) if outs is not None else None
    rc = vq.lib.vq_diffuse_irradiance_multi_signal(None, C.byref(p) if p is not None else None, hdri, arr,
                                                   len(outs) if n is None else n, rows[0], rows[1],
                                                   C.byref(sig) if sig is not None else None, None)
    return rc, _msg()


def _lut(outs, rows=(0, LH), sig=None, samples=64, n=None):
    arr = (vq.Image * max(len(outs), 1))(*outs) if outs is not None else None
    rc = vq.lib.vq_brdf_integration_lut_multi_signal(None, arr, len(outs) if n is None else n, samples, rows[0], rows[1],
                                                     C.byref(sig) if sig is not None else None, None)
    return rc, _msg()


def _blur(a, b):
    rc = vq.lib.vq_gaussian_blur_cube(None, a, b, None)
    return rc, _msg()


def _refused(rc, msg, reason):
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


DIFFUSE = [
    ("no destination list", lambda: dict(outs=None, n=2), "null destination list"),
    ("no destination", lambda: dict(outs=[]), "1..8 destinations"),
    ("nine destinations", lambda: dict(outs=_cubes(9)), "1..8 destinations"),
    ("no params", lambda: dict(outs=_cubes(2), params=None), "params is null"),
    ("no HDRI", lambda: dict(outs=_cubes(2), hdri=vq.Pyramid(None, 64, 32, 4)), "bad HDRI pyramid descriptor"),
    ("two mips", lambda: dict(outs=_cubes(2, mips=2)), "diffuse irradiance cubemap must have 1 mip"),
    ("null local cube", lambda: dict(outs=[vq.Cubemap(None, RES, 1)] + _cubes(1)), "diffuse irradiance cubemap must have 1 mip"),
    ("odd res", lambda: dict(outs=_cubes(2, res=7), rows=(0, 42)), "cubemap resolution must be even"),
    ("src_mip past the pyramid", lambda: dict(outs=_cubes(2), params=vq.DiffuseIrradianceParams(0.0, 16, 4, 4)), "src_mip outside the pyramid"),
    ("rows past the cube", lambda: dict(outs=_cubes(2), rows=(0, 6 * RES + 1)), "row range out of bounds"),
    ("negative first row", lambda: dict(outs=_cubes(2), rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", lambda: dict(outs=_cubes(2), rows=(9, 8)), "row range out of bounds"),
    ("empty grid", lambda: dict(outs=_cubes(2), params=vq.DiffuseIrradianceParams(0.0, 0, 4, 2)), "sample grid out of range"),
    ("grid past 2^24", lambda: dict(outs=_cubes(2), params=vq.DiffuseIrradianceParams(0.0, 4096, 4096, 2)), "sample grid out of range"),
    ("grid past shared memory", lambda: dict(outs=_cubes(2), params=vq.DiffuseIrradianceParams(0.0, 30000, 2, 2)),
     "sample grid does not fit shared memory"),
    ("peer of another res", lambda: dict(outs=_cubes(2) + [vq.Cubemap(12 << 24, RES + 2, 1)]), "every destination cubemap must have the same shape"),
    ("peer with two mips", lambda: dict(outs=_cubes(1) + [vq.Cubemap(12 << 24, RES, 2)]), "every destination cubemap must have the same shape"),
    ("null peer", lambda: dict(outs=_cubes(1) + [vq.Cubemap(None, RES, 1)]), "every destination cubemap must have the same shape"),
    ("peer is the local cube", lambda: dict(outs=_cubes(2) + _cubes(1)), "a peer destination must not be the local cubemap"),
    ("signal with one destination", lambda: dict(outs=_cubes(1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", lambda: dict(outs=_cubes(2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal index", lambda: dict(outs=_cubes(2), sig=_signal(2, my_index=2)), "bad peer signal descriptor"),
    ("nine ranks", lambda: dict(outs=_cubes(2), sig=_signal(9)), "bad peer signal descriptor"),
]


@pytest.mark.parametrize("case,kw,reason", DIFFUSE, ids=[c[0] for c in DIFFUSE])
def test_diffuse_refusals(case, kw, reason):
    _refused(*_diffuse(**kw()), reason)


LUT = [
    ("no destination list", lambda: dict(outs=None, n=2), "null destination list"),
    ("no destination", lambda: dict(outs=[]), "1..8 destinations"),
    ("nine destinations", lambda: dict(outs=_luts(9)), "1..8 destinations"),
    ("null local LUT", lambda: dict(outs=[vq.Image(None, LW, LH, LW * 8)] + _luts(1)), "bad LUT image descriptor"),
    ("misaligned peer", lambda: dict(outs=_luts(1) + [vq.Image((3 << 24) + 4, LW, LH, LW * 8)]), "bad LUT image descriptor"),
    ("short pitch", lambda: dict(outs=_luts(1) + [vq.Image(3 << 24, LW, LH, LW * 8 - 8)]), "bad LUT image descriptor"),
    ("wider peer", lambda: dict(outs=_luts(2) + [vq.Image(12 << 24, LW + 1, LH, LW * 8 + 8)]), "every destination must have the size of the first"),
    ("shorter peer", lambda: dict(outs=_luts(1) + [vq.Image(12 << 24, LW, LH - 1, LW * 8)]), "every destination must have the size of the first"),
    ("peer is the local LUT", lambda: dict(outs=_luts(2) + _luts(1)), "a peer destination must not be the local LUT"),
    ("no samples", lambda: dict(outs=_luts(2), samples=0), "num_samples out of range"),
    ("too many samples", lambda: dict(outs=_luts(2), samples=8193), "num_samples out of range"),
    ("rows past the LUT", lambda: dict(outs=_luts(2), rows=(0, LH + 1)), "row range out of bounds"),
    ("negative first row", lambda: dict(outs=_luts(2), rows=(-1, 4)), "row range out of bounds"),
    ("reversed rows", lambda: dict(outs=_luts(2), rows=(9, 8)), "row range out of bounds"),
    ("signal with one destination", lambda: dict(outs=_luts(1), sig=_signal()), "a rendezvous only makes sense with peer destinations"),
    ("rendezvous over no rows", lambda: dict(outs=_luts(2), rows=(5, 5), sig=_signal()), "a rendezvous needs a non-empty row range"),
    ("bad signal index", lambda: dict(outs=_luts(2), sig=_signal(2, my_index=-1)), "bad peer signal descriptor"),
    ("nine ranks", lambda: dict(outs=_luts(2), sig=_signal(9)), "bad peer signal descriptor"),
]


@pytest.mark.parametrize("case,kw,reason", LUT, ids=[c[0] for c in LUT])
def test_lut_refusals(case, kw, reason):
    _refused(*_lut(**kw()), reason)


@pytest.mark.parametrize("which", ["diffuse", "lut"])
def test_signal_without_a_peer_flag_array(which):
    sig = _signal(3)
    sig.flags[2] = None
    _refused(*(_diffuse(_cubes(3), sig=sig) if which == "diffuse" else _lut(_luts(3), sig=sig)), "null flag array in the peer signal")


CUBE = 6 * 16 * 16 * 16                          # bytes of a 16-texel cube
BLUR = [
    ("null input", lambda: (vq.Cubemap(None, 16, 1), vq.Cubemap(1 << 30, 16, 1)), "null cubemap"),
    ("null output", lambda: (vq.Cubemap(1 << 30, 16, 1), vq.Cubemap(None, 16, 1)), "null cubemap"),
    ("input with two mips", lambda: (vq.Cubemap(1 << 30, 16, 2), vq.Cubemap(1 << 31, 16, 1)), "exactly 1 mip"),
    ("output with no mip", lambda: (vq.Cubemap(1 << 30, 16, 1), vq.Cubemap(1 << 31, 16, 0)), "exactly 1 mip"),
    ("face past the limit", lambda: (vq.Cubemap(1 << 30, 130, 1), vq.Cubemap(1 << 31, 130, 1)), "the face edge must be 1..128"),
    ("empty face", lambda: (vq.Cubemap(1 << 30, 0, 1), vq.Cubemap(1 << 31, 0, 1)), "the face edge must be 1..128"),
    ("resolutions differ", lambda: (vq.Cubemap(1 << 30, 16, 1), vq.Cubemap(1 << 31, 32, 1)), "the same resolution"),
    ("misaligned", lambda: (vq.Cubemap((1 << 30) + 8, 16, 1), vq.Cubemap(1 << 31, 16, 1)), "16-byte aligned"),
    ("output overlaps the input's end", lambda: (vq.Cubemap(1 << 30, 16, 1), vq.Cubemap((1 << 30) + CUBE - 16, 16, 1)),
     "the same cube or not overlap"),
    ("input overlaps the output's end", lambda: (vq.Cubemap((1 << 30) + 16, 16, 1), vq.Cubemap(1 << 30, 16, 1)),
     "the same cube or not overlap"),
]


@pytest.mark.parametrize("case,args,reason", BLUR, ids=[c[0] for c in BLUR])
def test_blur_cube_refusals(case, args, reason):
    _refused(*_blur(*args()), reason)


def test_valid_arguments_reach_the_context():
    """with every argument valid (empty ranges, one-rank signals, adjacent and identical cubes) the only refusal is the missing
    context"""
    for kw in (dict(outs=_cubes(1)), dict(outs=_cubes(8), rows=(3, 11)), dict(outs=_cubes(3), rows=(7, 7)),
               dict(outs=_cubes(1), sig=_signal(1)), dict(outs=_cubes(2), rows=(0, 1), sig=_signal(2, 1)),
               dict(outs=_cubes(2), params=vq.DiffuseIrradianceParams(0.010, 0, 0, 3))):
        _refused(*_diffuse(**kw), "null context")
    for kw in (dict(outs=_luts(1)), dict(outs=_luts(8), rows=(3, 11)), dict(outs=_luts(3), rows=(7, 7)),
               dict(outs=_luts(2), rows=(0, 1), sig=_signal(2, 1)), dict(outs=_luts(1) + [vq.Image(12 << 24, LW, LH, LW * 8 + 64)])):
        _refused(*_lut(**kw), "null context")
    for a, b in ((1 << 30, 1 << 30), (1 << 30, (1 << 30) + CUBE), ((1 << 30) + CUBE, 1 << 30)):
        _refused(*_blur(vq.Cubemap(a, 16, 1), vq.Cubemap(b, 16, 1)), "null context")
    _refused(*_blur(vq.Cubemap(1 << 30, 128, 1), vq.Cubemap(1 << 31, 128, 1)), "null context")
    _refused(*_blur(vq.Cubemap(1 << 30, 1, 1), vq.Cubemap(1 << 31, 1, 1)), "null context")


def test_exported_and_bound():
    """every symbol vqcuda_prefilter_multi.h declares is listed, exported and bound, and vqcuda.h includes the header"""
    hdr = open(os.path.join(ROOT, "include", "vqcuda_prefilter_multi.h")).read()
    declared = sorted(set(re.findall(r"VQ_API\s+[\w\s\*]+?\b(vq_\w+)\s*\(", hdr)))
    assert declared == sorted(vq.PREFILTER_MULTI_SYMBOLS) == sorted(["vq_diffuse_irradiance_multi_signal",
                                                                     "vq_brdf_integration_lut_multi_signal", "vq_gaussian_blur_cube"])
    assert not set(declared) & set(vq.ABI_SYMBOLS)
    for name in declared:
        assert hasattr(vq.lib, name) and getattr(vq.lib, name).argtypes, name
    assert '#include "vqcuda_prefilter_multi.h"' in open(os.path.join(ROOT, "include", "vqcuda.h")).read()
    for m in ("diffuse_irradiance_multi", "brdf_integration_lut_multi", "gaussian_blur_cube"):
        assert hasattr(vq.Context, m)


def test_environment_step_plan():
    """EnvironmentStep's bands: equal diffuse rows and the interleaved specular plan's ranges; each rendezvous its own epoch"""
    world = 3
    cubes = _cubes(world, res=16)
    spec = [vq.Cubemap((k + 20) << 24, 32, 6) for k in range(world)]
    plan = vd.InterleavedSpecularPlan(32, 6, world)
    for r in range(world):
        st = vd.EnvironmentStep(None, HDRI, cubes, cubes[0], spec, r, world)
        assert st.rows == vd.equal_tiles(96, world)[r]
        assert st.spec_ranges == plan.row_ranges(r)
    sig = _signal(3, 1)
    assert vd._signal_at(sig, 0xFFFFFFFF).epoch == 0xFFFFFFFF and vd._signal_at(sig, 1 << 32).epoch == 0
    assert vd._signal_at(sig, 5).my_index == 1 and sig.epoch == 1 and vd._signal_at(None, 5) is None
