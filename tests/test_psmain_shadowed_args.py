"""No GPU needed: vq_forward_lighting_shadowed_from_materials checks every argument before it touches the device, so everything
vq_forward_lighting_from_materials refuses, a null VqShadowMaps, caster counts beyond the cbuffer arrays and shadow maps whose
dimensions the PCF kernel cannot index are refused with VQ_ERR_INVALID_ARG and a message naming the cause, even without a context
(nothing can have been launched)."""
import ctypes as C

import pytest

import vqengine_b200 as vq
from test_psmain_args import DUMMY_TABLE, H, W, _img

MAP = 1 << 24                                    # shadow-map addresses: never dereferenced by the argument checks


def _maps(**kw):
    sm = vq.ShadowMaps()
    sm.point_cubes, sm.point_res = MAP, 8
    sm.spot_maps, sm.spot_width, sm.spot_height = 2 * MAP, 16, 16
    sm.directional_map, sm.directional_width, sm.directional_height = 3 * MAP, 32, 32
    for k, v in kw.items():
        setattr(sm, k, v)
    return sm


def _call(inputs, out, table, sm, row_begin=0, row_end=H, pf=None):
    pf = pf or vq.PerFrameData()
    pv, env = vq.PerViewLightingData(), vq.EnvironmentMaps()
    rc = vq.lib.vq_forward_lighting_shadowed_from_materials(None, C.byref(pf), C.byref(pv), C.byref(inputs), table, 0, C.byref(env),
                                                            C.byref(sm) if sm is not None else None, out, row_begin, row_end, None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


@pytest.mark.parametrize("case,reason", [
    ("null table", "null argument"),
    ("normal plane height", "attribute planes differ in size"),
    ("tangent plane width", "attribute planes differ in size"),
    ("ssao plane size", "bad SSAO plane"),
    ("output height", "the output must have the size"),
    ("output width", "the output must have the size"),
    ("row end past the image", "row range out of bounds"),
    ("negative row begin", "row range out of bounds"),
    ("reversed rows", "row range out of bounds"),
])
def test_refusals_of_the_unshadowed_call_hold(case, reason):
    ins = vq.SurfaceInputs(_img(0), _img(1), _img(2), _img(3, texel=4))
    out, table, rows = _img(4), C.cast(DUMMY_TABLE, C.c_void_p), (0, H)
    if case == "null table":
        table = None
    elif case == "normal plane height":
        ins.normal_v = _img(1, h=H - 1)
    elif case == "tangent plane width":
        ins.tangent_m = _img(2, w=W + 1)
    elif case == "ssao plane size":
        ins.ssao = _img(3, w=W - 1, texel=4)
    elif case == "output height":
        out = _img(4, h=H + 1)
    elif case == "output width":
        out = _img(4, w=W - 2)
    elif case == "row end past the image":
        rows = (0, H + 1)
    elif case == "negative row begin":
        rows = (-1, 4)
    elif case == "reversed rows":
        rows = (5, 4)
    rc, msg = _call(ins, out, table, _maps(), *rows)
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


@pytest.mark.parametrize("case,reason", [
    ("null shadow maps", "null shadow maps"),
    ("point casters beyond the array", "caster counts exceed the cbuffer arrays"),
    ("spot casters beyond the array", "caster counts exceed the cbuffer arrays"),
    ("negative caster count", "caster counts exceed the cbuffer arrays"),
    ("point_res 0", "point shadow cubes need a resolution in 1..16384"),
    ("point_res 16385", "point shadow cubes need a resolution in 1..16384"),
    ("spot width 0", "spot shadow maps need positive dimensions (< 2^31 texels)"),
    ("spot height 0", "spot shadow maps need positive dimensions (< 2^31 texels)"),
    ("spot 2^31 texels", "spot shadow maps need positive dimensions (< 2^31 texels)"),
    ("directional width 0", "directional shadow map needs positive dimensions (< 2^31 texels)"),
    ("directional height 0", "directional shadow map needs positive dimensions (< 2^31 texels)"),
    ("directional 2^31 texels", "directional shadow map needs positive dimensions (< 2^31 texels)"),
])
def test_shadow_arguments_refused_before_the_device(case, reason):
    ins = vq.SurfaceInputs(_img(0), _img(1), _img(2), _img(3, texel=4))
    out, table = _img(4), C.cast(DUMMY_TABLE, C.c_void_p)
    pf = vq.PerFrameData()
    sm = _maps()
    if case == "null shadow maps":
        sm = None
    elif case == "point casters beyond the array":
        pf.Lights.numPointCasters = 6                  # the cbuffer holds 5
    elif case == "spot casters beyond the array":
        pf.Lights.numSpotCasters = 6
    elif case == "negative caster count":
        pf.Lights.numPointCasters = -1
    elif case == "point_res 0":
        sm.point_res = 0
    elif case == "point_res 16385":
        sm.point_res = 16385
    elif case == "spot width 0":
        sm.spot_width = 0
    elif case == "spot height 0":
        sm.spot_height = 0
    elif case == "spot 2^31 texels":
        sm.spot_width, sm.spot_height = 1 << 16, 1 << 15
    elif case == "directional width 0":
        sm.directional_width = 0
    elif case == "directional height 0":
        sm.directional_height = 0
    elif case == "directional 2^31 texels":
        sm.directional_width, sm.directional_height = 1 << 15, 1 << 16
    rc, msg = _call(ins, out, table, sm, pf=pf)
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


def test_unbound_maps_are_not_checked():
    """a map that is not bound is not read, so its dimensions do not matter: the call gets past the shadow checks (and is refused
    later, at the stand-in material table)"""
    ins = vq.SurfaceInputs(_img(0), _img(1), _img(2), _img(3, texel=4))
    sm = _maps(point_cubes=None, point_res=0, spot_maps=None, spot_width=0, directional_map=None, directional_height=-3)
    rc, msg = _call(ins, _img(4), C.cast(DUMMY_TABLE, C.c_void_p), sm)
    assert rc != vq.VQ_OK and "shadow" not in msg and "caster" not in msg, (rc, msg)


def test_exported_and_bound():
    assert "vq_forward_lighting_shadowed_from_materials" in vq.ABI_SYMBOLS
    assert hasattr(vq.Context, "forward_lighting_shadowed_from_materials")
