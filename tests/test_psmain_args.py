"""No GPU needed: vq_forward_lighting_from_materials checks its arguments before it touches the device, so a null material
table, attribute planes or an output of different sizes, and a row range outside the image are refused with
VQ_ERR_INVALID_ARG and a message naming the cause, even without a context (nothing can have been launched)."""
import ctypes as C

import pytest

import vqengine_b200 as vq

W, H = 64, 32
BASE = 1 << 20                                   # descriptor addresses: never dereferenced by the argument checks


def _img(k, w=W, h=H, texel=16):
    return vq.Image(BASE * (k + 1), w, h, w * texel)


def _call(inputs, out, table, row_begin=0, row_end=H):
    pf, pv = vq.PerFrameData(), vq.PerViewLightingData()
    env = vq.EnvironmentMaps()
    rc = vq.lib.vq_forward_lighting_from_materials(None, C.byref(pf), C.byref(pv), C.byref(inputs), table, 0, C.byref(env),
                                                   out, row_begin, row_end, None)
    return rc, (vq.lib.vq_last_error() or b"").decode()


DUMMY_TABLE = C.create_string_buffer(64)         # stands in for a table handle; the cases below are refused before it is read


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
def test_refused_before_the_device(case, reason):
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
    rc, msg = _call(ins, out, table, *rows)
    assert rc == vq.VQ_ERR_INVALID_ARG and reason in msg, (rc, msg)


def test_exported_and_bound():
    assert "vq_forward_lighting_from_materials" in vq.ABI_SYMBOLS
    assert hasattr(vq.Context, "forward_lighting_from_materials")
