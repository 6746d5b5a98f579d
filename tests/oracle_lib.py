"""ctypes/numpy front end of the scalar oracle (oracle/liboracle.so) and of the reference-built
FidelityFX setup functions (oracle/_ref/libffxref.so). TEST INFRASTRUCTURE ONLY: imported by tests/,
__graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs — never by the product.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIB = os.path.join(ORACLE_DIR, "liboracle.so")
REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libffxref.so")

f32 = C.c_float
u32 = C.c_uint32
_fp = np.ctypeslib.ndpointer(dtype=np.float32, flags="C_CONTIGUOUS")


def build(force: bool = False) -> None:
    if force or not os.path.exists(LIB) or any(
            os.path.getmtime(os.path.join(ORACLE_DIR, f)) > os.path.getmtime(LIB)
            for f in os.listdir(ORACLE_DIR) if f.endswith((".cpp", ".h"))):
        subprocess.check_call(["make", "-C", ORACLE_DIR, "-s", "all"])


_lib = None
_ref = None


def lib() -> C.CDLL:
    global _lib
    if _lib is None:
        build()
        _lib = C.CDLL(LIB)
        _lib.orc_ndf_ggx.restype = f32
        _lib.orc_geometry_smith.restype = f32
        _lib.orc_spotlight_intensity.restype = f32
        _lib.orc_aprx.restype = f32
        _lib.orc_cubemap_texel_count.restype = C.c_uint64
        _lib.orc_pyramid_texel_count.restype = C.c_uint64
    return _lib


def ref():
    """The reference's own A_CPU FidelityFX setup functions, or None if oracle/_ref was not built."""
    global _ref
    if _ref is None and os.path.exists(REF_LIB):
        _ref = C.CDLL(REF_LIB)
    return _ref


def _f(a) -> np.ndarray:
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a: np.ndarray):
    return a.ctypes.data_as(C.POINTER(f32))


def cpu_threads() -> int:
    return max(1, os.cpu_count() or 1)


# ---- whole passes ------------------------------------------------------------------------------
def forward_lighting(pf, pv, planes, diff_cube, diff_res, spec_cube, spec_res, spec_mips, lut,
                     row_begin=0, row_end=None, threads=None, out=None) -> np.ndarray:
    pos, nrm, alb = (_f(p) for p in planes[:3])
    em = _f(planes[3]) if len(planes) > 3 else None
    h, w = pos.shape[:2]
    out = np.zeros((h, w, 4), np.float32) if out is None else out
    lutc = _f(lut)
    lib().orc_forward_lighting(C.byref(pf), C.byref(pv), _p(pos), _p(nrm), _p(alb),
                               _p(em) if em is not None else None, w, h,
                               _p(_f(diff_cube)), diff_res, _p(_f(spec_cube)), spec_res, spec_mips,
                               _p(lutc), lutc.shape[1], lutc.shape[0], _p(out),
                               row_begin, h if row_end is None else row_end, threads or cpu_threads())
    return out


def sample_cube(cube, res, mips, dirs, mip) -> np.ndarray:
    """SampleCubeLevel over n directions: dirs (n, 3), mip an int or (n,) ints -> (n, 4)"""
    d = _f(dirs).reshape(-1, 3)
    m = np.ascontiguousarray(np.broadcast_to(np.asarray(mip, dtype=np.int32), (d.shape[0],)))
    out = np.zeros((d.shape[0], 4), np.float32)
    lib().orc_sample_cube_n(_p(_f(cube)), res, mips, _p(d), m.ctypes.data_as(C.POINTER(C.c_int)), C.c_int64(d.shape[0]), _p(out))
    return out


def sample_lut(lut, u, v) -> np.ndarray:
    """SampleLUT (bilinear CLAMP) of a [H, W, 2] LUT at n coordinates -> (n, 2)"""
    l = _f(lut)
    uv = _f(np.stack(np.broadcast_arrays(np.asarray(u, np.float32).ravel(), np.asarray(v, np.float32).ravel()), axis=1))
    out = np.zeros((uv.shape[0], 2), np.float32)
    lib().orc_sample_lut_n(_p(l), l.shape[1], l.shape[0], _p(uv), C.c_int64(uv.shape[0]), _p(out))
    return out


def hdri_build_mips(level0: np.ndarray, levels: int) -> np.ndarray:
    h, w = level0.shape[:2]
    n = int(lib().orc_pyramid_texel_count(w, h, levels))
    pyr = np.zeros((n, 4), np.float32)
    pyr[: w * h] = _f(level0).reshape(-1, 4)
    lib().orc_hdri_build_mips(_p(pyr), w, h, levels)
    return pyr


def diffuse_irradiance(pyr, w, h, levels, res, step=0.0, n_phi=64, n_theta=16, src_mip=3,
                       row_begin=0, row_end=None, threads=None, f64_accum=False) -> np.ndarray:
    out = np.zeros((6 * res * res, 4), np.float32)
    lib().orc_diffuse_irradiance(_p(_f(pyr)), w, h, levels, f32(step), n_phi, n_theta, src_mip, _p(out), res,
                                 row_begin, 6 * res if row_end is None else row_end, threads or cpu_threads(), int(f64_accum))
    return out


def specular_prefilter(pyr, w, h, levels, res, mips, num_samples=512, row_begin=0, row_end=None, threads=None):
    n = int(lib().orc_cubemap_texel_count(res, mips))
    out = np.zeros((n, 4), np.float32)
    total = lib().orc_cubemap_row_count(res, mips)
    lib().orc_specular_prefilter(_p(_f(pyr)), w, h, levels, _p(out), res, mips, num_samples,
                                 row_begin, total if row_end is None else row_end, threads or cpu_threads())
    return out


def specular_prefilter_texels(pyr, w, h, levels, res, mips, texels, num_samples=512, threads=None) -> np.ndarray:
    """K3 on a list of flattened texel indices of the packed cube -> (n, 4)"""
    t = np.ascontiguousarray(texels, dtype=np.int64)
    out = np.zeros((t.size, 4), np.float32)
    lib().orc_specular_prefilter_texels(_p(_f(pyr)), w, h, levels, res, mips, num_samples,
                                        t.ctypes.data_as(C.POINTER(C.c_int64)), int(t.size), _p(out), threads or cpu_threads())
    return out


def specular_prefilter_sensitivity(pyr, w, h, levels, res, mips, texels, num_samples=512, rel_eps=2.0 ** -21, threads=None) -> np.ndarray:
    """per texel: how far the oracle's own K3 result moves under a few-ulp (rel_eps radians) tilt of the look direction -> (n,)"""
    t = np.ascontiguousarray(texels, dtype=np.int64)
    out = np.zeros((t.size,), np.float32)
    lib().orc_specular_prefilter_sensitivity(_p(_f(pyr)), w, h, levels, res, mips, num_samples,
                                             t.ctypes.data_as(C.POINTER(C.c_int64)), int(t.size), f32(rel_eps), _p(out),
                                             threads or cpu_threads())
    return out


def brdf_integration_lut(w, h, samples=2048, row_begin=0, row_end=None, threads=None) -> np.ndarray:
    out = np.zeros((h, w, 2), np.float32)
    lib().orc_brdf_integration_lut(_p(out), w, h, samples, row_begin, h if row_end is None else row_end,
                                   threads or cpu_threads())
    return out


def gaussian_blur(img, vertical: bool, threads=None) -> np.ndarray:
    img = _f(img)
    out = np.zeros_like(img)
    lib().orc_gaussian_blur(_p(img), _p(out), img.shape[1], img.shape[0], int(vertical), threads or cpu_threads())
    return out


def tonemap(params, img, threads=None) -> np.ndarray:
    img = _f(img)
    out = np.zeros_like(img)
    lib().orc_tonemap(C.byref(params), _p(img), _p(out), img.shape[1], img.shape[0], threads or cpu_threads())
    return out


def cas(con, img, threads=None) -> np.ndarray:
    img = _f(img)
    out = np.zeros_like(img)
    lib().orc_cas(con, _p(img), _p(out), img.shape[1], img.shape[0], threads or cpu_threads())
    return out


def fsr_easu(con, img, out_w, out_h, address_mode=0, threads=None) -> np.ndarray:
    img = _f(img)
    out = np.zeros((out_h, out_w, 4), np.float32)
    lib().orc_fsr_easu(con, address_mode, _p(img), img.shape[1], img.shape[0], _p(out), out_w, out_h,
                       threads or cpu_threads())
    return out


def fsr_rcas(con, img, threads=None) -> np.ndarray:
    img = _f(img)
    out = np.zeros_like(img)
    lib().orc_fsr_rcas(con, _p(img), _p(out), img.shape[1], img.shape[0], threads or cpu_threads())
    return out


def spd_downsample(img, mips: int):
    img = _f(img)
    h, w = img.shape[:2]
    sizes = [(w >> l, h >> l) for l in range(1, mips + 1) if (w >> l) >= 1 and (h >> l) >= 1]
    packed = np.zeros((sum(a * b for a, b in sizes), 4), np.float32)
    lib().orc_spd_downsample(_p(img), w, h, mips, _p(packed))
    out, o = [], 0
    for (lw, lh) in sizes:
        out.append(packed[o:o + lw * lh].reshape(lh, lw, 4))
        o += lw * lh
    return out


# ---- setup functions ---------------------------------------------------------------------------
def cas_setup(sharp, iw, ih, ow, oh, which="oracle"):
    con = (u32 * 8)()
    fn = lib().orc_cas_setup if which == "oracle" else ref().ref_cas_setup
    fn(con, f32(sharp), f32(iw), f32(ih), f32(ow), f32(oh))
    return con


def fsr_easu_con(vw, vh, iw, ih, ow, oh, which="oracle"):
    con = (u32 * 16)()
    fn = lib().orc_fsr_easu_con if which == "oracle" else ref().ref_fsr_easu_con
    fn(con, f32(vw), f32(vh), f32(iw), f32(ih), f32(ow), f32(oh))
    return con


def fsr_rcas_con(stops, which="oracle"):
    con = (u32 * 4)()
    fn = lib().orc_fsr_rcas_con if which == "oracle" else ref().ref_fsr_rcas_con
    fn(con, f32(stops))
    return con


def spd_setup(rect, mips=-1, which="oracle"):
    d, o, n = (u32 * 2)(), (u32 * 2)(), (u32 * 2)()
    r = (u32 * 4)(*rect)
    fn = lib().orc_spd_setup if which == "oracle" else ref().ref_spd_setup
    fn(d, o, n, r, mips)
    return list(d), list(o), list(n)


# ---- SURVEY §8(f).1 surface producer ---------------------------------------------------------------
class _OrcTexture2D(C.Structure):
    _fields_ = [("ptr", C.c_void_p), ("width", C.c_int32), ("height", C.c_int32), ("levels", C.c_int32)]


class _OrcMaterialTextures(C.Structure):
    _fields_ = [("t", _OrcTexture2D * 7)]


def texture_mip_chain(level0: np.ndarray, levels: int = None) -> np.ndarray:
    """[H,W,4] uint8 -> packed RGBA8 mip chain (flat uint8), DXGIUtils.cpp:263-287 box filter"""
    h, w = level0.shape[:2]
    import vqengine_b200 as vq
    levels = vq.mip_level_count(w, h) if levels is None else levels
    n = vq.pyramid_texel_count(w, h, levels)
    buf = np.zeros(n * 4, np.uint8)
    buf[: w * h * 4] = np.ascontiguousarray(level0).reshape(-1)
    lib().orc_texture_build_mips(buf.ctypes.data_as(C.c_void_p), w, h, levels)
    return buf


def gbuffer_from_materials(planes, materials, chains, ambient_factor: float, alpha_mask: bool = False, emissive: bool = True,
                           init=None, row_begin=0, row_end=None, threads=None):
    """planes = [position_u, normal_v, tangent_m(, ssao)]; chains = list of dict slot -> (packed uint8 chain, w, h, levels) or None.
    Returns [position_ao, normal_roughness, albedo_metalness(, emissive)]; `init` pre-fills the outputs (alpha-mask discard)."""
    import vqengine_b200 as vq
    h, w = planes[0].shape[:2]
    n = len(materials)
    mats = (vq.MaterialData * n)(*materials)
    tex = (_OrcMaterialTextures * n)()
    for i, d in enumerate(chains):
        for k, slot in enumerate(vq.MATERIAL_TEXTURE_SLOTS):
            e = d.get(slot)
            if e is not None:
                buf, tw, th, tl = e
                tex[i].t[k] = _OrcTexture2D(buf.ctypes.data, tw, th, tl)
    outs = [np.zeros((h, w, 4), np.float32) if init is None else np.array(init[i], np.float32, copy=True)
            for i in range(4 if emissive else 3)]
    ssao = planes[3] if len(planes) > 3 and planes[3] is not None else None
    fp = lambda a: a.ctypes.data_as(C.c_void_p) if a is not None else None
    p0, p1, p2 = _f(planes[0]), _f(planes[1]), _f(planes[2])
    ssao = _f(ssao) if ssao is not None else None
    lib().orc_gbuffer_from_materials(fp(p0), fp(p1), fp(p2), fp(ssao), w, h,
                                     mats, tex, n, C.c_float(ambient_factor), 1 if alpha_mask else 0,
                                     fp(outs[0]), fp(outs[1]), fp(outs[2]), fp(outs[3]) if emissive else None,
                                     row_begin, h if row_end is None else row_end, threads or cpu_threads())
    return outs


def sample_texture8(chain, w, h, levels, u, v, ddx=(0.0, 0.0), ddy=(0.0, 0.0), bias=0.0):
    out = np.zeros(4, np.float32)
    lod = C.c_float(0)
    ptr = chain.ctypes.data_as(C.c_void_p) if chain is not None else None
    lib().orc_sample_texture8(ptr, w, h, levels, f32(u), f32(v), f32(ddx[0]), f32(ddx[1]), f32(ddy[0]), f32(ddy[1]),
                              f32(bias), _p(out), C.byref(lod))
    return out, lod.value


def unpack_normal(sampled, n, t):
    out = np.zeros(3, np.float32)
    lib().orc_unpack_normal(_p(_f(sampled)), _p(_f(n)), _p(_f(t)), _p(out))
    return out


# ---- §8(f).2 Radiance .hdr codec / §8(f).3 skydome + ApplyReflections (oracle_frame.cpp) ---------------------------
STB_REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libstbref.so")
_stb = None


def stb_ref():
    """The reference's own vendored stb_image / stb_image_write .hdr codec (oracle/_ref/libstbref.so), or None."""
    global _stb
    if _stb is None and os.path.exists(STB_REF_LIB):
        _stb = C.CDLL(STB_REF_LIB)
        _stb.stbref_write_hdr.restype = C.c_uint64
    return _stb


def _bytes_ptr(b: np.ndarray):
    return b.ctypes.data_as(C.POINTER(C.c_uint8))


def hdr_decode(file_bytes, which: str = "oracle"):
    """-> (rc, rgba float32 [h,w,4] or None, max_luminance). rc: 0 ok, else the stb failure class (oracle) / 1 (ref)."""
    buf = np.frombuffer(bytes(file_bytes), dtype=np.uint8).copy()
    w, h = C.c_int(0), C.c_int(0)
    if which == "ref":
        r = stb_ref()
        if not r.stbref_loadf(_bytes_ptr(buf), C.c_int(buf.size), C.byref(w), C.byref(h), None):
            return 1, None, None
        out = np.empty((h.value, w.value, 4), dtype=np.float32)
        r.stbref_loadf(_bytes_ptr(buf), C.c_int(buf.size), C.byref(w), C.byref(h), _p(out))
        return 0, out, None
    L = lib()
    rc = L.orc_hdr_decode(_bytes_ptr(buf), C.c_uint64(buf.size), C.byref(w), C.byref(h), None, None)
    if rc:
        return rc, None, None
    out = np.empty((h.value, w.value, 4), dtype=np.float32)
    lum = f32(0)
    L.orc_hdr_decode(_bytes_ptr(buf), C.c_uint64(buf.size), C.byref(w), C.byref(h), _p(out), C.byref(lum))
    return 0, out, lum.value


def hdr_encode(rgba, which: str = "oracle") -> bytes:
    a = _f(rgba)
    h, w = a.shape[:2]
    cap = 256 + w * h * 6 + h * 8
    out = np.empty(cap, dtype=np.uint8)
    if which == "ref":
        n = stb_ref().stbref_write_hdr(_p(a), C.c_int(w), C.c_int(h), _bytes_ptr(out), C.c_uint64(cap))
    else:
        L = lib()
        L.orc_hdr_encode.restype = C.c_uint64
        n = L.orc_hdr_encode(_p(a), C.c_int(w), C.c_int(h), _bytes_ptr(out), C.c_uint64(cap))
    assert n <= cap
    return out[:n].tobytes()


def linear_to_rgbe(rgba) -> np.ndarray:
    a = _f(rgba).reshape(-1, 4)
    out = np.empty((a.shape[0], 4), dtype=np.uint8)
    lib().orc_linear_to_rgbe(_p(a), C.c_int(a.shape[0]), _bytes_ptr(out))
    return out.reshape(np.asarray(rgba).shape[:-1] + (4,))


def skydome(hdri_pyramid, hw, hh, levels, inv_view_proj, scene, normal_mask=None, rows=None, threads=0):
    """scene [h,w,4] is updated in place where normal_mask.xyz == 0 (everywhere if normal_mask is None)."""
    import vqengine_b200 as vq  # struct definitions only (VqMatrix)
    h, w = scene.shape[:2]
    m = vq.Matrix((f32 * 16)(*[float(x) for x in np.asarray(inv_view_proj, dtype=np.float32).reshape(16)]))
    rb, re = rows if rows else (0, h)
    py = _f(hdri_pyramid)
    nm = _f(normal_mask) if normal_mask is not None else None
    lib().orc_skydome(_p(py), C.c_int(hw), C.c_int(hh), C.c_int(levels), C.byref(m), _p(nm) if nm is not None else None,
                      _p(scene), C.c_int(w), C.c_int(h), C.c_int(rb), C.c_int(re), C.c_int(threads or (os.cpu_count() or 1)))
    return scene


def apply_reflections(scene, reflection, bounding_volumes=None, threads=0):
    h, w = scene.shape[:2]
    refl = _f(reflection)
    bv = _f(bounding_volumes) if bounding_volumes is not None else None
    lib().orc_apply_reflections(_p(scene), _p(refl), _p(bv) if bv is not None else None, C.c_int(w), C.c_int(h),
                                C.c_int(threads or (os.cpu_count() or 1)))
    return scene


def resize_downsample(img, ow: int, oh: int, which: str = "oracle"):
    """Image::CreateResizedImage (stbir_resize_float, 4 channels) for ow <= w, oh <= h -> [oh, ow, 4] float32"""
    a = _f(img)
    h, w = a.shape[:2]
    out = np.zeros((oh, ow, 4), dtype=np.float32)
    if which == "ref":
        rc = stb_ref().stbref_resize_float(_p(a), C.c_int(w), C.c_int(h), _p(out), C.c_int(ow), C.c_int(oh))
        assert rc == 1
    else:
        rc = lib().orc_resize_downsample(_p(a), C.c_int(w), C.c_int(h), _p(out), C.c_int(ow), C.c_int(oh))
        assert rc == 0
    return out


# ---- A25 / §8(f).4 groundwork: shadow tests (oracle_shadow.cpp) ------------------------------------------------------------
def forward_lighting_shadowed(pf, pv, planes, diff_cube, diff_res, spec_cube, spec_res, spec_mips, lut,
                              point_cubes=None, point_res=0, spot_maps=None, dir_map=None, threads=None) -> np.ndarray:
    pos, nrm, alb = (_f(p) for p in planes[:3])
    h, w = pos.shape[:2]
    out = np.zeros((h, w, 4), np.float32)
    lutc = _f(lut)
    pc = _f(point_cubes) if point_cubes is not None else None
    sm = _f(spot_maps) if spot_maps is not None else None
    dm = _f(dir_map) if dir_map is not None else None
    lib().orc_forward_lighting_shadowed(
        C.byref(pf), C.byref(pv), _p(pos), _p(nrm), _p(alb), C.c_int(w), C.c_int(h),
        _p(_f(diff_cube)), C.c_int(diff_res), _p(_f(spec_cube)), C.c_int(spec_res), C.c_int(spec_mips),
        _p(lutc), C.c_int(lutc.shape[1]), C.c_int(lutc.shape[0]),
        _p(pc) if pc is not None else None, C.c_int(point_res),
        _p(sm) if sm is not None else None, C.c_int(sm.shape[2] if sm is not None else 0), C.c_int(sm.shape[1] if sm is not None else 0),
        _p(dm) if dm is not None else None, C.c_int(dm.shape[1] if dm is not None else 0), C.c_int(dm.shape[0] if dm is not None else 0),
        _p(out), C.c_int(threads or cpu_threads()))
    return out


def shadow_test_pcf(light_space_pos, depth_bias, ndotl, shadow_map, directional=False) -> float:
    m = _f(shadow_map)
    lib().orc_shadow_test_pcf.restype = f32
    return float(lib().orc_shadow_test_pcf((f32 * 4)(*[float(x) for x in light_space_pos]), f32(depth_bias), f32(ndotl), _p(m),
                                           C.c_int(m.shape[1]), C.c_int(m.shape[0]), C.c_int(int(directional))))


def shadow_test_omni(lw, depth_bias, view_distance, far_plane, cube) -> float:
    c = _f(cube)
    lib().orc_shadow_test_omni.restype = f32
    return float(lib().orc_shadow_test_omni((f32 * 3)(*[float(x) for x in lw]), f32(depth_bias), f32(view_distance), f32(far_plane),
                                            _p(c), C.c_int(c.shape[1])))


# ---- the reference's OWN Image class (Libs/VQUtils/Source/Image.cpp compiled unmodified: oracle/_ref/libvqimageref.so) ----
IMG_REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libvqimageref.so")
_img = None


def image_ref():
    global _img
    if _img is None and os.path.exists(IMG_REF_LIB):
        _img = C.CDLL(IMG_REF_LIB)
    return _img


def ref_image_load(path: str):
    """Image::LoadFromFile(path) -> (rgba float32 [h,w,4], Image::MaxLuminance) or (None, None)"""
    r = image_ref()
    w, h, lum = C.c_int(0), C.c_int(0), f32(0)
    if r.vqimg_load(path.encode(), C.byref(w), C.byref(h), C.byref(lum), None) != 2:
        return None, None
    out = np.empty((h.value, w.value, 4), dtype=np.float32)
    r.vqimg_load(path.encode(), C.byref(w), C.byref(h), C.byref(lum), _p(out))
    return out, lum.value


def ref_image_resize(img, ow: int, oh: int):
    a = _f(img)
    out = np.zeros((oh, ow, 4), dtype=np.float32)
    assert image_ref().vqimg_resize(_p(a), C.c_int(a.shape[1]), C.c_int(a.shape[0]), _p(out), C.c_int(ow), C.c_int(oh)) == 1
    return out


def ref_image_save(path: str, img) -> bool:
    a = _f(img)
    return image_ref().vqimg_save(path.encode(), _p(a), C.c_int(a.shape[1]), C.c_int(a.shape[0])) == 1


def ref_mip_level_count(w: int, h: int) -> int:
    return int(image_ref().vqimg_mip_level_count(C.c_ulonglong(w), C.c_ulonglong(h)))


# ---- the reference's OWN VQ_DXGI_UTILS::MipImage (DXGIUtils.cpp compiled unmodified: oracle/_ref/libvqmipref.so) --------
MIP_REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libvqmipref.so")
_mip = None


def mip_ref():
    global _mip
    if _mip is None and os.path.exists(MIP_REF_LIB):
        _mip = C.CDLL(MIP_REF_LIB)
    return _mip


def ref_mip_image(level: np.ndarray) -> np.ndarray:
    """one MipImage step on an even-sized level: [H,W,4] float32 (RGB MIN, A = 1) or uint8 (box, truncating) -> [H/2,W/2,4]"""
    a = np.ascontiguousarray(level)
    h, w = a.shape[:2]
    assert w % 2 == 0 and h % 2 == 0, "the reference indexes (x+1, y+1) unconditionally"
    out = np.zeros((h // 2, w // 2, 4), dtype=a.dtype)
    mip_ref().vqmip_image(a.ctypes.data_as(C.c_void_p), out.ctypes.data_as(C.c_void_p), C.c_uint(w), C.c_uint(h),
                          C.c_uint(16 if a.dtype == np.float32 else 4))
    return out


# ---- the reference's OWN FPostProcessParameters wrappers (PostProcess.cpp compiled unmodified: oracle/_ref/libvqppref.so) ----
PP_REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libvqppref.so")
_pp = None


def pp_ref():
    global _pp
    if _pp is None and os.path.exists(PP_REF_LIB):
        _pp = C.CDLL(PP_REF_LIB)
        _pp.vqpp_rcas_linear_from_stops.restype = f32
        _pp.vqpp_rcas_stops_from_linear.restype = f32
    return _pp


# ---- the reference's SHADER TEXT compiled as C++ (oracle/_ref/libhlslref.so; ref_shim/hlsl_ref_shim.cpp) -----------------------
HLSL_REF_LIB = os.path.join(ORACLE_DIR, "_ref", "libhlslref.so")
_hlsl = None


def hlsl_ref():
    """Shaders/*.hlsl of the reference compiled with g++ on top of ref_shim/hlsl_compat.h, or None if oracle/_ref was not built."""
    global _hlsl
    if _hlsl is None and os.path.exists(HLSL_REF_LIB):
        lib()                                   # liboracle.so first: libhlslref.so resolves its samplers from it
        _hlsl = C.CDLL(HLSL_REF_LIB)
        for n in ("hlslref_ndf_ggx", "hlslref_geometry_smith", "hlslref_spotlight_intensity"):
            getattr(_hlsl, n).restype = f32
    return _hlsl


def hlsl_forward_image(pf, pv, planes, materials, chains, env, alpha_mask=False, point_cubes=None, point_res=0, spot_maps=None,
                       dir_map=None):
    """ForwardLighting.hlsl PSMain (compiled reference text) over the interpolated-attribute planes of the surface producer.
    Returns (color [H,W,4], discarded [H,W] bool)."""
    import vqengine_b200 as vq
    h, w = planes[0].shape[:2]
    n = len(materials)
    mats = (vq.MaterialData * n)(*materials)
    tex = (_OrcMaterialTextures * n)()
    for i, d in enumerate(chains):
        for k, slot in enumerate(vq.MATERIAL_TEXTURE_SLOTS):
            e = d.get(slot)
            if e is not None:
                buf, tw, th, tl = e
                tex[i].t[k] = _OrcTexture2D(buf.ctypes.data, tw, th, tl)
    p0, p1, p2 = _f(planes[0]), _f(planes[1]), _f(planes[2])
    ssao = _f(planes[3]) if len(planes) > 3 and planes[3] is not None else None
    out = np.zeros((h, w, 4), np.float32)
    disc = np.zeros((h, w), np.uint8)
    lutc = _f(env["lut"])
    pc = _f(point_cubes) if point_cubes is not None else None
    sm = _f(spot_maps) if spot_maps is not None else None
    dm = _f(dir_map) if dir_map is not None else None
    q = lambda a: _p(a) if a is not None else None
    hlsl_ref().hlslref_forward_image(
        C.byref(pf), C.byref(pv), _p(p0), _p(p1), _p(p2), q(ssao), C.c_int(w), C.c_int(h), mats, tex, C.c_int(n), C.c_int(int(alpha_mask)),
        _p(_f(env["diff"])), C.c_int(env["diff_res"]), _p(_f(env["spec"])), C.c_int(env["spec_res"]), C.c_int(env["spec_mips"]),
        _p(lutc), C.c_int(lutc.shape[1]), C.c_int(lutc.shape[0]),
        q(pc), C.c_int(point_res), q(sm), C.c_int(sm.shape[2] if sm is not None else 0), C.c_int(sm.shape[1] if sm is not None else 0),
        q(dm), C.c_int(dm.shape[1] if dm is not None else 0), C.c_int(dm.shape[0] if dm is not None else 0),
        _p(out), disc.ctypes.data_as(C.c_void_p))
    return out, disc.astype(bool)


def forward_lighting_shadowed_e(pf, pv, planes, diff_cube, diff_res, spec_cube, spec_res, spec_mips, lut,
                                point_cubes=None, point_res=0, spot_maps=None, dir_map=None, threads=None) -> np.ndarray:
    """orc_forward_lighting_shadowed with the emissive plane (planes[3]) passed through."""
    pos, nrm, alb = (_f(p) for p in planes[:3])
    em = _f(planes[3]) if len(planes) > 3 and planes[3] is not None else None
    h, w = pos.shape[:2]
    out = np.zeros((h, w, 4), np.float32)
    lutc = _f(lut)
    pc = _f(point_cubes) if point_cubes is not None else None
    sm = _f(spot_maps) if spot_maps is not None else None
    dm = _f(dir_map) if dir_map is not None else None
    q = lambda a: _p(a) if a is not None else None
    lib().orc_forward_lighting_shadowed_e(
        C.byref(pf), C.byref(pv), _p(pos), _p(nrm), _p(alb), q(em), C.c_int(w), C.c_int(h),
        _p(_f(diff_cube)), C.c_int(diff_res), _p(_f(spec_cube)), C.c_int(spec_res), C.c_int(spec_mips),
        _p(lutc), C.c_int(lutc.shape[1]), C.c_int(lutc.shape[0]),
        q(pc), C.c_int(point_res), q(sm), C.c_int(sm.shape[2] if sm is not None else 0), C.c_int(sm.shape[1] if sm is not None else 0),
        q(dm), C.c_int(dm.shape[1] if dm is not None else 0), C.c_int(dm.shape[0] if dm is not None else 0),
        _p(out), C.c_int(threads or cpu_threads()))
    return out


def depth_min_pyramid(depth):
    """[H,W] float32 depth -> list of levels (level 0 = copy, then 2x2 MIN, D3D mip-chain sizes), oracle_shadow.cpp DepthMinPyramid"""
    d = _f(depth)
    h, w = d.shape
    dims = []
    l = 0
    while True:
        dims.append((max(1, w >> l), max(1, h >> l)))
        if dims[-1] == (1, 1) or l == 12:
            break
        l += 1
    buf = np.zeros(sum(a * b for a, b in dims), np.float32)
    n = lib().orc_depth_min_pyramid(_p(d), C.c_int(w), C.c_int(h), _p(buf), C.c_int(len(dims)))
    out, o = [], 0
    for (lw, lh) in dims[:n]:
        out.append(buf[o:o + lw * lh].reshape(lh, lw))
        o += lw * lh
    return out


def hlsl_forward_gbuffer(pf, pv, planes, diff_cube, diff_res, spec_cube, spec_res, spec_mips, lut, row_begin=0, row_end=None, out=None):
    """ForwardLighting.hlsl PSMain (compiled reference text) driven from a G-buffer: rows [row_begin,row_end) -> out [H,W,4]"""
    pos, nrm, alb = (_f(p) for p in planes[:3])
    em = _f(planes[3]) if len(planes) > 3 and planes[3] is not None else None
    h, w = pos.shape[:2]
    out = np.zeros((h, w, 4), np.float32) if out is None else out
    lutc = _f(lut)
    hlsl_ref().hlslref_forward_gbuffer_rows(C.byref(pf), C.byref(pv), _p(pos), _p(nrm), _p(alb), _p(em) if em is not None else None,
                                            C.c_int(w), C.c_int(row_begin), C.c_int(h if row_end is None else row_end),
                                            _p(_f(diff_cube)), C.c_int(diff_res), _p(_f(spec_cube)), C.c_int(spec_res), C.c_int(spec_mips),
                                            _p(lutc), C.c_int(lutc.shape[1]), C.c_int(lutc.shape[0]), _p(out))
    return out
