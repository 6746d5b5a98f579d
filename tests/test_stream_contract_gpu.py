"""The C-ABI's stream and thread contract (include/vqcuda.h, top of the file):
  * a call that takes `stream` only ENQUEUES work on it: it returns without waiting for earlier work on that stream, reads its
    inputs and writes its outputs only after that work, and runs nothing on another stream (except the calls that grow context
    scratch, which wait for the device once and then enqueue);
  * the blocking calls (vq_forward_lighting_host, vq_hdr_load_host, vq_hdr_save_host, vq_material_table_create) are ordered after
    all device work enqueued before them, on any stream, and return with their own work complete;
  * the calls the header does not list as exceptions are re-entrant: threads that share one context, each on its own stream, get
    the bits a serial run gets, and vq_last_error is per thread.

The tests hold a stream with a GATE (tests/device_check/stream_gate.cu): one thread that polls a word of mapped host memory, with a
10 s %globaltimer bound, and then writes "opened" or "timed out" to a status word the host reads without a CUDA call. A keeper
thread opens the gate when the test says so, or after a fixed delay; it is joined in a `finally`, so no call can wait on a gate
for longer than the bound, and every test asserts that its gate was opened, not timed out.

Part 1: every entry point with a `void* stream` parameter (the CPU test below checks the table against vqcuda.h). Each row runs
once ungated (its reference, which also sizes the context's scratch and loads its kernels). Then its inputs are set to one
sentinel and its outputs to a NaN-payload sentinel, the gate is closed on a non-blocking stream s, and the copies that put the real
inputs back, then the call, are enqueued on s behind it. The call must (i) return while the gate is still closed, (ii) leave every
output and in-place buffer at its sentinel, as a snapshot taken on a second non-blocking stream after the legacy stream is drained
shows, and (iii) once the gate opens, produce the reference bits. One more case per scratch owner grows that scratch behind the
gate: the call waits for the device, so it returns only after the gate opened (the keeper opens it after a delay).
Part 2: each blocking call with a gate on the legacy stream and on a non-blocking stream, and behind the gate the kernel that
writes the call's device inputs (or, for vq_hdr_load_host, copies the output it is about to overwrite).
Part 3: 4 and 8 threads on one context (and 4 on two contexts), 50 rounds of a fixed mix of the re-entrant calls each."""
import contextlib
import ctypes as C
import os
import re
import subprocess
import threading
import time

import numpy as np
import pytest
import torch

import frame_domain as fd
import vqengine_b200 as vq
from envmaps import small_env
from test_multi_shading_gpu import Frame
from test_post_fused_gpu import fsr_consts, hdr
from test_psmain_fused_gpu import _env_maps
from test_psmain_shadowed_gpu import _maps, _shadow_scene
from vqengine_b200 import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "vqcuda.h")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC"]
GATE_NS = 10_000_000_000           # a gate nobody opens gives up after 10 s (and says so)
DELAY = 0.4                        # the keeper's delay where a call is expected to wait for the gate
ARMED, WAITING, OPENED, TIMED_OUT = 1, 2, 3, 4
STATUS = {0: "never closed", ARMED: "armed", WAITING: "waiting", OPENED: "opened", TIMED_OUT: "timed out"}
OUT_SENTINEL = 0x7FC0DEAD          # a quiet NaN with a payload no kernel computes
IN_SENTINEL = 0x4B1D4B1D           # 1.03e7: a finite input the real one never holds


# ---- the table: one row per entry point that takes a stream -----------------------------------------------------------------
def _words(t):
    return t.reshape(-1).view(torch.int32)


def _fill(t, bits):
    _words(t).fill_(bits)


class Row:
    """ins: device tensors the call reads (their contents now are the real ones); outs: device tensors it writes (in-place buffers
    are in both); run(ctx, stream) enqueues the call(s)"""

    def __init__(self, ins, outs, run, pre=None, keep=()):
        self.ins, self.outs, self.run, self.pre, self.keep = ins, outs, run, pre, keep
        self.real = [t.clone() for t in ins]
        self.inplace = [t for t in ins if any(t is o for o in outs)]

    def prime(self, stream, inplace_only=False):
        """on `stream`: every output to the sentinel, then the real inputs into place"""
        with torch.cuda.stream(stream):
            for o in self.outs:
                _fill(o, OUT_SENTINEL)
            for t, r in zip(self.ins, self.real):
                if not inplace_only or any(t is i for i in self.inplace):
                    t.copy_(r)


def _img(t, ch=4):
    return vq.image_of(t, ch)


def _f32(h, w, ch=4):
    return torch.empty((h, w, ch), dtype=torch.float32, device="cuda")


def _sp(s):
    return vq._stream_ptr(s)


class Scene:
    """one small shadowed frame: attribute planes, material table, environment, shadow maps and the G-buffer they produce"""

    def __init__(self, ctx):
        planes, mats, chains, env, pf, pv, maps = _shadow_scene(64, 18)
        self.f = Frame(ctx, planes, mats, chains, env, pf, pv, _maps(maps))
        self.mats, self.chains = mats, chains
        self.maps = [t for t in self.f.maps.values() if t is not None]
        self.env = list(self.f.env_keep)

    def close(self):
        self.f.close()


def _env_ins(S, reg):
    return [] if reg else S.env


def _use_env(c, S, reg):
    if not reg:
        c.environment_invalidate()


def r_forward(S, seed, reg=False):
    f, o, gb = S.f, _f32(S.f.h, S.f.w), S.f.gbuffer()

    def run(c, s):
        _use_env(c, S, reg)
        c.forward_lighting(f.pf, f.pv, gb, f.em, o, stream=s)
    return Row(f.gbt + _env_ins(S, reg), [o], run, keep=(gb,))


def r_forward_multi(S, seed, reg=False, signal_form=False):
    f, outs, gb = S.f, [_f32(S.f.h, S.f.w) for _ in range(2)], S.f.gbuffer()
    arr = (vq.Image * 2)(*[_img(o) for o in outs])

    def run(c, s):
        _use_env(c, S, reg)
        if signal_form:
            vq._check(vq.lib.vq_forward_lighting_multi_signal(c._h, C.byref(f.pf), C.byref(f.pv), C.byref(gb), C.byref(f.em), arr, 2,
                                                              0, 0, f.h, None, _sp(s)))
        else:
            vq._check(vq.lib.vq_forward_lighting_multi(c._h, C.byref(f.pf), C.byref(f.pv), C.byref(gb), C.byref(f.em), arr, 2, 0, 0,
                                                       f.h, _sp(s)))
    return Row(f.gbt + _env_ins(S, reg), outs, run, keep=(gb, arr))


def r_shadowed(S, seed, multi=False):
    f, outs, gb = S.f, [_f32(S.f.h, S.f.w) for _ in range(2 if multi else 1)], S.f.gbuffer()

    def run(c, s):
        c.environment_invalidate()
        if multi:
            c.forward_lighting_shadowed_multi(f.pf, f.pv, gb, f.em, [_img(o) for o in outs], 0, stream=s, **f.maps)
        else:
            c.forward_lighting_shadowed(f.pf, f.pv, gb, f.em, outs[0], stream=s, **f.maps)
    return Row(f.gbt + S.env + S.maps, outs, run, keep=(gb,))


def r_from_materials(S, seed, reg=False, shadowed=False, multi=False):
    f, outs, si = S.f, [_f32(S.f.h, S.f.w) for _ in range(2 if multi else 1)], S.f.inputs()
    maps = f.maps if shadowed else {}

    def run(c, s):
        _use_env(c, S, reg)
        if multi:
            c.forward_lighting_from_materials_multi(f.pf, f.pv, si, f.table, f.em, [_img(o) for o in outs], 0, stream=s, **maps)
        elif shadowed:
            c.forward_lighting_shadowed_from_materials(f.pf, f.pv, si, f.table, f.em, outs[0], stream=s, **maps)
        else:
            c.forward_lighting_from_materials(f.pf, f.pv, si, f.table, f.em, outs[0], stream=s)
    return Row(f.dp + _env_ins(S, reg) + (S.maps if shadowed else []), outs, run, keep=(si,))


def r_gbuffer_from_materials(S, seed):
    f, outs, si = S.f, [_f32(S.f.h, S.f.w) for _ in range(4)], S.f.inputs()
    gb = vq.GBuffer(*(_img(o) for o in outs))

    def run(c, s):
        c.gbuffer_from_materials(si, f.table, f.pf.fAmbientLightingFactor, gb, stream=s)
    return Row(list(f.dp), outs, run, keep=(si, gb))


def r_prepare_forward(S, seed):
    f, o, gb = S.f, _f32(S.f.h, S.f.w), S.f.gbuffer()

    def run(c, s):
        c.environment_prepare(f.em, stream=s)
        c.forward_lighting(f.pf, f.pv, gb, f.em, o, stream=s)
    return Row(f.gbt + S.env, [o], run, keep=(gb,))


def _hdri(w, h, seed):
    levels = vq.mip_level_count(w, h)
    d = torch.zeros((vq.pyramid_texel_count(w, h, levels), 4), dtype=torch.float32, device="cuda")
    d[: w * h] = torch.from_numpy(synth.hdri(w, h, seed=seed)).cuda().reshape(-1, 4)
    return d, vq.pyramid_of(d, w, h, levels)


def r_hdri_mips(S, seed, w=64, h=32):
    """w, h <= 4096: one SPD launch; wider: one launch per level"""
    d, p = _hdri(w, h, seed)
    return Row([d], [d], lambda c, s: c.hdri_build_mips(p, stream=s), keep=(p,))


def _mipped_hdri(ctx, seed):
    d, p = _hdri(64, 32, seed)
    ctx.hdri_build_mips(p)
    torch.cuda.synchronize()
    return d, p


def r_diffuse(S, seed):
    d, p = _mipped_hdri(S.ctx, seed)
    o = torch.empty((vq.cubemap_texel_count(8, 1), 4), dtype=torch.float32, device="cuda")
    cube = vq.cubemap_of(o, 8, 1)
    return Row([d], [o], lambda c, s: c.diffuse_irradiance(p, cube, n_phi=16, n_theta=4, src_mip=2, stream=s), keep=(p, cube))


def r_specular(S, seed, form="single"):
    d, p = _mipped_hdri(S.ctx, seed)
    res, mips = 8, 4
    outs = [torch.empty((vq.cubemap_texel_count(res, mips), 4), dtype=torch.float32, device="cuda") for _ in range(1 if form == "single" else 2)]
    cubes = [vq.cubemap_of(o, res, mips) for o in outs]
    rows = vq.cubemap_row_count(res, mips)

    def run(c, s):
        if form == "single":
            c.specular_prefilter(p, cubes[0], 64, stream=s)
        elif form == "multi":
            c.specular_prefilter_multi(p, cubes, 64, stream=s)
        else:
            c.specular_prefilter_ranges(p, cubes, [(0, rows // 3), (rows // 2, rows)], 64, stream=s)
    return Row([d], outs, run, keep=(p, cubes))


def r_brdf_lut(S, seed):
    o = _f32(16, 24, 2)
    return Row([], [o], lambda c, s: c.brdf_integration_lut(o, 64, stream=s))


def _ldr(h, w, seed):
    return torch.clamp(hdr(h, w, seed) / 4.0, 0.0, 1.0).contiguous()


def r_blur(S, seed, vertical):
    src = hdr(20, 37, seed)
    o = _f32(20, 37)
    return Row([src], [o], lambda c, s: c.gaussian_blur(src, o, vertical, stream=s))


def _post_pass(kind, seed):
    """(source, output shape, single call, multi call) of one post pass"""
    tm = synth.default_tonemapper()
    if kind == "tonemap":
        return hdr(20, 37, seed), (20, 37), lambda c, i, o, s: c.tonemap(tm, i, o, stream=s), \
            lambda c, i, os_, s: c.tonemap_multi(tm, i, os_, stream=s)
    if kind == "cas":
        con = vq.cas_setup(0.6, 37, 20, 37, 20)
        return _ldr(20, 37, seed), (20, 37), lambda c, i, o, s: c.cas(con, i, o, stream=s), \
            lambda c, i, os_, s: c.cas_multi(con, i, os_, stream=s)
    if kind == "fsr_easu":
        con = vq.fsr_easu_con(37, 23, 37, 23, 74, 46)
        return _ldr(23, 37, seed), (46, 74), lambda c, i, o, s: c.fsr_easu(con, i, o, stream=s), \
            lambda c, i, os_, s: c.fsr_easu_multi(con, i, os_, stream=s)
    con = vq.fsr_rcas_con(0.2)
    return _ldr(20, 37, seed), (20, 37), lambda c, i, o, s: c.fsr_rcas(con, i, o, stream=s), \
        lambda c, i, os_, s: c.fsr_rcas_multi(con, i, os_, stream=s)


def r_post_pass(S, seed, kind, multi=False):
    src, (oh, ow), single, many = _post_pass(kind, seed)
    outs = [_f32(oh, ow) for _ in range(2 if multi else 1)]
    if multi:
        return Row([src], outs, lambda c, s: many(c, src, [_img(o) for o in outs], s))
    return Row([src], outs, lambda c, s: single(c, src, outs[0], s))


POST_BRANCHES = {"fsr 2x": (23, 37, 46, 74), "fsr up": (41, 73, 54, 95), "cas": (20, 37, 20, 37), "tonemap": (20, 37, 20, 37)}


def r_post_process(S, seed, branch, multi=False):
    ih, iw, oh, ow = POST_BRANCHES[branch]
    src, tm = hdr(ih, iw, seed), synth.default_tonemapper()
    kw = {}
    if branch.startswith("fsr"):
        kw["easu"], kw["rcas"] = fsr_consts(ih, iw, oh, ow)
    elif branch == "cas":
        kw["cas"] = vq.cas_setup(0.5, iw, ih, iw, ih)
    outs = [_f32(oh, ow) for _ in range(2 if multi else 1)]

    def run(c, s):
        if multi:
            c.post_process_multi(tm, src, [_img(o) for o in outs], stream=s, **kw)
        else:
            c.post_process(tm, src, outs[0], stream=s, **kw)
    return Row([src], outs, run)


def r_spd(S, seed):
    """256 x 256: 8 levels, so the last CTA also runs the tail above mip 6 on its ticket"""
    src = hdr(256, 256, seed)
    _, con = vq.spd_setup(256, 256)
    assert con.mips == 8
    mips = [_f32(256 >> (i + 1), 256 >> (i + 1)) for i in range(con.mips)]
    return Row([src], mips, lambda c, s: c.spd_downsample(con, src, mips, stream=s), keep=(con,))


def r_texture_mips(S, seed):
    w, h = 48, 20
    levels = vq.mip_level_count(w, h)
    t = torch.zeros((vq.pyramid_texel_count(w, h, levels) * 4,), dtype=torch.uint8, device="cuda")
    t[: w * h * 4] = torch.from_numpy(np.random.default_rng(seed).integers(0, 256, w * h * 4, dtype=np.uint8)).cuda()
    tex = vq.texture_of(t, w, h, levels)
    return Row([t], [t], lambda c, s: c.texture_build_mips(tex, stream=s), keep=(tex,))


def r_depth_pyramid(S, seed, w=200, h=130):
    """8 levels: two launches, the second from the padded level 6 in context scratch"""
    d = torch.from_numpy(np.random.default_rng(seed).uniform(0.05, 1.0, (h, w)).astype(np.float32)).cuda()
    n = vq.depth_pyramid_level_count(w, h)
    lv = torch.empty((vq.depth_pyramid_texel_count(w, h, n),), dtype=torch.float32, device="cuda")
    return Row([d], [lv], lambda c, s: c.depth_min_pyramid(d, lv, stream=s))


def r_hdr_decode(S, seed):
    src = hdr(20, 37, seed)
    rgbe = S.ctx.hdr_encode_rgbe(src).cpu().numpy()
    data = vq.hdr_pack_file(rgbe)
    info, offs = vq.hdr_parse(data)
    assert offs is not None, "the file is run-length encoded"
    n = len(data)
    dfile = torch.zeros(((n + 15) // 16 * 16 + 16,), dtype=torch.uint8, device="cuda")
    dfile[:n] = torch.frombuffer(bytearray(data), dtype=torch.uint8).cuda()
    doffs = torch.from_numpy(offs.view(np.int64).copy()).cuda()
    out, lum = _f32(20, 37), torch.zeros((1,), dtype=torch.float32, device="cuda")

    def run(c, s):
        vq._check(vq.lib.vq_hdr_decode(c._h, dfile.data_ptr(), n, C.byref(info), doffs.data_ptr(), _img(out), lum.data_ptr(), _sp(s)))
    return Row([dfile, doffs, lum], [out, lum], run, keep=(info,))


def r_hdr_encode(S, seed):
    src = hdr(20, 37, seed)
    out = torch.empty((20, 37, 4), dtype=torch.uint8, device="cuda")
    return Row([src], [out], lambda c, s: vq._check(vq.lib.vq_hdr_encode_rgbe(c._h, _img(src), out.data_ptr(), _sp(s))))


def r_resize(S, seed, new_pair=False):
    """40 x 50 -> 23 x 17. new_pair: the context's last pair is 40 x 30 (its tables are at least as large), so the gated call
    rebuilds the tables and uploads them from pageable vectors on the stream"""
    src, o, other = hdr(40, 50, seed), _f32(17, 23), _f32(30, 40)
    pre = (lambda c, s: c.image_resize(src, other, stream=s)) if new_pair else None
    return Row([src], [o], lambda c, s: c.image_resize(src, o, stream=s), pre=pre, keep=(other,))


def _sky(w, h, seed):
    m = fd.view_proj(fd.yaw_pitch(0.9, 0.25), 1.2, w / h)
    hdri = torch.from_numpy(np.ascontiguousarray(fd.sky_hdri(64, 32, seed=seed))).cuda()
    rng = np.random.default_rng(seed)
    mask = rng.uniform(-1, 1, (h, w, 4)).astype(np.float32)
    mask[rng.uniform(size=(h, w)) < 0.5, :3] = 0.0
    return m, hdri, vq.pyramid_of(hdri, 64, 32, 1), torch.from_numpy(mask).cuda()


def r_skydome(S, seed, multi=False):
    h, w = 18, 37
    m, hdri, pyr, mask = _sky(w, h, seed)
    scene, peer = hdr(h, w, seed + 1), _f32(h, w)

    def run(c, s):
        if multi:
            c.skydome_multi(m, pyr, [_img(scene), _img(peer)], 0, normal_mask=mask, stream=s)
        else:
            c.skydome(m, pyr, scene, normal_mask=mask, stream=s)
    return Row([hdri, mask, scene], [scene, peer] if multi else [scene], run, keep=(pyr,))


def r_composite(S, seed, multi=False):
    h, w = 18, 37
    scene, refl, bv, peer = hdr(h, w, seed), hdr(h, w, seed + 1), _ldr(h, w, seed + 2), _f32(h, w)

    def run(c, s):
        if multi:
            c.apply_reflections_multi(refl, [_img(scene), _img(peer)], 0, bounding_volumes=bv, stream=s)
        else:
            c.apply_reflections(scene, refl, bv, stream=s)
    return Row([scene, refl, bv], [scene, peer] if multi else [scene], run)


# name -> (the entry points the row calls, builder(scene, seed))
ROWS = {
    "forward": (("vq_forward_lighting",), r_forward),
    "forward multi": (("vq_forward_lighting_multi",), r_forward_multi),
    "forward multi_signal": (("vq_forward_lighting_multi_signal",), lambda S, k: r_forward_multi(S, k, signal_form=True)),
    "prepare + forward": (("vq_environment_prepare", "vq_forward_lighting"), r_prepare_forward),
    "shadowed": (("vq_forward_lighting_shadowed",), r_shadowed),
    "shadowed multi_signal": (("vq_forward_lighting_shadowed_multi_signal",), lambda S, k: r_shadowed(S, k, multi=True)),
    "from_materials": (("vq_forward_lighting_from_materials",), r_from_materials),
    "shadowed_from_materials": (("vq_forward_lighting_shadowed_from_materials",), lambda S, k: r_from_materials(S, k, shadowed=True)),
    "from_materials multi_signal": (("vq_forward_lighting_from_materials_multi_signal",),
                                    lambda S, k: r_from_materials(S, k, multi=True)),
    "shadowed_from_materials multi_signal": (("vq_forward_lighting_from_materials_multi_signal",),
                                             lambda S, k: r_from_materials(S, k, shadowed=True, multi=True)),
    "gbuffer_from_materials": (("vq_gbuffer_from_materials",), r_gbuffer_from_materials),
    "texture_build_mips": (("vq_texture_build_mips",), r_texture_mips),
    "hdri_build_mips spd": (("vq_hdri_build_mips",), r_hdri_mips),
    "hdri_build_mips per level": (("vq_hdri_build_mips",), lambda S, k: r_hdri_mips(S, k, 4098, 4)),
    "diffuse_irradiance": (("vq_diffuse_irradiance",), r_diffuse),
    "specular_prefilter": (("vq_specular_prefilter",), r_specular),
    "specular_prefilter_multi": (("vq_specular_prefilter_multi",), lambda S, k: r_specular(S, k, "multi")),
    "specular_prefilter_ranges": (("vq_specular_prefilter_ranges",), lambda S, k: r_specular(S, k, "ranges")),
    "brdf_integration_lut": (("vq_brdf_integration_lut",), r_brdf_lut),
    "gaussian_blur_x": (("vq_gaussian_blur_x",), lambda S, k: r_blur(S, k, False)),
    "gaussian_blur_y": (("vq_gaussian_blur_y",), lambda S, k: r_blur(S, k, True)),
    "tonemap": (("vq_tonemap",), lambda S, k: r_post_pass(S, k, "tonemap")),
    "cas": (("vq_cas",), lambda S, k: r_post_pass(S, k, "cas")),
    "fsr_easu": (("vq_fsr_easu",), lambda S, k: r_post_pass(S, k, "fsr_easu")),
    "fsr_rcas": (("vq_fsr_rcas",), lambda S, k: r_post_pass(S, k, "fsr_rcas")),
    "tonemap multi_signal": (("vq_tonemap_multi_signal",), lambda S, k: r_post_pass(S, k, "tonemap", True)),
    "cas multi_signal": (("vq_cas_multi_signal",), lambda S, k: r_post_pass(S, k, "cas", True)),
    "fsr_easu multi_signal": (("vq_fsr_easu_multi_signal",), lambda S, k: r_post_pass(S, k, "fsr_easu", True)),
    "fsr_rcas multi_signal": (("vq_fsr_rcas_multi_signal",), lambda S, k: r_post_pass(S, k, "fsr_rcas", True)),
    **{f"post_process {b}": (("vq_post_process",), (lambda b: lambda S, k: r_post_process(S, k, b))(b)) for b in POST_BRANCHES},
    "post_process multi_signal": (("vq_post_process_multi_signal",), lambda S, k: r_post_process(S, k, "fsr 2x", True)),
    "spd_downsample": (("vq_spd_downsample",), r_spd),
    "depth_min_pyramid": (("vq_depth_min_pyramid",), r_depth_pyramid),
    "hdr_decode": (("vq_hdr_decode",), r_hdr_decode),
    "hdr_encode_rgbe": (("vq_hdr_encode_rgbe",), r_hdr_encode),
    "image_resize": (("vq_image_resize",), r_resize),
    "image_resize new pair": (("vq_image_resize",), lambda S, k: r_resize(S, k, new_pair=True)),
    "skydome": (("vq_skydome",), r_skydome),
    "skydome multi_signal": (("vq_skydome_multi_signal",), lambda S, k: r_skydome(S, k, multi=True)),
    "apply_reflections": (("vq_apply_reflections",), r_composite),
    "apply_reflections multi_signal": (("vq_apply_reflections_multi_signal",), lambda S, k: r_composite(S, k, multi=True)),
}


def stream_entry_points():
    """every VQ_API function of vqcuda.h with a `void* stream` parameter"""
    text = re.sub(r"/\*.*?\*/", " ", open(HEADER).read(), flags=re.S)
    names = set()
    for m in re.finditer(r"VQ_API\s+[\w\s\*]*?\b(vq_\w+)\s*\(([^;]*)\)\s*;", text):
        if re.search(r"\bvoid\s*\*\s*stream\b", m.group(2)):
            names.add(m.group(1))
    return names


def test_every_stream_entry_point_has_a_row():
    """CPU: the table above names every entry point of vqcuda.h that takes a stream, and nothing else"""
    want = stream_entry_points()
    assert {"vq_forward_lighting", "vq_post_process", "vq_image_resize", "vq_environment_prepare"} <= want, sorted(want)
    have = set().union(*(covers for covers, _ in ROWS.values()))
    assert not sorted(want - have), f"entry points with a stream and no row: {sorted(want - have)}"
    assert not sorted(have - want), f"rows for names that are not stream entry points of vqcuda.h: {sorted(have - want)}"


# ---- the gate, the streams, the fixtures ---------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def sg(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out = tmp_path_factory.mktemp("devicecheck") / "libstreamgate.so"
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), *FLAGS, "-o", str(out),
                           os.path.join(ROOT, "tests", "device_check", "stream_gate.cu")])
    torch.cuda.init()
    lib = C.CDLL(str(out))
    vp = C.c_void_p
    lib.sg_gate_new.argtypes = [C.POINTER(vp)]
    lib.sg_gate_free.argtypes = [vp]
    lib.sg_gate_words.argtypes = [vp]
    lib.sg_gate_words.restype = vp
    lib.sg_gate_close.argtypes = [vp, vp, C.c_ulonglong]
    lib.sg_stream_create.argtypes = [C.POINTER(vp)]
    lib.sg_stream_flags.argtypes = [vp, C.POINTER(C.c_uint)]
    lib.sg_stream_destroy.argtypes = [vp]
    return lib


class Gate:
    def __init__(self, lib):
        self.lib, self.h = lib, C.c_void_p()
        assert lib.sg_gate_new(C.byref(self.h)) == 0
        self.words = (C.c_uint32 * 2).from_address(lib.sg_gate_words(self.h))
        self.opened_at = None

    def status(self):
        return STATUS[self.words[1]]

    @contextlib.contextmanager
    def closed(self, stream, delay=None):
        """the gate closed on `stream`; the keeper opens it when the block sets the yielded event, after `delay` seconds, or on exit"""
        self.opened_at = None
        assert self.lib.sg_gate_close(self.h, C.c_void_p(stream.cuda_stream), GATE_NS) == 0
        go = threading.Event()

        def keep():
            go.wait(delay)
            self.opened_at = time.monotonic()
            self.words[0] = 1
        keeper = threading.Thread(target=keep, name="gate keeper")
        keeper.start()
        try:
            yield go
        finally:
            go.set()
            keeper.join()

    def free(self):
        self.lib.sg_gate_free(self.h)


@pytest.fixture(scope="module")
def gate(sg):
    g = Gate(sg)
    yield g
    torch.cuda.synchronize()
    g.free()


def make_streams(lib, n):
    out = []
    for _ in range(n):
        h = C.c_void_p()
        assert lib.sg_stream_create(C.byref(h)) == 0
        flags = C.c_uint(7)
        assert lib.sg_stream_flags(h, C.byref(flags)) == 0 and flags.value == 1, "cudaStreamNonBlocking"
        out.append(torch.cuda.ExternalStream(h.value))
    return out


@pytest.fixture(scope="module")
def streams(sg):
    ss = make_streams(sg, 2)
    yield ss
    torch.cuda.synchronize()
    for s in ss:
        sg.sg_stream_destroy(C.c_void_p(s.cuda_stream))


def legacy():
    s = torch.cuda.default_stream()
    assert s.cuda_stream == 0, "torch's default stream is the legacy stream"
    return s


@pytest.fixture(scope="module")
def sctx(sg):
    c = vq.Context(0)
    yield c
    torch.cuda.synchronize()
    c.close()


@pytest.fixture(scope="module")
def scene(sctx):
    S = Scene(sctx)
    S.ctx = sctx
    yield S
    S.close()


def reference(row, ctx, s):
    torch.cuda.synchronize()           # the row's tensors were made on the legacy stream, which s does not wait for
    if row.pre is not None:
        row.pre(ctx, s)
    row.prime(s)
    row.run(ctx, s)
    s.synchronize()
    return [o.clone() for o in row.outs]


def assert_bits(what, outs, refs):
    for k, (o, r) in enumerate(zip(outs, refs)):
        a, b = _words(o), _words(r)
        if not torch.equal(a, b):
            pytest.fail(f"{what}: output {k}: {int((a != b).sum())} of {a.numel()} words differ from the ungated call")


def _snapshot(snaps, outs, s2):
    """copies of `outs` taken on s2 -> which of them still hold the output sentinel"""
    with torch.cuda.stream(s2):
        for snap, o in zip(snaps, outs):
            snap.copy_(o)
        return [bool((_words(snap) == OUT_SENTINEL).all()) for snap in snaps]


def _sentinels(row):
    for t in row.ins:
        _fill(t, IN_SENTINEL)
    for o in row.outs:
        _fill(o, OUT_SENTINEL)
    torch.cuda.synchronize()


# ---- part 1: every entry point that takes a stream only enqueues on it ----------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", list(ROWS))
def test_enqueues_behind_earlier_work(sctx, scene, gate, streams, name):
    s, s2 = streams
    row = ROWS[name][1](scene, 7)
    ref = reference(row, sctx, s)
    if row.pre is not None:
        row.pre(sctx, s)
        s.synchronize()
    snaps = [torch.empty_like(o) for o in row.outs]
    _sentinels(row)
    # once without the gate: the first launch of a kernel loads its module (lazy loading), which waits for running kernels
    assert all(_snapshot(snaps, row.outs, s2))
    with gate.closed(s) as go:
        row.prime(s)
        row.run(sctx, s)
        st = gate.status()
        assert st in ("armed", "waiting"), f"{name}: the call returned with the gate {st}: it waited for earlier work on its stream"
        legacy().synchronize()
        held = _snapshot(snaps, row.outs, s2)
        assert all(held), f"{name}: outputs {[k for k, h in enumerate(held) if not h]} were written before the gate opened"
        go.set()
    s.synchronize()
    assert gate.status() == "opened"
    assert_bits(name, row.outs, ref)


def _shadow_small(S):
    def first(c):
        f = S.f
        o = _f32(f.h, f.w)
        c.forward_lighting_shadowed(f.pf, f.pv, f.gbuffer(), f.em, o, row_begin=0, row_end=1, **f.maps)
    return first


def _env_small(S):
    env = small_env(hdri_w=32, hdri_h=16, diff_res=4, spec_res=8, spec_mips=4, lut=8)
    em, keep = _env_maps(env)
    planes = [torch.from_numpy(p).cuda() for p in synth.gbuffer(16, 8, seed=3)]
    pf, pv = synth.scene_constants(16, 8, 4, seed=3)
    assert sum(t.numel() for t in keep) < sum(t.numel() for t in S.env)

    def first(c, keep=keep):
        o = _f32(8, 16)
        c.environment_invalidate()
        c.forward_lighting(pf, pv, vq.GBuffer(_img(planes[0]), _img(planes[1]), _img(planes[2]), vq.null_image()), em, o)
        torch.cuda.synchronize()
    return first


def _resize_small(S):
    def first(c):
        c.image_resize(hdr(40, 50, 1), _f32(4, 5))
    return first


def _depth_small(S):
    def first(c):
        c.depth_min_pyramid(torch.ones((4, 4), device="cuda"), torch.empty((64,), device="cuda"))
    return first


# scratch owner -> (the row whose gated call grows it, the ungated call that allocates it smaller first)
GROWTH = {
    "env_per_call": ("forward", _env_small),
    "shadow_rec": ("shadowed", _shadow_small),
    "resize_mid and resize_tab": ("image_resize", _resize_small),
    "depth_pad": ("depth_min_pyramid", _depth_small),
}


@pytest.mark.gpu
@pytest.mark.parametrize("owner", list(GROWTH))
def test_scratch_growth_waits_for_the_device(sctx, scene, gate, streams, owner):
    """a call that grows context scratch waits for all earlier device work (the old buffer may still be read) and then enqueues"""
    s, _ = streams
    name, small = GROWTH[owner]
    row = ROWS[name][1](scene, 7)
    ref = reference(row, sctx, s)
    c = vq.Context(0)
    try:
        small(scene)(c)
        torch.cuda.synchronize()
        _sentinels(row)
        with gate.closed(s, delay=DELAY):
            row.prime(s)
            row.run(c, s)
            returned, opened = time.monotonic(), gate.opened_at
        s.synchronize()
        assert gate.status() == "opened"
        assert opened is not None and returned >= opened, f"{owner}: the growing call returned before the gate opened"
        assert_bits(f"{owner} growth", row.outs, ref)
    finally:
        torch.cuda.synchronize()
        c.close()


def _host_gbuffer(f):
    planes = [t.cpu() for t in f.gbt]
    return planes, vq.GBuffer(*(_img(p) for p in planes))


@pytest.mark.gpu
def test_stage_growth_waits_for_the_device(scene, gate, streams):
    """vq_ctx_resize growing the host-call staging waits for earlier device work; the host call then shades as before"""
    s, _ = streams
    f = scene.f
    planes, hgb = _host_gbuffer(f)
    want, got = torch.empty((f.h, f.w, 4)), torch.empty((f.h, f.w, 4))
    c, c2 = vq.Context(0), vq.Context(0)
    try:
        c.forward_lighting_host(f.pf, f.pv, hgb, f.em, want)
        c2.resize(8, 8)
        with gate.closed(s, delay=DELAY):
            c2.resize(f.w * 2, f.h * 2)
            returned, opened = time.monotonic(), gate.opened_at
        s.synchronize()
        assert gate.status() == "opened"
        assert opened is not None and returned >= opened, "vq_ctx_resize grew the staging before the gate opened"
        c2.forward_lighting_host(f.pf, f.pv, hgb, f.em, got)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32))
    finally:
        torch.cuda.synchronize()
        c.close()
        c2.close()


@pytest.mark.gpu
def test_gate_on_the_legacy_stream(gate, streams):
    """the gate itself: closed on the legacy stream it holds a copy enqueued there, and a non-blocking stream runs past it"""
    s, _ = streams
    a = torch.full((1024,), 1.0, device="cuda")
    b = torch.zeros_like(a)
    c = torch.zeros_like(a)
    assert bool((c == 0.0).all()) and not bool((b == 1.0).all())     # the comparison kernels loaded before the gate
    torch.cuda.synchronize()
    with gate.closed(legacy()) as go:
        with torch.cuda.stream(legacy()):
            b.copy_(a)
        with torch.cuda.stream(s):
            c.copy_(a)
        s.synchronize()
        assert gate.status() in ("armed", "waiting")
        with torch.cuda.stream(s):
            assert bool((c == 1.0).all()) and bool((b == 0.0).all()), "the copy behind the gate ran"
        go.set()
    torch.cuda.synchronize()
    assert gate.status() == "opened"
    assert bool((b == 1.0).all())


# ---- part 2: the blocking calls are ordered after all earlier device work -------------------------------------------------------
WHERE = ["legacy", "non-blocking"]


def _gate_stream(where, streams):
    return legacy() if where == "legacy" else streams[0]


def _behind_gate(gate, gs, writes, call):
    """closes the gate on gs, enqueues the copies `writes` [(dst, src)] behind it, makes the blocking call; the keeper opens the gate
    after DELAY. -> (the call's result, the time it returned, the time the gate opened before that or None)"""
    with gate.closed(gs, delay=DELAY):
        with torch.cuda.stream(gs):
            for dst, src in writes:
                dst.copy_(src)
        result = call()
        returned, opened = time.monotonic(), gate.opened_at
    torch.cuda.synchronize()
    assert gate.status() == "opened"
    return result, returned, opened


def _after_gate(what, returned, opened):
    assert opened is not None and returned >= opened, f"{what} returned before the gate opened: it did not wait for earlier device work"


@pytest.mark.gpu
@pytest.mark.parametrize("where", WHERE)
def test_forward_lighting_host_after_earlier_work(scene, gate, streams, where):
    """the environment maps are written behind the gate; the call (unregistered environment: it rebuilds the sampling copies from
    them) must shade from what was written"""
    f = scene.f
    planes, hgb = _host_gbuffer(f)
    want, got = torch.empty((f.h, f.w, 4)), torch.full((f.h, f.w, 4), float("nan"))
    c = vq.Context(0)
    try:
        c.resize(f.w, f.h)
        c.forward_lighting_host(f.pf, f.pv, hgb, f.em, want)      # also sizes the staging: no regrow below
        real = [t.clone() for t in scene.env]
        for t in scene.env:
            _fill(t, IN_SENTINEL)
        torch.cuda.synchronize()
        _, returned, opened = _behind_gate(gate, _gate_stream(where, streams), list(zip(scene.env, real)),
                                           lambda: c.forward_lighting_host(f.pf, f.pv, hgb, f.em, got))
        _after_gate("vq_forward_lighting_host", returned, opened)
        assert torch.equal(got.view(torch.int32), want.view(torch.int32)), "vq_forward_lighting_host shaded from the maps' old contents"
    finally:
        torch.cuda.synchronize()
        c.close()


@pytest.mark.gpu
@pytest.mark.parametrize("where", WHERE)
def test_hdr_save_host_after_earlier_work(sctx, gate, streams, where):
    src, real = _f32(20, 37), hdr(20, 37, 3)
    src.copy_(real)
    want = sctx.hdr_save_host(src)
    _fill(src, IN_SENTINEL)
    torch.cuda.synchronize()
    got, returned, opened = _behind_gate(gate, _gate_stream(where, streams), [(src, real)], lambda: sctx.hdr_save_host(src))
    _after_gate("vq_hdr_save_host", returned, opened)
    assert got == want, "vq_hdr_save_host encoded the image before it was written"


@pytest.mark.gpu
@pytest.mark.parametrize("where", WHERE)
def test_hdr_load_host_after_earlier_work(sctx, gate, streams, where):
    """behind the gate a copy reads the image the call overwrites: it must still see the old contents"""
    data = vq.hdr_pack_file(sctx.hdr_encode_rgbe(hdr(20, 37, 4)).cpu().numpy())
    out = _f32(20, 37)
    want_lum = sctx.hdr_load_host(data, out)
    want = out.clone()
    old = hdr(20, 37, 5)
    out.copy_(old)
    snap = torch.full_like(out, float("nan"))
    torch.cuda.synchronize()
    lum, returned, opened = _behind_gate(gate, _gate_stream(where, streams), [(snap, out)], lambda: sctx.hdr_load_host(data, out))
    _after_gate("vq_hdr_load_host", returned, opened)
    assert torch.equal(_words(snap), _words(old)), "vq_hdr_load_host overwrote the image while earlier work was still reading it"
    assert torch.equal(_words(out), _words(want)) and np.float32(lum) == np.float32(want_lum)


@pytest.mark.gpu
@pytest.mark.parametrize("where", WHERE)
def test_material_table_create_after_earlier_work(sctx, scene, gate, streams, where):
    """the material textures are written behind the gate; the table (and its sampling copies, where a material has them) must hold
    what was written: the G-buffer produced with it equals the one produced with the scene's table"""
    f = scene.f
    si = f.inputs()
    want = [_f32(f.h, f.w) for _ in range(4)]
    sctx.gbuffer_from_materials(si, f.table, f.pf.fAmbientLightingFactor, vq.GBuffer(*(_img(o) for o in want)))
    tex, writes = [], []
    for d in scene.chains:
        mt = vq.MaterialTextures()
        for slot in vq.MATERIAL_TEXTURE_SLOTS:
            e = d.get(slot)
            if e is not None:
                buf, w, h, levels = e
                real = torch.from_numpy(buf).cuda()
                t = torch.empty_like(real)
                _fill(t, IN_SENTINEL)
                writes.append((t, real))
                setattr(mt, slot, vq.texture_of(t, w, h, levels))
        tex.append(mt)
    torch.cuda.synchronize()
    table, returned, opened = _behind_gate(gate, _gate_stream(where, streams), writes, lambda: sctx.material_table(scene.mats, tex))
    try:
        _after_gate("vq_material_table_create", returned, opened)
        got = [_f32(f.h, f.w) for _ in range(4)]
        sctx.gbuffer_from_materials(si, table, f.pf.fAmbientLightingFactor, vq.GBuffer(*(_img(o) for o in got)))
        torch.cuda.synchronize()
        assert_bits("G-buffer from the gated table", got, want)
    finally:
        torch.cuda.synchronize()
        table.close()


# ---- part 3: threads sharing a context, each on its own stream ------------------------------------------------------------------
# the calls the header does not list as exceptions; the shading calls use the environment registered before the threads start
THREAD_MIX = {
    "forward": lambda S, k: r_forward(S, k, reg=True),
    "forward multi_signal": lambda S, k: r_forward_multi(S, k, reg=True, signal_form=True),
    "from_materials": lambda S, k: r_from_materials(S, k, reg=True),
    "shadowed_from_materials": lambda S, k: r_from_materials(S, k, reg=True, shadowed=True),
    "from_materials multi_signal": lambda S, k: r_from_materials(S, k, reg=True, multi=True),
    "shadowed_from_materials multi_signal": lambda S, k: r_from_materials(S, k, reg=True, shadowed=True, multi=True),
    **{name: ROWS[name][1] for name in (
        "skydome", "skydome multi_signal", "apply_reflections", "apply_reflections multi_signal",
        "post_process fsr 2x", "post_process fsr up", "post_process cas", "post_process tonemap", "post_process multi_signal",
        "tonemap", "cas", "fsr_easu", "fsr_rcas", "tonemap multi_signal", "cas multi_signal", "fsr_easu multi_signal",
        "fsr_rcas multi_signal", "gaussian_blur_x", "gaussian_blur_y", "spd_downsample", "hdri_build_mips spd",
        "hdri_build_mips per level", "diffuse_irradiance", "specular_prefilter", "specular_prefilter_multi",
        "specular_prefilter_ranges", "brdf_integration_lut", "hdr_decode", "hdr_encode_rgbe", "texture_build_mips",
        "gbuffer_from_materials")},
}
ROUNDS = 50


def _refusals(sctx):
    """refused calls (as the *_args tests make them), one message each: -> [(call(ctx), message)]"""
    a, b = _f32(4, 4), _f32(4, 5)
    ia, ib = _img(a), _img(b)
    tm = synth.default_tonemapper()
    cas = vq.cas_setup(0.5, 4, 4, 4, 4)
    easu = vq.fsr_easu_con(4, 4, 4, 4, 8, 8)
    m = vq.Matrix((vq.f32 * 16)(*([1.0] + [0.0] * 4) * 3 + [1.0]))
    pyr = vq.pyramid_of(torch.zeros((1, 4), device="cuda"), 1, 1, 1)
    calls = [
        lambda c: vq.lib.vq_tonemap(c._h, C.byref(tm), ia, ib, None),
        lambda c: vq.lib.vq_cas(c._h, cas, ia, ia, None),
        lambda c: vq.lib.vq_fsr_easu(c._h, easu, 7, ia, ib, None),
        lambda c: vq.lib.vq_skydome(c._h, C.byref(m), pyr, None, ia, 0, 9, None),
    ]
    out = []
    for call in calls:
        assert call(sctx) == vq.VQ_ERR_INVALID_ARG
        out.append((call, vq.lib.vq_last_error()))
    assert len({msg for _, msg in out}) == len(out) and all(msg for _, msg in out), [msg for _, msg in out]
    return out, (a, b, pyr)


class Kit:
    """one thread's rows (its own outputs; inputs seeded by the thread, the shading rows' inputs shared) and their serial bits"""

    def __init__(self, S, seed, ctx, stream):
        self.rows = {name: build(S, seed) for name, build in THREAD_MIX.items()}
        self.ctx, self.stream = ctx, stream
        n0 = vq.launch_count()
        self.refs = {name: reference(row, ctx, stream) for name, row in self.rows.items()}
        self.launches = vq.launch_count() - n0

    def round(self):
        s = self.stream
        for row in self.rows.values():
            row.prime(s, inplace_only=True)
            row.run(self.ctx, s)
        s.synchronize()

    def check(self, what):
        with torch.cuda.stream(self.stream):
            for name, row in self.rows.items():
                assert_bits(f"{what} {name}", row.outs, self.refs[name])


def run_threads(sg, S, contexts, n_threads, rounds):
    streams = make_streams(sg, n_threads)
    try:
        for c in contexts:
            c.environment_prepare(S.f.em)
        kits = [Kit(S, 100 + k, contexts[k % len(contexts)], streams[k]) for k in range(n_threads)]
        refusals, keep = _refusals(contexts[0])
        torch.cuda.synchronize()
        barrier = threading.Barrier(n_threads)
        errors = []

        def work(k):
            kit = kits[k]
            try:
                for r in range(rounds):
                    barrier.wait()
                    kit.round()
                    kit.check(f"thread {k} round {r}:")
                    if k % 2:
                        call, msg = refusals[(k // 2) % len(refusals)]
                        assert call(kit.ctx) == vq.VQ_ERR_INVALID_ARG
                    else:
                        msg = b""
                    got = vq.lib.vq_last_error()
                    assert got == msg, f"thread {k} round {r}: vq_last_error is {got!r}, want {msg!r}"
            except BaseException as e:       # noqa: BLE001  (reported by the main thread)
                errors.append(e)
                barrier.abort()

        n0 = vq.launch_count()
        threads = [threading.Thread(target=work, args=(k,), name=f"caller {k}") for k in range(n_threads)]
        for t in threads:
            t.start()
        for t in threads:
            t.join()
        if errors:
            raise next((e for e in errors if not isinstance(e, threading.BrokenBarrierError)), errors[0])
        assert vq.launch_count() - n0 == rounds * sum(kit.launches for kit in kits), "launches in the threads"
    finally:
        torch.cuda.synchronize()
        for c in contexts:
            c.environment_invalidate()
        for s in streams:
            sg.sg_stream_destroy(C.c_void_p(s.cuda_stream))


@pytest.mark.gpu
@pytest.mark.parametrize("n_threads", [4, 8])
def test_threads_share_one_context(sg, sctx, scene, n_threads):
    run_threads(sg, scene, [sctx], n_threads, ROUNDS)


@pytest.mark.gpu
def test_threads_on_two_contexts(sg, sctx, scene):
    c = vq.Context(0)
    try:
        run_threads(sg, scene, [sctx, c], 4, ROUNDS)
    finally:
        c.close()
