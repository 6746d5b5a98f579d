"""-m gpu: no pixel's result depends on where it is shaded. K1 (forward_kernel: plain, SHADOWED, MULTI) and the one-pass PSMain
kernel (psmain_kernel: plain, SHADOWED) pick their light loop per warp (the TINY vote), exchange gather data between lane pairs,
and shade pixels they never store (ragged tiles, discarded pixels, the second row of an odd height). The bit identity of the
fused, multi-destination and host calls with the two-pass path rests on each pixel's bits depending on that pixel alone.

Metamorphic and bit for bit, on domain frames (forward_domain adversarial G-buffers, a light_domain mixed frame) with map-less
materials, whose G-buffer texels do not depend on their neighbours: permute the pixels, shade, undo the permutation, compare."""
import numpy as np
import pytest
import torch

import forward_domain as fd
import light_domain as ld
import psmain_domain as pd
import vqengine_b200 as vq
from gpu_util import dev, host
from test_forward_domain_gpu import _env
from test_psmain_domain_gpu import tall_frame
from vqengine_b200.shader_data import TEXCFG_DIFFUSE

pytestmark = pytest.mark.gpu

SENTINEL = 12345.0
CAM = (0.0, 5.0, -17.0)
KERNELS = ["k1", "k1 shadowed", "k1 multi", "psmain", "psmain shadowed"]


def _frame(kind):
    """512 x 8 domain frames with their lights and environment, and a 512 x 300 one ("tall": more row pairs than psmain's grid has
    CTAs per column, so CTAs shade a second tile from a stage holding their first tile's texels); fAmbientLightingFactor = 1 (the
    adapted inputs' ao is exact)"""
    if kind == "tall":
        planes, env, pf, pv = tall_frame(300)
        sm = torch.cuda.get_device_properties(0).multi_processor_count
        assert planes[0].shape[0] // 2 > pd.ps_ctas_per_column(512, sm), "the tall frame must give some CTA a second tile"
    elif kind == "adversarial":
        planes, _ = fd.adversarial_gbuffer(512, 8, 31, CAM, emissive=True)
        env = fd.make_env(16, 33, (48, 20), seed=31)
        pf, pv = fd.constants(CAM, env["spec_mips"], 0.0, lights=fd.lights(512, 8, 31, 0.0))
    else:
        p = pd.crop(ld.mixed_frame("one of each", seed=702), 512)
        planes, env, pf, pv = [np.ascontiguousarray(x[:8]) for x in p["planes"]], p["env"], p["pf"], p["pv"]
    pf = ld.with_dark_caster(pf)
    pf.fAmbientLightingFactor = 1.0
    return planes, env, pf, pv


def shade(ctx, kernel, planes, env, pf, pv, materials=None, alpha_mask=False):
    """one kernel on the G-buffer planes (K1) or their adapted interpolants (psmain); `materials` = (surface planes, materials,
    textures) replaces the adaptation"""
    h, w = planes[0].shape[:2]
    em, tk = _env(vq, env)
    out = dev(np.full((h, w, 4), SENTINEL, np.float32))
    cubes = dev(np.full((pf.Lights.numPointCasters, 6, 2, 2), np.inf, np.float32))
    if kernel.startswith("k1"):
        d = [dev(p) for p in planes]
        gb = vq.GBuffer(*(vq.image_of(t) for t in d[:3]), vq.image_of(d[3]) if len(d) > 3 else vq.null_image())
        if kernel == "k1":
            ctx.forward_lighting(pf, pv, gb, em, out)
        elif kernel == "k1 shadowed":
            ctx.forward_lighting_shadowed(pf, pv, gb, em, out, point_cubes=cubes)
        else:                                                     # two destinations: forward_kernel<MULTI>
            out2 = dev(np.full((h, w, 4), SENTINEL, np.float32))
            ctx.forward_lighting_multi(pf, pv, gb, em, [vq.image_of(out), vq.image_of(out2)], dst_row_offset=0)
            a, b = host(out), host(out2)
            assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
            return a
        return host(out)
    sp, mats, tex = materials if materials is not None else (*pd.adapt(planes), None)
    d = [dev(p) for p in sp]
    si = vq.SurfaceInputs(vq.image_of(d[0]), vq.image_of(d[1]), vq.image_of(d[2]), vq.image_of(d[3], 1))
    table = ctx.material_table(mats, tex or [vq.MaterialTextures() for _ in mats])
    if kernel == "psmain":
        ctx.forward_lighting_from_materials(pf, pv, si, table, em, out, alpha_mask=alpha_mask)
    else:
        ctx.forward_lighting_shadowed_from_materials(pf, pv, si, table, em, out, point_cubes=cubes, alpha_mask=alpha_mask)
    got = host(out)
    table.close()
    return got


def same(tag, a, b):
    bad = (a.view(np.uint32) != b.view(np.uint32)).any(-1)
    assert not bad.any(), f"{tag}: {int(bad.sum())} pixels changed with their placement, first {np.argwhere(bad)[0]}"


FRAMES = ["adversarial", "mixed"]


def test_gbuffer_texels_do_not_depend_on_neighbours(ctx):
    """the precondition: the producer's texels of a permuted frame are the permuted texels (two-pass G-buffer)"""
    planes, env, pf, pv = _frame("adversarial")
    h, w = planes[0].shape[:2]
    perm = np.random.default_rng(1).permutation(h * w)

    def produce(pl):
        sp, mats = pd.adapt(pl)
        d = [dev(p) for p in sp]
        si = vq.SurfaceInputs(vq.image_of(d[0]), vq.image_of(d[1]), vq.image_of(d[2]), vq.image_of(d[3], 1))
        table = ctx.material_table(mats, [vq.MaterialTextures() for _ in mats])
        gbt = [dev(np.zeros((h, w, 4), np.float32)) for _ in range(4)]
        ctx.gbuffer_from_materials(si, table, 1.0, vq.GBuffer(*(vq.image_of(t) for t in gbt)))
        out = [host(t) for t in gbt]
        table.close()
        return out

    a = produce(planes)
    b = produce([p.reshape(-1, 4)[perm].reshape(h, w, 4) for p in planes])
    for x, y in zip(a, b):
        assert np.array_equal(x.reshape(-1, 4)[perm].view(np.uint32), y.reshape(-1, 4).view(np.uint32))


@pytest.mark.parametrize("frame", FRAMES)
@pytest.mark.parametrize("kernel", KERNELS)
def test_permutations(ctx, kernel, frame):
    """a random permutation; K1's A and B halves swapped / psmain's rows y and y+1 swapped; column shifts by 1, 31, 32, 127, 128
    (ragged last tiles); fold against unfold"""
    planes, env, pf, pv = _frame(frame)
    h, w = planes[0].shape[:2]
    base = shade(ctx, kernel, planes, env, pf, pv)
    assert (base != SENTINEL).all()
    perm = np.random.default_rng(7).permutation(h * w)
    got = shade(ctx, kernel, [p.reshape(-1, 4)[perm].reshape(h, w, 4) for p in planes], env, pf, pv)
    back = np.empty_like(got.reshape(-1, 4))
    back[perm] = got.reshape(-1, 4)
    same(f"{kernel}/{frame}: random permutation", back.reshape(h, w, 4), base)
    if kernel.startswith("k1"):
        idx = np.arange(w) ^ 128                                  # A <-> B within each 256-pixel tile
        sw = [np.ascontiguousarray(p[:, idx]) for p in planes]
        same(f"{kernel}/{frame}: halves swapped", shade(ctx, kernel, sw, env, pf, pv)[:, idx], base)
    else:
        idx = np.arange(h) ^ 1                                    # rows y <-> y+1 within each tile
        sw = [np.ascontiguousarray(p[idx]) for p in planes]
        same(f"{kernel}/{frame}: rows swapped", shade(ctx, kernel, sw, env, pf, pv)[idx], base)
    for s in (1, 31, 32, 127, 128):
        pad = [np.ascontiguousarray(np.concatenate([p[:, w - s:], p], 1)) for p in planes]
        same(f"{kernel}/{frame}: shifted by {s}", shade(ctx, kernel, pad, env, pf, pv)[:, s:], base)
    folded = shade(ctx, kernel, [pd.fold(p) for p in planes], env, pf, pv)
    same(f"{kernel}/{frame}: folded", pd.unfold(folded), base)


@pytest.mark.parametrize("frame", ["mixed", "tall"])
@pytest.mark.parametrize("kernel", KERNELS)
def test_tiny_vote_does_not_change_other_pixels(ctx, kernel, frame):
    """every pixel rough (no warp votes TINY), then a roughness-0 pixel in every 32 columns of every row (every warp of both
    kernels votes TINY): the pixels that were not changed keep their bits, so shade_light2<true> and <false> round a pixel that
    does not escape alike"""
    planes, env, pf, pv = _frame(frame)
    planes = [p.copy() for p in planes]
    planes[1][..., 3] = np.maximum(planes[1][..., 3], np.float32(0.05))
    assert not pd.tiny_pixels(planes).any()
    none = shade(ctx, kernel, planes, env, pf, pv)
    marked = np.zeros(planes[0].shape[:2], bool)
    marked[:, 5::32] = True
    tiny = [p.copy() for p in planes]
    tiny[1][marked, 3] = 0.0
    warps = pd.k1_warps(marked.shape) if kernel.startswith("k1") else pd.ps_warps(marked.shape)
    assert (pd.per_warp(marked, warps) > 0).all()
    every = shade(ctx, kernel, tiny, env, pf, pv)
    same(f"{kernel}: TINY in every warp", every[~marked], none[~marked])


def _discard_material():
    """a material whose 1x1 single-level diffuse map has alpha 0: discarded under the alpha mask at any LOD"""
    m = pd.material((1.0, 1.0, 1.0), 0.0, 0.5, (0.0, 0.0, 0.0), 0.0)
    m.textureConfig = float(TEXCFG_DIFFUSE)
    t = torch.tensor([255, 255, 255, 0], dtype=torch.uint8, device="cuda")
    mt = vq.MaterialTextures()
    mt.diffuse = vq.texture_of(t, 1, 1, 1)
    return m, mt, t


@pytest.mark.parametrize("frame", ["mixed", "tall"])
@pytest.mark.parametrize("kernel", ["psmain", "psmain shadowed"])
def test_discarded_pixels_do_not_change_other_pixels(ctx, kernel, frame):
    """discarded pixels (whose stage holds zeros, roughness 0 and a zero normal, on a CTA's first tile; the previous tile's
    texels on the later tiles of the tall frame) sit in warps of ordinary pixels: the produced pixels equal the frame without
    discards, and the discarded ones are not written"""
    planes, env, pf, pv = _frame(frame)
    sp, mats = pd.adapt(planes)
    m, mt, keep = _discard_material()
    tex = [vq.MaterialTextures() for _ in mats] + [mt]
    full = shade(ctx, kernel, planes, env, pf, pv, materials=(sp, mats + [m], tex), alpha_mask=True)
    rng = np.random.default_rng(3)
    disc = rng.uniform(0, 1, planes[0].shape[:2]) < 0.15
    disc[1, :] = True                                      # a whole tile row: the second row of every pair of tiles
    disc[4, 64:96] = True                                  # one warp's 32 columns of a row
    disc[7, :200] = True
    disc[-1, 300:] = True                                  # the last tile row (on the tall frame, a CTA's later tile)
    sp2 = [p.copy() for p in sp]
    sp2[2][disc, 3] = float(len(mats))
    got = shade(ctx, kernel, planes, env, pf, pv, materials=(sp2, mats + [m], tex), alpha_mask=True)
    assert (got[disc] == SENTINEL).all()
    same(f"{kernel}: discards", got[~disc], full[~disc])


HOST_HEIGHTS = [1, 15, 16, 17, 255, 256, 257, 263]


@pytest.mark.parametrize("h", HOST_HEIGHTS)
def test_host_call_equals_device_call(ctx, h):
    """vq_forward_lighting_host (rows cut into 1, 4 or 8 row chunks over three streams) equals vq_forward_lighting bit for bit,
    with packed and pitched host planes, with and without the emissive plane"""
    w = 300
    planes, _ = fd.adversarial_gbuffer(w, h, 40 + h, CAM, emissive=True)
    env = fd.make_env(8, 16, (20, 48), seed=h)
    pf, pv = fd.constants(CAM, env["spec_mips"], 0.0, lights=fd.lights(w, h, 40 + h, 0.0))
    em, tk = _env(vq, env)
    for emissive in (False, True):
        pl = planes if emissive else planes[:3]
        d = [dev(p) for p in pl]
        gb = vq.GBuffer(*(vq.image_of(t) for t in d[:3]), vq.image_of(d[3]) if emissive else vq.null_image())
        want = dev(np.zeros((h, w, 4), np.float32))
        ctx.forward_lighting(pf, pv, gb, em, want)
        want = host(want)
        for pitched in (False, True):
            pad = 7 if pitched else 0
            hp = []
            for p in pl:
                t = torch.zeros((h, w + pad, 4), dtype=torch.float32)
                t[:, :w] = torch.from_numpy(p)
                hp.append(t[:, :w])
            hout = torch.full((h, w + pad, 4), SENTINEL, dtype=torch.float32)
            hgb = vq.GBuffer(*(vq.image_of(t) for t in hp[:3]), vq.image_of(hp[3]) if emissive else vq.null_image())
            ctx.forward_lighting_host(pf, pv, hgb, em, hout[:, :w])
            got = hout.numpy()
            same(f"host h={h} emissive={emissive} pitched={pitched}", got[:, :w], want)
            assert (got[:, w:] == SENTINEL).all()
