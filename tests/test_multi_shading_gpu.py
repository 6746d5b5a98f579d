"""-m gpu: the multi-destination forms of the shadowed and the from-materials shading calls
(vq_forward_lighting_shadowed_multi_signal, vq_forward_lighting_from_materials_multi_signal). Into every destination each call must
store, bit for bit, what its single-destination call stores into its one output, at rows offset by dst_row_offset, and touch nothing
else. Simulated worlds (every "rank" on this one GPU, its peers' frames being local destinations) must assemble the frame one
full-frame call computes, from whole-frame attribute planes with row ranges and from per-rank band planes. The tests here pass no
signal. tests/test_rendezvous_gpu.py runs these calls with one, on one GPU, on flag words whose waits are already satisfied. A
rendezvous between ranks running at the same time needs two or more GPUs (tools/perf_multi_shading.py under torchrun)."""
import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from gpu_util import dev, host, report
from shader_cases import _pixel_scene, _shadow_setup
from test_psmain_fused_gpu import SENTINEL, _env_maps, _table
from test_psmain_shadowed_gpu import SUBSETS, _maps, _shadow_scene
from vqengine_b200.distributed import even_tiles

pytestmark = pytest.mark.gpu
CALLS = ("shadowed", "from_materials", "shadowed_from_materials")


class Frame:
    """one frame's inputs on the device: attribute planes, material table, registered environment, constants, shadow maps, and the
    G-buffer the surface producer makes of the planes (with an emissive plane) for the G-buffer call"""

    def __init__(self, ctx, planes, mats, chains, env, pf, pv, maps, alpha_mask=False):
        self.ctx, self.pf, self.pv, self.alpha_mask = ctx, pf, pv, alpha_mask
        self.h, self.w = planes[0].shape[:2]
        self.dp = [dev(p) for p in planes]
        self.table, self.keep = _table(ctx, mats, chains)
        self.em, self.env_keep = _env_maps(env)
        ctx.environment_prepare(self.em)
        self.maps = {k: (dev(v) if v is not None else None) for k, v in maps.items()}
        self.gbt = [dev(np.zeros((self.h, self.w, 4), np.float32)) for _ in range(4)]
        ctx.gbuffer_from_materials(self.inputs(), self.table, pf.fAmbientLightingFactor, self.gbuffer(), alpha_mask=alpha_mask)

    def inputs(self, a=0, b=None):
        p = [t[a:b] for t in self.dp]
        return vq.SurfaceInputs(vq.image_of(p[0]), vq.image_of(p[1]), vq.image_of(p[2]),
                                vq.image_of(p[3], 1) if len(p) > 3 else vq.null_image())

    def gbuffer(self, a=0, b=None):
        return vq.GBuffer(*(vq.image_of(t[a:b]) for t in self.gbt))

    def single(self, call, rows=None):
        """the single-destination call over rows (default: the whole frame) into a SENTINEL frame -> host array"""
        rb, re = rows or (0, self.h)
        out = dev(np.full((self.h, self.w, 4), SENTINEL, np.float32))
        c = self.ctx
        if call == "forward":
            c.forward_lighting(self.pf, self.pv, self.gbuffer(), self.em, out, row_begin=rb, row_end=re)
        elif call == "shadowed":
            c.forward_lighting_shadowed(self.pf, self.pv, self.gbuffer(), self.em, out, row_begin=rb, row_end=re, **self.maps)
        elif call == "from_materials":
            c.forward_lighting_from_materials(self.pf, self.pv, self.inputs(), self.table, self.em, out, alpha_mask=self.alpha_mask,
                                              row_begin=rb, row_end=re)
        else:
            c.forward_lighting_shadowed_from_materials(self.pf, self.pv, self.inputs(), self.table, self.em, out,
                                                       alpha_mask=self.alpha_mask, row_begin=rb, row_end=re, **self.maps)
        return host(out)

    def multi(self, call, images, dst_row_offset, rows=None, band=None, signal=None, stream=None):
        """the multi-destination call: rows of the whole-frame inputs, or (band = (a, b)) inputs holding just rows [a, b)"""
        a, b = band or (0, self.h)
        rb, re = rows or (0, b - a)
        c = self.ctx
        if call == "forward":
            c.forward_lighting_multi(self.pf, self.pv, self.gbuffer(a, b), self.em, images, dst_row_offset, row_begin=rb, row_end=re,
                                     signal=signal, stream=stream)
        elif call == "shadowed":
            c.forward_lighting_shadowed_multi(self.pf, self.pv, self.gbuffer(a, b), self.em, images, dst_row_offset, row_begin=rb,
                                              row_end=re, signal=signal, stream=stream, **self.maps)
        else:
            maps = self.maps if call == "shadowed_from_materials" else {}
            c.forward_lighting_from_materials_multi(self.pf, self.pv, self.inputs(a, b), self.table, self.em, images, dst_row_offset,
                                                    alpha_mask=self.alpha_mask, row_begin=rb, row_end=re, signal=signal, stream=stream,
                                                    **maps)

    def world(self, call, n, layout):
        """n simulated ranks, rank r shading its even_tiles band into all n frames (its own first, then the others in rotated
        order, as the multi-GPU step orders them) -> the n frames as host arrays"""
        frames = [dev(np.full((self.h, self.w, 4), SENTINEL, np.float32)) for _ in range(n)]
        imgs = [vq.image_of(f) for f in frames]
        for r, (a, b) in enumerate(even_tiles(self.h, n)):
            if a == b:
                continue
            order = imgs[r:] + imgs[:r]
            if layout == "rows":
                self.multi(call, order, 0, rows=(a, b))
            else:
                self.multi(call, order, a, band=(a, b))
        return [host(f) for f in frames]

    def close(self):
        torch.cuda.synchronize()
        self.table.close()
        self.ctx.environment_invalidate()


def _bits_equal(tag, got, want):
    bad = (got.view(np.uint32) != want.view(np.uint32)).any(-1)
    assert not bad.any(), f"{tag}: {int(bad.sum())} pixels differ, first {np.argwhere(bad)[0]}, {report(tag, got, want)}"


def _shadow_frame(ctx, w=150, h=33, bind=("point", "spot", "dir"), **kw):
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(w, h, **kw)
    return Frame(ctx, planes, mats, chains, env, pf, pv, _maps(maps, bind))


# ---- 1. local destinations at an offset ---------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_dest", [1, 2, 3, 8])
@pytest.mark.parametrize("call", CALLS)
def test_local_destinations(ctx, call, n_dest):
    """1, 2, 3 and 8 destinations taller than the frame, at an even offset, a row range from an odd row: each destination's band
    equals the single-destination call bit for bit, and its rows above and below the band keep their contents"""
    f = _shadow_frame(ctx)
    off, rows = 6, (3, 30)
    want = f.single(call, rows)
    frames = [dev(np.full((off + f.h + 5, f.w, 4), SENTINEL, np.float32)) for _ in range(n_dest)]
    f.multi(call, [vq.image_of(t) for t in frames], off, rows=rows)
    for k, t in enumerate(frames):
        got = host(t)
        _bits_equal(f"{call} destination {k}", got[off:off + f.h], want)
        assert (got[:off] == SENTINEL).all() and (got[off + f.h:] == SENTINEL).all(), f"{call} destination {k}: rows outside written"
    f.close()


# ---- 2. simulated worlds ----------------------------------------------------------------------------------------------------------
def _check_world(f, call, n, layout):
    want = f.single(call)
    for r, got in enumerate(f.world(call, n, layout)):
        _bits_equal(f"{call} world {n} {layout} frame {r}", got, want)


@pytest.mark.parametrize("layout", ["rows", "bands"])
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("call", CALLS)
@pytest.mark.parametrize("records", [True, False])
def test_world_assembles_the_frame(ctx, call, n, layout, records, monkeypatch):
    """record and map-by-map materials, a ragged width and an odd height (257 x 41: 8 ranks get bands of 4 and 6 rows)"""
    monkeypatch.setenv("VQ_SURFACE_RECORDS", "1" if records else "0")
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(257, 41)
    if layout == "bands":
        planes = planes[:3]          # a band's SSAO plane wraps at the band's last row, not the frame's
    f = Frame(ctx, planes, mats, chains, env, pf, pv, _maps(maps))
    _check_world(f, call, n, layout)
    f.close()


@pytest.mark.parametrize("layout", ["rows", "bands"])
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("call", CALLS)
def test_world_alpha_mask(ctx, call, n, layout):
    """pixels the alpha mask discards stay untouched in every frame"""
    env, mats, chains, planes, pf, pv = _pixel_scene(96, 48, 7, casters=True)
    kw = _shadow_setup(pf, 110)
    if layout == "bands":
        planes = planes[:3]
    f = Frame(ctx, planes, mats, chains, env, pf, pv, _maps(kw), alpha_mask=True)
    if call != "shadowed":           # the G-buffer call shades every texel of its G-buffer
        assert (f.single(call) == SENTINEL).all(-1).any(), "the scene discards nothing"
    _check_world(f, call, n, layout)
    f.close()


@pytest.mark.parametrize("layout", ["rows", "bands"])
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("call", CALLS)
def test_world_rotated(ctx, call, n, layout):
    """a non-zero HDRI yaw: the ROT instantiations of the multi-destination kernels"""
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(300, 40, uv_scale=0.03)
    pf.fHDRIOffsetInRadians = 0.7
    f = Frame(ctx, planes[:3], mats, chains, env, pf, pv, _maps(maps))
    _check_world(f, call, n, layout)
    f.close()


@pytest.mark.parametrize("bind", SUBSETS, ids=["+".join(b) for b in SUBSETS])
@pytest.mark.parametrize("call", ["shadowed", "shadowed_from_materials"])
def test_world_caster_configurations(ctx, call, bind):
    """each map type bound alone and every pair, over 3 ranks with band planes"""
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(160, 36)
    f = Frame(ctx, planes[:3], mats, chains, env, pf, pv, _maps(maps, bind))
    _check_world(f, call, 3, "bands")
    f.close()


@pytest.mark.parametrize("case", ["no maps", "cubes without point casters", "maps without spot casters", "directional not shadowing"])
@pytest.mark.parametrize("call", ["shadowed", "shadowed_from_materials"])
def test_world_no_test_runs(ctx, call, case):
    """no PCF test to run: the unshadowed kernels, the frame of the single-destination call (and, from materials, one launch)"""
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(96, 20)
    L = pf.Lights
    bind = ()
    if case == "cubes without point casters":
        L.numPointCasters, bind = 0, ("point",)
    elif case == "maps without spot casters":
        L.numSpotCasters, bind = 0, ("spot",)
    elif case == "directional not shadowing":
        L.directional.shadowing, bind = 0, ("dir",)
    f = Frame(ctx, planes, mats, chains, env, pf, pv, _maps(maps, bind))
    _check_world(f, call, 2, "rows")
    if call == "shadowed_from_materials":
        out = [dev(np.full((f.h, f.w, 4), SENTINEL, np.float32)) for _ in range(2)]
        before = vq.launch_count()
        f.multi(call, [vq.image_of(t) for t in out], 0)
        assert vq.launch_count() - before == 1
    f.close()


# ---- 3. launches ------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("call,launches", [("shadowed", 2), ("from_materials", 1), ("shadowed_from_materials", 1)])
def test_launches_per_call(ctx, call, launches):
    f = _shadow_frame(ctx, 64, 32)
    out = [dev(np.full((f.h, f.w, 4), SENTINEL, np.float32)) for _ in range(3)]
    f.multi(call, [vq.image_of(t) for t in out], 0)        # warm: nothing lazy is left for the counted call
    before = vq.launch_count()
    f.multi(call, [vq.image_of(t) for t in out], 0)
    assert vq.launch_count() - before == launches
    f.close()
