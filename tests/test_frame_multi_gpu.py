"""-m gpu: the band forms of the skydome and the reflection composite (vq_skydome_multi_signal, vq_apply_reflections_multi_signal).

Into every destination each call must store, bit for bit, what its single call leaves in the local frame outs[0] on the band's
frame rows, and touch no other row (the peers' frames start as NaN). Inputs hold the whole frame (offset 0) or just the band, at odd
and even offsets. Simulated worlds (tests/test_rendezvous_gpu.py: every rank on this one GPU, flag words whose waits are already
satisfied) run one rank's scene-colour step as the multi-GPU frame does: its shading call into its local frame alone, then the sky into
every rank's frame with the signal; every frame must equal the single-GPU frame. One world goes on through the composite and the fused
post chain. A rendezvous between ranks running at the same time needs two or more GPUs (tools/perf_frame_multi.py under torchrun)."""
import numpy as np
import pytest
import torch

import frame_domain as fd
import vqengine_b200 as vq
from gpu_util import dev
from test_multi_shading_gpu import Frame
from test_post_fused_gpu import chain, fsr_consts
from test_psmain_shadowed_gpu import _maps, _shadow_scene
from test_rendezvous_gpu import ORDERS, Case, SimWorld, pw, rank_dests, run_world  # noqa: F401 (pw: fixture)
from vqengine_b200 import synth
from vqengine_b200.distributed import even_tiles

pytestmark = pytest.mark.gpu
NAN = float("nan")


def _same(name, got, want):
    g, w = got.view(torch.int32), want.view(torch.int32)
    if not torch.equal(g, w):
        bad = (g != w).reshape(got.shape[0], -1).any(-1)
        pytest.fail(f"{name}: {int(bad.sum())} rows differ, first {torch.nonzero(bad).flatten()[:6].tolist()}")


def _peers(n, h, w, base, pitched):
    """outs[0] = a copy of `base` (the local frame), then n - 1 NaN frames; every other one a view into a wider allocation"""
    outs = [dev(base)]
    for k in range(1, n):
        if pitched and k % 2:
            big = torch.full((h, w + 5, 4), NAN, device="cuda")
            outs.append(big[:, 2:2 + w])
        else:
            outs.append(torch.full((h, w, 4), NAN, device="cuda"))
    return outs


def _check_dests(name, outs, ref, base, rows):
    """outs[0] == the single call's frame; every peer: the band rows of it, NaN elsewhere"""
    a, b = rows
    _same(f"{name} local frame", outs[0].contiguous(), ref)
    for k, o in enumerate(outs[1:], 1):
        want = torch.full_like(ref, NAN)
        want[a:b] = ref[a:b]
        _same(f"{name} destination {k}", o.contiguous(), want)


# layouts of a band's inputs: (frame rows [a, b), the plane's first frame row): whole = rows of the whole-frame plane at offset 0;
# band = a plane holding rows [a, b) at offset a; margin = a plane holding rows [a - 3, b + 2) at offset a - 3
def _plane_rows(layout, a, b, h):
    if layout == "whole":
        return 0, h
    if layout == "band":
        return a, b
    return max(a - 3, 0), min(b + 2, h)


def _band_args(layout, plane, a, b, h):
    p0, p1 = _plane_rows(layout, a, b, h)
    return np.ascontiguousarray(plane[p0:p1]), p0, (a - p0, b - p0)


# ---- the skydome -------------------------------------------------------------------------------------------------------------------
W, H = 67, 33                          # a ragged width (64 + 3) and an odd height
BANDS = [(0, 17), (7, 20), (6, 33), (10, 11), (13, 14), (32, 33)]    # offsets 0, odd and even; one-row bands; the last row


def _sky(w, h, m=None, hw=128, hh=64):
    m = fd.view_proj(fd.yaw_pitch(0.9, 0.25), 1.2, w / h) if m is None else m
    hdri = dev(fd.sky_hdri(hw, hh, seed=5))
    return m, hdri, vq.pyramid_of(hdri, hw, hh, 1)


def _sky_single(ctx, m, pyr, base, mask, rows):
    out = dev(base)
    ctx.skydome(m, pyr, out, normal_mask=dev(mask) if mask is not None else None, row_begin=rows[0], row_end=rows[1])
    return out


@pytest.mark.parametrize("mask_kind", [None, "holes", "signed"], ids=["no-mask", "holes", "signed"])
@pytest.mark.parametrize("layout", ["whole", "band", "margin"])
@pytest.mark.parametrize("n_dest", [1, 2, 3, 8])
def test_skydome_band_equals_single(ctx, n_dest, layout, mask_kind):
    """every band of BANDS; the signed mask has -0 (no surface) and NaN (a surface) normals; peers 1, 3, 5, 7 are pitched"""
    m, keep, pyr = _sky(W, H)
    base = np.random.default_rng(1).random((H, W, 4), dtype=np.float32)
    mask = fd.sky_mask(mask_kind, W, H, seed=3)
    for a, b in BANDS:
        ref = _sky_single(ctx, m, pyr, base, mask, (a, b))
        outs = _peers(n_dest, H, W, base, pitched=True)
        off = _plane_rows(layout, a, b, H)[0]
        rows = (a - off, b - off)
        kw = {"normal_mask": dev(_band_args(layout, mask, a, b, H)[0])} if mask is not None else {}
        n0 = vq.launch_count()
        ctx.skydome_multi(m, pyr, [vq.image_of(o) for o in outs], off, row_begin=rows[0], row_end=rows[1], **kw)
        assert vq.launch_count() - n0 == 1
        _check_dests(f"sky {layout} rows {a}-{b}", outs, ref, base, (a, b))


def test_skydome_pitched_mask_and_frame(ctx):
    """a mask and a local frame that are views into wider allocations"""
    m, keep, pyr = _sky(W, H)
    base = np.random.default_rng(2).random((H, W, 4), dtype=np.float32)
    mask = fd.sky_mask("signed", W, H, seed=4)
    ref = _sky_single(ctx, m, pyr, base, mask, (5, 30))
    big_m = torch.zeros((H, W + 3, 4), device="cuda")
    big_m[:, 1:1 + W] = dev(mask)
    big_f = torch.full((H, W + 9, 4), -3.0, device="cuda")
    big_f[:, 4:4 + W] = dev(base)
    outs = [big_f[:, 4:4 + W]] + _peers(3, H, W, base, pitched=True)[1:]
    ctx.skydome_multi(m, pyr, [vq.image_of(o) for o in outs], 0, normal_mask=big_m[:, 1:1 + W], row_begin=5, row_end=30)
    _check_dests("sky pitched", outs, ref, base, (5, 30))
    assert bool((big_f[:, :4] == -3.0).all()) and bool((big_f[:, 4 + W:] == -3.0).all())


def _crossing_camera(kind, w, h):
    """a camera whose clip-space w (or ray) crosses a limit of the fast division inside a row pair: w = ny * m7 + m15 varies by row"""
    m = fd.view_proj(fd.yaw_pitch(0.4, 0.3), 1.1, w / h).copy()
    ys = np.float32(1.0) - ((np.arange(h, dtype=np.float32) + np.float32(0.5)) / np.float32(h)) * np.float32(2.0)
    m[3] = m[11] = 0.0
    if kind == "w-zero":                             # w rounds to exactly 0 on row h // 2 - 3
        m[7], m[15] = 1.0, -ys[h // 2 - 3]
    elif kind == "w-tiny":                           # |w| < 1e-15 on a few rows
        m[7], m[15] = 1e-14, -1e-14 * float(ys[h // 3])
    elif kind == "w-huge":                           # |w| >= 1e15 away from the centre rows
        m[7], m[15] = 3e15, 0.0
    else:                                            # ray-huge: |ray.x| >= 1e15 away from the centre rows
        m[7], m[15] = 0.0, 1.0
        m[4], m[8], m[12] = 5e15, 0.0, 0.0
    m = m.astype(np.float32)
    slow = fd.sky_fallback(fd.sky_ray(m, w, h)).any(axis=1)
    cross = [y for y in range(h - 1) if slow[y] != slow[y + 1]]
    assert cross, (kind, "no row pair straddles a fast-path limit")
    return m, cross


@pytest.mark.parametrize("kind", ["w-zero", "w-tiny", "w-huge", "ray-huge"])
def test_skydome_partner_row_independence(ctx, kind):
    """bands that start on every row around a fast-path crossing pair their rows differently from the full-frame call, so one pixel of
    a pair takes the other branch there: every band equals the full-frame call's rows bit for bit"""
    w, h = 37, 41
    m, cross = _crossing_camera(kind, w, h)
    m, keep, pyr = _sky(w, h, m)
    base = np.zeros((h, w, 4), np.float32)
    full = _sky_single(ctx, m, pyr, base, None, (0, h))
    for y in cross:
        for a in range(max(y - 2, 0), min(y + 3, h)):
            for b in sorted({a + 1, a + 2, a + 5, min(a + 8, h)}):
                if b > h:
                    continue
                outs = _peers(2, h, w, base, pitched=False)
                ctx.skydome_multi(m, pyr, [vq.image_of(o) for o in outs], a, row_begin=0, row_end=b - a)
                torch.cuda.synchronize()
                for k, o in enumerate(outs):
                    _same(f"{kind} band {a}-{b} destination {k}", o[a:b], full[a:b])


# ---- the reflection composite ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("bv", [False, True], ids=["plain", "bounding-volumes"])
@pytest.mark.parametrize("layout", ["whole", "band", "margin"])
@pytest.mark.parametrize("n_dest", [1, 2, 3, 8])
def test_composite_band_equals_single(ctx, n_dest, layout, bv):
    """the special values of frame_domain.composite_planes; peers 1, 3, 5, 7 pitched"""
    s, r, b = fd.composite_planes(W, H, seed=7)
    ref = dev(s)
    ctx.apply_reflections(ref, dev(r), dev(b) if bv else None)
    for a, e in BANDS:
        want = dev(s)
        want[a:e] = ref[a:e]
        outs = _peers(n_dest, H, W, s, pitched=True)
        rp, off, rows = _band_args(layout, r, a, e, H)
        bp = _band_args(layout, b, a, e, H)[0] if bv else None
        n0 = vq.launch_count()
        ctx.apply_reflections_multi(dev(rp), [vq.image_of(o) for o in outs], off, bounding_volumes=dev(bp) if bv else None,
                                    row_begin=rows[0], row_end=rows[1])
        assert vq.launch_count() - n0 == 1
        _check_dests(f"composite {layout} rows {a}-{e}", outs, want, s, (a, e))


@pytest.mark.parametrize("bv", [False, True], ids=["plain", "bounding-volumes"])
def test_composite_large_band(ctx, bv):
    """3840 wide, a 1000-row band: more row groups than the capped grid, so each CTA strides the band"""
    w, h = 3840, 1080
    s, r, b = fd.composite_planes(w, h, seed=9)
    ref = dev(s)
    ctx.apply_reflections(ref, dev(r), dev(b) if bv else None)
    want = dev(s)
    want[37:1037] = ref[37:1037]
    outs = _peers(2, h, w, s, pitched=False)
    ctx.apply_reflections_multi(dev(r[37:1037]), [vq.image_of(o) for o in outs], 37, bounding_volumes=dev(b[37:1037]) if bv else None)
    _check_dests("composite 3840x1080", outs, want, s, (37, 1037))


# ---- simulated worlds: shade into the local frame, then the sky into every frame ------------------------------------------------------
def _sky_frame(ctx, w, h):
    """the shading scene with its top 40 % and a scatter of pixels cleared (normal 0: sky), in the G-buffer and the interpolants"""
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(w, h)
    sky = np.zeros((h, w), bool)
    sky[:int(0.4 * h)] = True
    sky |= np.random.default_rng(w + h).random((h, w)) < 0.05
    planes = [p.copy() for p in planes]
    planes[1][sky, :3] = 0.0
    f = Frame(ctx, planes, mats, chains, env, pf, pv, _maps(maps, ()))
    f.gbt[1][torch.from_numpy(sky).cuda(), :3] = 0.0
    return f


def _scene_ref(ctx, f, call, m, pyr):
    """the single-GPU scene colour: the full-frame shading call, then the full-frame sky under the call's mask"""
    ref = torch.from_numpy(f.single(call)).cuda()
    ctx.skydome(m, pyr, ref, normal_mask=_mask(f, call))
    return ref


def _mask(f, call):
    return f.gbt[1] if call == "forward" else f.dp[1]


def _sky_case(ctx, f, call, n, m, pyr, name):
    ref = _scene_ref(ctx, f, call, m, pyr)
    bands = even_tiles(f.h, n)
    mask = _mask(f, call)

    def run(r, dests, signal, stream):
        a, b = bands[r]
        f.multi(call, [vq.image_of(dests[0])], 0, rows=(a, b), stream=stream)
        if call == "forward":        # whole-frame mask, offset 0
            ctx.skydome_multi(m, pyr, [vq.image_of(d) for d in dests], 0, normal_mask=mask, row_begin=a, row_end=b, stream=stream,
                              signal=signal)
        else:                        # the band's rows of the mask, at the band's offset
            ctx.skydome_multi(m, pyr, [vq.image_of(d) for d in dests], a, normal_mask=mask[a:b], stream=stream, signal=signal)
    return Case(name, n, ref, NAN, [[band] for band in bands], run)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("call", ["forward", "from_materials"])
def test_scene_colour_world(ctx, pw, call, n, order):
    """257 x 41: a ragged width; even_tiles gives 8 ranks bands of 4 and 6 rows, some starting on odd rows"""
    f = _sky_frame(ctx, 257, 41)
    m, keep, pyr = _sky(257, 41)
    run_world(pw, _sky_case(ctx, f, call, n, m, pyr, f"sky {call} n{n}"), SimWorld(n, order))
    f.close()


def _composite_case(ctx, n, w, h, name):
    s, r, b = fd.composite_planes(w, h, seed=n)
    ref = dev(s)
    ctx.apply_reflections(ref, dev(r), dev(b))
    bands = even_tiles(h, n)
    st, rt, bt = dev(s), dev(r), dev(b)

    def run(r_, dests, signal, stream):
        a, e = bands[r_]
        dests[0][a:e] = st[a:e]                      # the rank's band of the scene colour, in its local frame
        stream.wait_stream(torch.cuda.current_stream())
        ctx.apply_reflections_multi(rt[a:e], [vq.image_of(d) for d in dests], a, bounding_volumes=bt[a:e], stream=stream,
                                    signal=signal)
    return Case(name, n, ref, NAN, [[band] for band in bands], run)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
def test_composite_world(ctx, pw, n, order):
    """each rank composites its band (band-local reflection and bounding-volume planes) into every frame"""
    run_world(pw, _composite_case(ctx, n, 131, 37, f"composite n{n}"), SimWorld(n, order))


@pytest.mark.parametrize("n", [2, 3, 8])
def test_frame_chain_world(ctx, n):
    """shade -> sky -> composite -> post, stage by stage over every rank (the post pass reads the neighbours' rows, so each stage
    waits for the one before, as the rendezvous makes it wait on several GPUs): every rank's display frame equals the single-GPU
    chain, and every signalled call stores its epoch"""
    w, h = 257, 41
    f = _sky_frame(ctx, w, h)
    m, keep, pyr = _sky(w, h)
    ref = _scene_ref(ctx, f, "from_materials", m, pyr)
    _, r, bvol = fd.composite_planes(w, h, seed=11)
    rt, bt = dev(r), dev(bvol)
    ctx.apply_reflections(ref, rt, bt)
    tm = synth.default_tonemapper()
    oh, ow = 2 * h, 2 * w
    easu, rcas = fsr_consts(h, w, oh, ow)
    want = chain(ctx, ref, tm, (oh, ow), easu=easu, rcas=rcas, cas=None, mode=vq.VQ_ADDRESS_WRAP)
    bands, out_bands = even_tiles(h, n), even_tiles(oh, n)
    world = SimWorld(n, "scrambled")
    scene = [torch.full((h, w, 4), NAN, device="cuda") for _ in range(n)]
    display = [torch.full((oh, ow, 4), NAN, device="cuda") for _ in range(n)]
    # one epoch per rendezvous, through 2^32; every stage starts from flag words that satisfy its own waits (SimWorld.preset), since
    # the simulated ranks run one after another
    for sky_e, comp_e, post_e in ((0xFFFFFFFB, 0xFFFFFFFC, 0xFFFFFFFD), (0xFFFFFFFE, 0, 1), (2, 3, 4)):
        for t in scene + display:
            t.fill_(NAN)
        world.preset(sky_e)
        for r_ in range(n):
            a, b = bands[r_]
            f.multi("from_materials", [vq.image_of(scene[r_])], 0, rows=(a, b))
            ctx.skydome_multi(m, pyr, [vq.image_of(d) for d in rank_dests(world, scene, r_)], a, normal_mask=f.dp[1][a:b],
                              signal=world.signal(r_, sky_e))
            world.ran(r_, sky_e)
        world.check(f"sky epoch {sky_e:#x}")
        world.preset(comp_e)
        for r_ in range(n):
            a, b = bands[r_]
            n0 = vq.launch_count()
            ctx.apply_reflections_multi(rt[a:b], [vq.image_of(d) for d in rank_dests(world, scene, r_)], a, bounding_volumes=bt[a:b],
                                        signal=world.signal(r_, comp_e))
            assert vq.launch_count() - n0 == 1
            world.ran(r_, comp_e)
        world.check(f"composite epoch {comp_e:#x}")
        for k in range(n):
            _same(f"scene frame {k} epoch {comp_e:#x}", scene[k], ref)
        world.preset(post_e)
        for r_ in range(n):
            ctx.post_process_multi(tm, scene[r_], [vq.image_of(d) for d in rank_dests(world, display, r_)], *out_bands[r_], easu=easu,
                                   rcas=rcas, signal=world.signal(r_, post_e))
            world.ran(r_, post_e)
        world.check(f"post epoch {post_e:#x}")
        for k in range(n):
            _same(f"display frame {k} epoch {post_e:#x}", display[k], want)
    f.close()


# ---- the ticket ring ----------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["skydome", "composite"])
def test_ticket_ring_wraps(ctx, family):
    """320 signalled calls of each new retirement block in a row, 2 ranks: every slot of the 128-slot ticket-pair ring comes back
    twice, and every call signals exactly its word"""
    w, h = 100, 8
    bands = even_tiles(h, 2)
    s, r, b = fd.composite_planes(w, h, seed=3)
    m, keep, pyr = _sky(w, h)
    mask = fd.sky_mask("holes", w, h, seed=5)
    if family == "skydome":
        ref = _sky_single(ctx, m, pyr, s, mask, (0, h))
    else:
        ref = dev(s)
        ctx.apply_reflections(ref, dev(r), dev(b))
    mt, rt, bt = dev(mask), dev(r), dev(b)
    world = SimWorld(2, "rotated")
    frames = [dev(s) for _ in range(2)]
    for e in range(1, 161):
        world.preset(e)
        for f_ in frames:
            f_.copy_(dev(s))
        for r_ in range(2):
            a, e2 = bands[r_]
            dests = rank_dests(world, frames, r_)
            if family == "skydome":
                ctx.skydome_multi(m, pyr, [vq.image_of(d) for d in dests], 0, normal_mask=mt, row_begin=a, row_end=e2,
                                  signal=world.signal(r_, e))
            else:
                ctx.apply_reflections_multi(rt[a:e2], [vq.image_of(d) for d in dests], a, bounding_volumes=bt[a:e2],
                                            signal=world.signal(r_, e))
            world.ran(r_, e)
            world.check(f"{family} ring epoch {e} rank {r_}")
    for k, f_ in enumerate(frames):
        _same(f"{family} ring frame {k}", f_, ref)
