"""-m gpu: the multi-destination post calls (vq_tonemap_multi_signal, vq_cas_multi_signal, vq_fsr_easu_multi_signal,
vq_fsr_rcas_multi_signal). Into every destination each call must store, bit for bit, what its single-destination call stores on
the requested rows, and touch no other row. Simulated worlds (every "rank" on this one GPU, its peers' display frames being local
destinations) must assemble the display frame the single-GPU chain computes, each rank running its distributed.post_chain_rows
plan into NaN-filled scratch, so that a row the plan misses would show up as NaN. The tests here pass no signal.
tests/test_rendezvous_gpu.py runs these calls with one, on one GPU, on flag words whose waits are already satisfied. A rendezvous
between ranks running at the same time needs two or more GPUs (tools/perf_post_multi.py under torchrun)."""
import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import equal_tiles, post_chain_rows

pytestmark = pytest.mark.gpu
SENTINEL = np.float32(-7.5e33)
TONEMAPS = [(vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_SRGB, 1), (vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_SRGB, 0),
            (vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_ST2084, 0), (vq.COLOR_SPACE_REC_2020, vq.DISPLAY_CURVE_ST2084, 0),
            (vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_LINEAR, 0), (vq.COLOR_SPACE_REC_709, 7, 0)]


def hdr(h, w, seed):
    """HDR scene colour with smooth gradients (so EASU's edge analysis sees structure), sharp edges and highlights"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([np.sin(xx * 0.31 + yy * 0.17) + 1.1, np.cos(xx * 0.07 - yy * 0.23) + 1.05, (xx + yy) % 7 / 3.0,
                    np.ones_like(xx)], axis=-1)
    img[..., :3] *= rng.uniform(0.2, 3.0, (h, w, 1)).astype(np.float32)
    img[rng.uniform(size=(h, w)) < 0.02, :3] = 40.0
    return torch.from_numpy(np.ascontiguousarray(img, np.float32)).cuda()


def filled(h, w, value=SENTINEL, n=1):
    return [torch.full((h, w, 4), float(value), dtype=torch.float32, device="cuda") for _ in range(n)]


def bits(t):
    torch.cuda.synchronize()
    return t.view(torch.int32).cpu().numpy()


class Pass:
    """one post pass: its single-destination call, its multi-destination call, and the output size for a source"""

    def __init__(self, ctx, kind, con=None, mode=vq.VQ_ADDRESS_WRAP, params=None, out_hw=None):
        self.ctx, self.kind, self.con, self.mode, self.params, self.out_hw = ctx, kind, con, mode, params, out_hw

    def out_size(self, src):
        return self.out_hw if self.kind == "fsr_easu" else tuple(src.shape[:2])

    def single(self, src, dst):
        c = self.ctx
        if self.kind == "tonemap":
            c.tonemap(self.params, src, dst)
        elif self.kind == "cas":
            c.cas(self.con, src, dst)
        elif self.kind == "fsr_easu":
            c.fsr_easu(self.con, src, dst, address_mode=self.mode)
        else:
            c.fsr_rcas(self.con, src, dst)

    def multi(self, src, dsts, rows, signal=None, stream=None):
        imgs = [vq.image_of(d) for d in dsts]
        c, kw = self.ctx, dict(signal=signal, stream=stream)
        if self.kind == "tonemap":
            c.tonemap_multi(self.params, src, imgs, *rows, **kw)
        elif self.kind == "cas":
            c.cas_multi(self.con, src, imgs, *rows, **kw)
        elif self.kind == "fsr_easu":
            c.fsr_easu_multi(self.con, src, imgs, *rows, address_mode=self.mode, **kw)
        else:
            c.fsr_rcas_multi(self.con, src, imgs, *rows, **kw)


def row_ranges(h):
    """row 0, the last row, single rows, odd starts, 8-row tile edges, the whole output and an empty range"""
    rr = [(0, h), (0, 1), (h - 1, h), (min(5, h - 1), min(6, h)), (min(3, h - 1), min(17, h)), (min(8, h - 1), min(16, h)),
          (min(7, h - 1), min(9, h)), (h // 3, h - h // 4), (h // 2, h // 2)]
    return sorted(set(rr))


def check_pass(p, src, n_dests):
    oh, ow = p.out_size(src)
    ref = filled(oh, ow)[0]
    p.single(src, ref)
    want = bits(ref)
    for rows in row_ranges(oh):
        dsts = filled(oh, ow, n=n_dests)
        n0 = vq.launch_count()
        p.multi(src, dsts, rows)
        assert vq.launch_count() - n0 == (1 if rows[1] > rows[0] else 0), rows
        a, b = rows
        for k, d in enumerate(dsts):
            got = bits(d)
            assert np.array_equal(got[a:b], want[a:b]), (p.kind, rows, k)
            untouched = np.full_like(got, np.float32(SENTINEL).view(np.int32))
            assert np.array_equal(got[:a], untouched[:a]) and np.array_equal(got[b:], untouched[b:]), (p.kind, rows, k)


@pytest.mark.parametrize("n_dests", [1, 2, 3, 8])
@pytest.mark.parametrize("cs,curve,gamma", TONEMAPS)
@pytest.mark.parametrize("h,w", [(37, 61), (64, 1100)])
def test_tonemap_multi_equals_single(ctx, n_dests, cs, curve, gamma, h, w):
    p = Pass(ctx, "tonemap", params=vq.TonemapperParams(cs, curve, 300.0, gamma, 1.0))
    check_pass(p, hdr(h, w, 1), n_dests)


@pytest.mark.parametrize("n_dests", [1, 2, 3, 8])
@pytest.mark.parametrize("kind", ["cas", "fsr_rcas"])
@pytest.mark.parametrize("h,w", [(37, 61), (48, 64), (9, 33)])
def test_sharpeners_multi_equal_single(ctx, n_dests, kind, h, w):
    src = torch.clamp(hdr(h, w, 2) / 4.0, 0.0, 1.0).contiguous()
    con = vq.cas_setup(0.6, w, h, w, h) if kind == "cas" else vq.fsr_rcas_con(0.2)
    check_pass(Pass(ctx, kind, con=con), src, n_dests)


EASU = [("2x", 23, 37, 46, 74), ("2x", 270, 480, 540, 960), ("preset 0.77", 41, 73, 54, 95), ("preset 0.67", 36, 64, 54, 96),
        ("preset 0.58", 31, 55, 54, 96), ("preset 0.50", 27, 48, 54, 96), ("near 1", 60, 60, 61, 61), ("down", 64, 64, 40, 41),
        ("ragged up", 29, 45, 43, 67)]


@pytest.mark.parametrize("mode", [vq.VQ_ADDRESS_WRAP, vq.VQ_ADDRESS_CLAMP])
@pytest.mark.parametrize("case,ih,iw,oh,ow", EASU, ids=[c[0] + f" {c[1]}x{c[2]}" for c in EASU])
@pytest.mark.parametrize("n_dests", [1, 2, 3, 8])
def test_easu_multi_equals_single(ctx, mode, case, ih, iw, oh, ow, n_dests):
    src = torch.clamp(hdr(ih, iw, 3) / 4.0, 0.0, 1.0).contiguous()
    con = vq.fsr_easu_con(iw, ih, iw, ih, ow, oh)
    check_pass(Pass(ctx, "fsr_easu", con=con, mode=mode, out_hw=(oh, ow)), src, n_dests)


# ---- simulated worlds: every rank's plan, whole frames in, its peers' display frames as local destinations --------------------
def reference_chain(ctx, src, tm, fsr, cas_con, out_hw, mode, rcas_con):
    """vq_tonemap -> [vq_cas] -> [vq_fsr_easu -> vq_fsr_rcas], as RenderPostProcess returns it (CAS's output unused with FSR on)"""
    h, w = src.shape[:2]
    t = filled(h, w)[0]
    ctx.tonemap(tm, src, t)
    if fsr is not None:
        e = filled(*out_hw)[0]
        ctx.fsr_easu(fsr, t, e, address_mode=mode)
        r = filled(*out_hw)[0]
        ctx.fsr_rcas(rcas_con, e, r)
        return r
    if cas_con is not None:
        c = filled(h, w)[0]
        ctx.cas(cas_con, t, c)
        return c
    return t


def run_world(ctx, n, src, tm, fsr, cas_con, out_hw, mode, rcas_con):
    in_h, in_w = src.shape[:2]
    oh, ow = out_hw
    frames = filled(oh, ow, n=n)
    for r, band in enumerate(equal_tiles(oh, n)):
        if band[0] == band[1]:
            continue
        dests = [vq.image_of(frames[(r + k) % n]) for k in range(n)]          # own frame first, then the peers' in rotated order
        plan = post_chain_rows(in_h, oh, band, fsr_con=fsr, address_mode=mode, cas=cas_con is not None)
        last = list(plan)[-1]
        tm_dst = filled(in_h, in_w, np.nan)[0] if last != "tonemap" else None
        n0 = vq.launch_count()
        for rows in plan["tonemap"]:
            ctx.tonemap_multi(tm, src, dests if last == "tonemap" else [vq.image_of(tm_dst)], *rows)
        if fsr is not None:
            easu = filled(oh, ow, np.nan)[0]
            ctx.fsr_easu_multi(fsr, tm_dst, [vq.image_of(easu)], *plan["fsr_easu"][0], address_mode=mode)
            ctx.fsr_rcas_multi(rcas_con, easu, dests, *plan["fsr_rcas"][0])
        elif last == "cas":
            ctx.cas_multi(cas_con, tm_dst, dests, *plan["cas"][0])
        assert vq.launch_count() - n0 == sum(len(v) for v in plan.values()) <= 4
    return frames


WORLDS = [("fsr wrap", 270, 480, 2.0, vq.VQ_ADDRESS_WRAP, False), ("fsr clamp", 270, 480, 2.0, vq.VQ_ADDRESS_CLAMP, False),
          ("fsr + cas", 270, 480, 2.0, vq.VQ_ADDRESS_WRAP, True), ("fsr preset ragged", 41, 73, 1 / 0.77, vq.VQ_ADDRESS_WRAP, False),
          ("fsr 2x ragged clamp", 23, 37, 2.0, vq.VQ_ADDRESS_CLAMP, False), ("cas", 270, 480, None, None, True),
          ("cas ragged", 37, 61, None, None, True), ("tonemap", 270, 480, None, None, False), ("tonemap ragged", 37, 61, None, None, False)]


@pytest.mark.parametrize("n", [1, 2, 3, 8])
@pytest.mark.parametrize("case,ih,iw,scale,mode,cas", WORLDS, ids=[w[0] for w in WORLDS])
def test_simulated_world_assembles_the_single_gpu_chain(ctx, n, case, ih, iw, scale, mode, cas):
    src = hdr(ih, iw, 4)
    tm = synth.default_tonemapper()
    if scale is not None:
        oh, ow = (2 * ih, 2 * iw) if scale == 2.0 else (round(ih * scale), round(iw * scale))
        fsr = vq.fsr_easu_con(iw, ih, iw, ih, ow, oh)
    else:
        oh, ow, fsr = ih, iw, None
    cas_con = vq.cas_setup(0.5, iw, ih, iw, ih) if cas else None
    rcas_con = vq.fsr_rcas_con(0.2)
    want = bits(reference_chain(ctx, src, tm, fsr, cas_con, (oh, ow), mode, rcas_con))
    for k, f in enumerate(run_world(ctx, n, src, tm, fsr, cas_con, (oh, ow), mode, rcas_con)):
        got = bits(f)
        assert np.array_equal(got, want), (case, n, k, int((got != want).any(-1).sum()))
