"""-m gpu: vq_gaussian_blur_multi_signal, one rank's band of vq_gaussian_blur into several frames. Into every destination it must
store, bit for bit, what vq_gaussian_blur stores on the band's rows and touch no other row; bands from equal_tiles for 1..8 ranks,
1-row bands and bands inside the top and bottom 10 rows assemble the single call's frame. A simulated world (every "rank" on this
one GPU, its peers' frames being local destinations, flag words preset so that every wait is already satisfied, as in
tests/test_rendezvous_gpu.py) runs the signalled blur band and then the post chain's band (vq_post_process_multi_signal) on the
blurred frames as distributed.blur_rows plans them, and must give what the single-GPU chain blur -> vq_post_process gives."""
import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import blur_rows, equal_tiles

pytestmark = pytest.mark.gpu
SENTINEL = np.float32(-7.5e33)


def hdr(h, w, seed):
    rng = np.random.default_rng(seed)
    img = rng.uniform(0.0, 4.0, (h, w, 4)).astype(np.float32)
    img[rng.uniform(size=(h, w)) < 0.02, :3] = 40.0
    return torch.from_numpy(img).cuda()


def filled(h, w, value=SENTINEL, n=1):
    return [torch.full((h, w, 4), float(value), dtype=torch.float32, device="cuda") for _ in range(n)]


def bits(t):
    torch.cuda.synchronize()
    return t.view(torch.int32).cpu().numpy()


def single(ctx, src, size=None):
    h, w = src.shape[:2]
    size = size or (w, h)
    out = filled(h, w)[0]
    ctx.gaussian_blur2d(vq.BlurParams(*size), src, out)
    return out


def bands(h):
    """1-row bands, bands inside the top and bottom 10 rows, bands across 64-row tile edges, the whole frame, an empty band"""
    rr = [(0, h), (0, 1), (h - 1, h), (min(3, h - 1), min(9, h)), (max(h - 9, 0), max(h - 2, 1)), (min(63, h - 1), min(65, h)),
          (min(5, h - 1), min(130, h)), (h // 3, h - h // 4), (h // 2, h // 2)]
    return sorted(set(rr))


@pytest.mark.parametrize("h,w", [(1, 1), (7, 33), (20, 64), (64, 64), (130, 97), (300, 211)])
@pytest.mark.parametrize("n_dests", [1, 2, 3, 8])
def test_band_into_every_destination(ctx, h, w, n_dests):
    src = hdr(h, w, h + w)
    want = bits(single(ctx, src))
    sent = SENTINEL.view(np.int32)
    for a, b in bands(h):
        dests = filled(h, w, n=n_dests)
        n0 = vq.launch_count()
        ctx.gaussian_blur_multi(vq.BlurParams(w, h), src, [vq.image_of(d) for d in dests], a, b)
        assert vq.launch_count() - n0 == (1 if b > a else 0)
        for d in dests:
            got = bits(d)
            assert np.array_equal(got[a:b], want[a:b]), ((a, b), int((got[a:b] != want[a:b]).any(-1).sum()))
            assert (got[:a] == sent).all() and (got[b:] == sent).all(), (a, b)


@pytest.mark.parametrize("n", [1, 2, 3, 4, 8])
@pytest.mark.parametrize("h,w", [(1, 5), (9, 40), (21, 64), (64, 100), (129, 70), (1080, 1920)])
def test_equal_tiles_assemble_the_single_call(ctx, n, h, w):
    src = hdr(h, w, 7 * n + h)
    want = bits(single(ctx, src))
    frame = filled(h, w)[0]
    for a, b in equal_tiles(h, n):
        ctx.gaussian_blur_multi(vq.BlurParams(w, h), src, [vq.image_of(frame)], a, b)
    assert np.array_equal(bits(frame), want)


def test_band_with_a_smaller_image_size(ctx):
    """rows and clamping follow iImageSize; columns and rows beyond it keep their sentinels"""
    h, w, sx, sy = 150, 120, 101, 133
    src = hdr(h, w, 5)
    want = bits(single(ctx, src, (sx, sy)))
    for a, b in [(0, sy), (120, sy), (0, 1), (sy - 1, sy), (40, 90)]:
        dests = filled(h, w, n=2)
        ctx.gaussian_blur_multi(vq.BlurParams(sx, sy), src, [vq.image_of(d) for d in dests], a, b)
        y = np.arange(h)[:, None, None]
        expect = np.where((y >= a) & (y < b), want, SENTINEL.view(np.int32))
        for d in dests:
            assert np.array_equal(bits(d), expect), (a, b)


class SimWorld:
    """n ranks' n x n flag words (row q = rank q's array), preset so that every wait of epoch e is already satisfied"""

    def __init__(self, n):
        self.n = n
        self.flags = torch.zeros((n, n), dtype=torch.int32, device="cuda")

    def signal(self, r, epoch):
        s = vq.PeerSignal()
        for i in range(self.n):
            s.flags[i] = self.flags.data_ptr() + 4 * ((r + i) % self.n) * self.n      # own array first, then the peers' rotated
        s.n_ranks, s.my_index, s.epoch = self.n, r, epoch
        self.flags.fill_(epoch + 1)
        return s


POST = [("tonemap", None, False, vq.VQ_ADDRESS_WRAP), ("cas", None, True, vq.VQ_ADDRESS_WRAP),
        ("fsr 2x wrap", 2.0, False, vq.VQ_ADDRESS_WRAP), ("fsr 2x clamp", 2.0, False, vq.VQ_ADDRESS_CLAMP),
        ("fsr 1.3x wrap", 1.3, False, vq.VQ_ADDRESS_WRAP)]


@pytest.mark.parametrize("n", [2, 3, 4, 8])
@pytest.mark.parametrize("case,scale,cas,mode", POST, ids=[p[0] for p in POST])
def test_simulated_world_blur_then_post_chain(ctx, n, case, scale, cas, mode):
    ih, iw = 90, 160
    src = hdr(ih, iw, n)
    tm = synth.default_tonemapper()
    if scale is not None:
        oh, ow = round(ih * scale), round(iw * scale)
        easu, rcas = vq.fsr_easu_con(iw, ih, iw, ih, ow, oh), vq.fsr_rcas_con(0.2)
    else:
        oh, ow, easu, rcas = ih, iw, None, None
    cas_con = vq.cas_setup(0.5, iw, ih, iw, ih) if cas else None
    p = vq.BlurParams(iw, ih)
    ref_display = filled(oh, ow)[0]
    ctx.post_process(tm, single(ctx, src), ref_display, cas=cas_con, easu=easu, rcas=rcas, address_mode=mode)
    want = bits(ref_display)

    world = SimWorld(n)
    blurred = filled(ih, iw, np.nan, n=n)          # a row no rank stores stays NaN and shows up in the display frame
    displays = filled(oh, ow, n=n)
    for r, band in enumerate(equal_tiles(oh, n)):
        if band[0] == band[1]:
            continue
        plan = blur_rows(ih, oh, band, fsr_con=easu, address_mode=mode, cas=cas)
        bdests = [vq.image_of(blurred[(r + k) % n]) for k in range(n)]
        for a, b in plan["gaussian_blur"]:
            ctx.gaussian_blur_multi(p, src, bdests, a, b, signal=world.signal(r, 2 * r))
        torch.cuda.synchronize()
    for r, band in enumerate(equal_tiles(oh, n)):
        if band[0] == band[1]:
            continue
        ddests = [vq.image_of(displays[(r + k) % n]) for k in range(n)]
        ctx.post_process_multi(tm, blurred[r], ddests, *band, cas=cas_con, easu=easu, rcas=rcas, address_mode=mode,
                               signal=world.signal(r, 2 * r + 1))
        torch.cuda.synchronize()
    for k in range(n):
        got = bits(displays[k])
        assert np.array_equal(got, want), (case, n, k, int((got != want).any(-1).sum()))
    # every rank's blurred frame holds every rank's band: the union of the plans' blur rows, and the blur of those rows
    ref_blur = bits(single(ctx, src))
    rows = sorted({y for band in equal_tiles(oh, n) for a, b in blur_rows(ih, oh, band, fsr_con=easu, address_mode=mode,
                                                                            cas=cas)["gaussian_blur"] for y in range(a, b)})
    for k in range(n):
        assert np.array_equal(bits(blurred[k])[rows], ref_blur[rows])
