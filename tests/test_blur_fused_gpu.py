"""-m gpu: vq_gaussian_blur (X then Y in one launch, no intermediate image) stores, bit for bit, what vq_gaussian_blur_x into a
temporary followed by vq_gaussian_blur_y stores: NaN positions compared as bits, on 1x1 / 1xN / Nx1 images, sizes on either side
of the kernel's 64 x 64 tiles and of its 16-row X chunks, heights below the 21 taps, iImageSize smaller than the images (the
pixels outside it must keep their sentinels), pitched images, +-Inf, NaN, subnormals and +-0, and a 4K synth.hdr_image frame."""
import ctypes as C

import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import synth

pytestmark = pytest.mark.gpu
SENTINEL = -7.5e33


def bits(t):
    torch.cuda.synchronize()
    return t.contiguous().view(torch.int32).cpu().numpy()


def image(h, w, seed, special=False, pitch_extra=0):
    """[h, w, 4] float32 on the GPU; with pitch_extra > 0 a column slice of a wider tensor (pitch > width * 16 bytes)"""
    rng = np.random.default_rng(seed)
    a = rng.uniform(-2.0, 6.0, (h, w + pitch_extra, 4)).astype(np.float32)
    if special:
        vals = np.array([np.inf, -np.inf, np.nan, 1e-40, -1e-40, 1e-45, 0.0, -0.0, 3e38, -3e38, 1.17e-38], np.float32)
        mask = rng.uniform(size=a.shape) < 0.08
        a[mask] = rng.choice(vals, int(mask.sum()))
        nanbits = a.view(np.uint32)
        nanbits[rng.uniform(size=a.shape) < 0.01] = 0x7FC01234      # NaN with a payload
    t = torch.from_numpy(a).cuda()
    return t[:, :w] if pitch_extra else t


def filled(h, w, pitch_extra=0):
    t = torch.full((h, w + pitch_extra, 4), SENTINEL, dtype=torch.float32, device="cuda")
    return t[:, :w] if pitch_extra else t


def two_calls(ctx, src, size, out_hw=None, pitch_extra=0):
    h, w = out_hw or src.shape[:2]
    tmp, out = filled(h, w, pitch_extra), filled(h, w, pitch_extra)
    p = vq.BlurParams(*size)
    vq._check(vq.lib.vq_gaussian_blur_x(ctx._h, C.byref(p), vq.image_of(src), vq.image_of(tmp), None))
    vq._check(vq.lib.vq_gaussian_blur_y(ctx._h, C.byref(p), vq.image_of(tmp), vq.image_of(out), None))
    return out


def fused(ctx, src, size, out_hw=None, pitch_extra=0):
    h, w = out_hw or src.shape[:2]
    out = filled(h, w, pitch_extra)
    ctx.gaussian_blur2d(vq.BlurParams(*size), src, out)
    return out


def check(ctx, src, size=None, out_hw=None, pitch_extra=0):
    size = size or (src.shape[1], src.shape[0])
    want = bits(two_calls(ctx, src, size, out_hw, pitch_extra))
    got = bits(fused(ctx, src, size, out_hw, pitch_extra))
    diff = np.argwhere(got != want)
    assert diff.size == 0, f"size {size}: {len(diff)} words differ, first at {diff[:4].tolist()}"
    sx, sy = size
    assert (got[sy:] == np.float32(SENTINEL).view(np.int32)).all() and (got[:, sx:] == np.float32(SENTINEL).view(np.int32)).all()
    assert (got[:sy, :sx, 3] == np.float32(1.0).view(np.int32)).all()


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (1, 300), (7, 1), (300, 1), (2, 2), (5, 13), (20, 20), (21, 21)])
def test_tiny_and_thin_images(ctx, h, w):
    check(ctx, image(h, w, h * 1000 + w))


EDGES = [63, 64, 65, 127, 128, 129]
@pytest.mark.parametrize("h", [1, 10, 11, 15, 16, 17, 20] + EDGES + [84, 85, 200])
def test_heights_around_tiles_and_chunks(ctx, h):
    check(ctx, image(h, 97, h))


@pytest.mark.parametrize("w", [1, 2, 3, 4, 5, 11, 12, 13, 24, 25] + EDGES + [88, 89, 191, 192, 193])
def test_widths_around_tiles(ctx, w):
    check(ctx, image(70, w, w + 7))


@pytest.mark.parametrize("size", [(1, 1), (17, 9), (64, 64), (65, 3), (3, 65), (90, 130), (100, 139), (139, 100)])
def test_image_size_smaller_than_the_images(ctx, size):
    """clamping follows iImageSize, not the image; pixels outside iImageSize keep their sentinels"""
    check(ctx, image(140, 100 if size[0] <= 100 else 150, 3), size=size)


def test_image_size_smaller_than_a_larger_destination(ctx):
    check(ctx, image(70, 80, 4), size=(61, 50), out_hw=(90, 100))


@pytest.mark.parametrize("extra", [1, 3, 64])
def test_pitched_images(ctx, extra):
    src = image(131, 77, extra, pitch_extra=extra)
    check(ctx, src, pitch_extra=extra + 2)
    check(ctx, src, size=(70, 100), pitch_extra=extra)


@pytest.mark.parametrize("h,w", [(1, 1), (3, 40), (40, 3), (64, 64), (150, 211)])
def test_special_values(ctx, h, w):
    """+-Inf, NaN (with payloads), subnormals, +-0 and near-overflow values: compared as bits"""
    check(ctx, image(h, w, 99 + h, special=True))


def test_full_4k_frame(ctx):
    src = torch.from_numpy(synth.hdr_image(3840, 2160)).cuda()
    check(ctx, src)


def test_two_streams_one_context(ctx):
    """no context scratch: calls on two streams of one context at once give each its own result"""
    a, b = image(300, 500, 1), image(300, 500, 2)
    want_a, want_b = bits(two_calls(ctx, a, (500, 300))), bits(two_calls(ctx, b, (500, 300)))
    oa, ob = filled(300, 500), filled(300, 500)
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    torch.cuda.synchronize()
    for _ in range(3):
        ctx.gaussian_blur2d(vq.BlurParams(500, 300), a, oa, stream=s1)
        ctx.gaussian_blur2d(vq.BlurParams(500, 300), b, ob, stream=s2)
    assert (bits(oa) == want_a).all() and (bits(ob) == want_b).all()
