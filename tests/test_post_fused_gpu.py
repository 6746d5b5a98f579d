"""-m gpu: RenderPostProcess in one launch (vq_post_process, vq_post_process_multi_signal). The display frame must equal, bit for bit,
what the separate calls compute (vq_tonemap -> vq_fsr_easu -> vq_fsr_rcas, vq_tonemap -> vq_cas, vq_tonemap) over every scale of
both EASU paths, both address modes, sizes at the fused tiles' edges, pitched images, every tonemapper branch, the sharpness
range and non-finite inputs; the band form must store those bits on its rows only; and the host mirror's RenderPostProcess,
which now makes the one call, must return what its three calls returned."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import synth
from vqengine_b200.distributed import equal_tiles

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SENTINEL = np.float32(-7.5e33)
TONEMAPS = [(vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_SRGB, 1), (vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_SRGB, 0),
            (vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_ST2084, 0), (vq.COLOR_SPACE_REC_2020, vq.DISPLAY_CURVE_ST2084, 0),
            (vq.COLOR_SPACE_REC_709, vq.DISPLAY_CURVE_LINEAR, 0), (vq.COLOR_SPACE_REC_709, 7, 0)]
MODES = [vq.VQ_ADDRESS_WRAP, vq.VQ_ADDRESS_CLAMP]


def hdr(h, w, seed, special=False):
    """HDR scene colour with gradients, edges and highlights; `special` adds negatives, values beyond 2^126, +-Inf and NaN"""
    rng = np.random.default_rng(seed)
    yy, xx = np.mgrid[0:h, 0:w].astype(np.float32)
    img = np.stack([np.sin(xx * 0.31 + yy * 0.17) + 1.1, np.cos(xx * 0.07 - yy * 0.23) + 1.05, (xx + yy) % 7 / 3.0,
                    np.ones_like(xx)], axis=-1)
    img[..., :3] *= rng.uniform(0.2, 3.0, (h, w, 1)).astype(np.float32)
    img[rng.uniform(size=(h, w)) < 0.02, :3] = 40.0
    if special:
        vals = np.array([-0.5, -3.0, 2.0 ** 127, 3e38, np.inf, -np.inf, np.nan, 0.0, -0.0, 1e-30], np.float32)
        mask = rng.uniform(size=(h, w, 3)) < 0.08
        img[..., :3][mask] = rng.choice(vals, size=int(mask.sum()))
    return torch.from_numpy(np.ascontiguousarray(img, np.float32)).cuda()


def filled(h, w, value=SENTINEL, n=1):
    return [torch.full((h, w, 4), float(value), dtype=torch.float32, device="cuda") for _ in range(n)]


def bits(t):
    torch.cuda.synchronize()
    return t.contiguous().view(torch.int32).cpu().numpy()


def tonemapper(cs=vq.COLOR_SPACE_REC_709, curve=vq.DISPLAY_CURVE_SRGB, gamma=1):
    return vq.TonemapperParams(cs, curve, 300.0, gamma, 1.0)


def chain(ctx, src, tm, out_hw, easu=None, rcas=None, cas=None, mode=vq.VQ_ADDRESS_WRAP):
    """the separate calls, as RenderPostProcess made them"""
    h, w = src.shape[:2]
    t = filled(h, w)[0]
    ctx.tonemap(tm, src, t)
    if easu is not None:
        e = filled(*out_hw)[0]
        ctx.fsr_easu(easu, t, e, address_mode=mode)
        r = filled(*out_hw)[0]
        ctx.fsr_rcas(rcas, e, r)
        return r
    if cas is not None:
        c = filled(h, w)[0]
        ctx.cas(cas, t, c)
        return c
    return t


def fused(ctx, src, tm, out_hw, easu=None, rcas=None, cas=None, mode=vq.VQ_ADDRESS_WRAP, dst=None):
    dst = filled(*out_hw)[0] if dst is None else dst
    n0 = vq.launch_count()
    ctx.post_process(tm, src, dst, cas=cas, easu=easu, rcas=rcas, address_mode=mode)
    assert vq.launch_count() - n0 == 1
    return dst


def assert_same(got, want, what):
    g, w = bits(got), bits(want)
    assert np.array_equal(g, w), (what, int((g != w).any(-1).sum()), np.argwhere((g != w).any(-1))[:4].tolist())


def fsr_consts(ih, iw, oh, ow, stops=0.2):
    return vq.fsr_easu_con(iw, ih, iw, ih, ow, oh), vq.fsr_rcas_con(stops)


def check_fsr(ctx, src, oh, ow, mode=vq.VQ_ADDRESS_WRAP, tm=None, stops=0.2):
    ih, iw = src.shape[:2]
    tm = tm or tonemapper()
    easu, rcas = fsr_consts(ih, iw, oh, ow, stops)
    want = chain(ctx, src, tm, (oh, ow), easu=easu, rcas=rcas, mode=mode)
    assert_same(fused(ctx, src, tm, (oh, ow), easu=easu, rcas=rcas, mode=mode), want, (ih, iw, oh, ow, mode, stops))


# every FSR preset (1/0.77 .. 1/0.5), 1:1, the exact 2x and ragged non-2x upscales
SCALES = [("2x", 37, 61, 74, 122), ("preset 0.77", 41, 73, 54, 95), ("preset 0.67", 36, 64, 54, 96), ("preset 0.58", 31, 55, 54, 96),
          ("preset 0.50 near 2x", 27, 49, 54, 96), ("1:1", 45, 67, 45, 67), ("ragged", 29, 45, 43, 67), ("ragged tall", 50, 23, 77, 40)]


@pytest.mark.parametrize("cs,curve,gamma", TONEMAPS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case,ih,iw,oh,ow", SCALES, ids=[s[0] for s in SCALES])
def test_fsr_equals_the_three_calls(ctx, cs, curve, gamma, mode, case, ih, iw, oh, ow):
    check_fsr(ctx, hdr(ih, iw, 1), oh, ow, mode, tonemapper(cs, curve, gamma))


# the 2x path's display tile is 62 x 14 (input 31 x 7 per tile); the up path's 30 x 14
SIZES_2X = [(1, 1), (2, 3), (3, 2), (1, 40), (40, 1), (13, 17), (6, 30), (7, 31), (8, 32), (13, 61), (14, 62), (15, 63), (21, 93), (29, 97)]
SIZES_UP = [(1, 1), (2, 3), (3, 2), (13, 29), (14, 30), (15, 31), (27, 59), (28, 60), (29, 61), (41, 89), (43, 97)]


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("ih,iw", SIZES_2X)
def test_fsr_2x_sizes(ctx, mode, ih, iw):
    check_fsr(ctx, hdr(ih, iw, 2), 2 * ih, 2 * iw, mode)


@pytest.mark.parametrize("ratio", [1.0, 0.67])
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("oh,ow", SIZES_UP)
def test_fsr_up_sizes(ctx, ratio, mode, oh, ow):
    ih, iw = max(1, round(oh * ratio)), max(1, round(ow * ratio))
    check_fsr(ctx, hdr(ih, iw, 3), oh, ow, mode)


@pytest.mark.parametrize("stops", [0.0, 0.2, 2.0])
@pytest.mark.parametrize("case,ih,iw,oh,ow", [SCALES[0], SCALES[2], SCALES[5]], ids=["2x", "preset 0.67", "1:1"])
def test_fsr_rcas_sharpness(ctx, stops, case, ih, iw, oh, ow):
    check_fsr(ctx, hdr(ih, iw, 4), oh, ow, stops=stops)


@pytest.mark.parametrize("cs,curve,gamma", TONEMAPS)
@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("case,ih,iw,oh,ow", [SCALES[0], SCALES[2], SCALES[5]], ids=["2x", "preset 0.67", "1:1"])
def test_fsr_non_finite_and_extreme_inputs(ctx, cs, curve, gamma, mode, case, ih, iw, oh, ow):
    """negatives, 2^127, 3e38, +-Inf, NaN, signed zeros: the same bits, NaN payloads and positions included"""
    check_fsr(ctx, hdr(ih, iw, 5, special=True), oh, ow, mode, tonemapper(cs, curve, gamma))


@pytest.mark.parametrize("path", ["2x", "up"])
def test_fsr_pitched_images(ctx, path):
    ih, iw = 23, 37
    oh, ow = (2 * ih, 2 * iw) if path == "2x" else (35, 56)
    big = hdr(ih, iw + 9, 6)
    src = big[:, 3:3 + iw]                                  # pitch of iw + 9 texels, offset by 3
    easu, rcas = fsr_consts(ih, iw, oh, ow)
    want = chain(ctx, src, tonemapper(), (oh, ow), easu=easu, rcas=rcas)
    dst_big = filled(oh, ow + 5)[0]
    dst = dst_big[:, 1:1 + ow]
    fused(ctx, src, tonemapper(), (oh, ow), easu=easu, rcas=rcas, dst=dst)
    assert_same(dst, want, path)
    b = bits(dst_big)
    assert (b[:, :1] == SENTINEL.view(np.int32)).all() and (b[:, 1 + ow:] == SENTINEL.view(np.int32)).all()


def test_fsr_4k_to_8k(ctx):
    for mode in MODES:
        check_fsr(ctx, torch.from_numpy(synth.hdr_image(3840, 2160)).cuda(), 4320, 7680, mode)
        torch.cuda.empty_cache()


def test_fsr_1440p_to_4k(ctx):
    check_fsr(ctx, torch.from_numpy(synth.hdr_image(2560, 1440)).cuda(), 2160, 3840)


# ---- tonemapper -> CAS, tonemapper alone ---------------------------------------------------------------------------------------
SIZES_CAS = [(1, 1), (2, 3), (3, 2), (7, 31), (8, 32), (9, 33), (37, 61), (64, 97)]


@pytest.mark.parametrize("cs,curve,gamma", TONEMAPS)
@pytest.mark.parametrize("sharp", [0.0, 0.8, 1.0])
@pytest.mark.parametrize("special", [False, True])
def test_cas_equals_the_two_calls(ctx, cs, curve, gamma, sharp, special):
    for h, w in SIZES_CAS:
        src, tm, con = hdr(h, w, 7, special), tonemapper(cs, curve, gamma), vq.cas_setup(sharp, w, h, w, h)
        assert_same(fused(ctx, src, tm, (h, w), cas=con), chain(ctx, src, tm, (h, w), cas=con), (h, w))


def test_cas_pitched_images(ctx):
    h, w = 19, 45
    src = hdr(h, w + 7, 8)[:, 2:2 + w]
    con = vq.cas_setup(0.8, w, h, w, h)
    dst = filled(h, w + 3)[0][:, 3:]
    fused(ctx, src, tonemapper(), (h, w), cas=con, dst=dst)
    assert_same(dst, chain(ctx, src, tonemapper(), (h, w), cas=con), "pitched")


@pytest.mark.parametrize("cs,curve,gamma", TONEMAPS)
def test_tonemapper_alone(ctx, cs, curve, gamma):
    for h, w in [(1, 1), (37, 61), (64, 1100)]:
        src, tm = hdr(h, w, 9, special=True), tonemapper(cs, curve, gamma)
        assert_same(fused(ctx, src, tm, (h, w)), chain(ctx, src, tm, (h, w)), (h, w))


# ---- one launch, no scratch -----------------------------------------------------------------------------------------------------
def test_two_streams_of_one_context(ctx):
    """no context scratch: the same call in flight on two streams gives the single-stream bits on both"""
    ih, iw = 270, 480
    src = hdr(ih, iw, 10)
    easu, rcas = fsr_consts(ih, iw, 2 * ih, 2 * iw)
    want = bits(fused(ctx, src, tonemapper(), (2 * ih, 2 * iw), easu=easu, rcas=rcas))
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    outs = filled(2 * ih, 2 * iw, n=2)
    torch.cuda.synchronize()
    for _ in range(4):
        for s, o in ((s1, outs[0]), (s2, outs[1])):
            ctx.post_process(tonemapper(), src, o, easu=easu, rcas=rcas, stream=s)
    torch.cuda.synchronize()
    for o in outs:
        assert np.array_equal(bits(o), want)


# ---- multi-destination form ----------------------------------------------------------------------------------------------------
BRANCHES = [("fsr 2x", 23, 37, 46, 74), ("fsr 2x tall", 61, 20, 122, 40), ("fsr preset", 41, 73, 54, 95), ("fsr 1:1", 37, 61, 37, 61),
            ("cas", 37, 61, None, None), ("tonemap", 37, 61, None, None)]


def branch_consts(case, ih, iw, oh, ow):
    if case.startswith("fsr"):
        easu, rcas = fsr_consts(ih, iw, oh, ow)
        return dict(easu=easu, rcas=rcas), (oh, ow)
    if case == "cas":
        return dict(cas=vq.cas_setup(0.6, iw, ih, iw, ih)), (ih, iw)
    return {}, (ih, iw)


def row_ranges(h):
    """row 0, the last row, single rows, both fused tile heights' edges, the whole output and an empty range"""
    rr = [(0, h), (0, 1), (h - 1, h), (min(5, h - 1), min(6, h)), (min(13, h - 1), min(15, h)), (min(14, h - 1), min(28, h)),
          (min(7, h - 1), min(9, h)), (h // 3, h - h // 4), (h // 2, h // 2)]
    return sorted(set(rr))


@pytest.mark.parametrize("mode", MODES)
@pytest.mark.parametrize("n_dests", [1, 2, 3, 8])
@pytest.mark.parametrize("case,ih,iw,oh,ow", BRANCHES, ids=[b[0] for b in BRANCHES])
def test_multi_equals_single(ctx, mode, n_dests, case, ih, iw, oh, ow):
    src = hdr(ih, iw, 11)
    kw, (h, w) = branch_consts(case, ih, iw, oh, ow)
    want = bits(fused(ctx, src, tonemapper(), (h, w), mode=mode, **kw))
    for a, b in row_ranges(h):
        dsts = filled(h, w, np.nan, n=n_dests)
        n0 = vq.launch_count()
        ctx.post_process_multi(tonemapper(), src, [vq.image_of(d) for d in dsts], a, b, address_mode=mode, **kw)
        assert vq.launch_count() - n0 == (1 if b > a else 0), (a, b)
        for k, d in enumerate(dsts):
            got = bits(d)
            assert np.array_equal(got[a:b], want[a:b]), (case, (a, b), k)
            assert np.isnan(d[:a].cpu().numpy()).all() and np.isnan(d[b:].cpu().numpy()).all(), (case, (a, b), k)


WORLDS = [("fsr wrap", 270, 480, 2.0, vq.VQ_ADDRESS_WRAP, False), ("fsr clamp", 270, 480, 2.0, vq.VQ_ADDRESS_CLAMP, False),
          ("fsr + cas", 270, 480, 2.0, vq.VQ_ADDRESS_WRAP, True), ("fsr preset ragged", 41, 73, 1 / 0.77, vq.VQ_ADDRESS_WRAP, False),
          ("fsr 2x ragged clamp", 23, 37, 2.0, vq.VQ_ADDRESS_CLAMP, False), ("cas", 270, 480, None, None, True),
          ("cas ragged", 37, 61, None, None, True), ("tonemap", 270, 480, None, None, False), ("tonemap ragged", 37, 61, None, None, False)]


@pytest.mark.parametrize("n", [1, 2, 3, 8])
@pytest.mark.parametrize("case,ih,iw,scale,mode,cas", WORLDS, ids=[w[0] for w in WORLDS])
def test_simulated_world_assembles_the_single_gpu_chain(ctx, n, case, ih, iw, scale, mode, cas):
    """every rank on this GPU, its peers' display frames as local destinations, ONE fused launch per rank into NaN-filled frames"""
    src = hdr(ih, iw, 4)
    tm = synth.default_tonemapper()
    if scale is not None:
        oh, ow = (2 * ih, 2 * iw) if scale == 2.0 else (round(ih * scale), round(iw * scale))
        easu, rcas = fsr_consts(ih, iw, oh, ow)
    else:
        oh, ow, easu, rcas = ih, iw, None, None
    cas_con = vq.cas_setup(0.5, iw, ih, iw, ih) if cas else None
    want = bits(chain(ctx, src, tm, (oh, ow), easu=easu, rcas=rcas, cas=cas_con, mode=mode or vq.VQ_ADDRESS_WRAP))
    frames = filled(oh, ow, np.nan, n=n)
    for r, band in enumerate(equal_tiles(oh, n)):
        if band[0] == band[1]:
            continue
        dests = [vq.image_of(frames[(r + k) % n]) for k in range(n)]
        n0 = vq.launch_count()
        ctx.post_process_multi(tm, src, dests, *band, cas=cas_con, easu=easu, rcas=rcas, address_mode=mode or vq.VQ_ADDRESS_WRAP)
        assert vq.launch_count() - n0 == 1
    for k, f in enumerate(frames):
        got = bits(f)
        assert np.array_equal(got, want), (case, n, k, int((got != want).any(-1).sum()))


# ---- the host mirror ------------------------------------------------------------------------------------------------------------
HOST_PROGRAM = r'''
#include "vq_renderer.hpp"
#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <vector>
// RenderPostProcess (one vq_post_process call) against the calls it made before, on the same scene colour
static std::vector<float> Read(const VqImage& im) {
    std::vector<float> v((size_t)im.width * im.height * 4);
    cudaDeviceSynchronize();
    cudaMemcpy2D(v.data(), (size_t)im.width * 16, im.ptr, im.pitch_bytes, (size_t)im.width * 16, im.height, cudaMemcpyDeviceToHost);
    return v;
}
int main() {
    const int W = 123, H = 69;
    vq::VQRenderer r;
    if (!r.Initialize(0) || !r.OnWindowSizeChanged(W, H, 2 * W, 2 * H)) return 2;
    std::vector<float> scene((size_t)W * H * 4);
    for (size_t i = 0; i < scene.size(); ++i) scene[i] = 2.5f * (1.0f + std::sin(0.37f * (float)i)) + ((i % 97) == 0 ? 30.0f : 0.0f);
    cudaMemcpy(r.SceneColor().mem.ptr, scene.data(), scene.size() * 4, cudaMemcpyHostToDevice);
    VqContext* ctx = r.Context();
    vq::FTexture2D t, c, e, o, bt, bo;
    if (!t.Create(W, H) || !c.Create(W, H) || !e.Create(2 * W, 2 * H) || !o.Create(2 * W, 2 * H) || !bt.Create(W, H) || !bo.Create(W, H)) return 3;
    const char* names[4] = {"fsr wrap", "cas only", "tonemapper only", "blur + fsr"};
    for (int cfg = 0; cfg < 4; ++cfg) {
        vq::FPostProcessParameters pp;
        pp.SceneRTWidth = W; pp.SceneRTHeight = H; pp.DisplayResolutionWidth = 2 * W; pp.DisplayResolutionHeight = 2 * H;
        pp.FSR_EASUParams.UpdateEASUConstantBlock(W, H, W, H, 2 * W, 2 * H);
        pp.FSR_RCASParams.UpdateRCASConstantBlock();
        pp.FFXCASParams.UpdateCASConstantBlock(W, H, W, H);
        pp.UpscalingAlgorithm = (cfg == 0 || cfg == 3) ? vq::FPostProcessParameters::FIDELITYFX_SUPER_RESOLUTION1 : vq::FPostProcessParameters::NONE;
        pp.bEnableCAS = cfg == 1;
        pp.bEnableGaussianBlur = cfg == 3;
        const VqImage* out = r.RenderPostProcess(nullptr, pp, false);
        if (!out) { std::printf("%s: %s\n", names[cfg], vq::LastError()); return 4; }
        const std::vector<float> got = Read(*out);
        // the calls RenderPostProcess made before
        VqImage in = r.SceneColor().View();
        if (cfg == 3) {
            const VqBlurParams bp{W, H};
            if (vq_gaussian_blur_x(ctx, &bp, in, bt.View(), nullptr) || vq_gaussian_blur_y(ctx, &bp, bt.View(), bo.View(), nullptr)) return 5;
            in = bo.View();
        }
        const VqTonemapperParams tp{0, 0, 200.0f, 1, 1.0f};
        if (vq_tonemap(ctx, &tp, in, t.View(), nullptr)) return 5;
        VqImage want = t.View();
        if (cfg == 1) { if (vq_cas(ctx, pp.FFXCASParams.CASConstantBlock, t.View(), c.View(), nullptr)) return 5; want = c.View(); }
        if (cfg == 0 || cfg == 3) {
            if (vq_fsr_easu(ctx, pp.FSR_EASUParams.EASUConstantBlock, VQ_ADDRESS_WRAP, t.View(), e.View(), nullptr) ||
                vq_fsr_rcas(ctx, pp.FSR_RCASParams.RCASConstantBlock, e.View(), o.View(), nullptr)) return 5;
            want = o.View();
        }
        const std::vector<float> ref = Read(want);
        const bool same = out->width == want.width && out->height == want.height && std::memcmp(got.data(), ref.data(), ref.size() * 4) == 0;
        std::printf("%s: %dx%d %s\n", names[cfg], out->width, out->height, same ? "same bits" : "DIFFERENT");
        if (!same) return 6;
    }
    return 0;
}
'''


def test_host_mirror_render_post_process(tmp_path):
    host = os.path.join(ROOT, "vqengine_b200", "host")
    assert shutil.which("g++") and os.path.exists(os.path.join(host, "libvqhost.so")), "host layer not built"
    src = tmp_path / "post.cpp"
    src.write_text(HOST_PROGRAM)
    exe = str(tmp_path / "post")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    subprocess.check_call(["g++", "-std=c++17", str(src), "-I", host, "-I", os.path.join(cuda, "include"), "-L", host, "-lvqhost",
                           "-L", os.path.join(ROOT, "vqengine_b200"), "-lvqcuda", "-L", os.path.join(cuda, "lib64"), "-lcudart",
                           f"-Wl,-rpath,{host}", f"-Wl,-rpath,{os.path.join(ROOT, 'vqengine_b200')}", f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}",
                           "-o", exe])
    r = subprocess.run([exe], capture_output=True, text=True, timeout=120)
    print(r.stdout, r.stderr)
    assert r.returncode == 0, (r.returncode, r.stdout, r.stderr)
    assert r.stdout.count("same bits") == 4
