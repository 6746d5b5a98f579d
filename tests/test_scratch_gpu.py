"""-m gpu: a context's scratch history does not change a single bit. Every call that grows context scratch (K1's sampling
copies, the registered environment, the resize tables and intermediate, the PCF records, the depth pyramid's pads, the host
call's staging) runs small -> large -> small on one context, and each result must equal the same call on a fresh context."""
import numpy as np
import pytest
import torch

import forward_domain as fd
from gpu_util import dev, host, assert_scaled
from shadow_util import fill_casters

pytestmark = [pytest.mark.gpu, pytest.mark.usefixtures("ctx")]

CAM = (0.0, 5.0, -17.0)


def _history_free(vq, calls):
    """runs `calls` (context -> array) in order on one context, then each on a fresh context: the results must agree"""
    ctx = vq.Context(0)
    try:
        seen = [f(ctx) for f in calls]
    finally:
        ctx.close()
    for k, (f, want) in enumerate(zip(calls, seen)):
        fresh = vq.Context(0)
        try:
            got = f(fresh)
        finally:
            fresh.close()
        assert np.array_equal(want, got, equal_nan=True), f"call {k} depends on the context's scratch history"
    return seen


def _envs():
    """two environments whose cubes differ in size and mip count (and whose LUTs differ in shape)"""
    return [fd.make_env(5, 16, (20, 48), seed=1), fd.make_env(33, 64, (48, 20), seed=2)]


def _maps(vq, env):
    t = [dev(env[k]) for k in ("diff", "spec", "lut")]
    return vq.EnvironmentMaps(vq.cubemap_of(t[0], env["diff_res"], env["diff_mips"]),
                              vq.cubemap_of(t[1], env["spec_res"], env["spec_mips"]), vq.image_of(t[2], 2)), t


def _gbuffer(vq, tensors):
    im = [vq.image_of(t) for t in tensors]
    return vq.GBuffer(im[0], im[1], im[2], im[3] if len(im) > 3 else vq.null_image())


def _frame(env, w, h, seed, emissive=False):
    planes, _ = fd.adversarial_gbuffer(w, h, seed, CAM, emissive=emissive)
    pf, pv = fd.constants(CAM, env["spec_mips"], 0.7, lights=fd.lights(w, h, seed, 0.7))
    return planes, pf, pv


def _oracle(orc, env, planes, pf, pv):
    return orc.forward_lighting(pf, pv, planes, env["diff"], env["diff_res"], env["spec"], env["spec_res"], env["spec_mips"],
                                env["lut"])


def _shade(vq, env, planes, pf, pv, prepare):
    def call(ctx):
        em, keep = _maps(vq, env)
        d = [dev(p) for p in planes]
        if prepare:
            ctx.environment_prepare(em)
        out = torch.zeros(planes[0].shape, dtype=torch.float32, device="cuda")
        ctx.forward_lighting(pf, pv, _gbuffer(vq, d), em, out)
        return host(out)
    return call


@pytest.mark.parametrize("prepare", [False, True], ids=["per_call", "prepared"])
def test_sampling_copies(vq, orc, prepare):
    """K1 with sampling copies built per call, and from vq_environment_prepare followed by a shade, for environment
    A -> B -> A: the copies regrow for B and A is built into the larger buffer"""
    envs = _envs()
    frames = [_frame(e, 256, 16, seed=40 + k) for k, e in enumerate(envs)]
    order = (0, 1, 0)
    got = _history_free(vq, [_shade(vq, envs[i], *frames[i], prepare) for i in order])
    for i, g in zip(order, got):
        assert_scaled(f"env {i}", g, _oracle(orc, envs[i], *frames[i]))


def test_image_resize(vq):
    rng = np.random.default_rng(3)
    pairs = [((100, 37), (41, 13)), ((1024, 512), (256, 128)), ((100, 37), (41, 13))]
    srcs = {wh: (rng.random((wh[1], wh[0], 4), dtype=np.float32) * 5) for wh, _ in pairs}

    def resize(wh, owh):
        def call(ctx):
            src = dev(srcs[wh])
            out = torch.zeros((owh[1], owh[0], 4), dtype=torch.float32, device="cuda")
            ctx.image_resize(src, out)
            return host(out)
        return call
    _history_free(vq, [resize(*p) for p in pairs])


def test_shadowed_pass_records(vq):
    """PCF records for rows [0, 8), then for all rows, then [0, 8) again"""
    env = _envs()[0]
    w, h = 300, 41
    planes, pf, pv = _frame(env, w, h, seed=50)
    fill_casters(pf, 5, 5, seed=2)
    pf.f2SpotLightShadowMapDimensions.x = pf.f2SpotLightShadowMapDimensions.y = 16.0
    rng = np.random.default_rng(51)
    cubes = rng.uniform(0.0, 1.2, (5, 6, 8, 8)).astype(np.float32)
    spots = rng.uniform(0.3, 0.7, (5, 16, 16)).astype(np.float32)

    def shadowed(rows):
        def call(ctx):
            em, keep = _maps(vq, env)
            d = [dev(p) for p in planes]
            out = torch.zeros((h, w, 4), dtype=torch.float32, device="cuda")
            ctx.forward_lighting_shadowed(pf, pv, _gbuffer(vq, d), em, out, point_cubes=dev(cubes), spot_maps=dev(spots),
                                          row_begin=rows[0], row_end=rows[1])
            return host(out)
        return call
    got = _history_free(vq, [shadowed(r) for r in ((0, 8), (0, h), (0, 8))])
    assert np.array_equal(got[0][:8], got[1][:8]) and (got[0][8:] == 0).all()


def test_depth_pyramid_pads(vq):
    rng = np.random.default_rng(5)
    depths = {wh: rng.uniform(0.05, 1.0, (wh[1], wh[0])).astype(np.float32) for wh in ((256, 200), (1920, 1080))}

    def pyramid(wh):
        def call(ctx):
            w, h = wh
            n = vq.depth_pyramid_level_count(w, h)
            levels = torch.full((vq.depth_pyramid_texel_count(w, h, n),), -1.0, dtype=torch.float32, device="cuda")
            d = dev(depths[wh])
            ctx.depth_min_pyramid(d, levels)
            return host(levels)
        return call
    _history_free(vq, [pyramid(wh) for wh in ((256, 200), (1920, 1080), (256, 200))])


def test_host_call_staging(vq, orc):
    """the blocking host-buffer call at 4 staging planes, then 5 (an emissive plane), then a smaller frame"""
    env = _envs()[0]
    frames = [_frame(env, 256, 40, seed=60), _frame(env, 256, 40, seed=61, emissive=True), _frame(env, 130, 21, seed=62)]

    def host_call(planes, pf, pv):
        def call(ctx):
            em, keep = _maps(vq, env)
            hp = [torch.from_numpy(p) for p in planes]
            hout = torch.zeros(planes[0].shape, dtype=torch.float32)
            ctx.forward_lighting_host(pf, pv, _gbuffer(vq, hp), em, hout)
            return hout.numpy().copy()
        return call
    got = _history_free(vq, [host_call(*f) for f in frames])
    for k, (g, f) in enumerate(zip(got, frames)):
        assert_scaled(f"host call {k}", g, _oracle(orc, env, *f))
