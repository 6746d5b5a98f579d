"""K1's domain inputs in the one-pass PSMain kernel's form (tests/psmain_domain.py), no GPU: the adapted interpolants and
materials through the oracle's surface producer give back the scene's G-buffer, and the fold keeps every warp-targeted
property of the probe frames."""
import numpy as np
import pytest

import forward_domain as fd
import light_domain as ld
import psmain_domain as pd

T_EXACT = 0.02


def _scenes():
    env = fd.make_env(5, 16, (20, 48), seed=3)
    yield "spec", fd.specular_probe(fd.probe_env("spec", env), env["spec_mips"], 2000, seed=1)["planes"]
    yield "diff", fd.diffuse_probe(fd.probe_env("diff", env), 2000, seed=2)["planes"]
    yield "lut", fd.lut_probe(fd.probe_env("lut", env), 0, 2000, seed=3)["planes"]
    yield "adversarial", fd.adversarial_gbuffer(515, 9, 4, ld.CAM, emissive=True)[0]
    yield "range", ld.range_probes()[0]["planes"]
    yield "spot", ld.spot_probes()[1]["planes"]
    yield "mirror", ld.mirror_probes()[0]["planes"]
    yield "near", ld.distance_probes()[0]["planes"]
    yield "directional", ld.directional_probe()[0]["planes"]
    yield "t sweep", ld.t_sweep_probe()["planes"]
    yield "view", ld.view_probe()["planes"]
    yield "mixed", ld.mixed_frame("one of each", 3)["planes"]


@pytest.mark.parametrize("name,planes", list(_scenes()), ids=[n for n, _ in _scenes()])
def test_adapted_inputs_reproduce_the_gbuffer(orc, name, planes):
    """position, ao, roughness, albedo, metalness and emissive bit for bit; the normal is the scene's renormalised (the
    producer's N * rsqrtf(N.N)), within 4 ulp of 1 per component"""
    sp, mats = pd.adapt(planes)
    h, w = planes[0].shape[:2]
    gb = orc.gbuffer_from_materials(sp, mats, [{}] * len(mats), 1.0, emissive=True)
    bits = lambda a: np.ascontiguousarray(a, np.float32).view(np.uint32)
    assert np.array_equal(bits(gb[0]), bits(planes[0])), name                       # P and ao = 1 * ssao
    assert np.array_equal(bits(gb[1][..., 3]), bits(planes[1][..., 3])), name       # roughness
    assert np.array_equal(bits(gb[2]), bits(planes[2])), name                       # albedo, metalness
    em = planes[3] if len(planes) > 3 else np.zeros((h, w, 4), np.float32)
    assert np.array_equal(bits(gb[3]), bits(em)), name
    n = pd.renormalised(planes)
    assert np.abs(gb[1][..., :3] - n).max() <= 4 * 2.0 ** -24, name


def test_fold_is_a_warp_preserving_bijection():
    rng = np.random.default_rng(0)
    a = rng.normal(size=(6, 768, 4)).astype(np.float32)
    f = pd.fold(a)
    assert f.shape == (12, 384, 4) and np.array_equal(pd.unfold(f), a)
    # K1 pixel (y, 256 j + 128 k + c) -> (2 y + k, 128 j + c)
    assert np.array_equal(f[2 * 3 + 1, 128 * 2 + 5], a[3, 256 * 2 + 128 + 5])
    # K1's warps are psmain's warps after the fold; unfolded, psmain puts the same pixels into other warps
    k1 = pd.k1_warps(a.shape[:2])
    assert np.array_equal(pd.fold(k1), pd.ps_warps(f.shape[:2]))
    assert not np.array_equal(pd.ps_warps(a.shape[:2]), k1)


def _votes(mask, warps):
    return pd.per_warp(mask, warps)


def test_fold_keeps_the_t_sweep():
    """after the fold, every psmain warp of the t sweep holds exactly the exact-path pixels its K1 warp held: one per 32 columns,
    evaluated on the renormalised normal the producer hands on"""
    p = ld.t_sweep_probe()
    wi = fd._unit(np.array([0.4, 1.0, 0.3]))
    cam = (0.0, 3.0, -4.0)
    t = pd.ggx_t(p["planes"], cam, wi)
    exact = t < T_EXACT
    assert (np.abs(t - T_EXACT) > 1e-6).all()                     # no pixel is near enough to the switch for rounding to move it
    k1 = _votes(exact, pd.k1_warps(exact.shape))
    q = pd.fold_probe(p)
    tf = pd.ggx_t(q["planes"], cam, wi)
    ps = _votes(tf < T_EXACT, pd.ps_warps(tf.shape))
    assert np.array_equal(ps, k1) and (ps == 2).all()               # one per row of 32 columns: two per warp
    print(f"t sweep: {int(exact.sum())} exact-N.H pixels in {len(ps)} warps, folded and unfolded")


def test_fold_keeps_the_tiny_and_escape_votes():
    """the adversarial G-buffer's lone roughness-1e-3 pixels and the mirror probes' escape roughness vote in the same warps after
    the fold; unfolded, psmain pairs them with other pixels"""
    planes, _ = fd.adversarial_gbuffer(512, 8, 5, ld.CAM)
    tiny = pd.tiny_pixels(planes)
    k1 = _votes(tiny, pd.k1_warps(tiny.shape))
    ps = _votes(pd.fold(tiny), pd.ps_warps((16, 256)))
    assert np.array_equal(ps, k1)
    assert (k1 == 0).any() and (k1 > 0).any()
    rough_rows = pd.fold(np.broadcast_to((np.arange(8) % 4 == 3)[:, None], (8, 512)))
    # the rough rows' warps vote TINY through their single 1e-3 pixel only
    ids = np.unique(pd.ps_warps((16, 256))[rough_rows & pd.fold(tiny)])
    assert len(ids) == 2 * 2                                        # two rough rows, two tiles each
    for p in ld.mirror_probes():
        esc = p["escape"]
        q = pd.fold_probe(p)
        assert np.array_equal(_votes(q["escape"], pd.ps_warps(q["escape"].shape)), _votes(esc, pd.k1_warps(esc.shape)))


def test_fold_probe_folds_every_per_pixel_array():
    p = ld.range_probes()[3]
    q = pd.fold_probe(p)
    assert np.array_equal(pd.unfold(q["lit"]), p["lit"]) and np.array_equal(pd.unfold(q["planes"][1]), p["planes"][1])
    assert q["range"] == p["range"]


def test_tiny_pixels_is_the_kernel_rule():
    """the vote's fp32 rule: roughness below 0.0298 votes, the ROUGH_MIX values 0, 1e-3, 0.0239 and 0.0241 do"""
    r = np.array([0.0, 1e-3, 0.0239, 0.0241, 0.0297, 0.03, 0.5, 1.0], np.float32)
    planes = [np.zeros((1, 8, 4), np.float32), np.zeros((1, 8, 4), np.float32)]
    planes[1][0, :, 3] = r
    assert pd.tiny_pixels(planes)[0].tolist() == [True, True, True, True, True, False, False, False]
