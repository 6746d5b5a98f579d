"""CPU: the renderer driver (tests/host_check/renderer_driver.cpp) builds against the in-tree libvqhost.so and reports a missing
device the way the layer documents it, and the host layer's pure-host constant helpers (PostProcess.cpp:37-99) equal the oracle's
FidelityFX setup functions bit for bit and float64 for the sharpness conversion."""
import math

import numpy as np
import pytest

import host_driver as hd


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    if not hd.available():
        pytest.skip("g++ / libvqhost.so not available")
    return hd.build(tmp_path_factory.mktemp("driver"))


def _has_device():
    import torch
    return torch.cuda.is_available()


def test_driver_links_and_reports_the_missing_device(driver, tmp_path):
    """VQRenderer::Initialize fails with vq_ctx_create's VQ_ERR_NO_DEVICE message, and the driver exits with its Initialize code"""
    if _has_device():
        pytest.skip("a CUDA device is present")
    out = hd.run(driver, tmp_path, ["init"], rc=hd.EXIT_INIT)
    fail = [l for l in out if l.startswith("FAIL init:")]
    assert len(fail) == 1, out
    assert "vq_ctx_create: no CUDA device available" in fail[0] and "this backend has no CPU path" in fail[0], fail[0]


def test_linear_sharpness_round_trip(driver, tmp_path):
    """SetLinearSharpness(S) stores log10(S) / log10(0.5) stops, GetLinearSharpness returns 0.5^stops: both within a few fp32 ulps of
    the float64 values, and the round trip gives S back"""
    values = [1.0, 0.999, 0.8, 0.5, 0.25, 0.2, 0.1, 0.05, 0.01, 1e-3, 0.7071]
    out = hd.run(driver, tmp_path, [f"host_helpers kind=sharpness linear={v!r}" for v in values])
    got = [l.split()[1:] for l in out if l.startswith("sharpness ")]
    assert len(got) == len(values)
    for v, (stops, linear) in zip(values, got):
        s32 = float(np.float32(v))
        want_stops = math.log10(s32) / math.log10(0.5)
        assert abs(float(stops) - want_stops) <= 4 * 2.0 ** -23 * max(1.0, abs(want_stops)), (v, stops, want_stops)
        assert abs(float(linear) - 0.5 ** float(stops)) <= 4 * 2.0 ** -24 * 0.5 ** float(stops), (v, linear)
        assert abs(float(linear) - s32) <= 8 * 2.0 ** -24 * max(s32, 2.0 ** -10), (v, linear)


def test_constant_blocks_equal_the_oracle(driver, tmp_path, orc):
    """UpdateCASConstantBlock, UpdateEASUConstantBlock and UpdateRCASConstantBlock against orc.cas_setup / fsr_easu_con /
    fsr_rcas_con over a sweep of sharpness, sizes and render / display ratios, word for word"""
    cas = [(s, iw, ih, ow, oh) for s in (0.0, 0.3, 0.8, 1.0) for (iw, ih, ow, oh) in ((70, 37, 70, 37), (1920, 1080, 1920, 1080),
                                                                                      (1280, 720, 1920, 1080), (1, 1, 1, 1))]
    easu = [(iw, ih, cw, ch, ow, oh) for (iw, ih, cw, ch, ow, oh) in (
        (70, 37, 70, 37, 140, 74), (70, 37, 70, 37, 105, 55), (1280, 720, 1280, 720, 1920, 1080), (1477, 831, 1477, 831, 2560, 1440),
        (960, 540, 1920, 1080, 3840, 2160), (3840, 2160, 3840, 2160, 3840, 2160), (1, 1, 1, 1, 2, 2))]
    rcas = [0.0, 0.2, 0.5, 1.0, 2.0, 0.123]
    lines = [f"host_helpers kind=cas sharp={s!r} iw={iw} ih={ih} ow={ow} oh={oh}" for (s, iw, ih, ow, oh) in cas]
    lines += [f"host_helpers kind=easu iw={a} ih={b} cw={c} ch={d} ow={e} oh={f}" for (a, b, c, d, e, f) in easu]
    lines += [f"host_helpers kind=rcas stops={s!r}" for s in rcas]
    out = hd.run(driver, tmp_path, lines)
    words = lambda kind: [[int(x) for x in l.split()[1:]] for l in out if l.startswith(kind + " ")]
    for (s, iw, ih, ow, oh), got in zip(cas, words("cas"), strict=True):
        assert got == list(orc.cas_setup(s, iw, ih, ow, oh)), ("cas", s, iw, ih, ow, oh)
    for (iw, ih, cw, ch, ow, oh), got in zip(easu, words("easu"), strict=True):
        assert got == list(orc.fsr_easu_con(iw, ih, cw, ch, ow, oh)), ("easu", iw, ih, cw, ch, ow, oh)
    for s, got in zip(rcas, words("rcas"), strict=True):
        assert got == list(orc.fsr_rcas_con(s)), ("rcas", s)
