"""CPU: the sampler-probe identities of tests/forward_domain.py hold on the oracle's PSMain, so that the GPU probes
(test_forward_domain_gpu.py) compare K1 with a statement that is known to be the reference's: a probe G-buffer's output is
exactly one specular sample, one diffuse sample or one LUT channel."""
import math

import numpy as np
import pytest

import forward_domain as fd
import sampling_ref as sr


def _oracle(orc, probe, env):
    out = orc.forward_lighting(probe["pf"], probe["pv"], probe["planes"], env["diff"], env["diff_res"], env["spec"],
                               env["spec_res"], env["spec_mips"], env["lut"])
    return out


def _check(name, got, probe):
    err = np.abs(got[..., :3].astype(np.float64) - probe["want"]).max(-1)
    worst = float((err / probe["tol"]).max())
    print(f"{name}: max |oracle - float64| = {err.max():.2e}, max error / bound = {worst:.3f}")
    assert np.isfinite(got).all() and worst <= 1.0, name


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_specular_probe_identity_on_oracle(orc, res):
    base = fd.make_env(5, res, (48, 20), seed=res)
    env = fd.probe_env("spec", base)
    for max_lod in (env["spec_mips"], env["spec_mips"] + 3, 4.7, 0):
        for offset in (0.0, 0.7):
            p = fd.specular_probe(env, max_lod, 4000, seed=res + 17, offset=offset)
            _check(f"spec {res} lod {max_lod} off {offset}", _oracle(orc, p, env), p)


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_diffuse_probe_identity_on_oracle(orc, res):
    env = fd.probe_env("diff", fd.make_env(res, 2, (20, 48), seed=res))
    for offset in (0.0, 0.7, math.pi):
        p = fd.diffuse_probe(env, 4000, seed=res + 3, offset=offset)
        _check(f"diff {res} off {offset}", _oracle(orc, p, env), p)


@pytest.mark.parametrize("wh", sr.LUT_SIZES)
def test_lut_probe_identity_on_oracle(orc, wh):
    for ch in (0, 1):
        env = fd.probe_env("lut", fd.make_env(2, 5, wh, seed=wh[0] + wh[1]), channel=ch)
        p = fd.lut_probe(env, ch, 6000, seed=wh[0] * 7 + ch)
        _check(f"lut {wh} channel {ch}", _oracle(orc, p, env), p)
