"""CPU: the oracle's cube and LUT samplers against the float64 restatement of DESIGN.md §3 (tests/sampling_ref.py).

Tolerance. Face selection compares absolute values of the same float32 components in both, which is exact, so both always
pick the same face, ties included. What differs is the texel-space coordinate: the oracle forms x = (sx*0.5+0.5)*N - 0.5
in fp32, |dx| <= N * 2^-22 (one rounded division for sx, one add, one multiply, one subtract), and likewise y. The seamless
sampler is continuous in (x, y) everywhere — across texel boundaries, face edges and corners — with slope at most the
largest texel difference, so even where the two put floor(x) on different sides of an integer the results differ by at
most (|dx| + |dy|) * max|texel difference|. The fp32 lerps and the corner mean add at most 16 * 2^-24 * max|texel|.
"""
import numpy as np
import pytest

import sampling_ref as sr

U24 = 2.0 ** -24


def _cube_bound(N, t):
    span = float(t.max() - t.min())
    return 2 * N * 4 * U24 * span + 16 * U24 * float(np.abs(t).max())


@pytest.mark.parametrize("res", sr.CUBE_RES)
def test_oracle_cube_sampler_matches_float64_rules(orc, res):
    rng = np.random.default_rng(100 + res)
    mips = sr.mip_count(res)
    cube = sr.random_cube(res, seed=res)
    uni = sr.uniform_directions(100_000, rng)
    worst = 0.0
    for mip in range(mips + 2):                         # the last two clamp to the last mip
        N = res >> min(mip, mips - 1)
        d = np.concatenate([uni, sr.special_directions(N, rng)])
        ref = sr.sample_cube(cube, res, mips, d, mip)
        got = orc.sample_cube(cube, res, mips, d, mip).astype(np.float64)
        err = np.abs(got - ref).max()
        worst = max(worst, err)
        assert err <= _cube_bound(N, cube), (res, mip, err)
    print(f"cube {res} x {mips} mips: max |oracle - float64| = {worst:.2e}")


def test_float64_rules_are_seamless_and_exact_at_texel_centres():
    """properties of the restatement itself: a texel-centre direction returns that texel; a direction on an edge or a
    corner returns the same value from either face (continuity of the seamless rule)"""
    rng = np.random.default_rng(7)
    for res in sr.CUBE_RES:
        cube = sr.random_cube(res, seed=res)
        N = res
        c = (2 * np.arange(N) + 1) / N - 1
        sx, sy = [a.ravel() for a in np.meshgrid(c, -c)]          # row 0 is the top (sy = +1) row
        for f in range(6):
            M, U, V = sr._FACES[f].astype(np.float64)
            d = M[None] + sx[:, None] * U[None] + sy[:, None] * V[None]
            got = sr.sample_cube(cube, res, sr.mip_count(res), d, 0)
            assert np.allclose(got, cube[f * N * N:(f + 1) * N * N], atol=1e-12)
        e = sr.special_directions(N, rng)[6:6 + 12 * 9 + 8]          # edges and corners
        for k in range(3):                                              # nudge each component off the tie
            a, b = e.astype(np.float64).copy(), e.astype(np.float64).copy()
            a[:, k] *= 1 + 1e-9; b[:, k] *= 1 - 1e-9
            va = sr.sample_cube(cube, res, sr.mip_count(res), a, 0)
            vb = sr.sample_cube(cube, res, sr.mip_count(res), b, 0)
            assert np.abs(va - vb).max() < 1e-6 * N


@pytest.mark.parametrize("w,h", sr.LUT_SIZES)
def test_oracle_lut_sampler_matches_float64_rules(orc, w, h):
    rng = np.random.default_rng(w * 100 + h)
    lut = sr.random_lut(w, h, seed=w + h)
    edges = np.concatenate([[0.0, 1.0, -0.25, 1.25, 0.5 / w, 1 - 0.5 / w], (np.arange(w) + 0.5) / w, np.arange(w + 1) / w])
    vedges = np.concatenate([[0.0, 1.0, -0.25, 1.25], (np.arange(h) + 0.5) / h, np.arange(h + 1) / h])
    eu, ev = [a.ravel() for a in np.meshgrid(edges, vedges)]
    u = np.concatenate([rng.uniform(0, 1, 100_000), eu]).astype(np.float32)
    v = np.concatenate([rng.uniform(0, 1, 100_000), ev]).astype(np.float32)
    ref = sr.sample_lut(lut, u, v)
    got = orc.sample_lut(lut, u, v).astype(np.float64)
    bound = (w + h) * 2 * U24 + 8 * U24
    err = np.abs(got - ref).max()
    print(f"LUT {w}x{h}: max |oracle - float64| = {err:.2e}")
    assert err <= bound
