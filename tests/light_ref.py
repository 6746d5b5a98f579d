"""float64 restatement of the discrete and ill-conditioned parts of K1's light loop (Lighting.hlsl:29-73 / :308-345 and the
`denom < EPSILON -> D = 1` escape of NormalDistributionGGX, BRDF.hlsl:65-79), for tests/test_light_domain*.py.

  * the range decision: the fp32 rule `sqrt_rn(dot(L, L)) < range` with the dot product unfused, (x*x + y*y) + z*z;
  * the spot intensity as an interval: the float64 angle widened by what an fp32 evaluation of its cosine can be off
    (the cosine error budget DELTA_C), pushed through acos and the ramp, which is monotone in theta, so that a hard or
    narrow cone yields a DECISION interval (an intensity that may be anything from 0 to 1 only near an edge);
  * GGX's t and the D = 1 escape from the fp32 N.H the shader sequence produces.
The continuous BRDF needs no restatement here: the oracle is pinned to the shader text bit for bit (tests/test_hlsl_ref.py).
"""
import math

import numpy as np

F32 = np.float32
U24 = 2.0 ** -24
PI32 = F32(3.14159265359)                  # hlsl_math.h PI
EPS32 = F32(0.000000000001)                # BRDF.hlsl:22
# Cosine error budget of an fp32 evaluation of dot(normalize(P - Lpos), normalize(spotDir)) with unit inputs, in units of
# 2^-24: the normalised spot direction (3 roundings + a division per component: 4), the squared length (3 roundings, half of
# it in the reciprocal square root: 1.5), rsqrt.approx (2^-22.9 relative: 2; the oracle's sqrt + division: 2), the three
# products and two sums (5), the final scaling (1). 16 covers K1's sequence and the oracle's alike.
DELTA_C = 16 * U24
ACOS_ULP = 4                               # device acosf: 2 ulp (CUDA C Programming Guide, table of single-precision errors)


def f32(x):
    return np.asarray(x, F32)


def dot_u(a, b):
    """HLSL dot on fp32 operands, every operation rounded on its own: (x*x' + y*y') + z*z'"""
    a, b = f32(a), f32(b)
    with np.errstate(all="ignore"):
        return (a[..., 0] * b[..., 0] + a[..., 1] * b[..., 1]) + a[..., 2] * b[..., 2]


def normalize_u(v):
    """v / sqrt(dot(v, v)) in fp32, correctly rounded (the oracle's normalize, K1's normalize_u)"""
    v = f32(v)
    with np.errstate(all="ignore"):
        return v / np.sqrt(dot_u(v, v))[..., None]


# ---- range ---------------------------------------------------------------------------------------------------------
def light_d2(P, Lpos):
    """the fp32 squared distance of CalculatePointLightIllumination: L = Lw - P rounded, then dot(L, L) unfused"""
    with np.errstate(all="ignore"):
        L = f32(Lpos)[None] - f32(P)
    return dot_u(L, L)


def in_range(P, Lpos, rng):
    """`length(Lw - P) < l.range` in fp32: the decision K1 must reproduce bit for bit"""
    with np.errstate(all="ignore"):
        return np.sqrt(light_d2(P, Lpos)) < F32(rng)


def distance64(P, Lpos):
    return np.linalg.norm(np.asarray(Lpos, np.float64)[None] - np.asarray(P, np.float64), axis=-1)


# ---- spot intensity --------------------------------------------------------------------------------------------------
def spot_theta64(P, Lpos, spot_dir):
    """angle between the pixel direction P - Lpos and the (normalised) spot direction, float64 from the fp32 inputs"""
    d = np.asarray(P, np.float64) - np.asarray(Lpos, np.float64)[None]
    u = d / np.linalg.norm(d, axis=-1, keepdims=True)
    s = np.asarray(spot_dir, np.float64)
    s = s / np.linalg.norm(s)
    return np.arccos(np.clip(u @ s, -1.0, 1.0))


def ramp64(theta, inner, outer):
    """SpotlightIntensity (Lighting.hlsl:57-73) on a float64 angle: 0 beyond outer, 1 up to inner, the linear ramp between"""
    inner, outer = float(F32(inner)), float(F32(outer))
    theta = np.asarray(theta, np.float64)
    with np.errstate(all="ignore"):
        lin = 1.0 - (theta - inner) / (outer - inner)
    return np.where(theta > outer, 0.0, np.where(theta <= inner, 1.0, lin))


def theta_interval(theta):
    """[lo, hi] of the angle an fp32 evaluation can produce: the cosine off by DELTA_C (which near the axis moves theta by up
    to sqrt(2 DELTA_C), elsewhere by about DELTA_C / sin(theta)), then acosf off by ACOS_ULP ulp"""
    c = np.cos(theta)
    lo = np.arccos(np.minimum(c + DELTA_C, 1.0))
    hi = np.arccos(np.maximum(c - DELTA_C, -1.0))
    pad = ACOS_ULP * U24 * 2.0 * np.maximum(np.abs(theta), 2.0 ** -126)
    return np.maximum(lo - pad, 0.0), hi + pad


def spot_interval(P, Lpos, spot_dir, inner, outer):
    """(lo, hi, theta64): the float64 bound on the intensity an fp32 evaluation may produce. The ramp is monotone
    (non-increasing) in theta, so its values at the ends of the angle interval bound it; the ramp's own fp32 rounding
    (1 - (theta - inner) * invCone with a rounded reciprocal) adds a few ulp of 1."""
    th = spot_theta64(P, Lpos, spot_dir)
    a, b = theta_interval(th)
    hi, lo = ramp64(a, inner, outer), ramp64(b, inner, outer)
    slack = 8 * U24
    return lo - slack, hi + slack, th


def decided(lo, hi):
    """an intensity that cannot flip: the interval does not reach across an edge (width of a normal ramp step aside)"""
    return (hi - lo) < 0.5


def oracle_spot_cos(P, Lpos, spot_dir):
    """the oracle's cosine bit for bit: dot(normalize(P - Lpos), normalize(spotDir)) (Lighting.hlsl:59-61); above 1 its
    acos is NaN"""
    with np.errstate(all="ignore"):
        d = f32(P) - f32(Lpos)[None]
    return dot_u(normalize_u(d), normalize_u(f32(spot_dir))[None])


# ---- GGX ----------------------------------------------------------------------------------------------------------------
def ggx_t(ndoth, roughness):
    """t = nh2 * (a2 - 1) + 1 in fp32, unfused (BRDF.hlsl:65-79)"""
    r = f32(roughness)
    nh = f32(ndoth)
    a = r * r
    a2 = a * a
    return (nh * nh) * (a2 - F32(1.0)) + F32(1.0)


def d_escape(ndoth, roughness):
    """the `PI * t * t < EPSILON -> D = 1` decision"""
    t = ggx_t(ndoth, roughness)
    with np.errstate(all="ignore"):
        return PI32 * (t * t) < EPS32


def escape_roughness_bound():
    """the largest roughness for which PI * r^8 < 1e-12 in real arithmetic: 0.0274..."""
    return (1e-12 / math.pi) ** 0.125
