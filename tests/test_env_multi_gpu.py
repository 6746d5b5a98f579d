"""-m gpu: the band forms of the environment prefilter (vq_diffuse_irradiance_multi_signal, vq_brdf_integration_lut_multi_signal)
and the one-launch cube blur (vq_gaussian_blur_cube), bit for bit against the single-GPU calls they replace:
  * K2 and K4 on 1, 2, 3 and 8 destinations, over empty, one-row, face-boundary, odd and whole row ranges, in both sampling modes,
    with several source mips and HDRI pyramids down to a 2 x 1 one; rows outside the range keep a NaN sentinel everywhere;
  * the cube blur against vq_gaussian_blur_x -> temporary -> vq_gaussian_blur_y per face, for every face edge 1..128, on inputs with
    negatives, denormals, +-Inf and NaN, and in place;
  * simulated worlds of 2, 3 and 8 ranks (tests/test_rendezvous_gpu.py's SimWorld, run_world and watcher) for each new retirement
    block, and distributed.EnvironmentStep's diffuse band, blur and specular ranges; 320 signalled calls in a row per block."""
import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import distributed as vd
from vqengine_b200.distributed import equal_tiles
from test_ibl_gpu import _pyr
from test_rendezvous_gpu import ORDERS, Case, SimWorld, _assert_frames, pw, rank_dests, run_world  # noqa: F401  (pw: fixture)

pytestmark = pytest.mark.gpu
SENTINEL = 0x7FC0DEAD              # a quiet NaN with a payload no kernel computes


def _nan_like(t):
    out = torch.empty_like(t)
    out.view(torch.int32).fill_(SENTINEL)
    return out


def _bits(t):
    return t.contiguous().view(torch.int32)


def _assert_rows(got, ref, a, b, what):
    """units [a, b) of `got` equal `ref` bit for bit, every other unit holds the sentinel"""
    torch.cuda.synchronize()
    g, r = _bits(got), _bits(ref)
    assert torch.equal(g[a:b], r[a:b]), (what, "inside the range")
    assert bool((g[:a] == SENTINEL).all()) and bool((g[b:] == SENTINEL).all()), (what, "outside the range")


# ---- K2 ----------------------------------------------------------------------------------------------------------------------
def _hdri(ctx, w, h):
    _, levels, d, p = _pyr(ctx, vq, None, w, h)
    return d, p, levels


def _diffuse_ref(ctx, p, res, kw):
    full = torch.zeros((6 * res * res, 4), dtype=torch.float32, device="cuda")
    full.view(torch.int32).fill_(SENTINEL)
    ctx.diffuse_irradiance(p, vq.cubemap_of(full, res, 1), **kw)
    return full


def _diffuse_ranges(res):
    return {"empty": (5, 5), "one row": (7, 8), "face boundary": (res - 2, res + 3), "odd": (3, 6 * res - 5),
            "whole": (0, 6 * res), "last row": (6 * res - 1, 6 * res)}


@pytest.mark.parametrize("n_dest", [1, 2, 3, 8])
def test_diffuse_multi_ranges(ctx, n_dest):
    res, kw = 16, dict(n_phi=48, n_theta=12, src_mip=2)
    d, p, _ = _hdri(ctx, 128, 64)
    ref = _diffuse_ref(ctx, p, res, kw)
    for name, (a, b) in _diffuse_ranges(res).items():
        dests = [_nan_like(ref) for _ in range(n_dest)]
        n0 = vq.launch_count()
        ctx.diffuse_irradiance_multi(p, [vq.cubemap_of(t, res, 1) for t in dests], row_begin=a, row_end=b, **kw)
        assert vq.launch_count() - n0 == (1 if b > a else 0)
        for k, t in enumerate(dests):
            _assert_rows(t, ref, a * res, b * res, f"{name} destination {k}")


@pytest.mark.parametrize("mode", ["grid", "step"])
@pytest.mark.parametrize("w,h,src_mip", [(256, 128, 3), (256, 128, 0), (64, 32, 5), (16, 8, 2), (4, 2, 1), (2, 1, 0)],
                         ids=lambda v: str(v))
def test_diffuse_multi_sampling(ctx, mode, w, h, src_mip):
    """both sampling modes, source mips from 0 to the pyramid's last level, HDRI pyramids down to one level"""
    res = 8
    kw = dict(n_phi=37, n_theta=11, src_mip=src_mip) if mode == "grid" else dict(step=0.05, src_mip=src_mip)
    d, p, levels = _hdri(ctx, w, h)
    assert src_mip < levels
    ref = _diffuse_ref(ctx, p, res, kw)
    for a, b in ((0, 6 * res), (3, 6 * res - 7), (res, 2 * res)):
        dests = [_nan_like(ref) for _ in range(3)]
        ctx.diffuse_irradiance_multi(p, [vq.cubemap_of(t, res, 1) for t in dests], row_begin=a, row_end=b, **kw)
        for k, t in enumerate(dests):
            _assert_rows(t, ref, a * res, b * res, f"rows {a}..{b} destination {k}")


def test_diffuse_multi_engine_step(ctx):
    """the engine's own step, 0.010 (629 x 158 samples per texel), and a 64-texel face, into 2 destinations"""
    res, kw = 64, dict(step=0.010, src_mip=3)
    d, p, _ = _hdri(ctx, 256, 128)
    ref = _diffuse_ref(ctx, p, res, kw)
    for a, b in equal_tiles(6 * res, 8)[2:4]:
        dests = [_nan_like(ref) for _ in range(2)]
        ctx.diffuse_irradiance_multi(p, [vq.cubemap_of(t, res, 1) for t in dests], row_begin=a, row_end=b, **kw)
        for k, t in enumerate(dests):
            _assert_rows(t, ref, a * res, b * res, f"rows {a}..{b} destination {k}")


# ---- K4 ----------------------------------------------------------------------------------------------------------------------
def _lut_ref(ctx, w, h, samples):
    ref = torch.zeros((h, w, 2), dtype=torch.float32, device="cuda")
    ref.view(torch.int32).fill_(SENTINEL)
    ctx.brdf_integration_lut(ref, samples)
    return ref


def _lut_dest(h, w, k):
    """destination k: every other one pitched (a view into a wider image)"""
    t = torch.empty((h, w + 3 * (k % 2), 2), dtype=torch.float32, device="cuda")
    t.view(torch.int32).fill_(SENTINEL)
    return t[:, :w]


@pytest.mark.parametrize("n_dest", [1, 2, 3, 8])
@pytest.mark.parametrize("w,h,samples", [(1, 1, 64), (37, 23, 333), (300, 9, 128), (1024, 1024, 512)], ids=lambda v: str(v))
def test_lut_multi_ranges(ctx, n_dest, w, h, samples):
    ref = _lut_ref(ctx, w, h, samples)
    ranges = {(0, h), (0, 0), (h // 2, h // 2 + 1), (h - 1, h), (h // 3, h - h // 4)}
    for a, b in sorted(ranges):
        dests = [_lut_dest(h, w, k) for k in range(n_dest)]
        n0 = vq.launch_count()
        ctx.brdf_integration_lut_multi([vq.image_of(t, 2) for t in dests], samples, row_begin=a, row_end=b)
        assert vq.launch_count() - n0 == (1 if b > a else 0)
        for k, t in enumerate(dests):
            _assert_rows(t.contiguous(), ref, a, b, f"{w}x{h} rows {a}..{b} destination {k}")


# ---- K5 on a whole cube --------------------------------------------------------------------------------------------------------
def _cube_input(res, seed):
    """normal values of both signs and wide range, with denormals, +-Inf and NaN sprinkled in"""
    g = np.random.default_rng(seed)
    x = (g.standard_normal((6 * res * res, 4)) * np.exp(g.uniform(-8, 8, (6 * res * res, 4)))).astype(np.float32)
    flat = x.reshape(-1)
    n = flat.size
    for v, frac in ((1e-40, 0.02), (-3e-42, 0.02), (np.inf, 0.004), (-np.inf, 0.004), (np.nan, 0.004), (-0.0, 0.01)):
        idx = g.choice(n, size=max(1, int(n * frac)), replace=False)
        flat[idx] = v
    return torch.from_numpy(x).cuda()


def _twelve_calls(ctx, src, res):
    """vq_gaussian_blur_x into a temporary, then vq_gaussian_blur_y, per face: the engine's blur of the diffuse cube"""
    out = _nan_like(src)
    tmp = torch.empty((res, res, 4), dtype=torch.float32, device="cuda")
    fi, fo = src.view(6, res, res, 4), out.view(6, res, res, 4)
    for f in range(6):
        ctx.gaussian_blur(fi[f], tmp, False)
        ctx.gaussian_blur(tmp, fo[f], True)
    return out


def test_blur_cube_every_size(ctx):
    """every face edge from 1 to the limit (128), odd ones included, out of place and in place"""
    for res in range(1, 129):
        src = _cube_input(res, res)
        ref = _twelve_calls(ctx, src, res)
        out = _nan_like(src)
        n0 = vq.launch_count()
        ctx.gaussian_blur_cube(vq.cubemap_of(src, res, 1), vq.cubemap_of(out, res, 1))
        assert vq.launch_count() - n0 == 1
        inplace = src.clone()
        ctx.gaussian_blur_cube(vq.cubemap_of(inplace, res, 1), vq.cubemap_of(inplace, res, 1))
        torch.cuda.synchronize()
        assert torch.equal(_bits(out), _bits(ref)), f"res {res}: {int((_bits(out) != _bits(ref)).sum())} words differ"
        assert torch.equal(_bits(inplace), _bits(ref)), f"res {res} in place"


def test_blur_cube_special_values_reach_the_output(ctx):
    """the inputs above do exercise the special values: the output holds NaN, and finite faces stay finite"""
    res = 64
    src = _cube_input(res, 5)
    out = _nan_like(src)
    ctx.gaussian_blur_cube(vq.cubemap_of(src, res, 1), vq.cubemap_of(out, res, 1))
    torch.cuda.synchronize()
    assert bool(torch.isnan(out[:, :3]).any()) and bool((out[:, 3] == 1.0).all())
    clean = torch.randn((6 * res * res, 4), device="cuda")
    ctx.gaussian_blur_cube(vq.cubemap_of(clean, res, 1), vq.cubemap_of(out, res, 1))
    torch.cuda.synchronize()
    assert bool(torch.isfinite(out).all())
    assert torch.equal(_bits(out), _bits(_twelve_calls(ctx, clean, res)))


def test_blur_cube_refusals_on_device(ctx):
    res = 16
    a = torch.zeros((6 * res * res + 8, 4), device="cuda")
    with pytest.raises(vq.VqError, match="the same cube or not overlap"):
        ctx.gaussian_blur_cube(vq.Cubemap(a.data_ptr(), res, 1), vq.Cubemap(a.data_ptr() + 16 * 8, res, 1))
    with pytest.raises(vq.VqError, match="1..128"):
        ctx.gaussian_blur_cube(vq.Cubemap(a.data_ptr(), 130, 1), vq.Cubemap(a.data_ptr(), 130, 1))


# ---- simulated worlds ----------------------------------------------------------------------------------------------------------
def diffuse_case(ctx, n, res, kw, name, hw=(128, 64)):
    d, p, _ = _hdri(ctx, *hw)
    ref = _diffuse_ref(ctx, p, res, kw)
    bands = equal_tiles(6 * res, n)
    assert all(b > a for a, b in bands)

    def run(r, dests, signal, stream):
        ctx.diffuse_irradiance_multi(p, [vq.cubemap_of(t, res, 1) for t in dests], row_begin=bands[r][0], row_end=bands[r][1],
                                     stream=stream, signal=signal, **kw)
    case = Case(name, n, ref, float("nan"), [[(a * res, b * res)] for a, b in bands], run)
    case.keep = d
    return case


def lut_case(ctx, n, w, h, samples, name):
    ref = _lut_ref(ctx, w, h, samples)
    bands = equal_tiles(h, n)
    assert all(b > a for a, b in bands)

    def run(r, dests, signal, stream):
        ctx.brdf_integration_lut_multi([vq.image_of(t, 2) for t in dests], samples, row_begin=bands[r][0], row_end=bands[r][1],
                                       stream=stream, signal=signal)
    return Case(name, n, ref, float("nan"), [[band] for band in bands], run)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
def test_diffuse_world(ctx, pw, n, order):
    run_world(pw, diffuse_case(ctx, n, 8, dict(n_phi=32, n_theta=8, src_mip=2), f"diffuse 8 n{n}"), SimWorld(n, order))


def test_diffuse_world_step(ctx, pw):
    """the step mode at a 16-texel face over 3 ranks (bands that start inside a face)"""
    run_world(pw, diffuse_case(ctx, 3, 16, dict(step=0.05, src_mip=3), "diffuse step 16 n3"), SimWorld(3, "scrambled"))


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
def test_lut_world(ctx, pw, n, order):
    """38 x 29: a LUT row is 304 bytes, whole 16-byte words for the watcher's copies (ragged widths: test_lut_multi_ranges)"""
    run_world(pw, lut_case(ctx, n, 38, 29, 128, f"lut 38x29 n{n}"), SimWorld(n, order))


def test_lut_world_1024(ctx, pw):
    run_world(pw, lut_case(ctx, 2, 1024, 1024, 256, "lut 1024 n2"), SimWorld(2, "rotated"))


@pytest.mark.parametrize("family", ["diffuse", "lut"])
def test_ticket_ring_wraps(ctx, family):
    """320 signalled calls of one new retirement block in a row, 2 ranks: every slot of the ticket-pair ring comes back twice"""
    case = (diffuse_case(ctx, 2, 4, dict(n_phi=8, n_theta=4, src_mip=1), "diffuse ring") if family == "diffuse"
            else lut_case(ctx, 2, 16, 6, 32, "lut ring"))
    world = SimWorld(2, "rotated")
    frames = case.dests()
    for e in range(1, 161):
        world.preset(e)
        for r in range(2):
            case.run(r, rank_dests(world, frames, r), world.signal(r, e), None)
            world.ran(r, e)
            world.check(f"{family} ring epoch {e} rank {r}")
    _assert_frames(case, frames, case.expected(range(2)), "after the ring")


# ---- distributed.EnvironmentStep: the diffuse band, the blur and the specular ranges -----------------------------------------------
class EnvWorld:
    """every rank's diffuse, blurred and specular cubes, and the single-GPU bits of each"""

    def __init__(self, ctx, n, dres=16, sres=32, mips=6, samples=128, kw=None):
        self.ctx, self.n, self.dres, self.sres, self.mips, self.samples = ctx, n, dres, sres, mips, samples
        self.kw = kw or dict(n_phi=32, n_theta=8, src_mip=2)
        self.d, self.p, _ = _hdri(ctx, 256, 128)
        self.diff_ref = _diffuse_ref(ctx, self.p, dres, self.kw)
        self.blur_ref = _twelve_calls(ctx, self.diff_ref, dres)
        self.spec_ref = torch.zeros((vq.cubemap_texel_count(sres, mips), 4), device="cuda")
        ctx.specular_prefilter(self.p, vq.cubemap_of(self.spec_ref, sres, mips), samples)
        self.diff = [_nan_like(self.diff_ref) for _ in range(n)]
        self.blur = [_nan_like(self.diff_ref) for _ in range(n)]
        self.spec = [_nan_like(self.spec_ref) for _ in range(n)]

    def steps(self, world):
        out = []
        for r in range(self.n):
            order = [r] + world.peers[r]
            out.append(vd.EnvironmentStep(self.ctx, self.p, [vq.cubemap_of(self.diff[q], self.dres, 1) for q in order],
                                          vq.cubemap_of(self.blur[r], self.dres, 1),
                                          [vq.cubemap_of(self.spec[q], self.sres, self.mips) for q in order], r, self.n,
                                          diffuse_params=self.kw, num_samples=self.samples))
        return out

    def reset(self):
        for t in self.diff + self.blur + self.spec:
            t.view(torch.int32).fill_(SENTINEL)

    def check(self, what):
        torch.cuda.synchronize()
        for r in range(self.n):
            assert torch.equal(_bits(self.diff[r]), _bits(self.diff_ref)), (what, "diffuse", r)
            assert torch.equal(_bits(self.blur[r]), _bits(self.blur_ref)), (what, "blurred", r)
            assert torch.equal(_bits(self.spec[r]), _bits(self.spec_ref)), (what, "specular", r)


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
def test_environment_step_world(ctx, n, order):
    """the ranks run one after another on one stream, in the order a real step's rendezvous imposes: every rank's diffuse band
    (epoch e), then every rank's blur and specular ranges (epoch e + 1); the flag words, the launch counts and every rank's three
    cubes are checked, through epochs across 2^32"""
    ew = EnvWorld(ctx, n)
    world = SimWorld(n, order)
    steps = ew.steps(world)
    s = torch.cuda.Stream()
    launches = []
    for st in steps:
        n0 = vq.launch_count()
        st.diffuse(0, None, s)
        launches.append(vq.launch_count() - n0)
    for st in steps:
        n0 = vq.launch_count()
        st.finish(0, None, s)
        launches.append(vq.launch_count() - n0)
    ew.check("without a signal")
    assert launches[:n] == [1] * n and launches[n:] == [2] * n
    for e in (0xFFFFFFFC, 0xFFFFFFFD, 0):
        ew.reset()
        for phase, e_p in (("diffuse", e), ("finish", (e + 1) & 0xFFFFFFFF)):
            world.preset(e_p)
            for r, st in enumerate(steps):
                n0 = vq.launch_count()
                getattr(st, phase)(e, world.sig[r], s)
                assert vq.launch_count() - n0 == (1 if phase == "diffuse" else 2), (phase, r)
                world.ran(r, e_p)
                world.check(f"env step {phase} epoch {e:#x} rank {r}")
        ew.check(f"epoch {e:#x}")


def test_environment_step_run_and_prepare(ctx):
    """run() on one rank of a world of one: diffuse, blur, specular and vq_environment_prepare in stream order, the next epoch back"""
    ew = EnvWorld(ctx, 1)
    lut = torch.zeros((32, 32, 2), device="cuda")
    ctx.brdf_integration_lut(lut, 64)
    world = SimWorld(1, "rotated")
    st = ew.steps(world)[0]
    st.env = vq.EnvironmentMaps(vq.cubemap_of(ew.blur[0], ew.dres, 1), vq.cubemap_of(ew.spec[0], ew.sres, ew.mips), vq.image_of(lut, 2))
    n0 = vq.launch_count()
    assert st.run(7, None, torch.cuda.current_stream()) == 9
    assert vq.launch_count() - n0 >= 4
    ew.check("run")
    ctx.environment_invalidate()
