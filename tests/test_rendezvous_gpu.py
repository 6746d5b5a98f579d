"""-m gpu: the in-kernel cross-rank rendezvous of every signalled call, on one GPU (vq::peer_rendezvous and the four retirement
blocks that run it: forward_kernel<MULTI>, psmain_kernel<MULTI>, specular_persistent_kernel, post_retire).

A SimWorld owns n x n int32 flag words, one row per rank, and gives each rank the VqPeerSignal a multi-GPU step would: flags[0]
is the rank's own row, flags[1..n-1] its peers' rows, in bench.py's rotated order or in a fixed scrambled one. The ranks run one
after another on one stream, each storing its band into all n frames. They never wait for each other: before every step with
epoch e, EVERY word of the array is set to e + 1, which satisfies the wait (a signed difference >= 0, and any unsigned >=), so the
last CTA's wait returns after one poll whichever word it reads. A word the kernel writes becomes exactly e. Every rank call is
checked for
  * the flag words: after rank j, word j of every other row is e and every other word keeps its value (a pure-Python model);
  * the frames: the band equals the single-GPU result bit for bit, rows no rank has written yet keep their fill, and the world
    assembles what the same world without a signal assembles;
  * the launches: as many as without the signal;
  * the watcher (tests/device_check/peer_watch.cu): one CTA on a second stream, launched before the call, polls the word the rank
    writes into its first peer's row until it equals e and then copies every destination's band. The copy must hold the final
    bits; a flag raised before every CTA's stores would show as missing rows. Whether the watcher saw the flag while the call was
    still running is counted and printed (never asserted: it depends on scheduling).
Every call runs at least three consecutive steps on one context and one set of frames, through epochs 0xFFFFFFFD, 0xFFFFFFFE, 0,
1: the descriptor carries epochs across 2^32 and stores them exactly. Each call takes its retire count from the context's 128-slot
ticket-pair ring (vq_ticket_pair), so the next step gets another slot: a count the last CTA does not reset shows only when the ring
comes back to its slot. So each retirement block also runs 320 signalled calls in a row, which reuses every slot twice.
Epoch 0xFFFFFFFF is left out, since its pre-set value e + 1 would wrap to 0, and only 0xFFFFFFFF itself satisfies an unsigned
reading of it.

The other direction of the wait, that a stale or wrapped flag must HOLD it, and ranks releasing each other while they run at the
same time, are tested in tests/test_rendezvous_hold_gpu.py (flag arrays in mapped host memory, peers played by a host thread).
Not tested: a real multi-GPU step (NVLink peer stores, fence.sys ordering across devices) needs two or more GPUs
(tools/perf_multi_shading.py, tools/perf_post_multi.py under torchrun); the 20 s watchdog, on purpose, since testing it means a
trap."""
import ctypes as C
import os
import random
import subprocess

import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import synth, distributed as vd
from vqengine_b200.distributed import equal_tiles, even_tiles, post_chain_rows
from test_ibl_gpu import _pyr
from test_multi_shading_gpu import Frame
from test_post_fused_gpu import chain, fsr_consts, hdr
from test_post_multi_gpu import Pass, reference_chain
from test_psmain_shadowed_gpu import _maps, _shadow_scene

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]
EPOCHS = (0xFFFFFFFD, 0xFFFFFFFE, 0, 1)
WATCH_NS = 500_000_000             # the watcher gives up (and reports it) after 0.5 s
ORDERS = ("rotated", "scrambled")
LIVE = {}                          # case -> [rank steps the watcher saw while the call ran, rank steps watched]


@pytest.fixture(scope="module")
def pw(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out = tmp_path_factory.mktemp("devicecheck") / "libpeerwatch.so"
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), *FLAGS, "-o", str(out),
                           os.path.join(ROOT, "tests", "device_check", "peer_watch.cu")])
    torch.cuda.init()
    lib = C.CDLL(str(out))
    vp, u64 = C.c_void_p, C.c_ulonglong
    lib.pw_watch.argtypes = [vp, vp, C.c_uint32, u64, C.c_int, vp * 8, vp * 8, u64 * 8, vp]
    lib.pw_stamp.argtypes = [vp, vp]
    lib.pw_rendezvous.argtypes = [vp, vp * 8, C.c_int, C.c_int, C.c_uint32]
    yield lib
    for case, (live, watched) in sorted(LIVE.items()):
        print(f"watcher live: {case}: {live}/{watched}")
    print(f"watcher live: total {sum(v[0] for v in LIVE.values())}/{sum(v[1] for v in LIVE.values())}")


def _i32(u):
    u &= 0xFFFFFFFF
    return u - (1 << 32) if u >= 1 << 31 else u


def peer_order(n, r, order):
    """the peers of rank r in its signal's flags[1..n-1]: bench.py's PeerFlags rotation, or a fixed scrambled permutation"""
    peers = [(r + k) % n for k in range(1, n)]
    if order == "scrambled":
        random.Random(1009 * n + r).shuffle(peers)
    return peers


class SimWorld:
    """n simulated ranks' flag arrays (row q = rank q's array) and their VqPeerSignals, with the model of what must be written"""

    def __init__(self, n, order):
        self.n = n
        self.flags = torch.zeros((n, n), dtype=torch.int32, device="cuda")
        self.peers = [peer_order(n, r, order) for r in range(n)]
        self.sig = []
        for r in range(n):
            s = vq.PeerSignal()
            for i, q in enumerate([r] + self.peers[r]):
                s.flags[i] = self.word(q, 0)
            s.n_ranks, s.my_index = n, r
            self.sig.append(s)
        self.model = None

    def word(self, row, col):
        return self.flags.data_ptr() + 4 * (row * self.n + col)

    def preset(self, e):
        """every word of every array to e + 1: every wait of the step is satisfied before any rank runs"""
        assert e != 0xFFFFFFFF, "e + 1 would wrap"
        self.flags.fill_(_i32(e + 1))
        self.model = np.full((self.n, self.n), (e + 1) & 0xFFFFFFFF, np.uint32)

    def signal(self, r, e):
        self.sig[r].epoch = e
        return self.sig[r]

    def ran(self, r, e):
        """rank r's call of epoch e has finished: word r of every other rank's array holds e"""
        self.model[[q for q in range(self.n) if q != r], r] = e

    def check(self, what):
        torch.cuda.synchronize()
        got = self.flags.cpu().numpy().view(np.uint32)
        assert np.array_equal(got, self.model), (what, "flag words", got.tolist(), "want", self.model.tolist())


class Case:
    """one call's simulated world: n destinations per world (frames [h, w, 4] or cubemaps [texels, 4], both indexed by their first
    dimension, the 'unit'), the fill they start from, the single-GPU result `ref`, the unit ranges rank r writes, and
    run(r, dests, signal, stream), which enqueues rank r's calls into `dests` (its own destination first, then its peers')"""

    def __init__(self, name, n, ref, fill, regions, run):
        self.name, self.n, self.ref, self.fill, self.regions, self.run = name, n, ref, fill, regions, run
        self.units = ref.shape[0]
        self.unit_bytes = ref[0].numel() * 4
        self.fill_t = torch.full_like(ref, fill)

    def dests(self):
        return [torch.full_like(self.ref, self.fill) for _ in range(self.n)]

    def mask(self, ranks):
        m = torch.zeros(self.units, dtype=torch.bool, device="cuda")
        for r in ranks:
            for a, b in self.regions[r]:
                m[a:b] = True
        return m

    def expected(self, ranks):
        """the destinations once `ranks` have run: the single-GPU bits on their units, the fill elsewhere"""
        m = self.mask(ranks).view(-1, *([1] * (self.ref.dim() - 1)))
        return torch.where(m, self.ref, self.fill_t)

    def span(self, r):
        """the bytes of a destination that rank r's call writes: from its first unit to its last"""
        a, b = min(a for a, _ in self.regions[r]), max(b for _, b in self.regions[r])
        return a * self.unit_bytes, (b - a) * self.unit_bytes


def _same(got, want):
    return torch.equal(got.view(torch.int32), want.view(torch.int32))


def _assert_frames(case, dests, want, what):
    torch.cuda.synchronize()
    for k, d in enumerate(dests):
        if not _same(d, want):
            bad = (d.view(torch.int32) != want.view(torch.int32)).reshape(case.units, -1).any(-1)
            idx = torch.nonzero(bad).flatten()
            pytest.fail(f"{case.name} {what} destination {k}: {int(bad.sum())} units differ, first {idx[:4].tolist()}")


def rank_dests(world, frames, r):
    return [frames[r]] + [frames[q] for q in world.peers[r]]


def run_world(pw, case, world, epochs=EPOCHS, watch=True):
    """the world without a signal, then one signalled step per epoch on the same frames; every check of the module docstring"""
    n = case.n
    s1, s2 = torch.cuda.Stream(), torch.cuda.Stream()
    frames = case.dests()
    torch.cuda.synchronize()
    launches = []
    for r in range(n):
        n0 = vq.launch_count()
        case.run(r, rank_dests(world, frames, r), None, s1)
        launches.append(vq.launch_count() - n0)
    _assert_frames(case, frames, case.expected(range(n)), "world without a signal")

    spans = [case.span(r) for r in range(n)]
    snaps = [torch.empty(max(s for _, s in spans), dtype=torch.uint8, device="cuda") for _ in range(n)]
    status = torch.zeros(2, dtype=torch.int64, device="cuda")
    stamp = torch.zeros(1, dtype=torch.int64, device="cuda")
    live = LIVE.setdefault(case.name, [0, 0])
    for e in epochs:
        world.preset(e)
        for f in frames:
            f.fill_(case.fill)
        for r in range(n):
            what = f"epoch {e:#x} rank {r}"
            dests = rank_dests(world, frames, r)
            off, size = spans[r]
            if watch:
                status.zero_()
                torch.cuda.synchronize()
                src = (C.c_void_p * 8)(*[d.data_ptr() + off for d in dests])
                dst = (C.c_void_p * 8)(*[s.data_ptr() for s in snaps])
                sizes = (C.c_ulonglong * 8)(*([size] * n))
                # the word rank r writes into its first peer's array
                assert pw.pw_watch(C.c_void_p(s2.cuda_stream), world.word(world.peers[r][0], r), e, WATCH_NS, n, src, dst, sizes,
                                   status.data_ptr()) == 0
            n0 = vq.launch_count()
            case.run(r, dests, world.signal(r, e), s1)
            assert vq.launch_count() - n0 == launches[r], (case.name, what, "launches with and without the signal")
            if watch:
                assert pw.pw_stamp(C.c_void_p(s1.cuda_stream), stamp.data_ptr()) == 0
            world.ran(r, e)
            world.check(f"{case.name} {what}")
            _assert_frames(case, dests, case.expected(range(r + 1)), what)
            if watch:
                st = status.cpu().tolist()
                assert st[0] == 1, (case.name, what, "the watcher never saw the flag")
                for k, d in enumerate(dests):
                    band = d.view(torch.uint8).flatten()[off:off + size]
                    assert torch.equal(snaps[k][:size], band), (case.name, what, f"destination {k} was not finished when the flag was seen")
                live[0] += int(st[1] < int(stamp.item()))
                live[1] += 1
    _assert_frames(case, frames, case.expected(range(n)), "signalled world")


def _rows(bands):
    return [[band] for band in bands]


# ---- vq::peer_rendezvous alone --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("order", ORDERS)
def test_peer_rendezvous_stores(pw, order):
    """n = 2..8, every my_index, epochs across 2^32: word my_index of every peer's array holds the epoch, nothing else changes"""
    s = torch.cuda.Stream()
    for n in range(2, 9):
        world = SimWorld(n, order)
        for e in (5, 0xFFFFFFFE, 0):
            world.preset(e)
            torch.cuda.synchronize()
            for r in range(n):
                sig = world.signal(r, e)
                flags = (C.c_void_p * 8)(*[sig.flags[i] for i in range(8)])
                assert pw.pw_rendezvous(C.c_void_p(s.cuda_stream), flags, n, r, e) == 0
                world.ran(r, e)
                world.check(f"n {n} rank {r} epoch {e:#x}")


# ---- forward_kernel<MULTI> and psmain_kernel<MULTI> -------------------------------------------------------------------------
def shading_case(ctx, call, n, w, h, name):
    planes, mats, chains, env, pf, pv, maps = _shadow_scene(w, h)
    bind = () if call == "shadowed no test" else ("point", "spot", "dir")
    f = Frame(ctx, planes, mats, chains, env, pf, pv, _maps(maps, bind))
    api = "shadowed" if call == "shadowed no test" else call
    ref = torch.from_numpy(f.single(api)).cuda()
    bands = even_tiles(h, n)
    assert all(b > a for a, b in bands)

    def run(r, dests, signal, stream):
        f.multi(api, [vq.image_of(d) for d in dests], 0, rows=bands[r], signal=signal, stream=stream)
    return f, Case(name, n, ref, float("nan"), _rows(bands), run)


# forward: vq_forward_lighting_multi_signal; shadowed: the shadowed call with PCF tests (shadow_pcf_kernel, then forward_kernel);
# shadowed no test: no map bound, the plain forward_kernel branch; from_materials / shadowed_from_materials: psmain_kernel
SHADING = ("forward", "shadowed", "shadowed no test", "from_materials", "shadowed_from_materials")


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("call", SHADING)
def test_shading_world(ctx, pw, call, n, order):
    """257 x 41: a ragged width (the second 256-pixel tile has one column), 8 ranks get bands of 4 and 6 rows"""
    f, case = shading_case(ctx, call, n, 257, 41, f"{call} 257x41 n{n}")
    run_world(pw, case, SimWorld(n, order))
    f.close()


@pytest.mark.parametrize("call", SHADING)
def test_shading_single_cta(ctx, pw, call):
    """100 x 3 over 2 ranks: rank 1's band is one row, a grid of one CTA"""
    f, case = shading_case(ctx, call, 2, 100, 3, f"{call} 100x3 n2")
    run_world(pw, case, SimWorld(2, "scrambled"))
    f.close()


@pytest.mark.parametrize("call", ["forward", "shadowed", "from_materials"])
def test_shading_1080p(ctx, pw, call):
    """1920 x 1080 over 2 ranks: 540-row bands, taller than the grid's gridDim.y (8 x 256-pixel tiles per row)"""
    f, case = shading_case(ctx, call, 2, 1920, 1080, f"{call} 1920x1080 n2")
    run_world(pw, case, SimWorld(2, "rotated"))
    f.close()


# ---- specular_persistent_kernel --------------------------------------------------------------------------------------------
def specular_case(ctx, n, res, mips, samples, ranges_of, name, hw=(256, 128)):
    _, _, d, p = _pyr(ctx, vq, None, *hw)
    n_tex = vq.cubemap_texel_count(res, mips)
    whole = torch.zeros((n_tex, 4), dtype=torch.float32, device="cuda")
    ctx.specular_prefilter(p, vq.cubemap_of(whole, res, mips), samples)
    ranges = [ranges_of(r) for r in range(n)]
    regions = [[(vd.specular_row_to_texel(res, mips, a), vd.specular_row_to_texel(res, mips, b)) for a, b in rr] for rr in ranges]

    def run(r, dests, signal, stream):
        ctx.specular_prefilter_ranges(p, [vq.cubemap_of(t, res, mips) for t in dests], ranges[r], samples, signal=signal, stream=stream)
    case = Case(name, n, whole, float("nan"), regions, run)
    case.keep = d
    return case


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
def test_specular_world(ctx, pw, n, order):
    """InterleavedSpecularPlan's row ranges: split mips, mips every rank computes, mip 0's thread-per-texel units"""
    plan = vd.InterleavedSpecularPlan(32, 6, n)
    run_world(pw, specular_case(ctx, n, 32, 6, 128, plan.row_ranges, f"specular 32x6 n{n}"), SimWorld(n, order))


def test_specular_512_samples(ctx, pw):
    plan = vd.InterleavedSpecularPlan(64, 7, 2)
    run_world(pw, specular_case(ctx, 2, 64, 7, 512, plan.row_ranges, "specular 64x7 512 samples n2"), SimWorld(2, "rotated"))


@pytest.mark.parametrize("n", [2, 3])
def test_specular_single_cta(ctx, pw, n):
    """each rank one row of mip 1 (4 texels: one work unit, a grid of one CTA)"""
    run_world(pw, specular_case(ctx, n, 8, 4, 64, lambda r: [(48 + r, 49 + r)], f"specular one unit n{n}"), SimWorld(n, "scrambled"))


# ---- post_retire: the single passes (tonemap_kernel, cas_kernel, rcas_kernel, easu_2x/easu_up/easu_kernel) ------------------
def pass_case(p, src, n, name):
    oh, ow = p.out_size(src)
    ref = torch.full((oh, ow, 4), float("nan"), device="cuda")
    p.single(src, ref)
    bands = equal_tiles(oh, n)
    assert all(b > a for a, b in bands)

    def run(r, dests, signal, stream):
        p.multi(src, dests, bands[r], signal=signal, stream=stream)
    return Case(name, n, ref, float("nan"), _rows(bands), run)


def _ldr(h, w, seed):
    return torch.clamp(hdr(h, w, seed) / 4.0, 0.0, 1.0).contiguous()


EASU = [("2x", 23, 37, 46, 74), ("up", 41, 73, 54, 95), ("1:1", 45, 67, 45, 67), ("down", 64, 64, 40, 41)]
MODES = {"wrap": vq.VQ_ADDRESS_WRAP, "clamp": vq.VQ_ADDRESS_CLAMP}


def post_pass(ctx, kind, h, w):
    if kind == "tonemap":
        return Pass(ctx, "tonemap", params=synth.default_tonemapper()), hdr(h, w, 1)
    if kind == "cas":
        return Pass(ctx, "cas", con=vq.cas_setup(0.6, w, h, w, h)), _ldr(h, w, 2)
    if kind == "fsr_rcas":
        return Pass(ctx, "fsr_rcas", con=vq.fsr_rcas_con(0.2)), _ldr(h, w, 2)
    path, mode = kind.split()[1:]
    _, ih, iw, oh, ow = next(c for c in EASU if c[0] == path)
    return Pass(ctx, "fsr_easu", con=vq.fsr_easu_con(iw, ih, iw, ih, ow, oh), mode=MODES[mode], out_hw=(oh, ow)), _ldr(ih, iw, 3)


PASSES = ["tonemap", "cas", "fsr_rcas"] + [f"fsr_easu {c[0]} {m}" for c in EASU for m in MODES]


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("kind", PASSES)
def test_post_pass_world(ctx, pw, kind, n, order):
    p, src = post_pass(ctx, kind, 37, 61)
    run_world(pw, pass_case(p, src, n, f"{kind} n{n}"), SimWorld(n, order))


@pytest.mark.parametrize("kind", ["tonemap", "cas", "fsr_rcas"])
def test_post_pass_single_cta(ctx, pw, kind):
    """3 x 29 over 3 ranks: one-row bands, each a grid of one CTA (ranks 1 and 2 start inside the frame)"""
    p, src = post_pass(ctx, kind, 3, 29)
    run_world(pw, pass_case(p, src, 3, f"{kind} 3x29 n3"), SimWorld(3, "scrambled"))


# ---- post_retire: the fused kernels (post_fsr2x_kernel, post_fsr_up_kernel, post_cas_kernel, tonemap_kernel) -----------------
def fused_case(ctx, branch, n, ih, iw, oh, ow, name):
    src = hdr(ih, iw, 4)
    tm = synth.default_tonemapper()
    kw = dict(easu=None, rcas=None, cas=None, mode=vq.VQ_ADDRESS_WRAP)
    if branch.startswith("fsr"):
        kw["easu"], kw["rcas"] = fsr_consts(ih, iw, oh, ow)
    elif branch == "cas":
        kw["cas"] = vq.cas_setup(0.5, iw, ih, iw, ih)
    ref = chain(ctx, src, tm, (oh, ow), **kw)
    bands = equal_tiles(oh, n)
    assert all(b > a for a, b in bands)

    def run(r, dests, signal, stream):
        ctx.post_process_multi(tm, src, [vq.image_of(d) for d in dests], *bands[r], cas=kw["cas"], easu=kw["easu"], rcas=kw["rcas"],
                               address_mode=kw["mode"], signal=signal, stream=stream)
    return Case(name, n, ref, float("nan"), _rows(bands), run)


FUSED = [("fsr 2x", 35, 63, 70, 126), ("fsr up", 41, 73, 54, 95), ("cas", 37, 61, 37, 61), ("tonemap", 37, 61, 37, 61)]


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("branch,ih,iw,oh,ow", FUSED, ids=[c[0] for c in FUSED])
def test_post_process_world(ctx, pw, branch, ih, iw, oh, ow, n, order):
    run_world(pw, fused_case(ctx, branch, n, ih, iw, oh, ow, f"post_process {branch} n{n}"), SimWorld(n, order))


@pytest.mark.parametrize("branch,ih,iw,oh,ow", [("fsr 2x", 2160, 3840, 4320, 7680), ("fsr up", 1440, 2560, 2160, 3840)],
                         ids=["4K to 8K", "1440p to 4K"])
def test_post_process_large(ctx, pw, branch, ih, iw, oh, ow):
    run_world(pw, fused_case(ctx, branch, 2, ih, iw, oh, ow, f"post_process {branch} {ow}x{oh} n2"), SimWorld(2, "rotated"))


# ---- distributed.post_chain_rows: three passes, the signal on the last ------------------------------------------------------
@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("mode", ["wrap", "clamp"])
def test_post_chain_world(ctx, pw, mode, n, order):
    ih, iw = 270, 480
    oh, ow = 2 * ih, 2 * iw
    src, tm = hdr(ih, iw, 4), synth.default_tonemapper()
    fsr, rcas = fsr_consts(ih, iw, oh, ow)
    ref = reference_chain(ctx, src, tm, fsr, None, (oh, ow), MODES[mode], rcas)
    bands = equal_tiles(oh, n)

    def run(r, dests, signal, stream):
        plan = post_chain_rows(ih, oh, bands[r], fsr_con=fsr, address_mode=MODES[mode])
        t = torch.full((ih, iw, 4), float("nan"), device="cuda")
        e = torch.full((oh, ow, 4), float("nan"), device="cuda")
        stream.wait_stream(torch.cuda.current_stream())     # no device-wide synchronisation: the watcher may be waiting
        for rows in plan["tonemap"]:
            ctx.tonemap_multi(tm, src, [vq.image_of(t)], *rows, stream=stream)
        ctx.fsr_easu_multi(fsr, t, [vq.image_of(e)], *plan["fsr_easu"][0], address_mode=MODES[mode], stream=stream)
        ctx.fsr_rcas_multi(rcas, e, [vq.image_of(d) for d in dests], *plan["fsr_rcas"][0], signal=signal, stream=stream)
        stream.synchronize()       # the scratch frames are freed on return
    run_world(pw, Case(f"post chain {mode} n{n}", n, ref, float("nan"), _rows(bands), run), SimWorld(n, order))


# ---- the ticket ring and concurrent worlds ----------------------------------------------------------------------------------
@pytest.mark.parametrize("family", ["tonemap", "forward", "from_materials", "specular"])
def test_ticket_ring_wraps(ctx, family):
    """320 signalled calls of one retirement block in a row (post_retire, forward_kernel, psmain_kernel, the persistent prefilter),
    2 ranks on small frames: every slot of the ticket-pair ring comes back twice, and every call signals exactly its word. The
    tonemap bands are each followed by an HDRI min pyramid, whose SPD kernel takes vq_spd_ticket from the same counter."""
    f = None
    if family == "tonemap":
        case = pass_case(*post_pass(ctx, "tonemap", 37, 61), 2, "tonemap ring")
        _, _, keep, pyr = _pyr(ctx, vq, None, 64, 32)
    elif family == "specular":
        case = specular_case(ctx, 2, 8, 4, 64, lambda r: [(48 + r, 49 + r)], "specular ring")
    else:
        f, case = shading_case(ctx, family, 2, 100, 8, f"{family} ring")
    world = SimWorld(2, "rotated")
    frames = case.dests()
    for e in range(1, 161):
        world.preset(e)
        for r in range(2):
            case.run(r, rank_dests(world, frames, r), world.signal(r, e), None)
            if family == "tonemap":
                ctx.hdri_build_mips(pyr)
            world.ran(r, e)
            world.check(f"{family} ring epoch {e} rank {r}")
    _assert_frames(case, frames, case.expected(range(2)), "after the ring")
    if f is not None:
        f.close()


def test_two_worlds_in_flight(ctx):
    """two worlds, each with its own flags and frames, enqueued on two streams before any synchronisation: every call signals"""
    cases = [pass_case(*post_pass(ctx, "tonemap", 1080, 1920), 3, f"tonemap world {k}") for k in range(2)]
    worlds = [SimWorld(3, order) for order in ORDERS]
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    frames = [c.dests() for c in cases]
    for e in (1, 2, 3):
        for k in range(2):
            worlds[k].preset(e)
            for f in frames[k]:
                f.fill_(float("nan"))
        torch.cuda.synchronize()
        for r in range(3):
            for k in range(2):
                cases[k].run(r, rank_dests(worlds[k], frames[k], r), worlds[k].signal(r, e), streams[k])
                worlds[k].ran(r, e)
        for k in range(2):
            worlds[k].check(f"world {k} epoch {e}")
            _assert_frames(cases[k], frames[k], cases[k].expected(range(3)), f"world {k} epoch {e}")
