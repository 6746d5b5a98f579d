"""-m gpu: the direction of the in-kernel rendezvous that makes it a barrier. A signalled call must not finish while a peer's word in
its own flag array is stale, it must finish once every peer has arrived, and ranks running at the same time must release each other.

The flag arrays live in mapped, pinned host memory (tests/device_check/peer_hold.cu): the kernels reach them with the same
ld.acquire.sys / st.release.sys as peer memory, and a native keeper thread, which makes no CUDA call, plays the peers from the host.
Every wait is released by design. Each keeper run is told every epoch the calls it guards may wait on; if its calls have not
finished within its bound, it RESCUES them: it cycles every word through e and e + 1 for each of those epochs until they have (one
of the two satisfies an ==, >= or > test, signed or unsigned, of a wait at e), and it ends within 10 s, well inside the kernels'
20 s watchdog. So a correct library finishes every call, and a wrong one finishes it too and fails an assertion. Every test asserts
that no rescue happened (the 8-rank concurrent worlds print their count).

Part 1, held calls: each signalled entry point (the CPU test below keeps the table in step with the headers) in worlds of 2, 3 and 8
ranks, rotated and scrambled peer orders. The world runs once without a signal and once with every wait satisfied (so every kernel
is loaded before a call is held), then one rank at a time: its own row stale (e - 1), every word it must not read (its own word,
words n and above, the other rows) stale garbage. The keeper waits until the rank has stored e into every peer row and a watcher CTA
on a second stream has copied the rank's band, then releases the peers one at a time, in ascending or scrambled order, 20 ms apart.
A stamp kernel queued after the call records how many releases had begun when the call finished. Asserted: the call returned to the
host while its stream was still busy; the stamp reads n - 1; the watcher's copy, taken while the call was provably held, is the
single-GPU band; the flag words, frames and launch counts are those of test_rendezvous_gpu.run_world. For one cheap call of each
retirement block, the full table of stale (must hold) and ahead (must not hold: stamp 0) words, across the 2^32 wrap and at a
signed difference of -2^31; for each block, a grid of many CTA waves, where a flag raised before the last CTA's stores would show
in the watcher's copy; and distributed.EnvironmentStep with each of its two rendezvous held in turn.
Part 2, ranks release each other: all ranks of a world enqueued at once, each on its own non-blocking stream, flags stale, no
preset, the keeper only watching; one context per rank and one shared context; epochs across 2^32. Also EnvironmentStep over three
HDRIs in flight, each step's cubes snapshotted on the rank's stream. 8-rank worlds run in a child process with
CUDA_DEVICE_MAX_CONNECTIONS=32, so that 8 streams do not share hardware queues (a held kernel would block the rank queued behind it).
Part 3: two stream gates (tests/device_check/stream_gate.cu) opened in one host step release two 4096^2 HDRI pyramids (SPD, one
ticket word each) and two specular prefilters (a ticket pair each) on one context at once: every output is its serial bits.

Not tested here: NVLink peer stores and fence.sys ordering across devices (two or more GPUs), and the 20 s watchdog (a trap)."""
import ctypes as C
import json
import os
import random
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import vqengine_b200 as vq
from vqengine_b200 import distributed as vd
from test_env_multi_gpu import SENTINEL, _diffuse_ref, _twelve_calls, diffuse_case, lut_case
from test_frame_multi_gpu import _composite_case, _sky, _sky_case, _sky_frame
from test_ibl_gpu import _pyr
from test_rendezvous_gpu import ORDERS, _assert_frames, fused_case, pass_case, peer_order, post_pass, rank_dests, shading_case, \
    specular_case

gpu = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADERS = [os.path.join(ROOT, "include", h) for h in ("vqcuda.h", "vqcuda_prefilter_multi.h")]
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-lineinfo", "-O3", "-std=c++17", "--shared", "-Xcompiler", "-fPIC",
         "--expt-relaxed-constexpr"]
M = 0xFFFFFFFF
SLOTS = 16                         # peer_hold.cu PH_SLOTS
DWELL_US = 20_000                  # the keeper's pause before each release
BOUND_US = 2_000_000               # a keeper that waits longer than this rescues (peer_hold.cu's PH_BOUND_MAX_US)
WATCH_NS = 5_000_000_000           # the watcher gives up (and says so) after 5 s
# rank r's epoch in the held worlds: across 2^32 and at the signed half-way point
EPOCHS = (0xFFFFFFFF, 0, 1, 0x80000000, 0x7FFFFFFF, 0xFFFFFFFE, 0x12345678, 2)


# ---- the table: one row per signalled entry point ----------------------------------------------------------------------------------
def _shading(call):
    def build(ctx, n):
        f, case = shading_case(ctx, call, n, 257, 41, f"{call} n{n}")
        return case, f.close
    return build


def _post(kind):
    return lambda ctx, n: (pass_case(*post_pass(ctx, kind, 37, 61), n, f"{kind} n{n}"), None)


def _specular(ctx, n, res=32, mips=6):
    plan = vd.InterleavedSpecularPlan(res, mips, n)
    return specular_case(ctx, n, res, mips, 128, plan.row_ranges, f"specular n{n}"), None


def _skydome(ctx, n, w=257, h=41):
    f = _sky_frame(ctx, w, h)
    m, keep, pyr = _sky(w, h)
    case = _sky_case(ctx, f, "from_materials", n, m, pyr, f"sky n{n}")
    case.keep = keep
    return case, f.close


ENTRY = {
    "vq_forward_lighting_multi_signal": _shading("forward"),
    "vq_forward_lighting_shadowed_multi_signal": _shading("shadowed"),
    "vq_forward_lighting_from_materials_multi_signal": _shading("from_materials"),
    "vq_specular_prefilter_ranges": _specular,
    "vq_tonemap_multi_signal": _post("tonemap"),
    "vq_cas_multi_signal": _post("cas"),
    "vq_fsr_easu_multi_signal": _post("fsr_easu 2x wrap"),
    "vq_fsr_rcas_multi_signal": _post("fsr_rcas"),
    "vq_post_process_multi_signal": lambda ctx, n: (fused_case(ctx, "fsr 2x", n, 35, 63, 70, 126, f"post_process n{n}"), None),
    "vq_skydome_multi_signal": _skydome,
    "vq_apply_reflections_multi_signal": lambda ctx, n: (_composite_case(ctx, n, 131, 37, f"composite n{n}"), None),
    "vq_diffuse_irradiance_multi_signal":
        lambda ctx, n: (diffuse_case(ctx, n, 8, dict(n_phi=32, n_theta=8, src_mip=2), f"diffuse n{n}"), None),
    "vq_brdf_integration_lut_multi_signal": lambda ctx, n: (lut_case(ctx, n, 38, 29, 128, f"lut n{n}"), None),
}


def signal_entry_points():
    """every VQ_API function of the two headers with a VqPeerSignal parameter"""
    names = set()
    for h in HEADERS:
        text = re.sub(r"/\*.*?\*/", " ", open(h).read(), flags=re.S)
        for m in re.finditer(r"VQ_API\s+[\w\s\*]*?\b(vq_\w+)\s*\(([^;]*)\)\s*;", text):
            if re.search(r"\bVqPeerSignal\b", m.group(2)):
                names.add(m.group(1))
    return names


def test_every_signalled_entry_point_has_a_row():
    """CPU: the held-call table names every entry point of vqcuda.h and vqcuda_prefilter_multi.h that takes a VqPeerSignal"""
    want = signal_entry_points()
    assert {"vq_tonemap_multi_signal", "vq_specular_prefilter_ranges", "vq_diffuse_irradiance_multi_signal"} <= want, sorted(want)
    assert not sorted(want - set(ENTRY)), f"signalled entry points with no row: {sorted(want - set(ENTRY))}"
    assert not sorted(set(ENTRY) - want), f"rows for names that take no VqPeerSignal: {sorted(set(ENTRY) - want)}"


# ---- the library and a world's flag arrays ---------------------------------------------------------------------------------------
def build_lib(out):
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), *FLAGS, "-o", str(out),
                           os.path.join(ROOT, "tests", "device_check", "peer_hold.cu")])


def load_lib(path):
    lib = C.CDLL(str(path))
    vp, u32, i64 = C.c_void_p, C.c_uint32, C.c_longlong
    lib.ph_new.argtypes = [C.POINTER(vp)]
    for f in (lib.ph_free, lib.ph_reset):
        f.argtypes = [vp]
    for f in (lib.ph_host_flags, lib.ph_dev_flags, lib.ph_host_ctl):
        f.argtypes, f.restype = [vp], vp
    lib.ph_stamp.argtypes = [vp, vp, C.c_int]
    lib.ph_watch.argtypes = [vp, vp, C.c_int, C.c_int, u32, C.c_ulonglong, C.c_int, vp * 8, vp * 8, C.c_ulonglong * 8]
    lib.ph_keeper_start.argtypes = [vp, C.c_int, C.c_int, u32, u32, C.POINTER(C.c_int), C.c_int, C.c_int, C.c_int, i64, i64,
                                    C.POINTER(u32), C.c_int]
    lib.ph_keeper_join.argtypes = [vp, C.c_int]
    # load the module's kernels now: a first launch while a held call spins would wait for that call
    w = HoldWorld(lib, 2, "rotated")
    s = torch.cuda.Stream()
    w.flags[0, 1] = 3
    nul = (vp * 8)()
    assert lib.ph_watch(w.h, C.c_void_p(s.cuda_stream), 0, 1, 3, WATCH_NS, 0, nul, nul, (C.c_ulonglong * 8)()) == 0
    assert lib.ph_stamp(w.h, C.c_void_p(s.cuda_stream), 0) == 0
    torch.cuda.synchronize()
    assert w.ctl[2] == 1 and w.ctl[4 + SLOTS] == 1
    w.free()
    return lib


@pytest.fixture(scope="module")
def ph(tmp_path_factory):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    out = tmp_path_factory.mktemp("devicecheck") / "libpeerhold.so"
    build_lib(out)
    torch.cuda.init()
    lib = load_lib(out)
    lib.path = str(out)
    return lib


class HoldWorld:
    """n ranks' flag arrays in mapped host memory (row q = rank q's array, wider than n) and their VqPeerSignals"""

    def __init__(self, lib, n, order):
        self.lib, self.n = lib, n
        self.h = C.c_void_p()
        assert lib.ph_new(C.byref(self.h)) == 0
        rows, stride = lib.ph_rows(), lib.ph_stride()
        self.flags = np.ctypeslib.as_array((C.c_uint32 * (rows * stride)).from_address(lib.ph_host_flags(self.h))).reshape(rows, stride)
        self.ctl = np.ctypeslib.as_array((C.c_uint32 * (4 + 2 * SLOTS)).from_address(lib.ph_host_ctl(self.h)))
        base = lib.ph_dev_flags(self.h)
        self.peers = [peer_order(n, r, order) for r in range(n)]
        self.sig = []
        for r in range(n):
            s = vq.PeerSignal()
            for i, q in enumerate([r] + self.peers[r]):
                s.flags[i] = base + 4 * stride * q
            s.n_ranks, s.my_index = n, r
            self.sig.append(s)

    def signal(self, r, e):
        self.sig[r].epoch = e & M
        return self.sig[r]

    def rescues(self):
        return int(self.ctl[1])

    def stamp(self, slot):
        assert self.ctl[4 + SLOTS + slot] == 1, "the stamp never ran"
        return int(self.ctl[4 + slot])

    def free(self):
        assert self.lib.ph_free(self.h) == 0


def release_order(n, r, scrambled):
    """the peers of rank r by rank index, ascending or in a fixed scrambled order"""
    out = [j for j in range(n) if j != r]
    if scrambled:
        random.Random(7919 * n + r).shuffle(out)
    return out


def held(ph, w, r, e, stale, order, enqueue, stream, watch=None):
    """one held call: rank r's own row holds `stale` at every peer word, every other word stale garbage (e - 1); the keeper
    releases the peers in `order` (a list of rank indices) once the rank's stores and the watcher's copy are in. `enqueue()` queues the
    call on `stream`; watch = (src, dst, sizes, n) starts the watcher first. Checks the stamp, the flag words and that no rescue
    happened; returns whether the call was still running when it returned to the host."""
    e &= M
    n = w.n
    w.flags[:] = (e - 1) & M
    for j in range(n):
        if j != r:
            w.flags[r, j] = stale & M
    model = w.flags.copy()
    for q in range(n):
        if q != r:
            model[q, r] = e
    for j in order:
        model[r, j] = e
    rescues = w.rescues()
    assert ph.ph_reset(w.h) == 0
    if watch is not None:
        src, dst, sizes, k = watch
        assert ph.ph_watch(w.h, C.c_void_p(watch_stream(stream).cuda_stream), w.peers[r][0], r, e, WATCH_NS, k, src, dst,
                           sizes) == 0
    arr = (C.c_int * max(len(order), 1))(*order)
    assert ph.ph_keeper_start(w.h, n, r, e, e, arr, len(order), int(watch is not None), 1, DWELL_US, BOUND_US, _u32s([e]), 1) == 0
    stop = 1
    try:
        enqueue()
        assert ph.ph_stamp(w.h, C.c_void_p(stream.cuda_stream), 0) == 0
        pending = not stream.query()
        stop = 0
    finally:
        got = ph.ph_keeper_join(w.h, stop)
    torch.cuda.synchronize()
    assert got == rescues, f"rank {r} epoch {e:#x}: the keeper had to rescue the call"
    if watch is not None:
        assert w.ctl[2] == 1, f"rank {r} epoch {e:#x}: the watcher never saw the flag"
    assert w.stamp(0) == len(order), (f"rank {r} epoch {e:#x} stale {stale & M:#x}: the call finished after {w.stamp(0)} of "
                                      f"{len(order)} releases")
    assert np.array_equal(w.flags, model), ("flag words", w.flags[:n, :n].tolist(), "want", model[:n, :n].tolist())
    return pending


def _u32s(values):
    return (C.c_uint32 * len(values))(*[v & M for v in values])


def guarded(ph, w, epochs, streams, enqueue, strict=True):
    """enqueue() queues signalled calls on `streams`, whose rendezvous wait on `epochs` (every one of them), each stream then gets a
    stamp; the keeper only watches, and rescues the calls if they have not all finished within its bound. strict: assert that no
    rescue was needed."""
    before = w.rescues()
    assert ph.ph_reset(w.h) == 0
    assert ph.ph_keeper_start(w.h, w.n, -1, epochs[-1] & M, 0, None, 0, 0, len(streams), 0, BOUND_US, _u32s(epochs), len(epochs)) == 0
    stop = 1
    try:
        enqueue()
        for k, s in enumerate(streams):
            assert ph.ph_stamp(w.h, C.c_void_p(s.cuda_stream), k) == 0
        stop = 0
    finally:
        ph.ph_keeper_join(w.h, stop)
    torch.cuda.synchronize()
    assert not strict or w.rescues() == before, f"epochs {[hex(e & M) for e in epochs]}: the keeper had to rescue calls"


_WATCH_STREAMS = {}


def watch_stream(stream):
    """the watcher's stream for a call stream: another non-blocking stream, made once"""
    if stream.cuda_stream not in _WATCH_STREAMS:
        _WATCH_STREAMS[stream.cuda_stream] = torch.cuda.Stream()
    return _WATCH_STREAMS[stream.cuda_stream]


def warm_world(ph, case, w, frames, stream):
    """the world without a signal (-> each rank's launch count), then signalled with every wait satisfied before it starts"""
    launches = []
    for r in range(case.n):
        n0 = vq.launch_count()
        case.run(r, rank_dests(w, frames, r), None, stream)
        launches.append(vq.launch_count() - n0)
    _assert_frames(case, frames, case.expected(range(case.n)), "world without a signal")
    w.flags[:] = 8
    guarded(ph, w, [7], [stream], lambda: [case.run(r, rank_dests(w, frames, r), w.signal(r, 7), stream) for r in range(case.n)])
    _assert_frames(case, frames, case.expected(range(case.n)), "world with its waits satisfied")
    return launches


class Watch:
    """the watcher's ranges for each rank of a case: the bytes of every destination that rank writes, and snapshot buffers"""

    def __init__(self, case, frames, w):
        self.case, self.frames, self.w = case, frames, w
        self.spans = [case.span(r) for r in range(case.n)]
        self.snaps = [torch.empty(max(s for _, s in self.spans), dtype=torch.uint8, device="cuda") for _ in range(case.n)]

    def args(self, r):
        off, size = self.spans[r]
        dests = rank_dests(self.w, self.frames, r)
        src = (C.c_void_p * 8)(*[d.data_ptr() + off for d in dests])
        dst = (C.c_void_p * 8)(*[s.data_ptr() for s in self.snaps])
        return src, dst, (C.c_ulonglong * 8)(*([size] * self.case.n)), self.case.n

    def check(self, r, what):
        off, size = self.spans[r]
        for k, d in enumerate(rank_dests(self.w, self.frames, r)):
            band = d.view(torch.uint8).flatten()[off:off + size]
            assert torch.equal(self.snaps[k][:size], band), (self.case.name, what, f"destination {k}: the copy taken while the call was "
                                                                                  "held is not the final band")


def held_world(ph, case, order, pairs):
    """the world warmed, then rank by rank a held call per (epoch, stale word, release order) of pairs(r)"""
    n = case.n
    w = HoldWorld(ph, n, order)
    s = torch.cuda.Stream()
    frames = case.dests()
    torch.cuda.synchronize()           # the reference and the fills ran on the legacy stream, which s does not wait for
    try:
        launches = warm_world(ph, case, w, frames, s)
        watch = Watch(case, frames, w)
        for k, per_rank in enumerate(pairs):
            for f in frames:
                f.fill_(case.fill)
            torch.cuda.synchronize()
            for r in range(n):
                e, stale, rel = per_rank(r)
                what = f"epoch {e & M:#x} stale {stale & M:#x} rank {r} releases {rel}"
                dests = rank_dests(w, frames, r)
                n0 = vq.launch_count()
                pending = held(ph, w, r, e, stale, rel, lambda: case.run(r, dests, w.signal(r, e), s), s, watch.args(r))
                assert vq.launch_count() - n0 == launches[r], (case.name, what, "launches with and without the signal")
                if rel:
                    assert pending, (case.name, what, "the call's stream was complete before any peer was released")
                _assert_frames(case, dests, case.expected(range(r + 1)), f"{case.name} {what}")
                watch.check(r, what)
        assert w.rescues() == 0
    finally:
        torch.cuda.synchronize()
        w.free()


# ---- Part 1: every signalled call holds until its last peer arrives -------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("entry", sorted(ENTRY))
def test_call_holds_until_every_peer(ctx, ph, entry, n, order):
    """every rank held in turn, its peers released in ascending (even ranks) or scrambled (odd ranks) order"""
    case, close = ENTRY[entry](ctx, n)

    def per_rank(r):
        e = EPOCHS[r % len(EPOCHS)]
        return e, e - 1, release_order(n, r, scrambled=r % 2 == 1)
    held_world(ph, case, order, [per_rank])
    if close:
        close()


# (epoch, word in the rank's own row): a stale word holds the wait, a word that has reached or passed the epoch does not
E = 0x9E3779B9
HOLD = [(E, E - 1), (0, 0xFFFFFFFF), (1, 0xFFFFFFFF), (0x80000000, 0), (E, E - 0x7FFFFFFF), (E, E - 0x80000000)]
AHEAD = [(E, E + 1), (E, E + 0x7FFFFFFF)]
BLOCKS = {
    "forward_kernel": lambda ctx: _shading("forward")(ctx, 3),
    "psmain_kernel": lambda ctx: _shading("from_materials")(ctx, 3),
    "specular_persistent_kernel": lambda ctx: _specular(ctx, 3, 8, 4),
    "cta_retire PostDests": lambda ctx: _post("tonemap")(ctx, 3),
    "cta_retire K2": lambda ctx: (diffuse_case(ctx, 3, 4, dict(n_phi=8, n_theta=4, src_mip=1), "diffuse n3"), None),
    "cta_retire K4": lambda ctx: (lut_case(ctx, 3, 16, 6, 32, "lut n3"), None),
}


@gpu
@pytest.mark.parametrize("block", list(BLOCKS))
def test_stale_and_ahead_words(ctx, ph, block):
    """3 ranks, every rank: each stale word of HOLD must hold the call until both peers are released (ascending or descending);
    each word of AHEAD must let it finish with no release (stamp 0)"""
    case, close = BLOCKS[block](ctx)
    pairs = [(lambda e, v, k: lambda r: (e, v, release_order(3, r, False)[::1 if (k + r) % 2 == 0 else -1]))(e, v, k)
             for k, (e, v) in enumerate(HOLD)]
    pairs += [(lambda e, v: lambda r: (e, v, []))(e, v) for e, v in AHEAD]
    held_world(ph, case, "scrambled", pairs)
    if close:
        close()


LARGE = {
    "forward_kernel": lambda ctx: _shading_large(ctx, "forward"),
    "psmain_kernel": lambda ctx: _shading_large(ctx, "from_materials"),
    "specular_persistent_kernel":
        lambda ctx: (specular_case(ctx, 2, 64, 7, 512, vd.InterleavedSpecularPlan(64, 7, 2).row_ranges, "specular 64x7 n2"), None),
    "cta_retire PostDests": lambda ctx: (pass_case(*post_pass(ctx, "tonemap", 1080, 1920), 2, "tonemap 1920x1080 n2"), None),
    "cta_retire K2": lambda ctx: (diffuse_case(ctx, 2, 64, dict(step=0.010, src_mip=3), "diffuse 64 n2", hw=(256, 128)), None),
    "cta_retire K4": lambda ctx: (lut_case(ctx, 2, 1024, 1024, 256, "lut 1024 n2"), None),
}


def _shading_large(ctx, call):
    f, case = shading_case(ctx, call, 2, 1920, 1080, f"{call} 1920x1080 n2")
    return case, f.close


@gpu
@pytest.mark.parametrize("block", list(LARGE))
def test_flag_follows_every_store(ctx, ph, block):
    """grids of many CTA waves, 2 ranks held: a flag raised by an early CTA instead of the last one would show in the watcher's
    copy (taken, back to front, before the call is released) as rows the later waves had not stored yet"""
    case, close = LARGE[block](ctx)
    held_world(ph, case, "rotated", [lambda r: (0xFFFFFFFF, 0xFFFFFFFE, release_order(2, r, False))])
    if close:
        close()


def _env_refs(ctx, seed, dres=16, sres=32, mips=6, samples=128, kw=None):
    kw = kw or dict(n_phi=32, n_theta=8, src_mip=2)
    _, _, d, p = _pyr(ctx, vq, None, 256, 128, seed=seed)
    diff = _diffuse_ref(ctx, p, dres, kw)
    spec = torch.zeros((vq.cubemap_texel_count(sres, mips), 4), device="cuda")
    ctx.specular_prefilter(p, vq.cubemap_of(spec, sres, mips), samples)
    return dict(keep=d, pyr=p, diff=diff, blur=_twelve_calls(ctx, diff, dres), spec=spec)


def _phase_epoch(phase, e):
    """the epoch of EnvironmentStep's rendezvous in diffuse(e) and in finish(e)"""
    return e if phase == "diffuse" else e + 1


class EnvRanks:
    """every rank's diffuse, blurred and specular cubes and its EnvironmentStep (on its own context)"""
    DRES, SRES, MIPS, SAMPLES, KW = 16, 32, 6, 128, dict(n_phi=32, n_theta=8, src_mip=2)

    def __init__(self, ctxs, w, pyr):
        n = len(ctxs)
        self.n = n
        like_d = torch.empty((6 * self.DRES ** 2, 4), device="cuda")
        like_s = torch.empty((vq.cubemap_texel_count(self.SRES, self.MIPS), 4), device="cuda")
        self.diff = [torch.empty_like(like_d) for _ in range(n)]
        self.blur = [torch.empty_like(like_d) for _ in range(n)]
        self.spec = [torch.empty_like(like_s) for _ in range(n)]
        self.reset()
        self.steps = []
        for r in range(n):
            order = [r] + w.peers[r]
            self.steps.append(vd.EnvironmentStep(ctxs[r], pyr, [vq.cubemap_of(self.diff[q], self.DRES, 1) for q in order],
                                                 vq.cubemap_of(self.blur[r], self.DRES, 1),
                                                 [vq.cubemap_of(self.spec[q], self.SRES, self.MIPS) for q in order], r, n,
                                                 diffuse_params=self.KW, num_samples=self.SAMPLES))

    def reset(self):
        for t in self.diff + self.blur + self.spec:
            t.view(torch.int32).fill_(SENTINEL)

    def check(self, ref, what, blur=None, spec=None):
        torch.cuda.synchronize()
        for r in range(self.n):
            b = self.blur[r] if blur is None else blur[r]
            s = self.spec[r] if spec is None else spec[r]
            assert torch.equal(b.view(torch.int32), ref["blur"].view(torch.int32)), (what, "blurred", r)
            assert torch.equal(s.view(torch.int32), ref["spec"].view(torch.int32)), (what, "specular", r)
            if blur is None:
                assert torch.equal(self.diff[r].view(torch.int32), ref["diff"].view(torch.int32)), (what, "diffuse", r)


@gpu
@pytest.mark.parametrize("n", [2, 3])
def test_environment_step_held(ctx, ph, n):
    """every rank's diffuse rendezvous (epoch e) held, then every rank's specular rendezvous (e + 1), through 2^32"""
    ref = _env_refs(ctx, 2)
    w = HoldWorld(ph, n, "scrambled")
    env = EnvRanks([ctx] * n, w, ref["pyr"])
    s = torch.cuda.Stream()
    torch.cuda.synchronize()
    try:
        for st in env.steps:
            st.diffuse(0, None, s)
        for st in env.steps:
            st.finish(0, None, s)
        env.check(ref, "without a signal")
        for phase in ("diffuse", "finish"):     # every word reaches both epochs (7, 8) before each phase
            w.flags[:] = 10
            guarded(ph, w, [_phase_epoch(phase, 7)], [s], lambda: [getattr(st, phase)(7, w.sig[r], s) for r, st in enumerate(env.steps)])
        env.check(ref, "with every wait satisfied")
        e = 0xFFFFFFFF
        env.reset()
        torch.cuda.synchronize()
        for phase, e_p in (("diffuse", e), ("finish", e + 1)):
            for r, st in enumerate(env.steps):
                pending = held(ph, w, r, e_p, e_p - 1, release_order(n, r, scrambled=r % 2 == 1),
                               (lambda st=st, r=r: getattr(st, phase)(e, w.sig[r], s)), s)
                assert pending, (phase, r, "the call's stream was complete before any peer was released")
        env.check(ref, "held")
        assert w.rescues() == 0
    finally:
        torch.cuda.synchronize()
        w.free()


# ---- Part 2: ranks release each other ------------------------------------------------------------------------------------------------
# shadowed calls are left out: their PCF records are context scratch, one buffer per context, so two of them may not be in flight on
# one context (vqcuda.h)
CONCURRENT = ["vq_forward_lighting_multi_signal", "vq_forward_lighting_from_materials_multi_signal", "vq_specular_prefilter_ranges",
              "vq_tonemap_multi_signal", "vq_post_process_multi_signal", "vq_skydome_multi_signal", "vq_apply_reflections_multi_signal",
              "vq_diffuse_irradiance_multi_signal", "vq_brdf_integration_lut_multi_signal"]
CONCURRENT_EPOCHS = (0xFFFFFFFE, 0xFFFFFFFF, 0, 1)


def concurrent_world(ph, entry, n, shared, order="scrambled", epochs=CONCURRENT_EPOCHS, strict=True):
    """all n ranks of `entry` enqueued at once, each on its own non-blocking stream, on one context per rank or one shared one;
    every frame is checked, and (strict) that no call needed a rescue and every flag word holds the epoch; returns the rescues"""
    ctxs = [vq.Context(0) for _ in range(1 if shared else n)]
    built = [ENTRY[entry](c, n) for c in ctxs]
    cases = [built[0 if shared else r][0] for r in range(n)]
    case = cases[0]
    for c in cases[1:]:
        assert torch.equal(c.ref.view(torch.int32), case.ref.view(torch.int32)), "the contexts disagree on the single-GPU bits"
    w = HoldWorld(ph, n, order)
    streams = [torch.cuda.Stream() for _ in range(n)]
    frames = case.dests()
    torch.cuda.synchronize()           # the references and the fills ran on the legacy stream, which the rank streams do not wait for
    try:
        # every rank's context sized and its kernels loaded: without a signal, then signalled with every wait satisfied
        for r in range(n):
            cases[r].run(r, rank_dests(w, frames, r), None, streams[r])
        torch.cuda.synchronize()
        w.flags[:] = 8
        guarded(ph, w, [7], streams, lambda: [cases[r].run(r, rank_dests(w, frames, r), w.signal(r, 7), streams[r]) for r in range(n)])
        _assert_frames(case, frames, case.expected(range(n)), "warm-up")
        w.flags[:] = (epochs[0] - 1) & M                 # stale, and never preset again
        for e in epochs:
            for f in frames:
                f.fill_(case.fill)
            torch.cuda.synchronize()
            guarded(ph, w, [e], streams, lambda: [cases[r].run(r, rank_dests(w, frames, r), w.signal(r, e), streams[r]) for r in range(n)],
                    strict)
            _assert_frames(case, frames, case.expected(range(n)), f"{case.name} epoch {e:#x}")
            off = w.flags[:n, :n][~np.eye(n, dtype=bool)]
            assert not strict or bool((off == e).all()), (f"epoch {e:#x}", w.flags[:n, :n].tolist())
        return w.rescues()
    finally:
        torch.cuda.synchronize()
        w.free()
        for _, close in built:
            if close:
                close()
        for c in ctxs:
            c.close()


@gpu
@pytest.mark.parametrize("shared", [False, True], ids=["context per rank", "shared context"])
@pytest.mark.parametrize("n", [2, 3])
@pytest.mark.parametrize("entry", CONCURRENT)
def test_ranks_release_each_other(ph, entry, n, shared):
    concurrent_world(ph, entry, n, shared)


def concurrent_env(ph, n, shared, base=0xFFFFFFFC, seeds=(2, 3, 4), strict=True):
    """three EnvironmentSteps over three HDRIs in flight on every rank's stream, each step's blurred and specular cubes copied into
    snapshots on the rank's stream after finish(): each snapshot must be that step's single-GPU environment, and (strict) no call
    may need a rescue; returns the rescues"""
    ctxs = [vq.Context(0) for _ in range(1 if shared else n)]
    refs = [_env_refs(ctxs[0], s) for s in seeds]
    w = HoldWorld(ph, n, "scrambled")
    env = EnvRanks([ctxs[0 if shared else r] for r in range(n)], w, refs[0]["pyr"])
    streams = [torch.cuda.Stream() for _ in range(n)]
    snaps = [([torch.empty_like(b) for b in env.blur], [torch.empty_like(s) for s in env.spec]) for _ in seeds]
    torch.cuda.synchronize()
    try:
        for st, s in zip(env.steps, streams):
            st.diffuse(0, None, s)
        torch.cuda.synchronize()
        for st, s in zip(env.steps, streams):
            st.finish(0, None, s)
        env.check(refs[0], "without a signal")
        for phase in ("diffuse", "finish"):     # every word reaches both epochs (7, 8) before each phase
            w.flags[:] = 10
            guarded(ph, w, [_phase_epoch(phase, 7)], streams,
                    lambda: [getattr(st, phase)(7, w.sig[r], s) for r, (st, s) in enumerate(zip(env.steps, streams))])
        env.check(refs[0], "with every wait satisfied")
        env.reset()
        w.flags[:] = (base - 1) & M
        torch.cuda.synchronize()

        def enqueue():
            for k, ref in enumerate(refs):
                for r, (st, s) in enumerate(zip(env.steps, streams)):
                    st.hdri = ref["pyr"]
                    st.run((base + 2 * k) & M, w.sig[r], s)
                    with torch.cuda.stream(s):
                        snaps[k][0][r].copy_(env.blur[r])
                        snaps[k][1][r].copy_(env.spec[r])
        guarded(ph, w, [base + k for k in range(2 * len(seeds))], streams, enqueue, strict)
        for k, ref in enumerate(refs):
            env.check(ref, f"step {k}", blur=snaps[k][0], spec=snaps[k][1])
        return w.rescues()
    finally:
        torch.cuda.synchronize()
        w.free()
        for c in ctxs:
            c.close()


@gpu
@pytest.mark.parametrize("shared", [False, True], ids=["context per rank", "shared context"])
@pytest.mark.parametrize("n", [2, 3])
def test_environment_steps_release_each_other(ph, n, shared):
    concurrent_env(ph, n, shared)


def child_main(lib_path):
    """the 8-rank concurrent worlds, in a process of their own: one JSON line per world"""
    torch.cuda.init()
    lib = load_lib(lib_path)
    for entry in CONCURRENT:
        for shared in (False, True):
            print(json.dumps({"world": f"{entry} n8 {'shared' if shared else 'per rank'}",
                              "rescues": concurrent_world(lib, entry, 8, shared, strict=False)}), flush=True)
    for shared in (False, True):
        print(json.dumps({"world": f"EnvironmentStep n8 {'shared' if shared else 'per rank'}",
                          "rescues": concurrent_env(lib, 8, shared, strict=False)}), flush=True)


@gpu
def test_eight_ranks_release_each_other(ph):
    """8 ranks: every frame must be the single-GPU frame; the rescue count is printed (8 streams and the watcherless keeper)"""
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32",
               PYTHONPATH=os.pathsep.join([ROOT, os.path.join(ROOT, "tests"), os.environ.get("PYTHONPATH", "")]))
    code = f"import test_rendezvous_hold_gpu as t; t.child_main({ph.path!r})"
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
    worlds = [json.loads(line) for line in p.stdout.splitlines() if line.startswith("{")]
    assert len(worlds) == 2 * len(CONCURRENT) + 2
    for wd in worlds:
        print(f"8-rank world {wd['world']}: {wd['rescues']} rescues")
    print(f"8-rank worlds: {sum(wd['rescues'] for wd in worlds)} rescues in {len(worlds)} worlds")


# ---- Part 3: the ticket ring's single words and pairs under overlap -----------------------------------------------------------------
@gpu
def test_tickets_under_overlap(ctx, tmp_path):
    """two 4096^2 HDRI pyramids (the SPD kernel, one ticket word each) and two specular prefilters (the persistent kernel, a ticket
    pair each) held behind two gates on two streams, released in one host step: every output equals its serial bits"""
    out = tmp_path / "libstreamgate.so"
    subprocess.check_call([os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc"), *FLAGS, "-o", str(out),
                           os.path.join(ROOT, "tests", "device_check", "stream_gate.cu")])
    sg = C.CDLL(str(out))
    vp = C.c_void_p
    sg.sg_gate_new.argtypes = [C.POINTER(vp)]
    sg.sg_gate_free.argtypes = [vp]
    sg.sg_gate_words.argtypes, sg.sg_gate_words.restype = [vp], vp
    sg.sg_gate_close.argtypes = [vp, vp, C.c_ulonglong]
    size, levels = 4096, vq.mip_level_count(4096, 4096)
    n_tex = vq.pyramid_texel_count(size, size, levels)
    g = torch.Generator(device="cuda")
    pyrs, pyr_refs, specs, spec_refs, srcs = [], [], [], [], []
    for k in range(2):
        g.manual_seed(11 + k)
        d = torch.zeros((n_tex, 4), device="cuda")
        d[:size * size] = torch.rand((size * size, 4), generator=g, device="cuda") * 16.0
        p = vq.pyramid_of(d, size, size, levels)
        ctx.hdri_build_mips(p)
        pyrs.append((d, p))
        pyr_refs.append(d.clone())
        _, _, sd, sp = _pyr(ctx, vq, None, 256, 128, seed=5 + k)
        cube = torch.zeros((vq.cubemap_texel_count(32, 6), 4), device="cuda")
        ctx.specular_prefilter(sp, vq.cubemap_of(cube, 32, 6), 128)
        srcs.append((sd, sp))
        specs.append(torch.empty_like(cube))
        spec_refs.append(cube)
    gates = []
    for _ in range(2):
        h = vp()
        assert sg.sg_gate_new(C.byref(h)) == 0
        gates.append((h, (C.c_uint32 * 2).from_address(sg.sg_gate_words(h))))
    streams = [torch.cuda.Stream(), torch.cuda.Stream()]
    try:
        for k in range(2):
            pyrs[k][0][size * size:].view(torch.int32).fill_(SENTINEL)
            specs[k].view(torch.int32).fill_(SENTINEL)
        torch.cuda.synchronize()
        try:
            for k in range(2):
                assert sg.sg_gate_close(gates[k][0], C.c_void_p(streams[k].cuda_stream), 10_000_000_000) == 0
            for k in range(2):
                ctx.hdri_build_mips(pyrs[k][1], stream=streams[k])
                ctx.specular_prefilter(srcs[k][1], vq.cubemap_of(specs[k], 32, 6), 128, stream=streams[k])
        finally:
            for _, words in gates:          # both gates open in one host step
                words[0] = 1
        torch.cuda.synchronize()
        for k in range(2):
            assert gates[k][1][1] == 3, f"gate {k} was not opened by the host (status {gates[k][1][1]})"
            assert torch.equal(pyrs[k][0].view(torch.int32), pyr_refs[k].view(torch.int32)), f"pyramid {k} differs from its serial bits"
            assert torch.equal(specs[k].view(torch.int32), spec_refs[k].view(torch.int32)), f"specular cube {k} differs from its serial bits"
    finally:
        torch.cuda.synchronize()
        for h, _ in gates:
            sg.sg_gate_free(h)
