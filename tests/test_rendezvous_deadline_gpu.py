"""-m gpu: a signalled call whose peer does not come back (include/vqcuda_rendezvous.h). With a deadline registered on its context,
the call's rendezvous gives up at the deadline, or when the host cancels, records the failure in the context's status and ends
normally: the process, the context and the device stay usable, and the group can meet again (vq_group_barrier).

The worlds are test_rendezvous_hold_gpu's: flag arrays in mapped host memory (tests/device_check/peer_hold.cu) that the host sets,
with the peer_hold keeper in watch mode around every call. A wait that the library failed to end would be rescued within the keeper's
bound (2 s) instead of reaching a trap; every test asserts that no rescue happened. No wait here is unregistered: every context that
runs a signalled call or a barrier has a deadline of at most 100 ms (5 s where the peers are released or the host cancels).

For every signalled entry point, in worlds of 2, 3 and 8 ranks, rank 0 runs on a context of its own:
  1. missing peer: one peer's word stale at e - 1, across 2^32 and at a signed difference of -2^31. The stream goes idle at or after
     the 100 ms deadline and within 1 s; the status holds one failure at e with exactly that rank in the mask; the rank's epoch is in
     every peer's array and every destination holds the rank's single-GPU band; the device synchronises and an unsignalled call gives
     its normal bits;
  2. cancel: a 5 s deadline, the host cancels after about 100 ms: the call ends within 1 s with the cancelled bit set; after a clear
     the next step succeeds;
  3. a late peer does not satisfy a later epoch: after a timeout at e the peer arrives at e; the call at e + 1 still times out. Then
     every rank's vq_group_barrier at a fresh epoch (in the 8-rank world rank 0's, its peers' arrivals played by the host, since eight
     waiting kernels need eight hardware queues) meets, and the next step is the single-GPU band with a clear status. All eight
     ranks' barriers, and seven giving up on a missing eighth, run in a child process with CUDA_DEVICE_MAX_CONNECTIONS=32;
  4. peers in time: test_rendezvous_hold_gpu's held runs with a 5 s deadline registered hold until the last release, with the same
     stamps, frames, flag words and launch counts, and the status stays clear.
The C++ front end's recovery (vq::VQRendererGroup) is tested in test_rendezvous_group_gpu.py."""
import time

import pytest
import torch

import vqengine_b200 as vq
from test_rendezvous_gpu import _assert_frames, rank_dests
from test_rendezvous_hold_gpu import BOUND_US, ENTRY, M, EPOCHS, HoldWorld, guarded, held_world, ph, release_order, warm_world  # noqa: F401

gpu = pytest.mark.gpu
DEADLINE_NS = 100_000_000
LONG_NS = 5_000_000_000
STALE = [(0x9E3779B9, 0x9E3779B8), (0, 0xFFFFFFFF), (0x80000000, 0)]    # (epoch, stale word): e - 1, across 2^32, -2^31


@pytest.fixture(scope="module")
def rctx():
    """rank 0's context (the deadline changes per test, so not the session's shared context) and the peers' contexts of a group"""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    torch.cuda.init()
    c = vq.Context(0)
    peers = [vq.Context(0) for _ in range(7)]
    for p in peers:
        p.set_rendezvous_deadline(1_000_000_000)
    yield c, peers
    torch.cuda.synchronize()
    for x in [c] + peers:
        x.close()


def _status(c, s):
    st = c.rendezvous_status(s)
    return (st.failures, st.first_epoch, st.last_epoch, st.missing_mask, st.cancelled)


def _call(ph, c, w, case, frames, s, e, words, action=None):
    """rank 0's call at epoch e with word j of its own row = words[j] (every other word e - 1), under the keeper in watch mode;
    returns the call's time on its stream in ms"""
    e &= M
    w.flags[:] = (e - 1) & M
    for j, v in words.items():
        w.flags[0, j] = v & M
    for f in frames:
        f.fill_(case.fill)
    torch.cuda.synchronize()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    dests = rank_dests(w, frames, 0)

    def enqueue():
        ev[0].record(s)
        case.run(0, dests, w.signal(0, e), s)
        ev[1].record(s)
        if action:
            action()
    guarded(ph, w, [e], [s], enqueue)
    return ev[0].elapsed_time(ev[1])


def _check_band(case, w, frames, what):
    _assert_frames(case, rank_dests(w, frames, 0), case.expected([0]), what)


@gpu
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("entry", sorted(ENTRY))
def test_missing_peer_cancel_and_late_peer(rctx, ph, entry, n):
    c, peer_ctxs = rctx
    case, close = ENTRY[entry](c, n)
    w = HoldWorld(ph, n, "rotated")
    s = torch.cuda.Stream()
    frames = case.dests()
    m = n - 1                                               # the missing peer
    torch.cuda.synchronize()
    try:
        warm_world(ph, case, w, frames, s)
        c.set_rendezvous_deadline(DEADLINE_NS)
        c.clear_rendezvous_status(s)
        # 1. missing peer
        for e, stale in STALE:
            what = f"{case.name}: peer {m} stale {stale:#x} at epoch {e:#x}"
            ms = _call(ph, c, w, case, frames, s, e, {j: (stale if j == m else e) for j in range(1, n)})
            assert DEADLINE_NS / 1e6 * 0.99 <= ms < 1000.0, (what, f"the call took {ms:.1f} ms")
            assert _status(c, s) == (1, e, e, 1 << m, 0), (what, _status(c, s))
            assert all(int(w.flags[q, 0]) == e for q in range(1, n)), (what, "the rank's epoch in its peers' arrays", w.flags[:n, :n])
            _check_band(case, w, frames, what)
            torch.cuda.synchronize()                        # the device and the context are healthy
            for f in frames:
                f.fill_(case.fill)
            case.run(0, rank_dests(w, frames, 0), None, s)
            _check_band(case, w, frames, what + ", then unsignalled")
            c.clear_rendezvous_status(s)
            assert _status(c, s) == (0, 0, 0, 0, 0)
        # 2. cancel under a 5 s deadline
        c.set_rendezvous_deadline(LONG_NS)
        e = 0x40000000
        ms = _call(ph, c, w, case, frames, s, e, {j: (e - 1 if j == m else e) for j in range(1, n)},
                   action=lambda: (time.sleep(0.1), c.cancel_rendezvous()))
        assert ms < 1000.0, (case.name, f"a cancelled call took {ms:.1f} ms")
        assert _status(c, s) == (1, e, e, 1 << m, 1), (case.name, "cancel", _status(c, s))
        _check_band(case, w, frames, "cancelled")
        c.clear_rendezvous_status(s)
        _call(ph, c, w, case, frames, s, e + 1, {j: e + 1 for j in range(1, n)})
        assert _status(c, s) == (0, 0, 0, 0, 0), (case.name, "the step after a cancel and a clear", _status(c, s))
        _check_band(case, w, frames, "after the cancel")
        # 3. a late peer does not satisfy a later epoch; a barrier at a fresh epoch does
        c.set_rendezvous_deadline(DEADLINE_NS)
        e = 0xFFFFFFF0
        _call(ph, c, w, case, frames, s, e, {j: (e - 1 if j == m else e) for j in range(1, n)})
        assert _status(c, s)[0] == 1
        c.clear_rendezvous_status(s)
        e1 = (e + 1) & M
        _call(ph, c, w, case, frames, s, e1, {j: (e if j == m else e1) for j in range(1, n)})
        assert _status(c, s) == (1, e1, e1, 1 << m, 0), (case.name, "peer late at e, call at e + 1", _status(c, s))
        c.clear_rendezvous_status(s)
        torch.cuda.synchronize()
        f_ep = (e + 8) & M
        ctxs = [c] + peer_ctxs[:n - 1]
        base = ph.ph_dev_flags(w.h)
        g = vq.Group(ctxs, [base + 4 * ph.ph_stride() * q for q in range(n)])
        try:
            w.flags[:] = (f_ep - 1) & M
            ranks = range(n) if n <= 3 else [0]
            if n > 3:
                w.flags[0, 1:n] = f_ep
            streams = [s] + [torch.cuda.Stream() for _ in range(n - 1)]
            guarded(ph, w, [f_ep], [streams[r] for r in ranks], lambda: [g.barrier(r, f_ep, streams[r]) for r in ranks])
            for r in ranks:
                assert _status(ctxs[r], streams[r]) == (0, 0, 0, 0, 0), (case.name, f"the barrier of rank {r}")
                assert all(int(w.flags[q, r]) == f_ep for q in range(n) if q != r), (case.name, f"rank {r}'s barrier arrival")
        finally:
            g.close()
        e2 = (f_ep + 1) & M
        _call(ph, c, w, case, frames, s, e2, {j: e2 for j in range(1, n)})
        assert _status(c, s) == (0, 0, 0, 0, 0), (case.name, "the step after the barrier", _status(c, s))
        _check_band(case, w, frames, "after the barrier")
        assert w.rescues() == 0
    finally:
        torch.cuda.synchronize()
        w.free()
        if close:
            close()


@gpu
@pytest.mark.parametrize("n", [2, 3, 8])
@pytest.mark.parametrize("entry", sorted(ENTRY))
def test_peers_in_time_under_a_deadline(rctx, ph, entry, n):
    """the held runs of test_rendezvous_hold_gpu (every rank held in turn, its peers released 20 ms apart) with a 5 s deadline: the
    same stamps, frames, flag words and launch counts, and no failure recorded"""
    c, _ = rctx
    c.set_rendezvous_deadline(LONG_NS)
    s = torch.cuda.Stream()
    c.clear_rendezvous_status(s)
    case, close = ENTRY[entry](c, n)

    def per_rank(r):
        e = EPOCHS[r % len(EPOCHS)]
        return e, e - 1, release_order(n, r, scrambled=r % 2 == 1)
    try:
        held_world(ph, case, "scrambled", [per_rank])
        assert _status(c, s) == (0, 0, 0, 0, 0), (case.name, _status(c, s))
    finally:
        if close:
            close()


@gpu
def test_context_refusals_and_clear(rctx):
    """cancel before a registration is refused; a registration makes status and clear device calls; a refused deadline leaves the
    registered one"""
    c = vq.Context(0)
    try:
        with pytest.raises(vq.VqError, match="no rendezvous deadline"):
            c.cancel_rendezvous()
        assert _status(c, None) == (0, 0, 0, 0, 0)
        for ns in (0, vq.RENDEZVOUS_MAX_DEADLINE_NS + 1):
            with pytest.raises(vq.VqError, match="deadline"):
                c.set_rendezvous_deadline(ns)
        with pytest.raises(vq.VqError, match="no rendezvous deadline"):
            c.cancel_rendezvous()
        c.set_rendezvous_deadline(vq.RENDEZVOUS_MAX_DEADLINE_NS)
        c.cancel_rendezvous()                                # a host store: no failure is recorded without a waiting call
        assert _status(c, None) == (0, 0, 0, 0, 0)
        c.clear_rendezvous_status()
        assert _status(c, None) == (0, 0, 0, 0, 0)
    finally:
        torch.cuda.synchronize()
        c.close()


def barrier8_child(lib_path):
    """all eight ranks' barriers on eight streams, then seven with the eighth missing; one JSON line"""
    import json
    from test_rendezvous_hold_gpu import load_lib
    torch.cuda.init()
    lib = load_lib(lib_path)
    n = 8
    ctxs = [vq.Context(0) for _ in range(n)]
    for c in ctxs:
        c.set_rendezvous_deadline(DEADLINE_NS)
    w = HoldWorld(lib, n, "rotated")
    streams = [torch.cuda.Stream() for _ in range(n)]
    g = vq.Group(ctxs, [lib.ph_dev_flags(w.h) + 4 * lib.ph_stride() * q for q in range(n)])
    out = {}
    try:
        f = 0x7FFFFFF0
        w.flags[:] = f - 1
        guarded(lib, w, [f], streams, lambda: [g.barrier(r, f, streams[r]) for r in range(n)])
        out["all"] = [_status(ctxs[r], streams[r]) for r in range(n)]
        out["words"] = all(int(w.flags[q, r]) == f for r in range(n) for q in range(n) if q != r)
        f += 1
        w.flags[:] = f - 1
        guarded(lib, w, [f], streams[:n - 1], lambda: [g.barrier(r, f, streams[r]) for r in range(n - 1)])
        out["missing"] = [_status(ctxs[r], streams[r]) for r in range(n - 1)]
        out["f"] = f
        out["rescues"] = w.rescues()
    finally:
        torch.cuda.synchronize()
        g.close()
        w.free()
        for c in ctxs:
            c.close()
    print(json.dumps(out), flush=True)


@gpu
def test_eight_rank_barrier(ph):
    """vq_group_barrier with all eight ranks waiting on the GPU: they meet with clear records; with the eighth missing, the other
    seven give up at the deadline and name it. In a child process with CUDA_DEVICE_MAX_CONNECTIONS=32, so that eight waiting
    one-thread kernels do not share hardware queues"""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32",
               PYTHONPATH=os.pathsep.join([root, os.path.join(root, "tests"), os.environ.get("PYTHONPATH", "")]))
    code = f"import test_rendezvous_deadline_gpu as t; t.barrier8_child({ph.path!r})"
    p = subprocess.run([sys.executable, "-c", code], env=env, capture_output=True, text=True, timeout=600)
    assert p.returncode == 0, p.stdout[-3000:] + p.stderr[-6000:]
    out = json.loads([line for line in p.stdout.splitlines() if line.startswith("{")][-1])
    assert out["rescues"] == 0
    assert all(tuple(st) == (0, 0, 0, 0, 0) for st in out["all"]), out["all"]
    assert out["words"], "a rank's barrier did not store its epoch into every peer's array"
    f = out["f"]
    assert all(tuple(st) == (1, f, f, 1 << 7, 0) for st in out["missing"]), out["missing"]
