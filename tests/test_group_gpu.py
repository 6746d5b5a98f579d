"""-m gpu: vq::VQRendererGroup (the C++ front end over a device group, include/vqcuda_group.h) against the single vq::VQRenderer, bit for
bit, through tests/host_check/group_driver.cpp.

Every group here is a simulated world on device 0: each rank has its own context, targets and stream, and the peer stores land in
the other ranks' buffers on the same GPU. The flag arrays live in tests/device_check/peer_hold.cu's mapped host memory, and every group
method runs under its keeper in watch mode: a rank that waits past the keeper's bound is rescued and counted, and the driver requires
zero rescues, so a wrong epoch or a missing arrival fails a check instead of reaching the kernels' 20 s trap. The driver checks:
  - rank orders and signals (flags[0] the rank's own array, the peers rotated, my_index = rank);
  - the LUT, the diffuse, blurred and specular cubes at steps 0.05 and 0.010, and the scene colour and display frame of every rank
    over the four scene-colour overloads x sky off / on x reflections off / on / with bounding volumes, at frame heights giving
    minimum (2-row), odd and even scene bands, through FSR 2x, FSR 1.5x, CAS and the tonemapper alone;
  - launches per rank: one per LUT, composite and post; shade 1 (2 for the shadowed G-buffer pass) + sky 1, and the one extra
    shade only on the first sky-less shadowed G-buffer frame at a size;
  - a larger size whose first sky-less shadowed frame runs no PCF test, then one that does: the records grow before the signalled
    call (rule 3 of DESIGN.md §6), with the launch counts that show it;
  - enqueue only: each steady frame method (RenderSceneColor* with and without the sky, ApplyReflections, RenderPostProcess) returns
    while a gate (tests/device_check/stream_gate.cu) holds every rank's stream, its outputs keep their previous bits until the gate
    opens, and then hold the single renderer's;
  - refusals: a size that empties a band and the Gaussian blur with no launch; one rank's invalid input returns false, every
    stream finishes and nothing is rescued; an environment the group did not register;
  - a long run of frames whose epochs cross 2^32 and reuse every slot of each context's ticket ring.
Peer stores across real devices and any multi-GPU timing are not covered by a one-GPU run; on a machine with more GPUs the same
driver takes a real device list (test_real_devices)."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

import host_driver as hd
from test_host_renderer_gpu import constant_materials, gbuffer_planes, lights_for, spot_hdri

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MAXW, MAXH, HW, HH = 96, 64, 64, 32
LONG_FRAMES = 200


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    assert hd.available(), "host layer not built"
    out = tmp_path_factory.mktemp("group_driver")
    exe = os.path.join(str(out), "group_driver")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "vqengine_b200")
    subprocess.check_call([os.path.join(cuda, "bin", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2",
                           "-Xcompiler", "-Wall,-Wextra,-Werror", "-I", hd.HOST, os.path.join(ROOT, "tests", "host_check", "group_driver.cpp"),
                           os.path.join(ROOT, "tests", "device_check", "peer_hold.cu"),
                           os.path.join(ROOT, "tests", "device_check", "stream_gate.cu"), "-L", hd.HOST, "-lvqhost", "-L", lib, "-lvqcuda",
                           "-Xlinker", f"-rpath,{hd.HOST}", "-Xlinker", f"-rpath,{lib}", "-o", exe])
    return exe


@pytest.fixture(scope="module")
def inputs(vq, tmp_path_factory):
    from vqengine_b200 import synth
    d = tmp_path_factory.mktemp("group_inputs")
    hd.put(d, "hdri.bin", spot_hdri(HW, HH))
    spec_mips = vq.mip_level_count(32, 32) - 1
    hd.put_bytes(d, "lights.bin", bytes(lights_for(vq, MAXW, MAXH, spec_mips)))
    hd.put_bytes(d, "lights_sh.bin", bytes(lights_for(vq, MAXW, MAXH, spec_mips, shadowing=True)))
    rng = np.random.default_rng(71)
    planes = gbuffer_planes(MAXW, MAXH, seed=72)
    planes[1][rng.uniform(0, 1, (MAXH, MAXW)) < 0.35, :3] = 0.0          # no surface there: the sky shows
    for i, p in enumerate(planes):
        hd.put(d, f"g{i}.bin", p)
    for i, p in enumerate(synth.surface_inputs(MAXW, MAXH, 3, seed=synth.SEED_BASE + 73, ssao=False)):
        hd.put(d, f"s{i}.bin", p)
    hd.put_bytes(d, "mats.bin", b"".join(bytes(m) for m in constant_materials(3)))
    hd.put(d, "dir.bin", rng.uniform(0.3, 0.7, (24, 16)))
    vp, _ = synth.sky_view_proj(0.8, -0.3, 1.1, MAXW / MAXH)
    hd.put(d, "vp.bin", vp)
    hd.put(d, "refl.bin", rng.uniform(0.0, 2.0, (MAXH, MAXW, 4)))
    hd.put(d, "bv.bin", rng.uniform(0.0, 1.0, (MAXH, MAXW, 4)))
    with open(os.path.join(str(d), "dims.txt"), "w") as f:
        f.write(f"{HW} {HH} {MAXW} {MAXH}\n")
    return str(d)


def _run(driver, inputs, devices, flags="mapped", long_frames=0, env=None, timeout=900):
    r = subprocess.run([driver, inputs, ",".join(map(str, devices)), flags, str(long_frames)], capture_output=True, text=True,
                       timeout=timeout, env=env)
    lines = r.stdout.splitlines()
    fails = [l for l in lines if l.startswith("FAIL")]
    assert r.returncode == 0 and not fails, f"exit {r.returncode}\n" + "\n".join(fails[:40]) + f"\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    assert lines and lines[-1] == "done 0 failures", lines[-5:]
    return lines


_guarded_passed = []


@pytest.mark.parametrize("n", [1, 2, 3])
def test_group_matches_single_renderer(driver, inputs, n):
    lines = _run(driver, inputs, [0] * n, long_frames=LONG_FRAMES if n == 2 else 0)
    assert sum(l.startswith("ok bits:") for l in lines) == 4 * 2 * 4 * 3 + 3 + 1
    assert sum(l.startswith("ok enqueue only:") for l in lines) == 4 * 3
    if n == 2:
        assert f"ok {LONG_FRAMES} frames keep the bits with no rescue" in lines and "ok the epoch wrapped past 2^32" in lines
    _guarded_passed.append(n)


def test_python_group(vq):
    """vqengine_b200.Group over three contexts on device 0: rank orders and signals as vqcuda_group.h states them"""
    ctxs = [vq.Context(0) for _ in range(3)]
    g = vq.Group(ctxs)
    try:
        own = [g.signal(r, 0).flags[0] for r in range(3)]
        assert all(own) and len(set(own)) == 3
        for r in range(3):
            order = g.rank_order(r)
            assert order == [(r + k) % 3 for k in range(3)] + [-1] * 5
            s = g.signal(r, 5)
            assert (s.n_ranks, s.my_index, s.epoch) == (3, r, 5)
            assert [s.flags[k] for k in range(3)] == [own[q] for q in order[:3]]
        with pytest.raises(vq.VqError):
            g.signal(3, 1)
        assert vq.lib.vq_group_arrive(g.h, 3, 1, None) == vq.VQ_ERR_INVALID_ARG
    finally:
        g.close()
        for c in ctxs:
            c.close()


def test_eight_ranks(driver, inputs):
    """8 streams need their own hardware queues: a signalled kernel that waits must not block the rank queued behind it"""
    _run(driver, inputs, [0] * 8, env=dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32"))
    _guarded_passed.append(8)


def test_group_owned_flags(driver, inputs):
    """flag_arrays == NULL: the group allocates zeroed device words. Run only once the guarded runs have passed, since nothing
    rescues a wait here"""
    if not {1, 2, 3, 8} <= set(_guarded_passed):
        pytest.skip("the guarded group runs did not all pass")
    _run(driver, inputs, [0, 0], flags="own")


def test_real_devices(driver, inputs):
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("one GPU: peer stores across devices are not exercised here")
    _run(driver, inputs, list(range(min(n, 8))), env=dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32"))


def _headless(args):
    exe = os.path.join(hd.HOST, "vq_headless_test")
    r = subprocess.run([exe, "-TestFrames=20", *args], capture_output=True, text=True, timeout=600,
                       env=dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32"))
    assert r.returncode == 0, f"{args}: exit {r.returncode}\n{r.stdout}\n{r.stderr}"
    return [l for l in r.stdout.splitlines() if l.startswith("frame ")]


def test_headless_group_smoke():
    """vq_headless_test -Devices=0,0 renders the smoke run's frames through a 2-rank group with the same per-frame means"""
    if not {2} <= set(_guarded_passed):
        pytest.skip("the guarded 2-rank run did not pass")
    single = _headless([])
    assert len(single) == 2
    assert _headless(["-Devices=0,0"]) == single
