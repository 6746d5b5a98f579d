"""-m gpu: vq::VQRendererGroup when a rank does not come back in time (vqcuda_rendezvous.h), through
tests/host_check/rendezvous_group_driver.cpp, in simulated worlds of 2 and 3 ranks on device 0. With a 100 ms deadline registered, a
frame whose last rank's stream is held behind a gate ends on the other ranks within the deadlines, RendezvousOK() names the held rank,
every signalled method refuses until Resync(), and the next frame is the single VQRenderer's bits on every rank;
PreFilterEnvironmentMap with a held rank returns false and succeeds after Resync(). Every group method runs under the peer_hold keeper
in watch mode, and the driver requires zero rescues."""
import os
import subprocess

import pytest

import host_driver as hd
from test_group_gpu import inputs  # noqa: F401  (the group driver's input files)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def driver(tmp_path_factory):
    assert hd.available(), "host layer not built"
    exe = os.path.join(str(tmp_path_factory.mktemp("rendezvous_group_driver")), "rendezvous_group_driver")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "vqengine_b200")
    subprocess.check_call([os.path.join(cuda, "bin", "nvcc"), "-gencode", "arch=compute_90a,code=sm_90a", "-std=c++17", "-O2",
                           "-Xcompiler", "-Wall,-Wextra,-Werror", "-I", hd.HOST,
                           os.path.join(ROOT, "tests", "host_check", "rendezvous_group_driver.cpp"),
                           os.path.join(ROOT, "tests", "device_check", "peer_hold.cu"),
                           os.path.join(ROOT, "tests", "device_check", "stream_gate.cu"), "-L", hd.HOST, "-lvqhost", "-L", lib, "-lvqcuda",
                           "-Xlinker", f"-rpath,{hd.HOST}", "-Xlinker", f"-rpath,{lib}", "-o", exe])
    return exe


@pytest.mark.parametrize("n", [2, 3])
def test_group_recovers_from_a_missing_rank(driver, inputs, n):  # noqa: F811
    r = subprocess.run([driver, inputs, ",".join(["0"] * n)], capture_output=True, text=True, timeout=600)
    lines = r.stdout.splitlines()
    fails = [line for line in lines if line.startswith("FAIL")]
    assert r.returncode == 0 and not fails, f"exit {r.returncode}\n" + "\n".join(fails) + f"\n{r.stdout[-3000:]}\n{r.stderr[-3000:]}"
    assert lines and lines[-1] == "done 0 failures", lines[-5:]
    assert sum(line.startswith("ok ") for line in lines) == 16, lines
