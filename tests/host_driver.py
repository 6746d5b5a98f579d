"""Builds and runs tests/host_check/renderer_driver.cpp: one scenario of the C++ host layer (vq::VQRenderer in libvqhost.so) per
run, every stage's output written as raw float32 or file bytes next to the scenario. Shared by test_host_renderer.py (CPU) and
test_host_renderer_gpu.py."""
import os
import shutil
import subprocess

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "vqengine_b200", "host")
SRC = os.path.join(ROOT, "tests", "host_check", "renderer_driver.cpp")

# the driver's exit codes (renderer_driver.cpp)
EXIT_NOT_REFUSED = 5
EXIT_INIT = 10


def available() -> bool:
    return bool(shutil.which("g++")) and os.path.exists(os.path.join(HOST, "libvqhost.so"))


def build(out_dir) -> str:
    exe = os.path.join(str(out_dir), "renderer_driver")
    cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
    lib = os.path.join(ROOT, "vqengine_b200")
    subprocess.check_call(["g++", "-std=c++17", "-O2", "-Wall", "-Wextra", "-Werror", SRC, "-I", HOST, "-I", os.path.join(cuda, "include"),
                           "-L", HOST, "-lvqhost", "-L", lib, "-lvqcuda", "-L", os.path.join(cuda, "lib64"), "-lcudart",
                           f"-Wl,-rpath,{HOST}", f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}", "-o", exe])
    return exe


def run(exe, work_dir, lines, rc=0, timeout=300):
    """writes the scenario into work_dir, runs it and returns its stdout lines; the exit code must be `rc`"""
    os.makedirs(str(work_dir), exist_ok=True)
    scen = os.path.join(str(work_dir), "scenario.txt")
    with open(scen, "w") as f:
        f.write("\n".join(lines) + "\n")
    r = subprocess.run([exe, scen], capture_output=True, text=True, timeout=timeout)
    assert r.returncode == rc, f"driver exit {r.returncode} (want {rc})\n{r.stdout}\n{r.stderr}"
    return r.stdout.splitlines()


def put(work_dir, name, arr) -> str:
    np.ascontiguousarray(arr, dtype=np.float32).tofile(os.path.join(str(work_dir), name))
    return name


def put_bytes(work_dir, name, data) -> str:
    with open(os.path.join(str(work_dir), name), "wb") as f:
        f.write(bytes(data))
    return name


def get(work_dir, name, shape=None, dtype=np.float32):
    a = np.fromfile(os.path.join(str(work_dir), name), dtype=dtype)
    return a.reshape(shape) if shape is not None else a


def get_bytes(work_dir, name) -> bytes:
    with open(os.path.join(str(work_dir), name), "rb") as f:
        return f.read()
