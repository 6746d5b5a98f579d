"""GPU-box helper: the C++ front end's device group (vq::VQRendererGroup) against the single vq::VQRenderer.

  python tools/perf_group.py [--frames 200] [--w 1920] [--h 1080] [--deadline-ns NS [--ranks 1,3]]

Builds a small timing program against libvqhost.so in a temporary directory and runs it. Workload: vq_headless_test's scene at the
given render size (a synthetic G-buffer, a 512x256 HDRI, a 64 diffuse / 128 specular cube), RenderSceneColor with the sky,
ApplyReflections and RenderPostProcess with FSR 2x, and PreFilterEnvironmentMap at the engine's step of 0.010. A frame's time comes from
CUDA events: `--frames` frames are enqueued back to back with no host wait, each rank's stream between its own start event (recorded
after the stream has waited for rank 0's) and its end event, and the slowest rank counts. The prefilter blocks like the engine's, so
it is the host clock around the call, which ends in a synchronise of every rank's stream. Each figure is given for `--repeats` runs
(min, median, max) so that the spread is visible. It reports:
  * a 1-rank group against VQRenderer (the group's own cost);
  * N = 2, 4, 8 ranks on device 0 (a simulated world: a cost figure, not a scaling figure);
  * with two or more GPUs, 1/2/4/8-rank strong scaling over real devices.
With --deadline-ns, each group of --ranks ranks on device 0 runs alternately without and with that rendezvous deadline registered
(vqcuda_rendezvous.h), --repeats times each, so that the cost of the policy in the wait loop shows against the run-to-run spread.
The card's name and power limit are read in the same run."""
import argparse, json, os, statistics, subprocess, sys, tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HOST = os.path.join(ROOT, "vqengine_b200", "host")

SRC = r'''
#include "vq_renderer.hpp"
#include <cuda_runtime_api.h>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>
using Clock = std::chrono::steady_clock;
static double ms(Clock::time_point a) { return std::chrono::duration<double, std::milli>(Clock::now() - a).count(); }
int main(int argc, char** argv) {
    const int frames = std::atoi(argv[1]), W = std::atoi(argv[2]), H = std::atoi(argv[3]);
    const unsigned long long deadline = std::strtoull(argv[4], nullptr, 10);     // 0: none registered
    std::vector<int> dev; for (int i = 5; i < argc; ++i) dev.push_back(std::atoi(argv[i]));
    const bool single = dev.empty();
    const int n = single ? 1 : (int)dev.size();
    vq::VQRenderer R; vq::VQRendererGroup G;
    if (single ? !R.Initialize(0) || !R.LoadDefaultResources()
               : !G.Initialize(dev) || (deadline && !G.SetRendezvousDeadline(deadline)) || !G.LoadDefaultResources()) return 2;
    const int EW = 512, EH = 256;
    std::vector<float> hdri((size_t)EW * EH * 4);
    for (size_t i = 0; i < hdri.size(); ++i) hdri[i] = 0.2f + 1.5f * std::fabs(std::sin(0.001f * (float)i));
    const vq::FEnvironmentMapDescriptor d{hdri.data(), EW, EH, 0.0f};
    std::vector<vq::FEnvironmentMapRenderingResources> envs(n);
    std::vector<vq::FEnvironmentMapRenderingResources*> ep;
    for (int r = 0; r < n; ++r) { if (!envs[r].CreateRenderingResources(single ? R : G.Rank(r), d, 64, 128)) return 3; ep.push_back(&envs[r]); }
    const std::vector<const vq::FEnvironmentMapRenderingResources*> ev(ep.begin(), ep.end());
    auto prefilter = [&] { return single ? R.PreFilterEnvironmentMap(envs[0], 0.010f) : G.PreFilterEnvironmentMap(ep, 0.010f); };
    if (!prefilter()) return 4;
    auto t0 = Clock::now();
    for (int i = 0; i < 5; ++i) prefilter();
    const double pre = ms(t0) / 5;
    std::vector<float> pos((size_t)W * H * 4), nrm(pos.size()), alb(pos.size());
    for (int y = 0; y < H; ++y) for (int x = 0; x < W; ++x) {
        const size_t o = ((size_t)y * W + x) * 4;
        pos[o] = -20.f + 40.f * x / W; pos[o + 1] = 0; pos[o + 2] = 20.f - 40.f * y / H; pos[o + 3] = 0.05f;
        nrm[o] = 0; nrm[o + 1] = y < H / 6 ? 0.f : 1.f; nrm[o + 2] = 0; nrm[o + 3] = 0.1f + 0.8f * (x % 7) / 7.f;
        alb[o] = 0.5f; alb[o + 1] = 0.4f; alb[o + 2] = 0.3f; alb[o + 3] = (x + y) % 5 == 0 ? 1.f : 0.f;
    }
    std::vector<vq::FTexture2D> gp(n), gn(n), ga(n), rf(n);
    std::vector<VqGBuffer> gb; std::vector<VqImage> refl;
    for (int r = 0; r < n; ++r) {
        cudaSetDevice(single ? 0 : G.Rank(r).Device());
        gp[r].Create(W, H); gn[r].Create(W, H); ga[r].Create(W, H); rf[r].Create(W, H);
        cudaMemcpy(gp[r].mem.ptr, pos.data(), pos.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(gn[r].mem.ptr, nrm.data(), nrm.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(ga[r].mem.ptr, alb.data(), alb.size() * 4, cudaMemcpyHostToDevice);
        cudaMemset(rf[r].mem.ptr, 0, (size_t)W * H * 16);
        gb.push_back(VqGBuffer{gp[r].View(), gn[r].View(), ga[r].View(), VqImage{}}); refl.push_back(rf[r].View());
    }
    vq::FPostProcessParameters pp;
    pp.SceneRTWidth = W; pp.SceneRTHeight = H; pp.DisplayResolutionWidth = 2 * W; pp.DisplayResolutionHeight = 2 * H;
    pp.FSR_EASUParams.UpdateEASUConstantBlock(W, H, W, H, 2 * W, 2 * H); pp.FSR_RCASParams.UpdateRCASConstantBlock();
    if (single ? !R.OnWindowSizeChanged(W, H, 2 * W, 2 * H) : !G.OnWindowSizeChanged(W, H, 2 * W, 2 * H)) return 5;
    vq::FSceneView view; view.cameraPosition = {0, 5, -17};
    view.GPULightingData.numPointLights = 4;
    for (int i = 0; i < 4; ++i) { auto& L = view.GPULightingData.point_lights[i]; L.position = {-15.f + 10.f * i, 9, -5}; L.range = 50; L.brightness = 500; L.color = {1, 1, 1}; }
    vq::FGraphicsSettings gfx;
    const float vp[16] = {1, 0, 0, 0, 0, 1.7f, 0, 0, 0, 0, 1, 1, 0, 0, -0.1f, 0};
    cudaStream_t s; cudaSetDevice(0); cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking);
    auto frame = [&](bool sync) {
        if (single) {
            R.RenderSceneColor(s, view, pp, gb[0], envs[0], gfx, false); R.RenderEnvironmentMap(s, vp, gb[0], envs[0]);
            R.ApplyReflections(s, refl[0]); R.RenderPostProcess(s, pp, false);
            if (sync) cudaStreamSynchronize(s);
        } else {
            G.RenderSceneColor(view, pp, gb, ev, gfx, false, vp); G.ApplyReflections(refl); G.RenderPostProcess(pp, false);
            for (int r = 0; sync && r < n; ++r) cudaStreamSynchronize(G.Stream(r));
        }
    };
    for (int i = 0; i < 20; ++i) frame(true);
    std::vector<cudaStream_t> streams;
    for (int r = 0; r < n; ++r) streams.push_back(single ? s : G.Stream(r));
    std::vector<cudaEvent_t> start(n), end(n);
    cudaEvent_t go;
    cudaSetDevice(single ? 0 : G.Rank(0).Device());
    cudaEventCreate(&go);
    cudaEventRecord(go, streams[0]);
    for (int r = 0; r < n; ++r) {
        cudaSetDevice(single ? 0 : G.Rank(r).Device());
        cudaEventCreate(&start[r]); cudaEventCreate(&end[r]);
        cudaStreamWaitEvent(streams[r], go, 0);
        cudaEventRecord(start[r], streams[r]);
    }
    for (int i = 0; i < frames; ++i) frame(false);
    float worst = 0.0f;
    for (int r = 0; r < n; ++r) {
        cudaSetDevice(single ? 0 : G.Rank(r).Device());
        cudaEventRecord(end[r], streams[r]);
        cudaEventSynchronize(end[r]);
        float t = 0.0f;
        cudaEventElapsedTime(&t, start[r], end[r]);
        worst = t > worst ? t : worst;
    }
    if (!single && !G.RendezvousOK()) return 6;
    std::printf("{\"ranks\": %d, \"single_renderer\": %s, \"deadline_ns\": %llu, \"frame_ms\": %.4f, \"prefilter_ms\": %.4f}\n", n,
                single ? "true" : "false", deadline, worst / frames, pre);
    cudaStreamDestroy(s);
    for (auto& e : envs) e.DestroyRenderingResources();
    return 0;
}
'''


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--w", type=int, default=1920)
    ap.add_argument("--h", type=int, default=1080)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--deadline-ns", type=int, default=0, help="compare groups without and with this rendezvous deadline")
    ap.add_argument("--ranks", default="1,3", help="with --deadline-ns: the group sizes on device 0")
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "perf_group.py needs a CUDA device"
    with tempfile.TemporaryDirectory() as tmp:
        src, exe = os.path.join(tmp, "perf_group.cpp"), os.path.join(tmp, "perf_group")
        open(src, "w").write(SRC)
        cuda = os.environ.get("CUDA_HOME", "/usr/local/cuda")
        lib = os.path.join(ROOT, "vqengine_b200")
        subprocess.check_call(["g++", "-std=c++17", "-O2", src, "-I", HOST, "-I", os.path.join(cuda, "include"), "-L", HOST, "-lvqhost",
                               "-L", lib, "-lvqcuda", "-L", os.path.join(cuda, "lib64"), "-lcudart", f"-Wl,-rpath,{HOST}",
                               f"-Wl,-rpath,{lib}", f"-Wl,-rpath,{os.path.join(cuda, 'lib64')}", "-o", exe])
        env = dict(os.environ, CUDA_DEVICE_MAX_CONNECTIONS="32")

        def once(devices, deadline=0):
            out = subprocess.run([exe, str(a.frames), str(a.w), str(a.h), str(deadline), *map(str, devices)], capture_output=True, text=True,
                                 env=env, timeout=1200)
            assert out.returncode == 0, out.stdout + out.stderr
            return json.loads(out.stdout.strip().splitlines()[-1])

        def summary(reps):
            spread = lambda k: [round(v, 4) for v in (min(x[k] for x in reps), statistics.median(x[k] for x in reps), max(x[k] for x in reps))]
            return {"ranks": reps[0]["ranks"], "single_renderer": reps[0]["single_renderer"], "deadline_ns": reps[0]["deadline_ns"],
                    "frame_ms_min_median_max": spread("frame_ms"), "prefilter_ms_min_median_max": spread("prefilter_ms")}

        def run(devices):
            return summary([once(devices) for _ in range(a.repeats)])

        card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True).stdout.strip().splitlines()
        if a.deadline_ns:
            res = {"card": card, "size": [a.w, a.h], "frames": a.frames, "deadline": []}
            for k in (int(x) for x in a.ranks.split(",")):
                without, with_ = [], []
                for _ in range(a.repeats):                  # alternated, so that both see the same drift of a shared host
                    without.append(once([0] * k))
                    with_.append(once([0] * k, a.deadline_ns))
                res["deadline"].append({"without": summary(without), "with": summary(with_)})
            print(json.dumps(res))
            return
        res = {"card": card, "size": [a.w, a.h], "frames": a.frames, "single": run([]), "one_device": [run([0] * k) for k in (1, 2, 4, 8)]}
        ngpu = torch.cuda.device_count()
        if ngpu >= 2:
            res["scaling"] = [run(list(range(k))) for k in (1, 2, 4, 8) if k <= ngpu]
        print(json.dumps(res))


if __name__ == "__main__":
    main()
