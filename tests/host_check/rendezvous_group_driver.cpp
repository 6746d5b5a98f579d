// rendezvous_group_driver.cpp — the recovery of a vq::VQRendererGroup whose rank does not come back in time, for
// tests/test_rendezvous_group_gpu.py. Linked with tests/device_check/peer_hold.cu (the flag arrays in mapped host memory, and its
// keeper in watch mode around every group method, which rescues a wait past 2 s and counts it) and tests/device_check/stream_gate.cu
// (a gate holds the last rank's stream, so that its calls start late).
//
//   rendezvous_group_driver <dir> <devices, e.g. 0,0,0>
//
// <dir> holds test_group_gpu.py's inputs. With a 100 ms deadline registered on the group:
//   - a frame (sky, reflections, post: three phases) while the last rank's stream is gated: the other ranks' streams finish after
//     three deadlines and within 1.5 s, the keeper rescues nothing, and once the gate opens RendezvousOK() is false and names the held rank in every other rank's record;
//   - every signalled method refuses with no launch until Resync(), which succeeds; the next frame is the single VQRenderer's bits on
//     every rank;
//   - PreFilterEnvironmentMap with the last rank's stream behind a gate that opens by itself after 500 ms returns false; after
//     Resync() it succeeds with the single renderer's cubes, and so does the next frame.
// Every line of output is "ok ..." or "FAIL ..."; the exit code is the number of FAIL lines, 200 on bad input.
#include "vq_renderer.hpp"

#include <cuda_runtime_api.h>
#include <array>
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <functional>
#include <string>
#include <vector>

extern "C" {
int ph_new(void** out);
int ph_free(void* world);
int ph_stride();
void* ph_dev_flags(void* world);
int ph_reset(void* world);
int ph_stamp(void* world, void* stream, int slot);
int ph_keeper_start(void* world, int n, int rank, uint32_t epoch, uint32_t value, const int* order, int n_order, int wait_watch,
                    int n_stamps, long long dwell_us, long long bound_us, const uint32_t* rescue, int n_rescue);
int ph_keeper_join(void* world, int stop);
int sg_gate_new(void** out_gate);
int sg_gate_free(void* gate);
void* sg_gate_words(void* gate);
int sg_gate_close(void* gate, void* stream, unsigned long long bound_ns);
}

namespace {

int g_fails = 0;
std::string g_dir;

void Check(bool ok, const std::string& what) {
    std::printf("%s %s\n", ok ? "ok" : "FAIL", what.c_str());
    std::fflush(stdout);
    if (!ok) ++g_fails;
}

std::vector<char> ReadFile(const std::string& name) {
    std::ifstream f(g_dir + "/" + name, std::ios::binary);
    if (!f) { std::fprintf(stderr, "cannot read %s\n", name.c_str()); std::exit(200); }
    return std::vector<char>((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
}
std::vector<char> Download(const VqImage& im) {
    const size_t row = (size_t)im.width * 16;
    std::vector<char> h(row * im.height);
    cudaDeviceSynchronize();
    cudaMemcpy2D(h.data(), row, im.ptr, im.pitch_bytes, row, im.height, cudaMemcpyDeviceToHost);
    return h;
}
std::vector<char> DownloadBytes(const void* p, size_t n) {
    std::vector<char> h(n);
    cudaDeviceSynchronize();
    cudaMemcpy(h.data(), p, n, cudaMemcpyDeviceToHost);
    return h;
}
bool Same(const std::vector<char>& a, const std::vector<char>& b) { return a.size() == b.size() && !std::memcmp(a.data(), b.data(), a.size()); }
void Upload(vq::FTexture2D& t, const std::vector<char>& b, int w, int h) { t.Create(w, h); cudaMemcpy(t.mem.ptr, b.data(), b.size(), cudaMemcpyHostToDevice); }
double Ms(std::chrono::steady_clock::time_point a) { return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - a).count(); }

}  // namespace

int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: %s <dir> <devices>\n", argv[0]); return 200; }
    g_dir = argv[1];
    std::vector<int> devices;
    for (const char* p = argv[2]; *p;) { char* end; devices.push_back((int)std::strtol(p, &end, 10)); p = *end == ',' ? end + 1 : end; }
    const int n = (int)devices.size(), held = n - 1;
    int HW, HH, MAXW, MAXH;
    { std::ifstream d(g_dir + "/dims.txt"); d >> HW >> HH >> MAXW >> MAXH; }
    const std::vector<char> hdri = ReadFile("hdri.bin"), lights = ReadFile("lights.bin"), vpb = ReadFile("vp.bin"), refl = ReadFile("refl.bin");
    std::vector<char> g[4];
    for (int i = 0; i < 4; ++i) g[i] = ReadFile("g" + std::to_string(i) + ".bin");
    if (lights.size() != sizeof(VqSceneLighting) || vpb.size() != 64) return 200;
    const float* vp = (const float*)vpb.data();

    void* world = nullptr;
    if (ph_new(&world) != 0) return 200;
    std::vector<uint32_t*> flags;
    for (int q = 0; q < n; ++q) flags.push_back((uint32_t*)ph_dev_flags(world) + q * ph_stride());
    vq::VQRenderer R;
    vq::VQRendererGroup G;
    if (!R.Initialize(devices[0]) || !R.LoadDefaultResources() || !G.Initialize(devices, flags.data())) return 200;
    cudaStream_t rs;
    cudaStreamCreateWithFlags(&rs, cudaStreamNonBlocking);
    int rescues = 0;
    // one group method under the keeper in watch mode: every rank's stream is stamped after it; `between` runs before the stamps
    auto guarded = [&](const std::function<bool()>& method, const std::function<void()>& between = nullptr) {
        const uint32_t e = G.Epoch(), epochs[3] = {e, e + 1, e + 2};
        ph_reset(world);
        if (ph_keeper_start(world, n, -1, e + 2, 0, nullptr, 0, 0, n, 0, 2000000, epochs, 3) != 0) std::exit(200);
        const bool ok = method();
        if (between) between();
        for (int r = 0; r < n; ++r) ph_stamp(world, G.Stream(r), r);
        rescues += ph_keeper_join(world, 0);
        return ok;
    };

    Check(G.SetRendezvousDeadline(100000000ull), "SetRendezvousDeadline(100 ms)");
    Check(!G.SetRendezvousDeadline(0) && G.SetRendezvousDeadline(100000000ull), "a deadline of 0 is refused");
    Check(guarded([&] { return G.LoadDefaultResources(); }), "LoadDefaultResources");
    const vq::FEnvironmentMapDescriptor desc{(const float*)hdri.data(), HW, HH, 0.0f};
    vq::FEnvironmentMapRenderingResources env;
    std::vector<vq::FEnvironmentMapRenderingResources> envs(n);
    std::vector<vq::FEnvironmentMapRenderingResources*> envPtrs;
    if (!env.CreateRenderingResources(R, desc, 8, 32) || !R.PreFilterEnvironmentMap(env, 0.05f)) return 200;
    for (int r = 0; r < n; ++r) { if (!envs[r].CreateRenderingResources(G.Rank(r), desc, 8, 32)) return 200; envPtrs.push_back(&envs[r]); }
    const std::vector<const vq::FEnvironmentMapRenderingResources*> envViews(envPtrs.begin(), envPtrs.end());
    Check(guarded([&] { return G.PreFilterEnvironmentMap(envPtrs, 0.05f); }), "PreFilterEnvironmentMap");

    // inputs, window, the single renderer's frame
    const int W = MAXW, H = 6 * n;
    vq::FTexture2D sg[4], sr;
    cudaSetDevice(devices[0]);
    for (int i = 0; i < 4; ++i) Upload(sg[i], g[i], MAXW, MAXH);
    Upload(sr, refl, MAXW, MAXH);
    std::vector<std::array<vq::FTexture2D, 5>> rt(n);        // per rank: the G-buffer planes, then the reflection radiance
    for (int r = 0; r < n; ++r) {
        cudaSetDevice(G.Rank(r).Device());
        for (int i = 0; i < 4; ++i) Upload(rt[r][i], g[i], MAXW, MAXH);
        Upload(rt[r][4], refl, MAXW, MAXH);
    }
    auto sub = [&](const vq::FTexture2D& t) { return VqImage{t.mem.ptr, W, H, (size_t)t.width * 16}; };
    vq::FPostProcessParameters pp;
    pp.SceneRTWidth = W; pp.SceneRTHeight = H; pp.DisplayResolutionWidth = W; pp.DisplayResolutionHeight = H;
    pp.UpscalingAlgorithm = vq::FPostProcessParameters::NONE;
    vq::FSceneView view;
    std::memcpy(&view.GPULightingData, lights.data(), sizeof(VqSceneLighting));
    view.cameraPosition = {3.5f, 6.0f, -14.0f};
    vq::FGraphicsSettings gfx;
    if (!R.OnWindowSizeChanged(W, H, W, H) || !G.OnWindowSizeChanged(W, H, W, H)) return 200;
    const VqGBuffer sgb{sub(sg[0]), sub(sg[1]), sub(sg[2]), sub(sg[3])};
    if (!R.RenderSceneColor(rs, view, pp, sgb, env, gfx, false) || !R.RenderEnvironmentMap(rs, vp, sgb, env) ||
        !R.ApplyReflections(rs, sub(sr)))
        return 200;
    const VqImage* sdisp = R.RenderPostProcess(rs, pp, false);
    if (!sdisp) return 200;
    std::vector<char> refScene = Download(R.SceneColor().View()), refDisp = Download(*sdisp);
    std::vector<VqGBuffer> gbs;
    std::vector<VqImage> rfs;
    for (int r = 0; r < n; ++r) { gbs.push_back(VqGBuffer{sub(rt[r][0]), sub(rt[r][1]), sub(rt[r][2]), sub(rt[r][3])}); rfs.push_back(sub(rt[r][4])); }
    const VqImage* disp = nullptr;
    auto scene = [&] { return G.RenderSceneColor(view, pp, gbs, envViews, gfx, false, vp); };
    auto rest = [&] { return G.ApplyReflections(rfs) && (disp = G.RenderPostProcess(pp, false)) != nullptr; };
    auto frameBits = [&](const std::string& what) {
        bool ok = guarded(scene) && guarded(rest) && G.RendezvousOK();
        for (int r = 0; ok && r < n; ++r) ok = Same(Download(G.Rank(r).SceneColor().View()), refScene) && Same(Download(disp[r]), refDisp);
        Check(ok && rescues == 0, "the single renderer's bits on every rank: " + what);
    };
    frameBits("a frame with every rank in time");

    // ---- a frame with the last rank's stream gated: the other ranks give up at the deadline
    void* gate = nullptr;
    if (sg_gate_new(&gate) != 0) return 200;
    volatile uint32_t* gw = (volatile uint32_t*)sg_gate_words(gate);
    const uint32_t e0 = G.Epoch();
    sg_gate_close(gate, G.Stream(held), 10000000000ull);
    double othersMs = 0.0;
    const bool enq = guarded([&] {
        const auto t0 = std::chrono::steady_clock::now();
        const bool ok = scene() && rest();
        for (int r = 0; r < n; ++r)
            if (r != held) cudaStreamSynchronize(G.Stream(r));
        othersMs = Ms(t0);
        return ok;
    }, [&] { gw[0] = 1u; });
    Check(enq && othersMs >= 300.0 && othersMs < 1500.0 && rescues == 0,
          "gated frame: the other ranks finish after three deadlines (sky, composite, post), within 1.5 s (" + std::to_string(othersMs) +
          " ms), no rescue");
    const bool rok = G.RendezvousOK();
    const std::string why = vq::LastError();
    bool named = !rok;
    for (int r = 0; r < n; ++r) {
        VqRendezvousStatus st;
        vq_ctx_rendezvous_status(G.Rank(r).Context(), G.Stream(r), &st);
        const bool want = r == held ? st.failures == 0
                                    : st.failures == 3 && st.first_epoch == e0 && st.last_epoch == e0 + 2 && st.missing_mask == (1u << held) && !st.cancelled;
        named = named && want;
        if (r != held) named = named && why.find("rank " + std::to_string(r) + ":") != std::string::npos;
    }
    named = named && why.find("missing rank(s) " + std::to_string(held)) != std::string::npos;
    Check(named, "RendezvousOK() is false and names rank " + std::to_string(held) + ": " + why);
    uint64_t b = vq_launch_count();
    Check(!scene() && !G.ApplyReflections(rfs) && !G.RenderPostProcess(pp, false) && !G.LoadDefaultResources() &&
          vq_launch_count() == b, "every signalled method refuses, with no launch, until Resync()");
    Check(guarded([&] { return G.Resync(); }) && rescues == 0, "Resync()");
    frameBits("the frame after Resync()");

    // ---- PreFilterEnvironmentMap with the last rank's stream behind a gate that opens by itself after 500 ms
    sg_gate_close(gate, G.Stream(held), 500000000ull);
    const bool pre = guarded([&] { return G.PreFilterEnvironmentMap(envPtrs, 0.010f); });
    Check(!pre && gw[1] == 4u && rescues == 0, "PreFilterEnvironmentMap with a held rank returns false: " + std::string(vq::LastError()));
    b = vq_launch_count();
    Check(!scene() && vq_launch_count() == b, "a frame is refused after the failed prefilter");
    Check(guarded([&] { return G.Resync(); }) && rescues == 0, "Resync() after the prefilter");
    if (!R.PreFilterEnvironmentMap(env, 0.010f)) return 200;
    Check(guarded([&] { return G.PreFilterEnvironmentMap(envPtrs, 0.010f); }) && rescues == 0, "PreFilterEnvironmentMap after Resync()");
    const size_t specBytes = vq_cubemap_texel_count(32, env.SpecMips) * 16, diffBytes = vq_cubemap_texel_count(8, 1) * 16;
    const auto ds = DownloadBytes(env.Tex_IrradianceDiffBlurred.ptr, diffBytes), ss = DownloadBytes(env.Tex_IrradianceSpec.ptr, specBytes);
    bool cubes = true;
    for (int r = 0; r < n; ++r)
        cubes = cubes && Same(DownloadBytes(envs[r].Tex_IrradianceDiffBlurred.ptr, diffBytes), ds) && Same(DownloadBytes(envs[r].Tex_IrradianceSpec.ptr, specBytes), ss);
    Check(cubes, "the cubes after Resync() are the single renderer's on every rank");
    if (!R.RenderSceneColor(rs, view, pp, sgb, env, gfx, false) || !R.RenderEnvironmentMap(rs, vp, sgb, env) || !R.ApplyReflections(rs, sub(sr)) ||
        !(sdisp = R.RenderPostProcess(rs, pp, false)))
        return 200;
    refScene = Download(R.SceneColor().View());
    refDisp = Download(*sdisp);
    frameBits("the frame after the recovered prefilter");

    cudaStreamSynchronize(rs);
    cudaStreamDestroy(rs);
    G.Destroy();
    sg_gate_free(gate);
    ph_free(world);
    std::printf("done %d failures\n", g_fails);
    return g_fails > 100 ? 100 : g_fails;
}
