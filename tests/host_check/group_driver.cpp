// group_driver.cpp — runs the same frames through one vq::VQRenderer and through a vq::VQRendererGroup and holds every rank of the
// group to the single renderer's bits, for tests/test_group_gpu.py. Linked with tests/device_check/stream_gate.cu, whose gates hold
// the ranks' streams to show that the frame methods only enqueue, and with tests/device_check/peer_hold.cu: unless the group
// owns its flags, they live in peer_hold's mapped host memory, and every group method runs under its keeper in watch mode, which
// rescues a rank that waits longer than its bound (a wrong epoch fails a check here instead of reaching the kernels' 20 s trap).
//
//   group_driver <dir> <devices, e.g. 0,0,0> <mapped|own> <long-run frames>
//
// <dir> holds the inputs test_group_gpu.py writes (raw float32 unless noted): hdri.bin (HW x HH), lights.bin / lights_sh.bin
// (VqSceneLighting bytes), g0..g3.bin and refl.bin, bv.bin (MAXW x MAXH planes), s0..s2.bin (surface inputs, MAXW x MAXH),
// mats.bin (VqMaterialData bytes), dir.bin (16 x 24 directional shadow map), vp.bin (16 floats), dims.txt ("HW HH MAXW MAXH").
// Every line of output is "ok ..." or "FAIL ..."; the exit code is the number of FAIL lines (capped at 100), 200 on bad input.
#include "vq_renderer.hpp"

#include <cuda_runtime_api.h>
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
void* ph_host_flags(void* world);
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

struct Inputs {                     // one copy of every per-device input on one device
    vq::FTexture2D g[4], s[3], refl, bv;
    vq::FDeviceBuffer dir;
    VqMaterialTable* table = nullptr;
    VqContext* ctx = nullptr;
    ~Inputs() { if (table) vq_material_table_destroy(ctx, table); }
};

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
VqImage Sub(const vq::FTexture2D& t, int w, int h) { return VqImage{t.mem.ptr, w, h, (size_t)t.width * 16}; }

struct Run {
    int MAXW = 0, MAXH = 0, HW = 0, HH = 0;
    std::vector<char> hdri, lights, lightsSh, mats, vp;
    std::vector<char> g[4], s[3], refl, bv, dir;
    void* world = nullptr;
    int rescues = 0;

    void Load() {
        std::ifstream d(g_dir + "/dims.txt");
        d >> HW >> HH >> MAXW >> MAXH;
        hdri = ReadFile("hdri.bin"); lights = ReadFile("lights.bin"); lightsSh = ReadFile("lights_sh.bin");
        mats = ReadFile("mats.bin"); vp = ReadFile("vp.bin"); refl = ReadFile("refl.bin"); bv = ReadFile("bv.bin"); dir = ReadFile("dir.bin");
        for (int i = 0; i < 4; ++i) g[i] = ReadFile("g" + std::to_string(i) + ".bin");
        for (int i = 0; i < 3; ++i) s[i] = ReadFile("s" + std::to_string(i) + ".bin");
        if (lights.size() != sizeof(VqSceneLighting) || lightsSh.size() != sizeof(VqSceneLighting) || vp.size() != 64) std::exit(200);
    }
    void Upload(vq::FTexture2D& t, const std::vector<char>& b) { t.Create(MAXW, MAXH); cudaMemcpy(t.mem.ptr, b.data(), b.size(), cudaMemcpyHostToDevice); }
    void Make(Inputs& in, vq::VQRenderer& r) {
        cudaSetDevice(r.Device());
        for (int i = 0; i < 4; ++i) Upload(in.g[i], g[i]);
        for (int i = 0; i < 3; ++i) Upload(in.s[i], s[i]);
        Upload(in.refl, refl); Upload(in.bv, bv);
        in.dir.Alloc(dir.size());
        cudaMemcpy(in.dir.ptr, dir.data(), dir.size(), cudaMemcpyHostToDevice);
        const int n = (int)(mats.size() / sizeof(VqMaterialData));
        std::vector<VqMaterialTextures> tex(n);
        std::memset(tex.data(), 0, tex.size() * sizeof(VqMaterialTextures));
        in.ctx = r.Context();
        if (vq_material_table_create(r.Context(), (const VqMaterialData*)mats.data(), tex.data(), n, &in.table) != VQ_OK) std::exit(200);
    }

    // runs one group method under the keeper: every rank's stream is stamped after it, and the keeper rescues a wait past 2 s
    bool Guarded(vq::VQRendererGroup& G, const std::function<bool()>& method) {
        if (!world) return method();
        const uint32_t e = G.Epoch();
        const uint32_t epochs[2] = {e, e + 1};
        ph_reset(world);
        if (ph_keeper_start(world, G.NumRanks(), -1, e + 1, 0, nullptr, 0, 0, G.NumRanks(), 0, 2000000, epochs, 2) != 0) std::exit(200);
        const bool ok = method();
        for (int r = 0; r < G.NumRanks(); ++r) ph_stamp(world, G.Stream(r), r);
        rescues = ph_keeper_join(world, 0);
        return ok;
    }
};

bool Same(const std::vector<char>& a, const std::vector<char>& b) { return a.size() == b.size() && !std::memcmp(a.data(), b.data(), a.size()); }

}  // namespace

int main(int argc, char** argv) {
    if (argc != 5) { std::fprintf(stderr, "usage: %s <dir> <devices> <mapped|own> <long-run frames>\n", argv[0]); return 200; }
    g_dir = argv[1];
    std::vector<int> devices;
    for (const char* p = argv[2]; *p;) { char* end; devices.push_back((int)std::strtol(p, &end, 10)); p = *end == ',' ? end + 1 : end; }
    const bool mapped = std::string(argv[3]) == "mapped";
    const int longFrames = std::atoi(argv[4]);
    const int n = (int)devices.size();
    Run run;
    run.Load();

    vq::VQRenderer R;
    if (!R.Initialize(devices[0]) || !R.LoadDefaultResources()) return 200;
    cudaStream_t rs;
    cudaStreamCreateWithFlags(&rs, cudaStreamNonBlocking);

    std::vector<uint32_t*> flags;
    if (mapped) {
        if (ph_new(&run.world) != 0) return 200;
        for (int q = 0; q < n; ++q) flags.push_back((uint32_t*)ph_dev_flags(run.world) + q * ph_stride());
    }
    vq::VQRendererGroup G;
    if (!G.Initialize(devices, mapped ? flags.data() : nullptr)) return 200;
    {
        VqPeerSignal sig;
        int order[8];
        bool ok = true;
        for (int r = 0; r < n; ++r) {
            vq_group_signal(G.Group(), r, 7, &sig);
            vq_group_rank_order(G.Group(), r, order);
            ok = ok && sig.n_ranks == n && sig.my_index == r && sig.epoch == 7;
            for (int k = 0; k < 8; ++k) ok = ok && order[k] == (k < n ? (r + k) % n : -1);
            for (int k = 0; mapped && k < n; ++k) ok = ok && sig.flags[k] == flags[(r + k) % n];
        }
        Check(ok, "rank orders and signals");
    }

    // ---- LoadDefaultResources
    uint64_t before = vq_launch_count();
    Check(run.Guarded(G, [&] { return G.LoadDefaultResources(); }) && run.rescues == 0, "LoadDefaultResources, no rescue");
    Check(vq_launch_count() - before == (uint64_t)n, "LoadDefaultResources: one launch per rank");
    const std::vector<char> lut = DownloadBytes(R.BRDFIntegrationLUT().mem.ptr, 1024 * 1024 * 8);
    for (int r = 0; r < n; ++r) Check(Same(DownloadBytes(G.Rank(r).BRDFIntegrationLUT().mem.ptr, 1024 * 1024 * 8), lut), "LUT bits, rank " + std::to_string(r));

    // ---- environment and PreFilterEnvironmentMap
    const vq::FEnvironmentMapDescriptor desc{(const float*)run.hdri.data(), run.HW, run.HH, 0.0f};
    vq::FEnvironmentMapRenderingResources env;
    std::vector<vq::FEnvironmentMapRenderingResources> envs(n);
    std::vector<vq::FEnvironmentMapRenderingResources*> envPtrs;
    if (!env.CreateRenderingResources(R, desc, 8, 32)) return 200;
    for (int r = 0; r < n; ++r) { if (!envs[r].CreateRenderingResources(G.Rank(r), desc, 8, 32)) return 200; envPtrs.push_back(&envs[r]); }
    const std::vector<const vq::FEnvironmentMapRenderingResources*> envViews(envPtrs.begin(), envPtrs.end());
    const size_t diffBytes = vq_cubemap_texel_count(8, 1) * 16, specBytes = vq_cubemap_texel_count(32, env.SpecMips) * 16;
    for (float step : {0.05f, 0.010f}) {
        if (!R.PreFilterEnvironmentMap(env, step)) return 200;
        before = vq_launch_count();
        Check(run.Guarded(G, [&] { return G.PreFilterEnvironmentMap(envPtrs, step); }) && run.rescues == 0, "PreFilterEnvironmentMap " + std::to_string(step));
        Check(vq_launch_count() - before >= (uint64_t)(3 * n), "PreFilterEnvironmentMap: K2, blur and K3 on every rank");
        const auto d = DownloadBytes(env.Tex_IrradianceDiff.ptr, diffBytes), b = DownloadBytes(env.Tex_IrradianceDiffBlurred.ptr, diffBytes),
                   s = DownloadBytes(env.Tex_IrradianceSpec.ptr, specBytes);
        for (int r = 0; r < n; ++r) {
            const std::string tag = " step " + std::to_string(step) + ", rank " + std::to_string(r);
            Check(Same(DownloadBytes(envs[r].Tex_IrradianceDiff.ptr, diffBytes), d), "diffuse cube bits" + tag);
            Check(Same(DownloadBytes(envs[r].Tex_IrradianceDiffBlurred.ptr, diffBytes), b), "blurred diffuse cube bits" + tag);
            Check(Same(DownloadBytes(envs[r].Tex_IrradianceSpec.ptr, specBytes), s), "specular cube bits" + tag);
        }
    }

    // ---- per-rank inputs
    Inputs single;
    run.Make(single, R);
    std::vector<std::unique_ptr<Inputs>> rin;
    for (int r = 0; r < n; ++r) { rin.emplace_back(new Inputs()); run.Make(*rin.back(), G.Rank(r)); }

    vq::FSceneView view;
    std::memcpy(&view.GPULightingData, run.lights.data(), sizeof(VqSceneLighting));
    view.cameraPosition = {3.5f, 6.0f, -14.0f}; view.HDRIYawOffset = 0.7f;
    vq::FSceneView viewSh = view;
    std::memcpy(&viewSh.GPULightingData, run.lightsSh.data(), sizeof(VqSceneLighting));
    vq::FGraphicsSettings gfx;
    const float* vp = (const float*)run.vp.data();

    struct Window { int w, h, dw, dh; const char* mode; };
    const std::vector<Window> windows = {
        {run.MAXW, 2 * n, 2 * run.MAXW, 4 * n, "fsr"},                    // minimum bands: 2 rows each, FSR 2x
        {run.MAXW, 4 * n + 1, run.MAXW * 3 / 2, (4 * n + 1) * 3 / 2, "fsr"},   // an odd last band, FSR "Quality" (1.5x)
        {run.MAXW, 6 * n, run.MAXW, 6 * n, "cas"},                          // even bands, CAS
        {run.MAXW - 16, 6 * n + 2, run.MAXW - 16, 6 * n + 2, "tonemap"}};   // the tonemapper alone
    enum { kGB, kGBShadowed, kMat, kMatShadowed };
    const char* kinds[] = {"gbuffer", "gbuffer shadowed", "materials", "materials shadowed"};

    auto setPost = [&](vq::FPostProcessParameters& pp, const Window& win) {
        pp.SceneRTWidth = win.w; pp.SceneRTHeight = win.h; pp.DisplayResolutionWidth = win.dw; pp.DisplayResolutionHeight = win.dh;
        pp.UpscalingAlgorithm = std::string(win.mode) == "fsr" ? vq::FPostProcessParameters::FIDELITYFX_SUPER_RESOLUTION1 : vq::FPostProcessParameters::NONE;
        pp.bEnableCAS = std::string(win.mode) == "cas";
        pp.FFXCASParams.UpdateCASConstantBlock(win.w, win.h, win.w, win.h);
        pp.FSR_EASUParams.UpdateEASUConstantBlock(win.w, win.h, win.w, win.h, win.dw, win.dh);
        pp.FSR_RCASParams.UpdateRCASConstantBlock();
    };
    // one frame through both; returns false when the group refused a method
    // shadowLights = false: the shadowed overloads with the maps bound but no shadowing light (no PCF test runs)
    auto frame = [&](const Window& win, const vq::FPostProcessParameters& pp, int kind, bool sky, int reflMode, bool compare,
                     uint64_t* sceneLaunches, bool shadowLights = true) -> bool {
        const bool sh = kind == kGBShadowed || kind == kMatShadowed, gb = kind == kGB || kind == kGBShadowed;
        const vq::FSceneView& v = sh && shadowLights ? viewSh : view;
        auto gbOf = [&](Inputs& in) { return VqGBuffer{Sub(in.g[0], win.w, win.h), Sub(in.g[1], win.w, win.h), Sub(in.g[2], win.w, win.h), Sub(in.g[3], win.w, win.h)}; };
        auto siOf = [&](Inputs& in) { return VqSurfaceInputs{Sub(in.s[0], win.w, win.h), Sub(in.s[1], win.w, win.h), Sub(in.s[2], win.w, win.h), VqImage{}}; };
        auto smOf = [&](Inputs& in) { VqShadowMaps m{}; m.directional_map = in.dir.ptr; m.directional_width = 16; m.directional_height = 24; return m; };
        // the single renderer
        const VqImage* sdisp = nullptr;
        if (compare) {
            const VqGBuffer g = gbOf(single);
            const VqSurfaceInputs si = siOf(single);
            const VqShadowMaps m = smOf(single);
            bool ok = kind == kGB ? R.RenderSceneColor(rs, v, pp, g, env, gfx, false)
                    : kind == kGBShadowed ? R.RenderSceneColor(rs, v, pp, g, env, gfx, false, m)
                    : kind == kMat ? R.RenderSceneColorFromMaterials(rs, v, pp, si, single.table, env, gfx, false)
                                   : R.RenderSceneColorFromMaterials(rs, v, pp, si, single.table, env, gfx, false, m);
            VqGBuffer mask{};
            mask.normal_roughness = gb ? g.normal_roughness : si.normal_v;
            if (sky) ok = ok && R.RenderEnvironmentMap(rs, vp, mask, env);
            const VqImage rf = Sub(single.refl, win.w, win.h), bvv = Sub(single.bv, win.w, win.h);
            if (reflMode) ok = ok && R.ApplyReflections(rs, rf, reflMode == 2 ? &bvv : nullptr);
            if (!ok || !(sdisp = R.RenderPostProcess(rs, pp, false))) { Check(false, "single renderer refused a frame"); return false; }
        }
        std::vector<VqGBuffer> gbs; std::vector<VqSurfaceInputs> sis; std::vector<const VqMaterialTable*> tabs; std::vector<VqShadowMaps> sms;
        std::vector<VqImage> rfs, bvs;
        for (auto& in : rin) {
            gbs.push_back(gbOf(*in)); sis.push_back(siOf(*in)); tabs.push_back(in->table); sms.push_back(smOf(*in));
            rfs.push_back(Sub(in->refl, win.w, win.h)); bvs.push_back(Sub(in->bv, win.w, win.h));
        }
        const float* skyVP = sky ? vp : nullptr;
        const uint64_t b0 = vq_launch_count();
        bool ok = run.Guarded(G, [&] {
            return kind == kGB ? G.RenderSceneColor(v, pp, gbs, envViews, gfx, false, skyVP)
                 : kind == kGBShadowed ? G.RenderSceneColor(v, pp, gbs, envViews, gfx, false, sms, skyVP)
                 : kind == kMat ? G.RenderSceneColorFromMaterials(v, pp, sis, tabs, envViews, gfx, false, skyVP)
                                : G.RenderSceneColorFromMaterials(v, pp, sis, tabs, envViews, gfx, false, sms, skyVP);
        });
        if (sceneLaunches) *sceneLaunches = vq_launch_count() - b0;
        int rescues = run.rescues;
        uint64_t b1 = vq_launch_count();
        if (ok && reflMode) { ok = run.Guarded(G, [&] { return G.ApplyReflections(rfs, reflMode == 2 ? &bvs : nullptr); }); rescues += run.rescues; }
        const bool reflLaunches = !reflMode || vq_launch_count() - b1 == (uint64_t)n;
        b1 = vq_launch_count();
        const VqImage* disp = nullptr;
        if (ok) { run.Guarded(G, [&] { disp = G.RenderPostProcess(pp, false); return disp != nullptr; }); rescues += run.rescues; }
        const bool postLaunches = vq_launch_count() - b1 == (uint64_t)n;
        if (!ok || !disp) return false;
        if (compare) {
            const std::string tag = std::string(kinds[kind]) + (sky ? ", sky" : "") + (reflMode == 1 ? ", reflections" : reflMode == 2 ? ", reflections+volumes" : "") +
                                    ", " + std::to_string(win.w) + "x" + std::to_string(win.h) + " " + win.mode;
            const auto scene = Download(R.SceneColor().View());
            const auto display = Download(*sdisp);
            bool same = true;
            for (int r = 0; r < n; ++r) same = same && Same(Download(G.Rank(r).SceneColor().View()), scene) && Same(Download(disp[r]), display);
            Check(same, "bits: " + tag);
            Check(rescues == 0 && reflLaunches && postLaunches, "no rescue, one composite and one post launch per rank: " + tag);
        }
        return true;
    };

    for (const Window& win : windows) {
        vq::FPostProcessParameters pp;
        setPost(pp, win);
        cudaStreamSynchronize(rs);
        if (!R.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh) || !G.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh)) { Check(false, "window"); continue; }
        for (int kind = 0; kind < 4; ++kind)
            for (int sky = 0; sky < 2; ++sky)
                for (int refl = 0; refl < 3; ++refl) {
                    uint64_t launches = 0;
                    frame(win, pp, kind, sky, refl, true, &launches);
                    const uint64_t shade = kind == kGBShadowed ? 2 : 1;
                    const uint64_t expect = n * (shade + (sky ? 1 : 0) + (kind == kGBShadowed && !sky && refl == 0 ? shade : 0));
                    Check(launches == expect, "scene launches " + std::to_string(launches) + " == " + std::to_string(expect) + " (" + kinds[kind] +
                                              (sky ? ", sky" : "") + ", refl " + std::to_string(refl) + ")");
                }
    }

    // ---- rule 3 with a frame that runs no PCF test: at a new, larger size the first sky-less shadowed frame has no shadowing light
    // (the records are not grown), the next one has: the records must be grown before the signalled call, not inside it
    {
        const Window win{run.MAXW, run.MAXH, run.MAXW, run.MAXH, "tonemap"};
        vq::FPostProcessParameters pp;
        setPost(pp, win);
        cudaStreamSynchronize(rs);
        R.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        G.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        uint64_t launches = 0;
        Check(frame(win, pp, kGBShadowed, false, 0, true, &launches, false) && launches == (uint64_t)n,
              "a shadowed frame without a PCF test: one launch per rank, no pre-pass");
        Check(frame(win, pp, kGBShadowed, false, 0, true, &launches) && launches == (uint64_t)(4 * n),
              "the next frame with a test sizes its records first: the pre-pass and the shade, two launches each");
        Check(frame(win, pp, kGBShadowed, false, 0, true, &launches) && launches == (uint64_t)(2 * n), "then steady: two launches per rank");
    }

    // ---- enqueue only: each steady frame method returns while a gate holds every rank's stream, and its outputs keep their
    // previous bits until the gate opens (under the keeper: mapped flags only)
    if (mapped) {
        const Window& win = windows[2];
        vq::FPostProcessParameters pp;
        setPost(pp, win);
        cudaStreamSynchronize(rs);
        R.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        G.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        cudaStream_t snap;                                       // snapshots: a stream of its own, no device-wide wait
        cudaSetDevice(devices[0]);
        cudaStreamCreateWithFlags(&snap, cudaStreamNonBlocking);
        std::vector<void*> gates(n);
        for (auto& g : gates) if (sg_gate_new(&g) != 0) return 200;
        auto snapshot = [&](const VqImage& im) {
            const size_t row = (size_t)im.width * 16;
            std::vector<char> h(row * im.height);
            cudaMemcpy2DAsync(h.data(), row, im.ptr, im.pitch_bytes, row, im.height, cudaMemcpyDeviceToHost, snap);
            cudaStreamSynchronize(snap);
            return h;
        };
        // method() under closed gates; `images(r)` are rank r's outputs, `before` their bits until the gate opens, `after` the bits
        // they must hold once it has
        auto gated = [&](const std::string& what, const std::function<bool()>& method, const std::function<VqImage(int)>& images,
                         const std::vector<char>& before, const std::vector<char>& after) {
            const uint32_t e = G.Epoch(), epochs[2] = {e, e + 1};
            ph_reset(run.world);
            if (ph_keeper_start(run.world, n, -1, e, 0, nullptr, 0, 0, n, 0, 2000000, epochs, 2) != 0) std::exit(200);
            for (int r = 0; r < n; ++r) sg_gate_close(gates[r], G.Stream(r), 10000000000ull);
            const bool ok = method();
            bool held = true, kept = true;
            for (int r = 0; r < n; ++r) held = held && ((volatile uint32_t*)sg_gate_words(gates[r]))[1] <= 2u;   // armed or waiting
            for (int r = 0; r < n; ++r) kept = kept && Same(snapshot(images(r)), before);
            for (int r = 0; r < n; ++r) ((volatile uint32_t*)sg_gate_words(gates[r]))[0] = 1u;
            for (int r = 0; r < n; ++r) ph_stamp(run.world, G.Stream(r), r);
            const int rescues = ph_keeper_join(run.world, 0);
            bool opened = true, same = true;
            for (int r = 0; r < n; ++r) opened = opened && cudaStreamSynchronize(G.Stream(r)) == cudaSuccess && ((volatile uint32_t*)sg_gate_words(gates[r]))[1] == 3u;
            for (int r = 0; r < n; ++r) same = same && Same(Download(images(r)), after);
            Check(ok && held && kept && opened && same && rescues == 0, "enqueue only: " + what);
        };
        std::vector<VqGBuffer> gbs; std::vector<VqSurfaceInputs> sis; std::vector<const VqMaterialTable*> tabs; std::vector<VqShadowMaps> sms;
        std::vector<VqImage> rfs;
        for (auto& in : rin) {
            gbs.push_back(VqGBuffer{Sub(in->g[0], win.w, win.h), Sub(in->g[1], win.w, win.h), Sub(in->g[2], win.w, win.h), Sub(in->g[3], win.w, win.h)});
            sis.push_back(VqSurfaceInputs{Sub(in->s[0], win.w, win.h), Sub(in->s[1], win.w, win.h), Sub(in->s[2], win.w, win.h), VqImage{}});
            tabs.push_back(in->table);
            VqShadowMaps m{}; m.directional_map = in->dir.ptr; m.directional_width = 16; m.directional_height = 24; sms.push_back(m);
            rfs.push_back(Sub(in->refl, win.w, win.h));
        }
        const VqGBuffer sg{Sub(single.g[0], win.w, win.h), Sub(single.g[1], win.w, win.h), Sub(single.g[2], win.w, win.h), Sub(single.g[3], win.w, win.h)};
        const VqSurfaceInputs ssi{Sub(single.s[0], win.w, win.h), Sub(single.s[1], win.w, win.h), Sub(single.s[2], win.w, win.h), VqImage{}};
        VqShadowMaps ssm{}; ssm.directional_map = single.dir.ptr; ssm.directional_width = 16; ssm.directional_height = 24;
        const VqImage srf = Sub(single.refl, win.w, win.h);
        const char* names[] = {"RenderSceneColor, sky", "RenderSceneColor", "RenderSceneColor shadowed", "RenderSceneColorFromMaterials, sky"};
        for (int c = 0; c < 4; ++c) {
            const bool sky = c == 0 || c == 3;
            auto scene = [&](bool group) {
                if (!group) {
                    VqGBuffer mask{};
                    mask.normal_roughness = c == 3 ? ssi.normal_v : sg.normal_roughness;
                    bool ok = c == 3 ? R.RenderSceneColorFromMaterials(rs, view, pp, ssi, single.table, env, gfx, false)
                            : c == 2 ? R.RenderSceneColor(rs, viewSh, pp, sg, env, gfx, false, ssm) : R.RenderSceneColor(rs, view, pp, sg, env, gfx, false);
                    return ok && (!sky || R.RenderEnvironmentMap(rs, vp, mask, env));
                }
                const float* skyVP = sky ? vp : nullptr;
                return c == 3 ? G.RenderSceneColorFromMaterials(view, pp, sis, tabs, envViews, gfx, false, skyVP)
                     : c == 2 ? G.RenderSceneColor(viewSh, pp, gbs, envViews, gfx, false, sms, skyVP) : G.RenderSceneColor(view, pp, gbs, envViews, gfx, false, skyVP);
            };
            // ungated first: kernels loaded, records sized, display targets known; then the single renderer's bits
            const VqImage* disp = nullptr;
            if (!run.Guarded(G, [&] { return scene(true) && G.ApplyReflections(rfs) && (disp = G.RenderPostProcess(pp, false)) != nullptr; })) {
                Check(false, std::string("ungated frame: ") + names[c]); continue;
            }
            std::vector<VqImage> displays(disp, disp + n);
            if (!scene(false)) return 200;
            const auto refScene = Download(R.SceneColor().View());
            R.ApplyReflections(rs, srf);
            const auto refRefl = Download(R.SceneColor().View());
            const auto refDisp = Download(*R.RenderPostProcess(rs, pp, false));
            std::vector<char> sentinel(refScene.size(), (char)0xFF), sentinelDisp(refDisp.size(), (char)0xFF);
            for (int r = 0; r < n; ++r) {
                cudaMemset2D(G.Rank(r).SceneColor().mem.ptr, (size_t)win.w * 16, 0xFF, (size_t)win.w * 16, win.h);
                cudaMemset2D(displays[r].ptr, displays[r].pitch_bytes, 0xFF, (size_t)displays[r].width * 16, displays[r].height);
            }
            cudaDeviceSynchronize();
            auto sceneOf = [&](int r) { return G.Rank(r).SceneColor().View(); };
            gated(names[c], [&] { return scene(true); }, sceneOf, sentinel, refScene);
            gated(std::string("ApplyReflections after ") + names[c], [&] { return G.ApplyReflections(rfs); }, sceneOf, refScene, refRefl);
            gated(std::string("RenderPostProcess after ") + names[c], [&] { return G.RenderPostProcess(pp, false) != nullptr; },
                  [&](int r) { return displays[r]; }, sentinelDisp, refDisp);
        }
        for (auto g : gates) sg_gate_free(g);
        cudaStreamDestroy(snap);
    }

    // ---- refusals
    {
        const Window& win = windows[2];
        vq::FPostProcessParameters pp;
        setPost(pp, win);
        cudaStreamSynchronize(rs);
        R.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        G.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        uint64_t b = vq_launch_count();
        // 2n - 2 rows are n - 1 row pairs: one rank's even band is empty
        if (n > 1) Check(!G.OnWindowSizeChanged(win.w, 2 * n - 2, win.w, 2 * n - 2) && vq_launch_count() == b, "a size that empties a band is refused, no launch");
        vq::FPostProcessParameters blur = pp;
        blur.bEnableGaussianBlur = true;
        b = vq_launch_count();
        Check(!G.RenderPostProcess(blur, false) && vq_launch_count() == b, "the Gaussian blur is refused, no launch");
        // the last rank alone gets a G-buffer without a position plane: its call is refused after its peers' calls were enqueued
        std::vector<VqGBuffer> gbs;
        for (auto& in : rin) gbs.push_back(VqGBuffer{Sub(in->g[0], win.w, win.h), Sub(in->g[1], win.w, win.h), Sub(in->g[2], win.w, win.h), VqImage{}});
        gbs.back().position_ao.ptr = nullptr;
        const bool refused = !run.Guarded(G, [&] { return G.RenderSceneColor(view, pp, gbs, envViews, gfx, false, nullptr); });
        bool finished = true;
        for (int r = 0; r < n; ++r) finished = cudaStreamSynchronize(G.Stream(r)) == cudaSuccess && finished;
        Check(refused && finished && run.rescues == 0, "one rank's invalid input: refused, every stream finishes, no rescue");
        // an environment the group did not register
        std::vector<const vq::FEnvironmentMapRenderingResources*> other(envViews);
        other[0] = &env;
        gbs.back().position_ao.ptr = rin.back()->g[0].mem.ptr;
        b = vq_launch_count();
        Check(!G.RenderSceneColor(view, pp, gbs, other, gfx, false, nullptr) && vq_launch_count() == b, "an unregistered environment is refused, no launch");
        // the group goes on after the refusals
        Check(frame(win, pp, kGB, true, 1, true, nullptr), "a frame after the refusals");
    }

    // ---- a long run: every slot of the ticket rings, and the epoch across 2^32 (a second group whose flags hold FirstEpoch - 1)
    if (longFrames > 0 && mapped) {
        void* w2 = nullptr;
        if (ph_new(&w2) != 0) return 200;
        const uint32_t first = 0xFFFFFFFFu - 3u * (uint32_t)longFrames / 2u;
        uint32_t* host = (uint32_t*)ph_host_flags(w2);
        std::vector<uint32_t*> f2;
        for (int q = 0; q < n; ++q) {
            for (int k = 0; k < ph_stride(); ++k) host[q * ph_stride() + k] = first - 1u;
            f2.push_back((uint32_t*)ph_dev_flags(w2) + q * ph_stride());
        }
        vq::VQRendererGroup L;
        Run run2 = run;
        run2.world = w2;
        if (!L.Initialize(devices, f2.data(), first)) return 200;
        bool ok = run2.Guarded(L, [&] { return L.LoadDefaultResources(); });
        std::vector<vq::FEnvironmentMapRenderingResources> envs2(n);
        std::vector<vq::FEnvironmentMapRenderingResources*> p2;
        for (int r = 0; r < n; ++r) { envs2[r].CreateRenderingResources(L.Rank(r), desc, 8, 32); p2.push_back(&envs2[r]); }
        const std::vector<const vq::FEnvironmentMapRenderingResources*> v2(p2.begin(), p2.end());
        ok = ok && run2.Guarded(L, [&] { return L.PreFilterEnvironmentMap(p2, 0.010f); });
        const Window& win = windows[0];
        vq::FPostProcessParameters pp;
        setPost(pp, win);
        cudaStreamSynchronize(rs);
        R.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        ok = ok && L.OnWindowSizeChanged(win.w, win.h, win.dw, win.dh);
        std::vector<VqGBuffer> gbs; std::vector<VqImage> rfs;
        for (auto& in : rin) { gbs.push_back(VqGBuffer{Sub(in->g[0], win.w, win.h), Sub(in->g[1], win.w, win.h), Sub(in->g[2], win.w, win.h), Sub(in->g[3], win.w, win.h)});
                               rfs.push_back(Sub(in->refl, win.w, win.h)); }
        const VqGBuffer g{Sub(single.g[0], win.w, win.h), Sub(single.g[1], win.w, win.h), Sub(single.g[2], win.w, win.h), Sub(single.g[3], win.w, win.h)};
        R.RenderSceneColor(rs, view, pp, g, env, gfx, false);
        R.RenderEnvironmentMap(rs, vp, g, env);
        R.ApplyReflections(rs, Sub(single.refl, win.w, win.h));
        const auto display = Download(*R.RenderPostProcess(rs, pp, false));
        bool wrapped = false, same = ok;
        int rescues = 0;
        for (int f = 0; f < longFrames && same; ++f) {
            const VqImage* disp = nullptr;
            same = run2.Guarded(L, [&] { return L.RenderSceneColor(view, pp, gbs, v2, gfx, false, vp); }); rescues += run2.rescues;
            same = same && run2.Guarded(L, [&] { return L.ApplyReflections(rfs); }); rescues += run2.rescues;
            same = same && run2.Guarded(L, [&] { disp = L.RenderPostProcess(pp, false); return disp != nullptr; }); rescues += run2.rescues;
            for (int r = 0; same && r < n; ++r) same = Same(Download(disp[r]), display);
            wrapped = wrapped || L.Epoch() < first;
        }
        Check(same && rescues == 0, std::to_string(longFrames) + " frames keep the bits with no rescue");
        Check(wrapped, "the epoch wrapped past 2^32");
        L.Destroy();
        ph_free(w2);
    }

    cudaStreamSynchronize(rs);
    cudaStreamDestroy(rs);
    G.Destroy();
    if (run.world) ph_free(run.world);
    std::printf("done %d failures\n", g_fails);
    return g_fails > 100 ? 100 : g_fails;
}
