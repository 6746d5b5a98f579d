// renderer_driver.cpp — runs one scenario through the C++ host layer (vq::VQRenderer, libvqhost.so) and writes what every
// stage produced, so that tests/test_host_renderer_gpu.py can hold each stage to an independent reference.
//
//   renderer_driver <scenario.txt>
//
// The scenario is one command per line: a name, then key=value words ('#' starts a comment). File names are relative to the
// scenario's directory. Inputs are raw float32 RGBA images (row-major, no header) unless a command says otherwise; outputs are
// raw float32 (or the file image's bytes). Every command that renders works on one non-default stream created by `init`.
// A command given `expect=fail` must be refused: the driver prints "refused <command>: <LastError>" and goes on.
//
// Exit codes: 0 ok, 2 bad scenario, 3 bad input file, 4 output not written, 5 a step that had to be refused was not,
// 10 + the step below when the layer refuses it (its LastError() goes to stderr and stdout).
#include "vq_renderer.hpp"

#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

namespace {

enum Step {
    kInit = 10, kLut, kEnvTexels, kEnvHdr, kPrefilter, kWindow, kScene, kSceneMaterials, kSky, kReflect, kReflectPass, kPost,
    kSave, kHiRes, kSpd, kBlurPass, kHostHelpers
};

struct Abort { int code; };
using Args = std::map<std::string, std::string>;

std::string g_dir;

std::string Need(const Args& a, const char* k) {
    auto it = a.find(k);
    if (it == a.end()) { std::fprintf(stderr, "missing key %s\n", k); throw Abort{2}; }
    return it->second;
}
std::string Opt(const Args& a, const char* k, const char* def) { auto it = a.find(k); return it == a.end() ? def : it->second; }
int NeedInt(const Args& a, const char* k) { return std::atoi(Need(a, k).c_str()); }
float OptFloat(const Args& a, const char* k, float def) { auto it = a.find(k); return it == a.end() ? def : std::strtof(it->second.c_str(), nullptr); }
std::vector<std::string> Split(const std::string& s, char sep) {
    std::vector<std::string> out; std::string cur; std::istringstream in(s);
    while (std::getline(in, cur, sep)) out.push_back(cur);
    return out;
}
std::string Path(const std::string& f) { return f.empty() || f[0] == '/' ? f : g_dir + "/" + f; }

std::vector<char> ReadFile(const std::string& name, size_t expect = 0) {
    std::ifstream f(Path(name), std::ios::binary);
    if (!f) { std::fprintf(stderr, "cannot read %s\n", name.c_str()); throw Abort{3}; }
    std::vector<char> b((std::istreambuf_iterator<char>(f)), std::istreambuf_iterator<char>());
    if (expect && b.size() != expect) { std::fprintf(stderr, "%s: %zu bytes, expected %zu\n", name.c_str(), b.size(), expect); throw Abort{3}; }
    return b;
}
void WriteFile(const std::string& name, const void* p, size_t n) {
    std::ofstream f(Path(name), std::ios::binary);
    f.write((const char*)p, (std::streamsize)n);
    if (!f) { std::fprintf(stderr, "cannot write %s\n", name.c_str()); throw Abort{4}; }
}

struct Driver {
    vq::VQRenderer r;
    cudaStream_t stream = nullptr;
    vq::FEnvironmentMapRenderingResources env;
    vq::FPostProcessParameters pp;
    const VqImage* lastPost = nullptr;
    std::vector<vq::FTexture2D*> owned;            // inputs of the current frame (freed at exit)
    VqMaterialTable* table = nullptr;

    ~Driver() {
        if (stream) cudaStreamSynchronize(stream);
        if (table) vq_material_table_destroy(r.Context(), table);
        for (auto* t : owned) delete t;
        env.DestroyRenderingResources();
        if (stream) cudaStreamDestroy(stream);
        r.Destroy();
    }

    [[noreturn]] void Refused(int step, const char* what) {
        std::fprintf(stderr, "FAIL %s: %s\n", what, vq::LastError());
        std::printf("FAIL %s: %s\n", what, vq::LastError());
        throw Abort{step};
    }
    vq::FTexture2D* Upload(const std::string& file, int w, int h, int texelBytes = 16) {
        const std::vector<char> b = ReadFile(file, (size_t)w * h * texelBytes);
        auto* t = new vq::FTexture2D();
        owned.push_back(t);
        if (!t->Create(w, h, texelBytes) || cudaMemcpy(t->mem.ptr, b.data(), b.size(), cudaMemcpyHostToDevice) != cudaSuccess) throw Abort{3};
        return t;
    }
    void* UploadRaw(const std::string& file, size_t bytes) {
        const std::vector<char> b = ReadFile(file, bytes);
        auto* t = new vq::FTexture2D();
        owned.push_back(t);
        if (!t->mem.Alloc(bytes) || cudaMemcpy(t->mem.ptr, b.data(), bytes, cudaMemcpyHostToDevice) != cudaSuccess) throw Abort{3};
        return t->mem.ptr;
    }
    void Dump(const std::string& file, const void* dptr, size_t bytes) {
        if (stream && cudaStreamSynchronize(stream) != cudaSuccess) throw Abort{4};
        std::vector<char> h(bytes);
        if (bytes && cudaMemcpy(h.data(), dptr, bytes, cudaMemcpyDeviceToHost) != cudaSuccess) throw Abort{4};
        WriteFile(file, h.data(), bytes);
    }
    std::vector<char> Download(const VqImage& im) {
        if (stream && cudaStreamSynchronize(stream) != cudaSuccess) throw Abort{4};
        const size_t row = (size_t)im.width * 16;
        std::vector<char> h(row * im.height);
        if (!h.empty() && cudaMemcpy2D(h.data(), row, im.ptr, im.pitch_bytes, row, im.height, cudaMemcpyDeviceToHost) != cudaSuccess)
            throw Abort{4};
        return h;
    }
    void DumpImage(const std::string& file, const VqImage& im) { const std::vector<char> h = Download(im); WriteFile(file, h.data(), h.size()); }

    // FSceneView / FGraphicsSettings of a scene command: the lights as raw VqSceneLighting bytes, the other fields as words
    void SceneInputs(const Args& a, vq::FSceneView& view, vq::FGraphicsSettings& gfx, bool& bHDR, VqShadowMaps& maps, bool& shadowed) {
        const std::vector<char> L = ReadFile(Need(a, "lights"), sizeof(VqSceneLighting));
        std::memcpy(&view.GPULightingData, L.data(), sizeof(VqSceneLighting));
        const auto cam = Split(Opt(a, "cam", "0,0,0"), ',');
        if (cam.size() != 3) throw Abort{2};
        view.cameraPosition = {std::strtof(cam[0].c_str(), nullptr), std::strtof(cam[1].c_str(), nullptr), std::strtof(cam[2].c_str(), nullptr)};
        view.HDRIYawOffset = OptFloat(a, "yaw", 0.0f);
        view.sceneRenderOptions.fAmbientLightingFactor = OptFloat(a, "ambient", 0.055f);
        gfx.Reflections = Opt(a, "ssr", "0") == "1" ? vq::EReflections::SCREEN_SPACE_REFLECTIONS__FFX : vq::EReflections::REFLECTIONS_OFF;
        bHDR = Opt(a, "hdr", "0") == "1";
        std::memset(&maps, 0, sizeof(maps));
        shadowed = false;
        if (a.count("point")) {
            maps.point_res = NeedInt(a, "point_res");
            maps.point_cubes = UploadRaw(Need(a, "point"), (size_t)6 * maps.point_res * maps.point_res * 4);
            shadowed = true;
        }
        if (a.count("spot")) {
            maps.spot_width = NeedInt(a, "spot_w"); maps.spot_height = NeedInt(a, "spot_h");
            maps.spot_maps = UploadRaw(Need(a, "spot"), (size_t)NeedInt(a, "spot_n") * maps.spot_width * maps.spot_height * 4);
            shadowed = true;
        }
        if (a.count("dir")) {
            maps.directional_width = NeedInt(a, "dir_w"); maps.directional_height = NeedInt(a, "dir_h");
            maps.directional_map = UploadRaw(Need(a, "dir"), (size_t)maps.directional_width * maps.directional_height * 4);
            shadowed = true;
        }
    }

    // returns false when the layer refused the step
    bool Run(const std::string& cmd, const Args& a) {
        if (cmd == "init") {
            if (!r.Initialize(std::atoi(Opt(a, "device", "0").c_str()))) return false;
            if (cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking) != cudaSuccess) { stream = nullptr; return false; }
            return true;
        }
        if (cmd == "lut") {                                                    // LoadDefaultResources
            if (!r.LoadDefaultResources()) return false;
            const vq::FTexture2D& t = r.BRDFIntegrationLUT();
            std::printf("lut %d %d %d\n", t.width, t.height, t.texelBytes);
            Dump(Need(a, "out"), t.mem.ptr, (size_t)t.width * t.height * t.texelBytes);
            return true;
        }
        if (cmd == "env_texels" || cmd == "env_hdr") {
            bool ok;
            if (cmd == "env_texels") {
                const int w = NeedInt(a, "w"), h = NeedInt(a, "h");
                const std::vector<char> b = ReadFile(Need(a, "file"), (size_t)w * h * 16);
                const vq::FEnvironmentMapDescriptor d{(const float*)b.data(), w, h, OptFloat(a, "maxcll", 0.0f)};
                ok = env.CreateRenderingResources(r, d, NeedInt(a, "diff"), NeedInt(a, "spec"));
            } else {
                const std::vector<char> b = ReadFile(Need(a, "file"));
                ok = env.CreateRenderingResourcesFromHDRFile(r, b.data(), b.size(), NeedInt(a, "diff"), NeedInt(a, "spec"));
            }
            if (!ok) return false;
            std::printf("env %d %d %d %d %d %d %d\n", env.HDRIWidth, env.HDRIHeight, env.HDRIMips, env.DiffuseRes, env.SpecRes, env.SpecMips,
                        env.MaxContentLightLevel);
            if (cudaDeviceSynchronize() != cudaSuccess) return false;
            Dump(Need(a, "out"), env.Tex_HDREnvironment.ptr, vq_pyramid_texel_count(env.HDRIWidth, env.HDRIHeight, env.HDRIMips) * 16);
            return true;
        }
        if (cmd == "prefilter") {                                              // PreFilterEnvironmentMap
            if (!r.PreFilterEnvironmentMap(env, OptFloat(a, "step", 0.010f))) return false;
            const size_t diff = vq_cubemap_texel_count(env.DiffuseRes, 1) * 16;
            Dump(Need(a, "diff"), env.Tex_IrradianceDiff.ptr, diff);
            Dump(Need(a, "blurred"), env.Tex_IrradianceDiffBlurred.ptr, diff);
            Dump(Need(a, "spec"), env.Tex_IrradianceSpec.ptr, vq_cubemap_texel_count(env.SpecRes, env.SpecMips) * 16);
            return true;
        }
        if (cmd == "window") {                                                 // OnWindowSizeChanged + the frame's PPParams
            const int w = NeedInt(a, "w"), h = NeedInt(a, "h"), dw = NeedInt(a, "dw"), dh = NeedInt(a, "dh");
            if (stream) cudaStreamSynchronize(stream);
            if (!r.OnWindowSizeChanged(w, h, dw, dh)) return false;
            pp.SceneRTWidth = w; pp.SceneRTHeight = h; pp.DisplayResolutionWidth = dw; pp.DisplayResolutionHeight = dh;
            return true;
        }
        if (cmd == "scene" || cmd == "scene_materials") {
            vq::FSceneView view; vq::FGraphicsSettings gfx; bool bHDR, shadowed; VqShadowMaps maps;
            SceneInputs(a, view, gfx, bHDR, maps, shadowed);
            const int w = pp.SceneRTWidth, h = pp.SceneRTHeight;
            bool ok;
            if (cmd == "scene") {
                const auto f = Split(Need(a, "planes"), ',');
                if (f.size() < 3 || f.size() > 4) throw Abort{2};
                VqGBuffer gb{Upload(f[0], w, h)->View(), Upload(f[1], w, h)->View(), Upload(f[2], w, h)->View(), VqImage{nullptr, 0, 0, 0}};
                if (f.size() == 4) gb.emissive = Upload(f[3], w, h)->View();
                ok = shadowed ? r.RenderSceneColor(stream, view, pp, gb, env, gfx, bHDR, maps) : r.RenderSceneColor(stream, view, pp, gb, env, gfx, bHDR);
            } else {
                const auto f = Split(Need(a, "surface"), ',');
                if (f.size() != 3) throw Abort{2};
                const VqSurfaceInputs si{Upload(f[0], w, h)->View(), Upload(f[1], w, h)->View(), Upload(f[2], w, h)->View(), VqImage{nullptr, 0, 0, 0}};
                const std::vector<char> m = ReadFile(Need(a, "materials"));
                const int n = (int)(m.size() / sizeof(VqMaterialData));
                if (n < 1 || m.size() % sizeof(VqMaterialData)) throw Abort{3};
                std::vector<VqMaterialTextures> tex(n);
                std::memset(tex.data(), 0, tex.size() * sizeof(VqMaterialTextures));
                if (table) { vq_material_table_destroy(r.Context(), table); table = nullptr; }
                if (vq_material_table_create(r.Context(), (const VqMaterialData*)m.data(), tex.data(), n, &table) != VQ_OK) throw Abort{3};
                ok = shadowed ? r.RenderSceneColorFromMaterials(stream, view, pp, si, table, env, gfx, bHDR, maps)
                              : r.RenderSceneColorFromMaterials(stream, view, pp, si, table, env, gfx, bHDR);
            }
            if (!ok) return false;
            DumpImage(Need(a, "out"), r.SceneColor().View());
            return true;
        }
        if (cmd == "sky") {                                                    // RenderEnvironmentMap
            const std::vector<char> m = ReadFile(Need(a, "vp"), 64);
            VqGBuffer gb{};
            gb.normal_roughness = Upload(Need(a, "normal"), pp.SceneRTWidth, pp.SceneRTHeight)->View();
            if (!r.RenderEnvironmentMap(stream, (const float*)m.data(), gb, env)) return false;
            DumpImage(Need(a, "out"), r.SceneColor().View());
            return true;
        }
        if (cmd == "reflect") {                                                // ApplyReflections
            const VqImage refl = Upload(Need(a, "refl"), pp.SceneRTWidth, pp.SceneRTHeight)->View();
            VqImage bv{};
            if (a.count("bv")) bv = Upload(Need(a, "bv"), pp.SceneRTWidth, pp.SceneRTHeight)->View();
            if (!r.ApplyReflections(stream, refl, a.count("bv") ? &bv : nullptr)) return false;
            DumpImage(Need(a, "out"), r.SceneColor().View());
            return true;
        }
        if (cmd == "reflect_pass") {                                           // ApplyReflectionsPass::RecordCommands
            const int w = NeedInt(a, "w"), h = NeedInt(a, "h");
            vq::ApplyReflectionsPass pass(r);
            vq::ApplyReflectionsPass::FDrawParameters p;
            p.pCmd = stream;
            p.UAVSceneRadiance = Upload(Need(a, "target"), w, h)->View();
            p.SRVReflectionRadiance = Upload(Need(a, "refl"), w, h)->View();
            if (a.count("bv")) p.SRVBoundingVolumes = Upload(Need(a, "bv"), w, h)->View();
            p.iSceneRTWidth = NeedInt(a, "rtw"); p.iSceneRTHeight = NeedInt(a, "rth");
            const std::string before = vq::LastError();
            pass.Initialize();
            pass.RecordCommands(&p);
            if (before != vq::LastError()) return false;
            DumpImage(Need(a, "out"), p.UAVSceneRadiance);
            return true;
        }
        if (cmd == "post") {                                                   // RenderPostProcess
            const std::string mode = Need(a, "mode");
            pp.bEnableGaussianBlur = Opt(a, "blur", "0") == "1";
            pp.bEnableCAS = mode == "cas";
            pp.UpscalingAlgorithm = mode == "fsr" ? vq::FPostProcessParameters::FIDELITYFX_SUPER_RESOLUTION1 : vq::FPostProcessParameters::NONE;
            pp.Sharpness = OptFloat(a, "sharpness", 0.8f);
            pp.FFXCASParams.CASSharpen = pp.Sharpness;
            pp.FFXCASParams.UpdateCASConstantBlock(pp.SceneRTWidth, pp.SceneRTHeight, pp.SceneRTWidth, pp.SceneRTHeight);
            pp.FSR_EASUParams.UpdateEASUConstantBlock(pp.SceneRTWidth, pp.SceneRTHeight, pp.SceneRTWidth, pp.SceneRTHeight,
                                                      pp.DisplayResolutionWidth, pp.DisplayResolutionHeight);
            pp.FSR_RCASParams.RCASSharpnessStops = OptFloat(a, "stops", 0.2f);
            pp.FSR_RCASParams.UpdateRCASConstantBlock();
            lastPost = r.RenderPostProcess(stream, pp, Opt(a, "hdr", "0") == "1");
            if (!lastPost) return false;
            std::printf("post %d %d\n", lastPost->width, lastPost->height);
            DumpImage(Need(a, "out"), *lastPost);
            return true;
        }
        if (cmd == "save") {                                                   // SaveToHDRFileImage of the display frame or scene colour
            const VqImage im = Opt(a, "src", "post") == "scene" ? r.SceneColor().View() : (lastPost ? *lastPost : VqImage{});
            const std::vector<unsigned char> f = r.SaveToHDRFileImage(im);
            if (f.empty()) return false;
            WriteFile(Need(a, "out"), f.data(), f.size());
            return true;
        }
        if (cmd == "hires") {                                                  // CreateEnvironmentMapFileImageFromHiRes
            const std::vector<char> b = ReadFile(Need(a, "file"));
            const std::vector<unsigned char> f = vq::CreateEnvironmentMapFileImageFromHiRes(r, b.data(), b.size(), NeedInt(a, "w"), NeedInt(a, "h"));
            if (f.empty()) return false;
            WriteFile(Need(a, "out"), f.data(), f.size());
            return true;
        }
        if (cmd == "spd" || cmd == "blur_pass") {
            const int w = NeedInt(a, "w"), h = NeedInt(a, "h");
            const VqImage in = Upload(Need(a, "file"), w, h)->View();
            const std::string before = vq::LastError();
            if (cmd == "spd") {                                                // SinglePassDownsamplerPass
                vq::SinglePassDownsamplerPass pass(r);
                pass.Initialize();
                pass.OnCreateWindowSizeDependentResources((unsigned)w, (unsigned)h);
                vq::SinglePassDownsamplerPass::FDrawParameters p; p.pCmd = stream; p.In = in;
                pass.RecordCommands(&p);
                if (before != vq::LastError()) return false;
                std::printf("spd %zu", pass.Mips().size());
                for (auto& m : pass.Mips()) std::printf(" %dx%d", m->width, m->height);
                std::printf("\n");
                std::vector<char> all;
                for (auto& m : pass.Mips()) {
                    const std::vector<char> part = Download(m->View());
                    all.insert(all.end(), part.begin(), part.end());
                }
                WriteFile(Need(a, "out"), all.data(), all.size());
                pass.Destroy();
            } else {                                                           // GaussianBlurPass
                vq::GaussianBlurPass pass(r);
                pass.Initialize();
                pass.OnCreateWindowSizeDependentResources((unsigned)w, (unsigned)h);
                vq::FTexture2D* out = new vq::FTexture2D(); owned.push_back(out);
                if (!out->Create(w, h)) throw Abort{3};
                vq::GaussianBlurPass::FDrawParameters p; p.pCmd = stream; p.In = in; p.Out = out->View();
                pass.RecordCommands(&p);
                if (before != vq::LastError()) return false;
                DumpImage(Need(a, "out"), out->View());
                pass.Destroy();
            }
            return true;
        }
        if (cmd == "host_helpers") {                                           // pure-host constant setup: no device needed
            const std::string kind = Need(a, "kind");
            vq::FPostProcessParameters p;
            if (kind == "sharpness") {
                p.FSR_RCASParams.SetLinearSharpness(OptFloat(a, "linear", 1.0f));
                std::printf("sharpness %.9g %.9g\n", p.FSR_RCASParams.RCASSharpnessStops, p.FSR_RCASParams.GetLinearSharpness());
            } else if (kind == "cas") {
                p.FFXCASParams.CASSharpen = OptFloat(a, "sharp", 0.8f);
                p.FFXCASParams.UpdateCASConstantBlock(NeedInt(a, "iw"), NeedInt(a, "ih"), NeedInt(a, "ow"), NeedInt(a, "oh"));
                std::printf("cas");
                for (unsigned v : p.FFXCASParams.CASConstantBlock) std::printf(" %u", v);
                std::printf("\n");
            } else if (kind == "easu") {
                p.FSR_EASUParams.UpdateEASUConstantBlock(NeedInt(a, "iw"), NeedInt(a, "ih"), NeedInt(a, "cw"), NeedInt(a, "ch"),
                                                         NeedInt(a, "ow"), NeedInt(a, "oh"));
                std::printf("easu");
                for (unsigned v : p.FSR_EASUParams.EASUConstantBlock) std::printf(" %u", v);
                std::printf("\n");
            } else if (kind == "rcas") {
                p.FSR_RCASParams.RCASSharpnessStops = OptFloat(a, "stops", 0.2f);
                p.FSR_RCASParams.UpdateRCASConstantBlock();
                std::printf("rcas");
                for (unsigned v : p.FSR_RCASParams.RCASConstantBlock) std::printf(" %u", v);
                std::printf("\n");
            } else {
                throw Abort{2};
            }
            return true;
        }
        std::fprintf(stderr, "unknown command %s\n", cmd.c_str());
        throw Abort{2};
    }
};

int StepCode(const std::string& cmd) {
    static const std::map<std::string, int> codes = {
        {"init", kInit}, {"lut", kLut}, {"env_texels", kEnvTexels}, {"env_hdr", kEnvHdr}, {"prefilter", kPrefilter},
        {"window", kWindow}, {"scene", kScene}, {"scene_materials", kSceneMaterials}, {"sky", kSky}, {"reflect", kReflect},
        {"reflect_pass", kReflectPass}, {"post", kPost}, {"save", kSave}, {"hires", kHiRes}, {"spd", kSpd},
        {"blur_pass", kBlurPass}, {"host_helpers", kHostHelpers}};
    auto it = codes.find(cmd);
    return it == codes.end() ? 2 : it->second;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 2) { std::fprintf(stderr, "usage: %s <scenario.txt>\n", argv[0]); return 2; }
    const std::string scenario = argv[1];
    const size_t slash = scenario.find_last_of('/');
    g_dir = slash == std::string::npos ? "." : scenario.substr(0, slash);
    std::ifstream in(scenario);
    if (!in) { std::fprintf(stderr, "cannot read %s\n", scenario.c_str()); return 2; }
    Driver d;
    std::string line;
    try {
        while (std::getline(in, line)) {
            const size_t hash = line.find('#');
            if (hash != std::string::npos) line.resize(hash);
            std::istringstream words(line);
            std::string cmd, w;
            if (!(words >> cmd)) continue;
            Args a;
            while (words >> w) {
                const size_t eq = w.find('=');
                if (eq == std::string::npos) { std::fprintf(stderr, "bad word %s\n", w.c_str()); return 2; }
                a[w.substr(0, eq)] = w.substr(eq + 1);
            }
            const bool expectFail = Opt(a, "expect", "ok") == "fail";
            const bool ok = d.Run(cmd, a);
            std::fflush(stdout);
            if (ok && expectFail) { std::printf("NOT REFUSED %s\n", cmd.c_str()); return 5; }
            if (!ok && expectFail) { std::printf("refused %s: %s\n", cmd.c_str(), vq::LastError()); continue; }
            if (!ok) d.Refused(StepCode(cmd), cmd.c_str());
            std::printf("ok %s\n", cmd.c_str());
        }
    } catch (const Abort& e) {
        std::fflush(stdout);
        return e.code;
    }
    return 0;
}
