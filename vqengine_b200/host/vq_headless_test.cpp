// vq_headless_test.cpp — the reference's only automated test is a smoke run: `VQE.exe -Test -TestFrames=<n>` renders n
// frames and exits 0 (Source/Engine/Main.cpp:65-84, VQEngine_Main.cpp:66-72,180; Scripts/TestVQE.bat:90-105).
// This is the headless equivalent over the CUDA backend: load an environment map (prefilter), then per frame
// RenderSceneColor + RenderPostProcess on a synthetic G-buffer, checking every frame for finite output.
// With -Devices=<d0>,<d1>,... the frames run through vq::VQRendererGroup, one rank per listed device (a device may repeat: -Devices=0,0
// is a 2-rank group on one GPU); every rank ends each frame holding the whole display frame, and rank 0's is checked and reported.
//   usage: vq_headless_test [-Test] [-TestFrames=<n>] [-W=<w>] [-H=<h>] [-Devices=<list>]
#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "vq_renderer.hpp"

static float frand(unsigned& s) { s = s * 1664525u + 1013904223u; return (float)(s >> 8) / 16777216.0f; }

int main(int argc, char** argv) {
    int frames = 100, W = 640, H = 360;    // NUM_TEST_FRAMES default 100 (VQEngine_Main.cpp:180)
    std::vector<int> devices;
    for (int i = 1; i < argc; ++i) {
        if (!std::strncmp(argv[i], "-TestFrames=", 12)) frames = std::atoi(argv[i] + 12);
        else if (!std::strncmp(argv[i], "-W=", 3)) W = std::atoi(argv[i] + 3);
        else if (!std::strncmp(argv[i], "-H=", 3)) H = std::atoi(argv[i] + 3);
        else if (!std::strncmp(argv[i], "-Devices=", 9)) {
            for (const char* p = argv[i] + 9; *p;) {
                char* end;
                devices.push_back((int)std::strtol(p, &end, 10));
                if (end == p) { std::fprintf(stderr, "bad -Devices list\n"); return 1; }
                p = *end == ',' ? end + 1 : end;
            }
        }
    }
    const bool grouped = !devices.empty();
    vq::VQRenderer single;
    vq::VQRendererGroup group;
    if (grouped ? !group.Initialize(devices) : !single.Initialize(0)) return 2;
    if (grouped ? !group.LoadDefaultResources() : !single.LoadDefaultResources()) return 3;
    const int nRanks = grouped ? group.NumRanks() : 1;
    vq::VQRenderer& renderer = grouped ? group.Rank(0) : single;

    // synthetic equirect HDRI 512x256
    const int EW = 512, EH = 256;
    std::vector<float> hdri((size_t)EW * EH * 4);
    unsigned seed = 0x5EED0001u;
    for (int y = 0; y < EH; ++y)
        for (int x = 0; x < EW; ++x) {
            float* t = &hdri[((size_t)y * EW + x) * 4];
            const float v = (y + 0.5f) / EH, sun = 12.0f * std::exp(-((x - 300.f) * (x - 300.f) + (y - 60.f) * (y - 60.f)) / 200.0f);
            t[0] = 0.1f + 1.2f * (1 - v) + sun; t[1] = 0.15f + 1.5f * (1 - v) + sun * 0.9f; t[2] = 0.3f + 1.9f * (1 - v) + sun * 0.7f; t[3] = 1.0f;
            t[0] *= 1.0f + 0.05f * (frand(seed) - 0.5f);
        }
    // The engine loads its environment maps from Radiance .hdr files (Data/Textures/EnvironmentMaps via EnvironmentMaps.ini):
    // write the synthetic panorama out as a .hdr file image through the backend (Image::SaveToDisk route) and load the
    // environment from THAT (Image::LoadFromFile route), so the smoke run covers both ends of the on-disk format.
    std::vector<vq::FEnvironmentMapRenderingResources> envs(nRanks);     // each rank decodes the file on its own device
    vq::FEnvironmentMapRenderingResources& env = envs[0];
    vq::FGraphicsSettings gfx; gfx.EnvironmentMapResolution = 128;
    {
        cudaSetDevice(renderer.Device());
        vq::FTexture2D staging;
        if (!staging.Create(EW, EH)) return 4;
        cudaMemcpy(staging.mem.ptr, hdri.data(), hdri.size() * 4, cudaMemcpyHostToDevice);
        const std::vector<unsigned char> file = renderer.SaveToHDRFileImage(staging.View());
        if (file.empty()) { std::fprintf(stderr, "SaveToHDRFileImage: %s\n", vq::LastError()); return 4; }
        for (int r = 0; r < nRanks; ++r)
            if (!envs[r].CreateRenderingResourcesFromHDRFile(grouped ? group.Rank(r) : single, file.data(), file.size(), 64,
                                                             gfx.EnvironmentMapResolution)) {
                std::fprintf(stderr, "CreateRenderingResourcesFromHDRFile: %s\n", vq::LastError()); return 4;
            }
        std::printf("environment map: %dx%d .hdr file image of %zu bytes, MaxContentLightLevel %d\n", env.HDRIWidth, env.HDRIHeight,
                    file.size(), env.MaxContentLightLevel);
    }
    std::vector<vq::FEnvironmentMapRenderingResources*> envPtrs;
    for (auto& e : envs) envPtrs.push_back(&e);
    const std::vector<const vq::FEnvironmentMapRenderingResources*> envViews(envPtrs.begin(), envPtrs.end());
    if (grouped ? !group.PreFilterEnvironmentMap(envPtrs, 0.05f) : !single.PreFilterEnvironmentMap(env, 0.05f)) return 5;

    // synthetic G-buffer
    std::vector<float> pos((size_t)W * H * 4), nrm(pos.size()), alb(pos.size());
    for (int y = 0; y < H; ++y)
        for (int x = 0; x < W; ++x) {
            const size_t o = ((size_t)y * W + x) * 4;
            const float fx = -20.f + 40.f * x / W, fz = 20.f - 40.f * y / H;
            pos[o] = fx; pos[o + 1] = 2.0f * std::sin(0.3f * fx) * std::cos(0.25f * fz); pos[o + 2] = fz; pos[o + 3] = 0.05f;
            float n[3] = {-0.6f * std::cos(0.3f * fx), 1.0f, 0.5f * std::sin(0.25f * fz)};
            const float l = std::sqrt(n[0] * n[0] + n[1] * n[1] + n[2] * n[2]);
            nrm[o] = n[0] / l; nrm[o + 1] = n[1] / l; nrm[o + 2] = n[2] / l; nrm[o + 3] = 0.04f + 0.9f * frand(seed);
            alb[o] = 0.1f + 0.8f * frand(seed); alb[o + 1] = 0.1f + 0.8f * frand(seed); alb[o + 2] = 0.1f + 0.8f * frand(seed);
            alb[o + 3] = frand(seed) < 0.2f ? 1.0f : 0.0f;
            if (y < H / 6) { nrm[o] = nrm[o + 1] = nrm[o + 2] = 0.0f; }       // the top band is sky: no surface, filled by the skydome pass
        }
    std::vector<vq::FTexture2D> gp(nRanks), gn(nRanks), ga(nRanks);
    std::vector<VqGBuffer> gbs;
    for (int r = 0; r < nRanks; ++r) {                                  // every rank's G-buffer on its own device
        cudaSetDevice(grouped ? group.Rank(r).Device() : 0);
        if (!gp[r].Create(W, H) || !gn[r].Create(W, H) || !ga[r].Create(W, H)) return 6;
        cudaMemcpy(gp[r].mem.ptr, pos.data(), pos.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(gn[r].mem.ptr, nrm.data(), nrm.size() * 4, cudaMemcpyHostToDevice);
        cudaMemcpy(ga[r].mem.ptr, alb.data(), alb.size() * 4, cudaMemcpyHostToDevice);
        gbs.push_back(VqGBuffer{gp[r].View(), gn[r].View(), ga[r].View(), VqImage{nullptr, 0, 0, 0}});
    }
    const VqGBuffer& gb = gbs[0];

    vq::FPostProcessParameters pp;
    pp.SceneRTWidth = W; pp.SceneRTHeight = H; pp.DisplayResolutionWidth = 2 * W; pp.DisplayResolutionHeight = 2 * H;
    pp.FSR_EASUParams.UpdateEASUConstantBlock(W, H, W, H, 2 * W, 2 * H);      // VQEngine_EventHandlers.cpp:298-306
    pp.FSR_RCASParams.UpdateRCASConstantBlock();
    if (grouped ? !group.OnWindowSizeChanged(W, H, 2 * W, 2 * H) : !renderer.OnWindowSizeChanged(W, H, 2 * W, 2 * H)) return 7;

    vq::FSceneView view;
    view.cameraPosition = {0.0f, 5.0f, -17.0f};
    VqSceneLighting& L = view.GPULightingData;
    L.numPointLights = 4;
    for (int i = 0; i < 4; ++i) {
        L.point_lights[i].position = {-15.f + 10.f * i, 9.0f, -5.0f + 4.f * i};
        L.point_lights[i].range = 50.0f; L.point_lights[i].brightness = 500.0f + 200.0f * i;
        L.point_lights[i].color = {1.0f, 0.9f - 0.1f * i, 0.6f + 0.1f * i};
    }
    L.directional.enabled = 1; L.directional.brightness = 0.9f; L.directional.color = {1, 1, 1};
    L.directional.lightDirection = {-0.5f, -0.83f, 0.25f};

    cudaSetDevice(renderer.Device());
    cudaStream_t pCmd = nullptr;
    if (!grouped) cudaStreamCreate(&pCmd);
    else pCmd = group.Stream(0);
    std::vector<float> readback((size_t)4 * W * H * 4);
    for (int f = 0; f < frames; ++f) {
        view.HDRIYawOffset = 0.01f * f;                         // the unit-test scene orbits; here the sky turns
        {   // skyCam at the origin, yaw following the HDRI offset (Scene.cpp:573-584): view = rotY(-yaw), LH perspective 60 degrees
            const float yaw = view.HDRIYawOffset, c = std::cos(yaw), s = std::sin(yaw);
            const float h = 1.0f / std::tan(0.5f * 1.0472f), w = h * (float)H / (float)W, q = 1000.0f / (1000.0f - 0.1f);
            const float viewM[16] = {c, 0, s, 0,  0, 1, 0, 0,  -s, 0, c, 0,  0, 0, 0, 1};
            const float proj[16] = {w, 0, 0, 0,  0, h, 0, 0,  0, 0, q, 1,  0, 0, -0.1f * q, 0};
            float vp[16];
            for (int r = 0; r < 4; ++r) for (int k = 0; k < 4; ++k) { float a = 0; for (int j = 0; j < 4; ++j) a += viewM[4 * r + j] * proj[4 * j + k]; vp[4 * r + k] = a; }
            if (grouped) {
                if (!group.RenderSceneColor(view, pp, gbs, envViews, gfx, false, vp)) return 8;
            } else if (!renderer.RenderSceneColor(pCmd, view, pp, gb, env, gfx, false) || !renderer.RenderEnvironmentMap(pCmd, vp, gb, env)) {
                return 8;
            }
        }
        const VqImage* out = grouped ? group.RenderPostProcess(pp, false) : renderer.RenderPostProcess(pCmd, pp, false);
        if (!out) return 9;
        if (f == frames - 1 || f == 0) {
            cudaStreamSynchronize(pCmd);
            cudaMemcpy(readback.data(), out->ptr, (size_t)out->width * out->height * 16, cudaMemcpyDeviceToHost);
            double sum = 0; for (float v : readback) { if (!std::isfinite(v)) { std::fprintf(stderr, "non-finite output\n"); return 10; } sum += v; }
            std::printf("frame %d: %dx%d mean %.6f\n", f, out->width, out->height, sum / readback.size());
        }
    }
    for (int r = 0; r < nRanks; ++r)
        if (cudaStreamSynchronize(grouped ? group.Stream(r) : pCmd) != cudaSuccess) return 11;
    if (!grouped) cudaStreamDestroy(pCmd);
    for (auto& e : envs) e.DestroyRenderingResources();
    std::printf("VQ headless test: %d frames OK, %llu kernel launches\n", frames, (unsigned long long)vq_launch_count());
    return 0;                                                   // PostQuitMessage(0)
}
