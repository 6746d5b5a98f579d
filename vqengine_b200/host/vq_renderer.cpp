// vq_renderer.cpp — C++ host layer: fills the constant blocks exactly where the engine does and dispatches the
// C-ABI passes in the engine's order. No pixel math here.
#include "vq_renderer.hpp"

#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <utility>

namespace vq {

static thread_local std::string g_err;
const char* LastError() { return g_err.c_str(); }
static bool Fail(const char* where) {
    g_err = std::string(where) + ": " + vq_last_error();
    std::fprintf(stderr, "[vq] error: %s\n", g_err.c_str());      // Log::Error + early return (Renderer.cpp:939-949)
    return false;
}
#define VQ_TRY(call, where) do { if ((call) != VQ_OK) return Fail(where); } while (0)

// ---- resources ---------------------------------------------------------------------------------
bool FDeviceBuffer::Alloc(size_t n) {
    if (bytes >= n && ptr) return true;
    Free();
    if (cudaMalloc(&ptr, n) != cudaSuccess) { cudaGetLastError(); ptr = nullptr; g_err = "cudaMalloc failed"; return false; }
    bytes = n;
    return true;
}
void FDeviceBuffer::Free() { if (ptr) cudaFree(ptr); ptr = nullptr; bytes = 0; }
bool FTexture2D::Create(int w, int h, int tb) {
    width = w; height = h; texelBytes = tb;
    return mem.Alloc((size_t)w * h * tb);
}

// ---- PostProcess.cpp:37-99 ------------------------------------------------------------------------
float FPostProcessParameters::FFSR1_RCAS::GetLinearSharpness() const { return std::pow(0.5f, RCASSharpnessStops); }
void FPostProcessParameters::FFSR1_RCAS::SetLinearSharpness(float S) { RCASSharpnessStops = std::log10(S) / std::log10(0.5f); }
void FPostProcessParameters::FFSR1_RCAS::UpdateRCASConstantBlock() { vq_fsr_rcas_con(RCASConstantBlock, RCASSharpnessStops); }
void FPostProcessParameters::FFSR1_EASU::UpdateEASUConstantBlock(unsigned iw, unsigned ih, unsigned cw, unsigned ch, unsigned ow, unsigned oh) {
    vq_fsr_easu_con(EASUConstantBlock, (float)iw, (float)ih, (float)cw, (float)ch, (float)ow, (float)oh);
}
void FPostProcessParameters::FFFXCAS::UpdateCASConstantBlock(unsigned iw, unsigned ih, unsigned ow, unsigned oh) {
    vq_cas_setup(CASConstantBlock, CASSharpen, (float)iw, (float)ih, (float)ow, (float)oh);
}

// ---- environment map resources (EnvironmentMapRendering.cpp:20-106) -----------------------------------
bool FEnvironmentMapRenderingResources::CreateRenderingResources(VQRenderer& Renderer, const FEnvironmentMapDescriptor& desc,
                                                                 int DiffuseRes_, int SpecRes_) {
    if (!desc.pHDRIData || desc.Width <= 0 || desc.Height <= 0) { g_err = "bad HDRI descriptor"; return false; }
    cudaSetDevice(Renderer.Device());                                       // the resources live on the renderer's device
    HDRIWidth = desc.Width; HDRIHeight = desc.Height;
    HDRIMips = vq_mip_level_count((uint64_t)desc.Width, (uint64_t)desc.Height);
    MaxContentLightLevel = (int)desc.MaxContentLightLevel;
    DiffuseRes = DiffuseRes_; SpecRes = SpecRes_;
    // "2x2 for the last mip level" (EnvironmentMapRendering.cpp:63)
    SpecMips = vq_mip_level_count((uint64_t)SpecRes_, (uint64_t)SpecRes_) - 1;
    if (!Tex_HDREnvironment.Alloc(vq_pyramid_texel_count(HDRIWidth, HDRIHeight, HDRIMips) * 16)) return false;
    if (cudaMemcpy(Tex_HDREnvironment.ptr, desc.pHDRIData, (size_t)HDRIWidth * HDRIHeight * 16, cudaMemcpyHostToDevice) != cudaSuccess) {
        g_err = "HDRI upload failed"; return false;
    }
    // CPU mips in the engine (TextureManager.cpp:714-727): here K11 on the device
    VQ_TRY(vq_hdri_build_mips(Renderer.Context(), HDRI(), nullptr), "vq_hdri_build_mips");
    const size_t diffBytes = vq_cubemap_texel_count(DiffuseRes, 1) * 16;
    return Tex_IrradianceDiff.Alloc(diffBytes) && Tex_IrradianceDiffBlurred.Alloc(diffBytes) &&
           Tex_BlurTemp.Alloc((size_t)DiffuseRes * DiffuseRes * 16) &&
           Tex_IrradianceSpec.Alloc(vq_cubemap_texel_count(SpecRes, SpecMips) * 16);
}
bool FEnvironmentMapRenderingResources::CreateRenderingResourcesFromHDRFile(VQRenderer& Renderer, const void* pFileBytes, size_t NumBytes,
                                                                            int DiffuseRes_, int SpecRes_) {
    VqHdrInfo info;
    VQ_TRY(vq_hdr_parse(pFileBytes, NumBytes, &info, nullptr), "vq_hdr_parse");          // "Error loading file" in the engine
    cudaSetDevice(Renderer.Device());
    HDRIWidth = info.width; HDRIHeight = info.height;
    HDRIMips = vq_mip_level_count((uint64_t)info.width, (uint64_t)info.height);
    DiffuseRes = DiffuseRes_; SpecRes = SpecRes_;
    SpecMips = vq_mip_level_count((uint64_t)SpecRes_, (uint64_t)SpecRes_) - 1;           // EnvironmentMapRendering.cpp:63
    if (!Tex_HDREnvironment.Alloc(vq_pyramid_texel_count(HDRIWidth, HDRIHeight, HDRIMips) * 16)) return false;
    float MaxLuminance = 0.0f;
    const VqImage level0{Tex_HDREnvironment.ptr, HDRIWidth, HDRIHeight, (size_t)HDRIWidth * 16};
    VQ_TRY(vq_hdr_load_host(Renderer.Context(), pFileBytes, NumBytes, level0, &MaxLuminance), "vq_hdr_load_host");
    MaxContentLightLevel = (int)MaxLuminance;
    VQ_TRY(vq_hdri_build_mips(Renderer.Context(), HDRI(), nullptr), "vq_hdri_build_mips");
    const size_t diffBytes = vq_cubemap_texel_count(DiffuseRes, 1) * 16;
    return Tex_IrradianceDiff.Alloc(diffBytes) && Tex_IrradianceDiffBlurred.Alloc(diffBytes) &&
           Tex_BlurTemp.Alloc((size_t)DiffuseRes * DiffuseRes * 16) &&
           Tex_IrradianceSpec.Alloc(vq_cubemap_texel_count(SpecRes, SpecMips) * 16);
}
void FEnvironmentMapRenderingResources::DestroyRenderingResources() {
    Tex_HDREnvironment.Free(); Tex_IrradianceDiff.Free(); Tex_IrradianceDiffBlurred.Free(); Tex_BlurTemp.Free(); Tex_IrradianceSpec.Free();
}

// ---- Data/EnvironmentMaps.ini ----------------------------------------------------------------------
std::vector<FEnvironmentMapFileDescriptor> ParseEnvironmentMapsINI(const std::string& text) {
    std::vector<FEnvironmentMapFileDescriptor> out;
    FEnvironmentMapFileDescriptor desc;
    bool sawEmptyLine = false, readingEnvMap = false;
    size_t pos = 0;
    while (pos <= text.size()) {
        size_t eol = text.find('\n', pos);
        if (eol == std::string::npos) eol = text.size();
        std::string line = text.substr(pos, eol - pos);
        pos = eol + 1;
        if (!line.empty() && line.back() == '\r') line.pop_back();
        if (!line.empty() && line[0] == ';') continue;                       // comment
        if (line.empty()) { sawEmptyLine = true; if (pos > text.size()) break; continue; }
        if (line.front() == '[') {                                          // section header: "[Name]"
            const size_t close = line.find(']');
            readingEnvMap = true;
            if (sawEmptyLine) { out.push_back(desc); desc = {}; sawEmptyLine = false; }
            desc.Name = line.substr(1, close == std::string::npos ? std::string::npos : close - 1);
            continue;
        }
        const size_t eq = line.find('=');
        if (eq != std::string::npos) {
            const std::string key = line.substr(0, eq), value = line.substr(eq + 1);
            if (key == "Path") desc.FilePath = value;
            if (key == "MaxCLL") desc.MaxContentLightLevel = std::strtof(value.c_str(), nullptr);
        }
        sawEmptyLine = false;
    }
    if (readingEnvMap) out.push_back(desc);
    return out;
}

std::vector<unsigned char> CreateEnvironmentMapFileImageFromHiRes(VQRenderer& Renderer, const void* pHiResFileBytes, size_t NumBytes,
                                                                  int TargetWidth, int TargetHeight) {
    VqHdrInfo info;
    if (vq_hdr_parse(pHiResFileBytes, NumBytes, &info, nullptr) != VQ_OK) { Fail("vq_hdr_parse"); return {}; }
    if (TargetWidth <= 0 || TargetHeight <= 0 || TargetWidth > info.width || TargetHeight > info.height) {
        g_err = "CreateEnvironmentMapFileImageFromHiRes: the target must not be larger than the source"; return {};
    }
    FTexture2D hi, lo;
    if (!hi.Create(info.width, info.height) || !lo.Create(TargetWidth, TargetHeight)) return {};
    float maxLuminance = 0.0f;
    if (vq_hdr_load_host(Renderer.Context(), pHiResFileBytes, NumBytes, hi.View(), &maxLuminance) != VQ_OK) { Fail("vq_hdr_load_host"); return {}; }
    if (vq_image_resize(Renderer.Context(), hi.View(), lo.View(), nullptr) != VQ_OK) { Fail("vq_image_resize"); return {}; }
    return Renderer.SaveToHDRFileImage(lo.View());                          // vq_hdr_save_host synchronises
}

// ---- renderer ------------------------------------------------------------------------------------
bool VQRenderer::Initialize(int DeviceIndex) {
    if (mCtx) return true;
    VQ_TRY(vq_ctx_create(DeviceIndex, &mCtx), "vq_ctx_create");
    mDevice = DeviceIndex;
    return true;
}
void VQRenderer::Destroy() {
    if (mCtx) { cudaSetDevice(mDevice); cudaDeviceSynchronize(); vq_ctx_destroy(mCtx); mCtx = nullptr; }
}
bool VQRenderer::LoadDefaultResources() {
    // CreateProceduralTextures LUT desc (Renderer.cpp:1026-1032): 1024x1024; ComputeBRDFIntegrationLUT: 2048 samples
    cudaSetDevice(mDevice);
    if (!mBRDFLUT.Create(1024, 1024, 8)) return false;
    VQ_TRY(vq_brdf_integration_lut(mCtx, mBRDFLUT.View(), 2048, 0, 1024, nullptr), "vq_brdf_integration_lut");
    return cudaStreamSynchronize(nullptr) == cudaSuccess;
}
bool VQRenderer::OnWindowSizeChanged(int rw, int rh, int dw, int dh) {
    cudaSetDevice(mDevice);
    return mSceneColor.Create(rw, rh) && mBlurTemp.Create(rw, rh) && mBlurOut.Create(rw, rh) && mPostOut.Create(rw, rh) &&
           mRCASOut.Create(dw, dh) && vq_ctx_resize(mCtx, rw, rh) == VQ_OK;
}

// K2's parameters: the given step over HDRI mip 3 (or the last one) (EnvironmentMapRendering.cpp:181-277)
static VqDiffuseIrradianceParams DiffuseParams(const FEnvironmentMapRenderingResources& env, float DiffuseIntegrationStep) {
    return VqDiffuseIrradianceParams{DiffuseIntegrationStep, 0, 0, 3 < env.HDRIMips ? 3 : env.HDRIMips - 1};
}

bool VQRenderer::PreFilterEnvironmentMap(FEnvironmentMapRenderingResources& env, float DiffuseIntegrationStep) {
    // Diffuse irradiance convolution (EnvironmentMapRendering.cpp:181-277): 6 per-face draws -> one launch
    const VqDiffuseIrradianceParams dp = DiffuseParams(env, DiffuseIntegrationStep);
    const VqCubemap diff{env.Tex_IrradianceDiff.ptr, env.DiffuseRes, 1};
    VQ_TRY(vq_diffuse_irradiance(mCtx, &dp, env.HDRI(), diff, 0, 6 * env.DiffuseRes, nullptr), "vq_diffuse_irradiance");
    // Blur diffuse irradiance, per face: X into temp, Y into the blurred cube (EnvironmentMapRendering.cpp:279-373)
    const VqBlurParams bp{env.DiffuseRes, env.DiffuseRes};
    const size_t faceBytes = (size_t)env.DiffuseRes * env.DiffuseRes * 16, pitch = (size_t)env.DiffuseRes * 16;
    for (int face = 0; face < 6; ++face) {
        const VqImage in{(char*)env.Tex_IrradianceDiff.ptr + face * faceBytes, env.DiffuseRes, env.DiffuseRes, pitch};
        const VqImage tmp{env.Tex_BlurTemp.ptr, env.DiffuseRes, env.DiffuseRes, pitch};
        const VqImage out{(char*)env.Tex_IrradianceDiffBlurred.ptr + face * faceBytes, env.DiffuseRes, env.DiffuseRes, pitch};
        VQ_TRY(vq_gaussian_blur_x(mCtx, &bp, in, tmp, nullptr), "vq_gaussian_blur_x");
        VQ_TRY(vq_gaussian_blur_y(mCtx, &bp, tmp, out, nullptr), "vq_gaussian_blur_y");
    }
    // Specular irradiance (EnvironmentMapRendering.cpp:386-472): mip x face draws, 512 samples
    VQ_TRY(vq_specular_prefilter(mCtx, env.HDRI(), env.Specular(), 512, 0, vq_cubemap_row_count(env.SpecRes, env.SpecMips), nullptr),
           "vq_specular_prefilter");
    // ExecuteCommandLists + CPU wait on the fence (EnvironmentMapRendering.cpp:477-485)
    if (cudaStreamSynchronize(nullptr) != cudaSuccess) { g_err = "PreFilterEnvironmentMap: device error"; return false; }
    return true;
}

// CopyPerFrameConstantBufferData / CopyPerViewConstantBufferData: the constant blocks PSMain reads
void VQRenderer::FillSceneConstants(const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                    const FEnvironmentMapRenderingResources& env, const FGraphicsSettings& GFXSettings,
                                    bool bHDRDisplay, VqPerFrameData& PerFrame, VqPerViewLightingData& PerView) const {
    // CopyPerFrameConstantBufferData (SceneRendering.cpp:429-450)
    std::memset(&PerFrame, 0, sizeof(PerFrame));
    PerFrame.Lights = SceneView.GPULightingData;
    PerFrame.fAmbientLightingFactor = SceneView.sceneRenderOptions.fAmbientLightingFactor;
    PerFrame.f2PointLightShadowMapDimensions = {1024.0f, 1024.0f};
    PerFrame.f2SpotLightShadowMapDimensions = {1024.0f, 1024.0f};
    PerFrame.f2DirectionalLightShadowMapDimensions = {2048.0f, 2048.0f};
    PerFrame.fHDRIOffsetInRadians = SceneView.HDRIYawOffset;
    if (bHDRDisplay) PerFrame.fAmbientLightingFactor *= 0.005f;
    // CopyPerViewConstantBufferData (SceneRendering.cpp:452-467)
    std::memset(&PerView, 0, sizeof(PerView));
    PerView.CameraPosition = SceneView.cameraPosition;
    PerView.ScreenDimensions = {(float)PPParams.SceneRTWidth, (float)PPParams.SceneRTHeight};
    PerView.MaxEnvMapLODLevels = (float)env.GetNumSpecularIrradianceCubemapLODLevels();
    PerView.EnvironmentMapDiffuseOnlyIllumination = GFXSettings.Reflections == EReflections::SCREEN_SPACE_REFLECTIONS__FFX;
}

// IBL SRVs (SceneRendering.cpp:1690-1717): blurred diffuse irradiance, prefiltered specular, BRDF LUT
VqEnvironmentMaps VQRenderer::EnvironmentMaps(const FEnvironmentMapRenderingResources& env) const {
    return VqEnvironmentMaps{env.DiffuseBlurred(), env.Specular(), mBRDFLUT.View()};
}

bool VQRenderer::RenderSceneColor(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                  const VqGBuffer& GBuffer, const FEnvironmentMapRenderingResources& env,
                                  const FGraphicsSettings& GFXSettings, bool bHDRDisplay) {
    VqPerFrameData PerFrame;
    VqPerViewLightingData PerView;
    FillSceneConstants(SceneView, PPParams, env, GFXSettings, bHDRDisplay, PerFrame, PerView);
    const VqEnvironmentMaps maps = EnvironmentMaps(env);
    VQ_TRY(vq_forward_lighting(mCtx, &PerFrame, &PerView, &GBuffer, &maps, mSceneColor.View(), 0, mSceneColor.height, pCmd),
           "vq_forward_lighting");
    return true;
}

bool VQRenderer::RenderSceneColorFromMaterials(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                               const VqSurfaceInputs& SurfaceInputs, const VqMaterialTable* MaterialTable,
                                               const FEnvironmentMapRenderingResources& env, const FGraphicsSettings& GFXSettings,
                                               bool bHDRDisplay, bool bAlphaMask) {
    VqPerFrameData PerFrame;
    VqPerViewLightingData PerView;
    FillSceneConstants(SceneView, PPParams, env, GFXSettings, bHDRDisplay, PerFrame, PerView);
    const VqEnvironmentMaps maps = EnvironmentMaps(env);
    VQ_TRY(vq_forward_lighting_from_materials(mCtx, &PerFrame, &PerView, &SurfaceInputs, MaterialTable, bAlphaMask ? 1 : 0, &maps,
                                              mSceneColor.View(), 0, mSceneColor.height, pCmd),
           "vq_forward_lighting_from_materials");
    return true;
}

// 4x4 inverse in double (row-major; the convention does not matter for an inverse), rounded to fp32 at the end
// the shadow-map sizes the shader divides by (Lighting.hlsl:190, :237) are those of the maps bound; a light type without a map
// keeps the engine's constant
static void SetShadowMapDimensions(const VqShadowMaps& maps, VqPerFrameData& PerFrame) {
    if (maps.point_cubes) PerFrame.f2PointLightShadowMapDimensions = {(float)maps.point_res, (float)maps.point_res};
    if (maps.spot_maps) PerFrame.f2SpotLightShadowMapDimensions = {(float)maps.spot_width, (float)maps.spot_height};
    if (maps.directional_map) PerFrame.f2DirectionalLightShadowMapDimensions = {(float)maps.directional_width, (float)maps.directional_height};
}

bool VQRenderer::RenderSceneColor(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                  const VqGBuffer& GBuffer, const FEnvironmentMapRenderingResources& env,
                                  const FGraphicsSettings& GFXSettings, bool bHDRDisplay, const VqShadowMaps& ShadowMaps) {
    VqPerFrameData PerFrame;
    VqPerViewLightingData PerView;
    FillSceneConstants(SceneView, PPParams, env, GFXSettings, bHDRDisplay, PerFrame, PerView);
    SetShadowMapDimensions(ShadowMaps, PerFrame);
    const VqEnvironmentMaps maps = EnvironmentMaps(env);
    VQ_TRY(vq_forward_lighting_shadowed(mCtx, &PerFrame, &PerView, &GBuffer, &maps, &ShadowMaps, mSceneColor.View(), 0,
                                        mSceneColor.height, pCmd),
           "vq_forward_lighting_shadowed");
    return true;
}

bool VQRenderer::RenderSceneColorFromMaterials(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                               const VqSurfaceInputs& SurfaceInputs, const VqMaterialTable* MaterialTable,
                                               const FEnvironmentMapRenderingResources& env, const FGraphicsSettings& GFXSettings,
                                               bool bHDRDisplay, const VqShadowMaps& ShadowMaps, bool bAlphaMask) {
    VqPerFrameData PerFrame;
    VqPerViewLightingData PerView;
    FillSceneConstants(SceneView, PPParams, env, GFXSettings, bHDRDisplay, PerFrame, PerView);
    SetShadowMapDimensions(ShadowMaps, PerFrame);
    const VqEnvironmentMaps maps = EnvironmentMaps(env);
    VQ_TRY(vq_forward_lighting_shadowed_from_materials(mCtx, &PerFrame, &PerView, &SurfaceInputs, MaterialTable, bAlphaMask ? 1 : 0,
                                                       &maps, &ShadowMaps, mSceneColor.View(), 0, mSceneColor.height, pCmd),
           "vq_forward_lighting_shadowed_from_materials");
    return true;
}

static bool Invert4x4(const float m[16], float out[16]) {
    double a[4][8];
    for (int r = 0; r < 4; ++r)
        for (int c = 0; c < 4; ++c) { a[r][c] = m[4 * r + c]; a[r][4 + c] = r == c ? 1.0 : 0.0; }
    for (int c = 0; c < 4; ++c) {
        int piv = c;
        for (int r = c + 1; r < 4; ++r) if (std::fabs(a[r][c]) > std::fabs(a[piv][c])) piv = r;
        if (std::fabs(a[piv][c]) < 1e-300) return false;
        if (piv != c) for (int k = 0; k < 8; ++k) std::swap(a[piv][k], a[c][k]);
        const double d = 1.0 / a[c][c];
        for (int k = 0; k < 8; ++k) a[c][k] *= d;
        for (int r = 0; r < 4; ++r)
            if (r != c) { const double f = a[r][c]; if (f != 0.0) for (int k = 0; k < 8; ++k) a[r][k] -= f * a[c][k]; }
    }
    for (int r = 0; r < 4; ++r) for (int c = 0; c < 4; ++c) out[4 * r + c] = (float)a[r][4 + c];
    return true;
}

bool VQRenderer::RenderEnvironmentMap(cudaStream_t pCmd, const float EnvironmentMapViewProj[16], const VqGBuffer& GBuffer,
                                      const FEnvironmentMapRenderingResources& env) {
    VqMatrix inv;
    if (!Invert4x4(EnvironmentMapViewProj, inv.m)) { g_err = "EnvironmentMapViewProj is singular"; return false; }
    const VqPyramid level0{env.Tex_HDREnvironment.ptr, env.HDRIWidth, env.HDRIHeight, 1};   // Skydome.hlsl samples mip 0 only
    VQ_TRY(vq_skydome(mCtx, &inv, level0, &GBuffer.normal_roughness, mSceneColor.View(), 0, mSceneColor.height, pCmd), "vq_skydome");
    return true;
}

bool VQRenderer::ApplyReflections(cudaStream_t pCmd, const VqImage& ReflectionRadiance, const VqImage* BoundingVolumes) {
    VQ_TRY(vq_apply_reflections(mCtx, mSceneColor.View(), ReflectionRadiance, BoundingVolumes, pCmd), "vq_apply_reflections");
    return true;
}

void ApplyReflectionsPass::RecordCommands(const IRenderPassDrawParameters* pDrawParameters) {
    const FDrawParameters* pParams = static_cast<const FDrawParameters*>(pDrawParameters);
    if (!pParams || !pParams->UAVSceneRadiance.ptr || !pParams->SRVReflectionRadiance.ptr) { g_err = "ApplyReflectionsPass: missing draw parameters"; return; }
    if (pParams->UAVSceneRadiance.width != pParams->iSceneRTWidth || pParams->UAVSceneRadiance.height != pParams->iSceneRTHeight) {
        g_err = "ApplyReflectionsPass: iSceneRTWidth/Height do not match the scene radiance target"; return;
    }
    const bool bCompositeColor2 = pParams->SRVBoundingVolumes.ptr != nullptr;                       // ApplyReflections.cpp:52
    if (vq_apply_reflections(mRenderer.Context(), pParams->UAVSceneRadiance, pParams->SRVReflectionRadiance,
                             bCompositeColor2 ? &pParams->SRVBoundingVolumes : nullptr, pParams->pCmd) != VQ_OK)
        g_err = std::string("vq_apply_reflections: ") + vq_last_error();
}

std::vector<unsigned char> VQRenderer::SaveToHDRFileImage(const VqImage& Image) {
    std::vector<unsigned char> file((size_t)256 + (size_t)Image.width * Image.height * 6 + (size_t)Image.height * 8);
    uint64_t n = 0;
    if (vq_hdr_save_host(mCtx, Image, file.data(), file.size(), &n) != VQ_OK) { Fail("vq_hdr_save_host"); return {}; }
    file.resize((size_t)n);
    return file;
}

const VqImage* VQRenderer::RenderPostProcess(cudaStream_t pCmd, const FPostProcessParameters& PPParams, bool /*bHDR*/) {
    auto fail = [&](const char* w) -> const VqImage* { Fail(w); return nullptr; };
    VqImage colorIn = mSceneColor.View();
    if (PPParams.bEnableGaussianBlur) {                                    // SceneRendering.cpp:2582-2638
        const VqBlurParams bp{PPParams.SceneRTWidth, PPParams.SceneRTHeight};
        if (vq_gaussian_blur_x(mCtx, &bp, colorIn, mBlurTemp.View(), pCmd) != VQ_OK) return fail("vq_gaussian_blur_x");
        if (vq_gaussian_blur_y(mCtx, &bp, mBlurTemp.View(), mBlurOut.View(), pCmd) != VQ_OK) return fail("vq_gaussian_blur_y");
        colorIn = mBlurOut.View();
    }
    const FPostPlan plan = PlanPostProcess(PPParams);
    mLastOutput = plan.Output;
    if (vq_post_process(mCtx, &plan.Tonemapper, plan.CAS, plan.EASU, VQ_ADDRESS_WRAP, plan.RCAS, colorIn, mLastOutput, pCmd) != VQ_OK)
        return fail("vq_post_process");
    return &mLastOutput;                                                   // "return pRscOutput" SceneRendering.cpp:2787
}

// "TonemapperCS" (SceneRendering.cpp:2640-2656), then "FFX-CAS CS" (2658-2693) or "FSR-EASU CS" + "FSR-RCAS CS" (2695-2783):
// one launch, no intermediate images
VQRenderer::FPostPlan VQRenderer::PlanPostProcess(const FPostProcessParameters& PPParams) const {
    const bool bFSR = PPParams.IsFSREnabled(), bCAS = PPParams.IsFFXCASEnabled() && PPParams.Sharpness > 0.0f;
    return FPostPlan{VqTonemapperParams{(int)PPParams.TonemapperParams.ContentColorSpace, (int)PPParams.TonemapperParams.OutputDisplayCurve,
                                        PPParams.TonemapperParams.DisplayReferenceBrightnessLevel,
                                        PPParams.TonemapperParams.ToggleGammaCorrection, PPParams.TonemapperParams.UIHDRBrightness},
                     bCAS ? PPParams.FFXCASParams.CASConstantBlock : nullptr, bFSR ? PPParams.FSR_EASUParams.EASUConstantBlock : nullptr,
                     bFSR ? PPParams.FSR_RCASParams.RCASConstantBlock : nullptr, bFSR ? mRCASOut.View() : mPostOut.View()};
}

// ---- IRenderPass-shaped passes ---------------------------------------------------------------------
void GaussianBlurPass::OnCreateWindowSizeDependentResources(unsigned W, unsigned H, const IRenderPassResourceCollection*) { mTemp.Create((int)W, (int)H); }
void GaussianBlurPass::OnDestroyWindowSizeDependentResources() { mTemp.mem.Free(); }
void GaussianBlurPass::RecordCommands(const IRenderPassDrawParameters* p) {
    const auto* dp = static_cast<const FDrawParameters*>(p);
    if (!dp) return;
    const VqBlurParams bp{dp->In.width, dp->In.height};
    if (vq_gaussian_blur_x(mRenderer.Context(), &bp, dp->In, mTemp.View(), dp->pCmd) != VQ_OK) { Fail("GaussianBlurPass X"); return; }
    if (vq_gaussian_blur_y(mRenderer.Context(), &bp, mTemp.View(), dp->Out, dp->pCmd) != VQ_OK) Fail("GaussianBlurPass Y");
}

void SinglePassDownsamplerPass::OnCreateWindowSizeDependentResources(unsigned W, unsigned H, const IRenderPassResourceCollection*) {
    uint32_t dispatch[2]; const uint32_t rect[4] = {0, 0, W, H};
    vq_spd_setup(dispatch, &mConstants, rect, -1);
    mMips.clear();
    for (uint32_t l = 1; l <= mConstants.mips; ++l) {
        if ((W >> l) < 1 || (H >> l) < 1) { mConstants.mips = l - 1; break; }
        mMips.emplace_back(new FTexture2D());
        mMips.back()->Create((int)(W >> l), (int)(H >> l));
    }
}
void SinglePassDownsamplerPass::RecordCommands(const IRenderPassDrawParameters* p) {
    const auto* dp = static_cast<const FDrawParameters*>(p);
    if (!dp || mMips.empty()) return;
    std::vector<VqImage> views;
    for (auto& m : mMips) views.push_back(m->View());
    if (vq_spd_downsample(mRenderer.Context(), &mConstants, dp->In, views.data(), dp->pCmd) != VQ_OK) Fail("SinglePassDownsamplerPass");
}

// ---- VQRendererGroup: one frame over several GPUs of one process (DESIGN.md §6) -------------------------------------------
// A signalled kernel spins in its last CTA until every peer's kernel of the same phase has arrived. Three rules keep a group from
// waiting forever: (1) each phase's signalled call is enqueued on EVERY rank before anything that can block the host (a scratch
// growth, a blocking call, the next phase); (2) what can be checked is checked for all ranks before the first launch, and a rank
// refused after its peers were enqueued arrives in their flag arrays anyway (Phase, vq_group_arrive); (3) no signalled call grows context
// scratch: environments are registered by the group's prefilter, the shadowed G-buffer pass sizes its PCF records in an unsignalled
// local pass first, and OnWindowSizeChanged pre-sizes the context.
static bool GroupFail(const std::string& what) {
    g_err = what;
    std::fprintf(stderr, "[vq] error: %s\n", g_err.c_str());
    return false;
}

bool VQRendererGroup::Initialize(const std::vector<int>& Devices, uint32_t* const* FlagArrays, uint32_t FirstEpoch) {
    if (mGroup) return true;
    if (Devices.empty() || Devices.size() > 8) return GroupFail("VQRendererGroup::Initialize: 1..8 devices");
    for (int d : Devices) {
        mRanks.emplace_back(new VQRenderer());
        if (!mRanks.back()->Initialize(d)) { Destroy(); return false; }
        cudaStream_t s = nullptr;
        if (cudaSetDevice(d) != cudaSuccess || cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking) != cudaSuccess) {
            cudaGetLastError(); Destroy(); return GroupFail("VQRendererGroup::Initialize: stream creation failed");
        }
        mStreams.push_back(s);
    }
    std::vector<VqContext*> ctxs;
    for (auto& r : mRanks) ctxs.push_back(r->Context());
    if (vq_group_create(ctxs.data(), (int)ctxs.size(), FlagArrays, &mGroup) != VQ_OK) { Fail("vq_group_create"); Destroy(); return false; }
    mPrepared.assign(mRanks.size(), VqEnvironmentMaps{});
    mShadowRecordsSized.assign(mRanks.size(), 0);
    mDisplay.assign(mRanks.size(), VqImage{});
    mEpoch = FirstEpoch;
    mRendezvousFailed = false;
    return true;
}

void VQRendererGroup::Destroy() {
    for (size_t r = 0; r < mStreams.size(); ++r) { cudaSetDevice(mRanks[r]->Device()); cudaStreamSynchronize(mStreams[r]); cudaStreamDestroy(mStreams[r]); }
    mStreams.clear();
    if (mGroup) { vq_group_destroy(mGroup); mGroup = nullptr; }
    mRanks.clear();                                              // ~VQRenderer destroys each context
    mPrepared.clear(); mDisplay.clear();
    mShadowRecordsSized.clear();
}

std::vector<VqImage> VQRendererGroup::Targets(int r, const FTexture2D VQRenderer::* member) const {
    const int n = NumRanks();
    std::vector<VqImage> outs;
    for (int k = 0; k < n; ++k) outs.push_back(((*mRanks[(r + k) % n]).*member).View());
    return outs;
}

bool VQRendererGroup::Usable(const char* what) const {
    if (!mGroup) return GroupFail("VQRendererGroup: not initialized");
    if (mRendezvousFailed) return GroupFail(std::string(what) + ": a rendezvous failed; Resync() first");
    return true;
}

bool VQRendererGroup::SetRendezvousDeadline(uint64_t ns) {
    if (!mGroup) return GroupFail("VQRendererGroup: not initialized");
    VQ_TRY(vq_group_set_rendezvous_deadline(mGroup, ns), "vq_group_set_rendezvous_deadline");
    return true;
}

bool VQRendererGroup::RendezvousOK() {
    if (!mGroup) return GroupFail("VQRendererGroup: not initialized");
    std::string why;
    for (int r = 0; r < NumRanks(); ++r) {
        cudaSetDevice(mRanks[r]->Device());
        VqRendezvousStatus st;
        if (cudaStreamSynchronize(mStreams[r]) != cudaSuccess) { cudaGetLastError(); return GroupFail("RendezvousOK: device error"); }
        if (vq_ctx_rendezvous_status(mRanks[r]->mCtx, mStreams[r], &st) != VQ_OK) return Fail("vq_ctx_rendezvous_status");
        if (!st.failures) continue;
        why += (why.empty() ? "" : "; ") + std::string("rank ") + std::to_string(r) + ": " + std::to_string(st.failures) +
               " rendezvous gave up (epochs " + std::to_string(st.first_epoch) + ".." + std::to_string(st.last_epoch) +
               (st.cancelled ? ", cancelled" : "") + "), missing rank(s)";
        for (int j = 0; j < 8; ++j)
            if (st.missing_mask >> j & 1u) why += " " + std::to_string(j);
    }
    if (why.empty()) return true;
    mRendezvousFailed = true;
    return GroupFail("RendezvousOK: " + why);
}

bool VQRendererGroup::Resync() {
    if (!mGroup) return GroupFail("VQRendererGroup: not initialized");
    const uint32_t e = mEpoch++;
    for (int r = 0; r < NumRanks(); ++r) {
        VQ_TRY(vq_ctx_rendezvous_clear(mRanks[r]->mCtx, mStreams[r]), "vq_ctx_rendezvous_clear");
        VQ_TRY(vq_group_barrier(mGroup, r, e, mStreams[r]), "vq_group_barrier");
    }
    mRendezvousFailed = false;
    return RendezvousOK();
}

template <class F> bool VQRendererGroup::Phase(uint32_t epoch, F issue) {
    for (int r = 0; r < NumRanks(); ++r) {
        VqPeerSignal sig;
        if (vq_group_signal(mGroup, r, epoch, &sig) != VQ_OK || issue(r, sig) != VQ_OK) {
            std::string why = std::string("rank ") + std::to_string(r) + ": " + vq_last_error();
            // the refused rank and the ranks after it arrive in their peers' arrays, ordered after their earlier work
            for (int q = r; q < NumRanks(); ++q)
                if (vq_group_arrive(mGroup, q, epoch, mStreams[q]) != VQ_OK)
                    why += std::string("; the arrival of rank ") + std::to_string(q) + " failed: " + vq_last_error();
            return GroupFail(why);
        }
    }
    return true;
}

bool VQRendererGroup::LoadDefaultResources() {
    if (!Usable("LoadDefaultResources")) return false;
    for (auto& r : mRanks) {
        cudaSetDevice(r->Device());
        if (!r->mBRDFLUT.Create(1024, 1024, 8)) return false;    // Renderer.cpp:1026-1032
    }
    const int n = NumRanks();
    for (auto& m : mPrepared) m = VqEnvironmentMaps{};           // the registered maps include the LUT: prefilter again to register
    const uint32_t e = mEpoch++;
    const bool ok = Phase(e, [&](int r, const VqPeerSignal& sig) {
        int a, b;
        vq_band_rows(1024, n, r, 0, &a, &b);
        const std::vector<VqImage> outs = Targets(r, &VQRenderer::mBRDFLUT);
        return vq_brdf_integration_lut_multi_signal(mRanks[r]->Context(), outs.data(), n, 2048, a, b, &sig, mStreams[r]);
    });
    bool synced = true;
    for (int r = 0; r < n; ++r) synced = cudaStreamSynchronize(mStreams[r]) == cudaSuccess && synced;
    return ok && (synced || GroupFail("LoadDefaultResources: device error")) && RendezvousOK();
}

bool VQRendererGroup::OnWindowSizeChanged(int rw, int rh, int dw, int dh) {
    if (!mGroup) return GroupFail("VQRendererGroup: not initialized");
    const int n = NumRanks();
    for (int r = 0; r < n; ++r) {
        int a, b, c, d;
        if (vq_band_rows(rh, n, r, 1, &a, &b) != VQ_OK || vq_band_rows(dh, n, r, 0, &c, &d) != VQ_OK) return Fail("vq_band_rows");
        if (b <= a || d <= c)
            return GroupFail("OnWindowSizeChanged: " + std::to_string(rw) + "x" + std::to_string(rh) + " -> " + std::to_string(dw) + "x" +
                             std::to_string(dh) + " leaves rank " + std::to_string(r) + " an empty band over " + std::to_string(n) + " ranks");
    }
    for (int r = 0; r < n; ++r) { cudaSetDevice(mRanks[r]->Device()); cudaStreamSynchronize(mStreams[r]); }
    for (auto& r : mRanks)
        if (!r->OnWindowSizeChanged(rw, rh, dw, dh)) return false;
    for (auto& s : mShadowRecordsSized) s = 0;
    return true;
}

bool VQRendererGroup::PreFilterEnvironmentMap(const PerRank<FEnvironmentMapRenderingResources*>& envs, float step) {
    if (!Usable("PreFilterEnvironmentMap")) return false;
    const int n = NumRanks();
    if ((int)envs.size() != n) return GroupFail("PreFilterEnvironmentMap: one environment per rank");
    for (int r = 0; r < n; ++r) {
        const FEnvironmentMapRenderingResources* e = envs[r];
        if (!e || !e->Tex_HDREnvironment.ptr || !e->Tex_IrradianceDiff.ptr || !e->Tex_IrradianceSpec.ptr)
            return GroupFail("PreFilterEnvironmentMap: rank " + std::to_string(r) + " has no environment resources");
        if (e->DiffuseRes != envs[0]->DiffuseRes || e->SpecRes != envs[0]->SpecRes || e->SpecMips != envs[0]->SpecMips)
            return GroupFail("PreFilterEnvironmentMap: the ranks' cubes differ in shape");
        if (!mRanks[r]->mBRDFLUT.mem.ptr) return GroupFail("PreFilterEnvironmentMap: LoadDefaultResources first (the LUT is registered with the maps)");
    }
    if (n > 1 && 6 * envs[0]->DiffuseRes < n) return GroupFail("PreFilterEnvironmentMap: fewer diffuse rows than ranks");
    const uint32_t e = mEpoch;
    mEpoch += 2;
    for (auto& m : mPrepared) m = VqEnvironmentMaps{};
    auto cubes = [&](int r, bool spec) {
        std::vector<VqCubemap> outs;
        for (int k = 0; k < n; ++k) {
            const FEnvironmentMapRenderingResources& q = *envs[(r + k) % n];
            outs.push_back(spec ? q.Specular() : VqCubemap{q.Tex_IrradianceDiff.ptr, q.DiffuseRes, 1});
        }
        return outs;
    };
    // K2: the rank's band of the (face, row) space into every rank's diffuse cube, epoch e
    bool ok = Phase(e, [&](int r, const VqPeerSignal& sig) {
        int a, b;
        vq_band_rows(6 * envs[r]->DiffuseRes, n, r, 0, &a, &b);
        const VqDiffuseIrradianceParams dp = DiffuseParams(*envs[r], step);
        const std::vector<VqCubemap> outs = cubes(r, false);
        return vq_diffuse_irradiance_multi_signal(mRanks[r]->Context(), &dp, envs[r]->HDRI(), outs.data(), n, a, b, &sig, mStreams[r]);
    });
    // the blur of the whole local cube, then K3 on the rank's ranges into every rank's specular cube, epoch e + 1
    ok = ok && Phase(e + 1, [&](int r, const VqPeerSignal& sig) {
        const FEnvironmentMapRenderingResources& env = *envs[r];
        int rc = vq_gaussian_blur_cube(mRanks[r]->Context(), VqCubemap{env.Tex_IrradianceDiff.ptr, env.DiffuseRes, 1}, env.DiffuseBlurred(), mStreams[r]);
        if (rc != VQ_OK) return rc;
        int ranges[2 * 16], count = 0;
        rc = vq_specular_rank_ranges(env.SpecRes, env.SpecMips, n, r, ranges, 16, &count);
        if (rc != VQ_OK) return rc;
        const std::vector<VqCubemap> outs = cubes(r, true);
        return vq_specular_prefilter_ranges(mRanks[r]->Context(), env.HDRI(), outs.data(), n, 512, ranges, count, &sig, mStreams[r]);
    });
    // every rank's K3 is enqueued: registering the maps may now grow scratch (and wait for the device)
    for (int r = 0; ok && r < n; ++r) {
        const VqEnvironmentMaps maps = mRanks[r]->EnvironmentMaps(*envs[r]);
        if (vq_environment_prepare(mRanks[r]->Context(), &maps, mStreams[r]) != VQ_OK) ok = Fail("vq_environment_prepare");
        else mPrepared[r] = maps;
    }
    bool synced = true;
    for (int r = 0; r < n; ++r) { cudaSetDevice(mRanks[r]->Device()); synced = cudaStreamSynchronize(mStreams[r]) == cudaSuccess && synced; }
    if (!synced) { for (auto& m : mPrepared) m = VqEnvironmentMaps{}; return GroupFail("PreFilterEnvironmentMap: device error"); }
    if (ok && !RendezvousOK()) { for (auto& m : mPrepared) m = VqEnvironmentMaps{}; return false; }
    return ok;
}

// the frame's maps must be the ones vq_environment_prepare registered on each rank's context, descriptor for descriptor (the key
// the forward pass compares): any other maps would make the signalled shading call rebuild sampling copies in scratch (rule 3)
static bool SameMaps(const VqEnvironmentMaps& a, const VqEnvironmentMaps& b) {
    auto cube = [](const VqCubemap& x, const VqCubemap& y) { return x.ptr == y.ptr && x.res == y.res && x.mips == y.mips; };
    return a.irradiance_diffuse.ptr && cube(a.irradiance_diffuse, b.irradiance_diffuse) && cube(a.irradiance_specular, b.irradiance_specular) &&
           a.brdf_lut.ptr == b.brdf_lut.ptr && a.brdf_lut.width == b.brdf_lut.width && a.brdf_lut.height == b.brdf_lut.height &&
           a.brdf_lut.pitch_bytes == b.brdf_lut.pitch_bytes;
}

bool VQRendererGroup::Prepared(const PerRank<const FEnvironmentMapRenderingResources*>& envs) const {
    if ((int)envs.size() != NumRanks()) return GroupFail("one environment per rank");
    for (int r = 0; r < NumRanks(); ++r)
        if (!envs[r] || !SameMaps(mPrepared[r], mRanks[r]->EnvironmentMaps(*envs[r])))
            return GroupFail("rank " + std::to_string(r) + ": the environment was not registered by the group's PreFilterEnvironmentMap");
    return true;
}

// whether vq_forward_lighting_shadowed runs its PCF pass, and so needs its records in scratch: some light type with casters has
// its map bound (a NULL map lights that type unshadowed, vqcuda.h)
static bool PCFTestRuns(const VqSceneLighting& L, const VqShadowMaps& m) {
    return (m.point_cubes && L.numPointCasters > 0) || (m.spot_maps && L.numSpotCasters > 0) ||
           (m.directional_map && L.directional.enabled && L.directional.shadowing);
}

struct VQRendererGroup::FSceneCall {
    const FSceneView* View; const FPostProcessParameters* PP; const FGraphicsSettings* GFX; bool bHDR;
    const PerRank<const FEnvironmentMapRenderingResources*>* Envs;
    const PerRank<VqGBuffer>* GBuffers;                         // G-buffer calls
    const PerRank<VqSurfaceInputs>* Surfaces;                   // ... or from-materials calls
    const PerRank<const VqMaterialTable*>* Tables;
    bool bAlphaMask;
    const PerRank<VqShadowMaps>* ShadowMaps;                    // nullptr: no shadow maps bound
    const float* EnvironmentMapViewProj;                        // nullptr: no sky
};

bool VQRendererGroup::RenderScene(const FSceneCall& c) {
    if (!Usable("RenderSceneColor")) return false;
    const int n = NumRanks();
    const bool gbuf = c.GBuffers != nullptr;
    if (!mRanks[0]->mSceneColor.mem.ptr) return GroupFail("RenderSceneColor: OnWindowSizeChanged first");
    if (!Prepared(*c.Envs)) return false;
    if ((gbuf ? (int)c.GBuffers->size() : (int)c.Surfaces->size()) != n || (!gbuf && (int)c.Tables->size() != n) ||
        (c.ShadowMaps && (int)c.ShadowMaps->size() != n))
        return GroupFail("RenderSceneColor: one input per rank");
    for (int r = 0; r < n; ++r) {
        const VqImage& plane = gbuf ? (*c.GBuffers)[r].normal_roughness : (*c.Surfaces)[r].normal_v;
        if (!plane.ptr || (!gbuf && !(*c.Tables)[r])) return GroupFail("RenderSceneColor: rank " + std::to_string(r) + " has a null input");
    }
    VqMatrix inv{};
    if (c.EnvironmentMapViewProj && !Invert4x4(c.EnvironmentMapViewProj, inv.m)) return GroupFail("EnvironmentMapViewProj is singular");

    std::vector<VqPerFrameData> pf(n);
    std::vector<VqPerViewLightingData> pv(n);
    std::vector<VqEnvironmentMaps> maps(n);
    std::vector<std::pair<int, int>> band(n);
    for (int r = 0; r < n; ++r) {
        const FEnvironmentMapRenderingResources& env = *(*c.Envs)[r];
        mRanks[r]->FillSceneConstants(*c.View, *c.PP, env, *c.GFX, c.bHDR, pf[r], pv[r]);
        if (c.ShadowMaps) SetShadowMapDimensions((*c.ShadowMaps)[r], pf[r]);
        maps[r] = mRanks[r]->EnvironmentMaps(env);
        vq_band_rows(mRanks[r]->mSceneColor.height, n, r, 1, &band[r].first, &band[r].second);
    }
    const VqShadowMaps* none = nullptr;
    auto shadow = [&](int r) { return c.ShadowMaps ? &(*c.ShadowMaps)[r] : none; };
    // the rank's band into its own frame only, no rendezvous
    auto shadeLocal = [&](int r) {
        VQRenderer& R = *mRanks[r];
        const VqImage local = R.mSceneColor.View();
        const int a = band[r].first, b = band[r].second;
        if (gbuf)
            return c.ShadowMaps ? vq_forward_lighting_shadowed(R.mCtx, &pf[r], &pv[r], &(*c.GBuffers)[r], &maps[r], shadow(r), local, a, b, mStreams[r])
                                : vq_forward_lighting(R.mCtx, &pf[r], &pv[r], &(*c.GBuffers)[r], &maps[r], local, a, b, mStreams[r]);
        return c.ShadowMaps ? vq_forward_lighting_shadowed_from_materials(R.mCtx, &pf[r], &pv[r], &(*c.Surfaces)[r], (*c.Tables)[r], c.bAlphaMask,
                                                                          &maps[r], shadow(r), local, a, b, mStreams[r])
                            : vq_forward_lighting_from_materials(R.mCtx, &pf[r], &pv[r], &(*c.Surfaces)[r], (*c.Tables)[r], c.bAlphaMask, &maps[r],
                                                                 local, a, b, mStreams[r]);
    };
    const uint32_t e = mEpoch++;
    bool ok;
    if (c.EnvironmentMapViewProj) {
        // shading into the local frame on every rank, then the sky into every frame: one writer per pixel, one crossing
        for (int r = 0; r < n; ++r)
            if (shadeLocal(r) != VQ_OK) return Fail("RenderSceneColor (local band)");
        ok = Phase(e, [&](int r, const VqPeerSignal& sig) {
            const FEnvironmentMapRenderingResources& env = *(*c.Envs)[r];
            const VqPyramid level0{env.Tex_HDREnvironment.ptr, env.HDRIWidth, env.HDRIHeight, 1};   // Skydome.hlsl samples mip 0 only
            const VqImage& mask = gbuf ? (*c.GBuffers)[r].normal_roughness : (*c.Surfaces)[r].normal_v;
            const std::vector<VqImage> outs = Targets(r, &VQRenderer::mSceneColor);
            return vq_skydome_multi_signal(mRanks[r]->mCtx, &inv, level0, &mask, outs.data(), n, 0, band[r].first, band[r].second, &sig, mStreams[r]);
        });
    } else {
        // the shadowed G-buffer pass grows its PCF records on the first frame at a size that runs a test: do that unsignalled on
        // every such rank first
        for (int r = 0; gbuf && c.ShadowMaps && r < n; ++r)
            if (!mShadowRecordsSized[r] && PCFTestRuns(pf[r].Lights, (*c.ShadowMaps)[r])) {
                if (shadeLocal(r) != VQ_OK) return Fail("vq_forward_lighting_shadowed");
                mShadowRecordsSized[r] = 1;
            }
        ok = Phase(e, [&](int r, const VqPeerSignal& sig) {
            VQRenderer& R = *mRanks[r];
            const std::vector<VqImage> outs = Targets(r, &VQRenderer::mSceneColor);
            const int a = band[r].first, b = band[r].second;
            if (gbuf)
                return c.ShadowMaps ? vq_forward_lighting_shadowed_multi_signal(R.mCtx, &pf[r], &pv[r], &(*c.GBuffers)[r], &maps[r], shadow(r),
                                                                                outs.data(), n, 0, a, b, &sig, mStreams[r])
                                    : vq_forward_lighting_multi_signal(R.mCtx, &pf[r], &pv[r], &(*c.GBuffers)[r], &maps[r], outs.data(), n, 0, a, b,
                                                                       &sig, mStreams[r]);
            return vq_forward_lighting_from_materials_multi_signal(R.mCtx, &pf[r], &pv[r], &(*c.Surfaces)[r], (*c.Tables)[r], c.bAlphaMask,
                                                                   &maps[r], shadow(r), outs.data(), n, 0, a, b, &sig, mStreams[r]);
        });
    }
    // with a sky the local shade sized the records wherever a test ran
    for (int r = 0; ok && gbuf && c.ShadowMaps && c.EnvironmentMapViewProj && r < n; ++r)
        if (PCFTestRuns(pf[r].Lights, (*c.ShadowMaps)[r])) mShadowRecordsSized[r] = 1;
    return ok;
}

bool VQRendererGroup::RenderSceneColor(const FSceneView& SceneView, const FPostProcessParameters& PPParams, const PerRank<VqGBuffer>& GBuffers,
                                       const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                                       bool bHDR, const float* EnvironmentMapViewProj) {
    return RenderScene(FSceneCall{&SceneView, &PPParams, &GFXSettings, bHDR, &envs, &GBuffers, nullptr, nullptr, false, nullptr,
                                  EnvironmentMapViewProj});
}
bool VQRendererGroup::RenderSceneColorFromMaterials(const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                                    const PerRank<VqSurfaceInputs>& SurfaceInputs, const PerRank<const VqMaterialTable*>& MaterialTables,
                                                    const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                                                    bool bHDR, const float* EnvironmentMapViewProj, bool bAlphaMask) {
    return RenderScene(FSceneCall{&SceneView, &PPParams, &GFXSettings, bHDR, &envs, nullptr, &SurfaceInputs, &MaterialTables, bAlphaMask,
                                  nullptr, EnvironmentMapViewProj});
}
bool VQRendererGroup::RenderSceneColor(const FSceneView& SceneView, const FPostProcessParameters& PPParams, const PerRank<VqGBuffer>& GBuffers,
                                       const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                                       bool bHDR, const PerRank<VqShadowMaps>& ShadowMaps, const float* EnvironmentMapViewProj) {
    return RenderScene(FSceneCall{&SceneView, &PPParams, &GFXSettings, bHDR, &envs, &GBuffers, nullptr, nullptr, false, &ShadowMaps,
                                  EnvironmentMapViewProj});
}
bool VQRendererGroup::RenderSceneColorFromMaterials(const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                                    const PerRank<VqSurfaceInputs>& SurfaceInputs, const PerRank<const VqMaterialTable*>& MaterialTables,
                                                    const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                                                    bool bHDR, const PerRank<VqShadowMaps>& ShadowMaps, const float* EnvironmentMapViewProj,
                                                    bool bAlphaMask) {
    return RenderScene(FSceneCall{&SceneView, &PPParams, &GFXSettings, bHDR, &envs, nullptr, &SurfaceInputs, &MaterialTables, bAlphaMask,
                                  &ShadowMaps, EnvironmentMapViewProj});
}

bool VQRendererGroup::ApplyReflections(const PerRank<VqImage>& ReflectionRadiance, const PerRank<VqImage>* BoundingVolumes) {
    if (!Usable("ApplyReflections")) return false;
    const int n = NumRanks();
    if (!mRanks[0]->mSceneColor.mem.ptr) return GroupFail("ApplyReflections: OnWindowSizeChanged first");
    if ((int)ReflectionRadiance.size() != n || (BoundingVolumes && (int)BoundingVolumes->size() != n))
        return GroupFail("ApplyReflections: one input per rank");
    for (int r = 0; r < n; ++r)
        if (!ReflectionRadiance[r].ptr) return GroupFail("ApplyReflections: rank " + std::to_string(r) + " has no reflection radiance");
    const uint32_t e = mEpoch++;
    return Phase(e, [&](int r, const VqPeerSignal& sig) {
        int a, b;
        vq_band_rows(mRanks[r]->mSceneColor.height, n, r, 1, &a, &b);
        const std::vector<VqImage> outs = Targets(r, &VQRenderer::mSceneColor);
        return vq_apply_reflections_multi_signal(mRanks[r]->mCtx, ReflectionRadiance[r], BoundingVolumes ? &(*BoundingVolumes)[r] : nullptr,
                                                 outs.data(), n, 0, a, b, &sig, mStreams[r]);
    });
}

const VqImage* VQRendererGroup::RenderPostProcess(const FPostProcessParameters& PPParams, bool /*bHDR*/) {
    if (!Usable("RenderPostProcess")) return nullptr;
    if (PPParams.bEnableGaussianBlur) { GroupFail("RenderPostProcess: the Gaussian blur has no band form in a group"); return nullptr; }
    if (!mRanks[0]->mSceneColor.mem.ptr) { GroupFail("RenderPostProcess: OnWindowSizeChanged first"); return nullptr; }
    const int n = NumRanks();
    std::vector<VQRenderer::FPostPlan> plan;
    for (auto& R : mRanks) plan.push_back(R->PlanPostProcess(PPParams));
    const uint32_t e = mEpoch++;
    const bool ok = Phase(e, [&](int r, const VqPeerSignal& sig) {
        const VQRenderer::FPostPlan& p = plan[r];
        std::vector<VqImage> outs;
        for (int k = 0; k < n; ++k) outs.push_back(plan[(r + k) % n].Output);
        int a, b;
        vq_band_rows(p.Output.height, n, r, 0, &a, &b);
        return vq_post_process_multi_signal(mRanks[r]->mCtx, &p.Tonemapper, p.CAS, p.EASU, VQ_ADDRESS_WRAP, p.RCAS, mRanks[r]->mSceneColor.View(),
                                            outs.data(), n, a, b, &sig, mStreams[r]);
    });
    if (!ok) return nullptr;
    for (int r = 0; r < n; ++r) mDisplay[r] = plan[r].Output;
    return mDisplay.data();
}

}  // namespace vq
