// vq_renderer.cpp — C++ host layer: fills the constant blocks exactly where the engine does and dispatches the
// C-ABI passes in the engine's order. No pixel math here.
#include "vq_renderer.hpp"

#include <cuda_runtime_api.h>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>

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
    return true;
}
void VQRenderer::Destroy() {
    if (mCtx) { cudaDeviceSynchronize(); vq_ctx_destroy(mCtx); mCtx = nullptr; }
}
bool VQRenderer::LoadDefaultResources() {
    // CreateProceduralTextures LUT desc (Renderer.cpp:1026-1032): 1024x1024; ComputeBRDFIntegrationLUT: 2048 samples
    if (!mBRDFLUT.Create(1024, 1024, 8)) return false;
    VQ_TRY(vq_brdf_integration_lut(mCtx, mBRDFLUT.View(), 2048, 0, 1024, nullptr), "vq_brdf_integration_lut");
    return cudaStreamSynchronize(nullptr) == cudaSuccess;
}
bool VQRenderer::OnWindowSizeChanged(int rw, int rh, int dw, int dh) {
    return mSceneColor.Create(rw, rh) && mBlurTemp.Create(rw, rh) && mBlurOut.Create(rw, rh) && mPostOut.Create(rw, rh) &&
           mRCASOut.Create(dw, dh) && vq_ctx_resize(mCtx, rw, rh) == VQ_OK;
}

bool VQRenderer::PreFilterEnvironmentMap(FEnvironmentMapRenderingResources& env, float DiffuseIntegrationStep) {
    // Diffuse irradiance convolution (EnvironmentMapRendering.cpp:181-277): 6 per-face draws -> one launch
    VqDiffuseIrradianceParams dp{DiffuseIntegrationStep, 0, 0, 3 < env.HDRIMips ? 3 : env.HDRIMips - 1};
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

bool VQRenderer::RenderSceneColor(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                  const VqGBuffer& GBuffer, const FEnvironmentMapRenderingResources& env,
                                  const FGraphicsSettings& GFXSettings, bool bHDRDisplay) {
    VqPerFrameData PerFrame;
    VqPerViewLightingData PerView;
    FillSceneConstants(SceneView, PPParams, env, GFXSettings, bHDRDisplay, PerFrame, PerView);
    // IBL SRVs (SceneRendering.cpp:1690-1717): blurred diffuse irradiance, prefiltered specular, BRDF LUT
    VqEnvironmentMaps maps{env.DiffuseBlurred(), env.Specular(), mBRDFLUT.View()};
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
    VqEnvironmentMaps maps{env.DiffuseBlurred(), env.Specular(), mBRDFLUT.View()};
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
    VqEnvironmentMaps maps{env.DiffuseBlurred(), env.Specular(), mBRDFLUT.View()};
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
    VqEnvironmentMaps maps{env.DiffuseBlurred(), env.Specular(), mBRDFLUT.View()};
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
    // "TonemapperCS" (SceneRendering.cpp:2640-2656), then "FFX-CAS CS" (2658-2693) or "FSR-EASU CS" + "FSR-RCAS CS" (2695-2783):
    // one launch, no intermediate images
    const VqTonemapperParams tp{(int)PPParams.TonemapperParams.ContentColorSpace, (int)PPParams.TonemapperParams.OutputDisplayCurve,
                                PPParams.TonemapperParams.DisplayReferenceBrightnessLevel, PPParams.TonemapperParams.ToggleGammaCorrection,
                                PPParams.TonemapperParams.UIHDRBrightness};
    const bool bFSR = PPParams.IsFSREnabled(), bCAS = PPParams.IsFFXCASEnabled() && PPParams.Sharpness > 0.0f;
    mLastOutput = bFSR ? mRCASOut.View() : mPostOut.View();
    if (vq_post_process(mCtx, &tp, bCAS ? PPParams.FFXCASParams.CASConstantBlock : nullptr,
                        bFSR ? PPParams.FSR_EASUParams.EASUConstantBlock : nullptr, VQ_ADDRESS_WRAP,
                        bFSR ? PPParams.FSR_RCASParams.RCASConstantBlock : nullptr, colorIn, mLastOutput, pCmd) != VQ_OK)
        return fail("vq_post_process");
    return &mLastOutput;                                                   // "return pRscOutput" SceneRendering.cpp:2787
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

}  // namespace vq
