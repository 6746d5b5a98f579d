// vq_renderer.hpp — C++ host layer over the C-ABI (include/vqcuda.h), shaped like the reference's
// renderer front end so that an engine integration reads like the original call sites:
//
//   reference (D3D12)                                              here (CUDA, headless)
//   -------------------------------------------------------------  ---------------------------------------------
//   VQRenderer::RenderSceneColor(pCmd, pCBufferHeap, SceneView,    vq::VQRenderer::RenderSceneColor(pCmd = stream,
//       PPParams, cbPerView, cbPerFrame, GFXSettings, bHDR)            SceneView, PPParams, GBuffer, GFXSettings, bHDR)
//       Renderer.h:470, SceneRendering.cpp:1619-1851
//   VQRenderer::RenderPostProcess(pCmd, pCBufferHeap, PPParams,    vq::VQRenderer::RenderPostProcess(pCmd, PPParams, bHDR)
//       bHDR) -> ID3D12Resource*     Renderer.h:482                    -> const VqImage* (the last image written)
//   VQRenderer::PreFilterEnvironmentMap(const Mesh&)               vq::VQRenderer::PreFilterEnvironmentMap()   (blocks)
//       Renderer.h:249, EnvironmentMapRendering.cpp:139-486
//   FEnvironmentMapRenderingResources::CreateRenderingResources    same name; HDRI comes from a host RGBA32F pointer
//       EnvironmentMapRendering.h:66
//   ComputeBRDFIntegrationLUT / LoadDefaultResources               vq::VQRenderer::LoadDefaultResources()
//       Renderer.cpp:871-974
//   IRenderPass (RenderPass.h:44-59)                               vq::IRenderPass + concrete passes below
//
// `pCmd` (ID3D12GraphicsCommandList*) becomes a cudaStream_t: recording == enqueueing; per-thread command
// lists == per-thread streams. `pCBufferHeap` disappears: constant blocks are passed by value.
// Errors follow the reference's conventions: bool / early return + Log::Error (here: vq::LastError()).
#pragma once
#include <cstdint>
#include <memory>
#include <string>
#include <vector>

#include "../../include/vqcuda.h"
#include "../../include/vqcuda_group.h"

typedef struct CUstream_st* cudaStream_t;

namespace vq {

const char* LastError();

// ---- device resources (replace TextureID / SRV_ID / UAV_ID; owned by the renderer like in the engine) ----
struct FDeviceBuffer {
    void* ptr = nullptr; size_t bytes = 0;
    bool Alloc(size_t n); void Free();
    ~FDeviceBuffer() { Free(); }
    FDeviceBuffer() = default; FDeviceBuffer(const FDeviceBuffer&) = delete; FDeviceBuffer& operator=(const FDeviceBuffer&) = delete;
};
struct FTexture2D {            // RGBA32F (texelBytes 16) or RG32F (8)
    FDeviceBuffer mem; int width = 0, height = 0, texelBytes = 16;
    bool Create(int w, int h, int texelBytes_ = 16);
    VqImage View() const { return VqImage{mem.ptr, width, height, (size_t)width * (size_t)texelBytes}; }
};

// ---- parameter bundles the engine hands to the renderer (reference: Source/Engine/...) ----
enum class EColorSpace { REC_709 = 0, REC_2020 };                               // Renderer/Rendering/HDR.h
enum class EDisplayCurve { sRGB = 0, ST2084, Linear };
enum class EReflections { REFLECTIONS_OFF = 0, SCREEN_SPACE_REFLECTIONS__FFX };  // Settings.h

struct FGraphicsSettings {                                                       // Settings.h:39-53 (used fields)
    EReflections Reflections = EReflections::REFLECTIONS_OFF;
    int EnvironmentMapResolution = 512;                                          // Data/EngineSettings.ini:11
};

struct FSceneView {                                                              // Scene/SceneViews.h:177 (used fields)
    VqSceneLighting GPULightingData{};
    VqFloat3 cameraPosition{0, 0, 0};
    float HDRIYawOffset = 0.0f;
    struct { float fAmbientLightingFactor = 0.055f; } sceneRenderOptions;
};

struct FPostProcessParameters {                                                  // PostProcess/PostProcess.h:74-172
    enum EUpscalingAlgorithm { NONE = 0, FIDELITYFX_SUPER_RESOLUTION1, NUM_UPSCALING_ALGORITHMS };
    struct FTonemapper {
        EColorSpace ContentColorSpace = EColorSpace::REC_709;
        EDisplayCurve OutputDisplayCurve = EDisplayCurve::sRGB;
        float DisplayReferenceBrightnessLevel = 200.0f;
        int ToggleGammaCorrection = 1;
        float UIHDRBrightness = 1.0f;
    };
    struct FBlurParams { int iImageSizeX, iImageSizeY; };
    struct FFFXCAS {
        float CASSharpen = 0.8f;
        void UpdateCASConstantBlock(unsigned InputWidth, unsigned InputHeight, unsigned OutputWidth, unsigned OutputHeight);
        unsigned CASConstantBlock[8]{};
    };
    struct FFSR1_EASU {
        void UpdateEASUConstantBlock(unsigned InputWidth, unsigned InputHeight, unsigned InputContainerWidth,
                                     unsigned InputContainerHeight, unsigned OutputWidth, unsigned OutputHeight);
        unsigned EASUConstantBlock[16]{};
    };
    struct FFSR1_RCAS {
        float GetLinearSharpness() const;
        void SetLinearSharpness(float Sharpness);
        void UpdateRCASConstantBlock();
        unsigned RCASConstantBlock[4]{};
        float RCASSharpnessStops = 0.2f;
    };
    bool IsFSREnabled() const { return UpscalingAlgorithm == FIDELITYFX_SUPER_RESOLUTION1; }
    bool IsFFXCASEnabled() const { return !IsFSREnabled() && bEnableCAS; }

    int SceneRTWidth = 0, SceneRTHeight = 0;
    int DisplayResolutionWidth = 0, DisplayResolutionHeight = 0;
    FTonemapper TonemapperParams{};
    FBlurParams BlurParams{};
    EUpscalingAlgorithm UpscalingAlgorithm = FIDELITYFX_SUPER_RESOLUTION1;
    FFSR1_EASU FSR_EASUParams{};
    FFSR1_RCAS FSR_RCASParams{};
    FFFXCAS FFXCASParams{};
    float Sharpness = 0.8f;
    bool bEnableCAS = false;            // compiled out in the engine (DISABLE_FIDELITYFX_CAS); selectable here
    bool bEnableGaussianBlur = false;   // `constexpr false` in the engine (SceneRendering.cpp:2526); selectable here
};

// ---- environment map bundle (EnvironmentMapRendering.h:26-68) ----
struct FEnvironmentMapDescriptor {      // the engine loads a file; headless callers hand over RGBA32F texels
    const float* pHDRIData = nullptr; int Width = 0, Height = 0; float MaxContentLightLevel = 0.0f;
};
class VQRenderer;
struct FEnvironmentMapRenderingResources {
    FDeviceBuffer Tex_HDREnvironment;          // equirect + min-filter mip pyramid
    FDeviceBuffer Tex_IrradianceDiff, Tex_IrradianceDiffBlurred, Tex_BlurTemp, Tex_IrradianceSpec;
    int HDRIWidth = 0, HDRIHeight = 0, HDRIMips = 0;
    int DiffuseRes = 0, SpecRes = 0, SpecMips = 0;
    int MaxContentLightLevel = 0;
    bool CreateRenderingResources(VQRenderer& Renderer, const FEnvironmentMapDescriptor& desc,
                                  int DiffuseIrradianceCubemapResolution, int SpecularMapMip0Resolution);
    // the engine's own route: a Radiance .hdr file image (Image::LoadFromFile, Libs/VQUtils/Source/Image.cpp:88-140, then
    // TextureManager upload). The file is decoded ON THE DEVICE straight into level 0 of the pyramid (vq_hdr_load_host);
    // MaxContentLightLevel = Image::MaxLuminance as the engine computes it.
    bool CreateRenderingResourcesFromHDRFile(VQRenderer& Renderer, const void* pFileBytes, size_t NumBytes,
                                             int DiffuseIrradianceCubemapResolution, int SpecularMapMip0Resolution);
    void DestroyRenderingResources();
    int GetNumSpecularIrradianceCubemapLODLevels() const { return SpecMips; }
    VqPyramid HDRI() const { return VqPyramid{Tex_HDREnvironment.ptr, HDRIWidth, HDRIHeight, HDRIMips}; }
    VqCubemap DiffuseBlurred() const { return VqCubemap{Tex_IrradianceDiffBlurred.ptr, DiffuseRes, 1}; }
    VqCubemap Specular() const { return VqCubemap{Tex_IrradianceSpec.ptr, SpecRes, SpecMips}; }
};

// ---- Data/EnvironmentMaps.ini (FileParser::ParseEnvironmentMapsFile, Source/Engine/Core/FileParser.cpp:264-321) ----
// "[Name]" sections with "Path=" and "MaxCLL=" keys, ';' comment lines. Host-only text parsing; the engine's quirk that a new
// section only closes the previous one after an empty line is kept.
struct FEnvironmentMapFileDescriptor {      // Source/Engine/EnvironmentMap.h:23-28
    std::string Name, FilePath; float MaxContentLightLevel = 0.0f;
};
std::vector<FEnvironmentMapFileDescriptor> ParseEnvironmentMapsINI(const std::string& FileContents);

// CreateEnvironmentMapTextureFromHiResAndSaveToDisk (Source/Engine/EnvironmentMap.cpp:142-209) on file images: decode the
// hi-res .hdr, Image::CreateResizedImage to TargetWidth x TargetHeight (the engine's table: 8k 8192x4096, 4k 4096x2048,
// 2k 2048x1024, 1k 1024x512), Image::SaveToDisk — all three steps on the device. Returns the smaller file image (empty on failure).
std::vector<unsigned char> CreateEnvironmentMapFileImageFromHiRes(VQRenderer& Renderer, const void* pHiResFileBytes, size_t NumBytes,
                                                                  int TargetWidth, int TargetHeight);

// ---- IRenderPass (RenderPass.h:25-59) ----
struct IRenderPassResourceCollection {};
struct IRenderPassDrawParameters {};
class IRenderPass {
public:
    virtual ~IRenderPass() = default;
    virtual bool Initialize() = 0;
    virtual void Destroy() = 0;
    virtual void OnCreateWindowSizeDependentResources(unsigned Width, unsigned Height, const IRenderPassResourceCollection* pRscParameters = nullptr) = 0;
    virtual void OnDestroyWindowSizeDependentResources() = 0;
    virtual void RecordCommands(const IRenderPassDrawParameters* pDrawParameters = nullptr) = 0;
};
class RenderPassBase : public IRenderPass {
protected:
    explicit RenderPassBase(VQRenderer& RendererIn) : mRenderer(RendererIn) {}
    VQRenderer& mRenderer;
};

// A compute pass in the reference's canonical shape (ApplyReflections.h:30-39): FDrawParameters carries the
// command list (stream) and the resources by handle.
class GaussianBlurPass : public RenderPassBase {
public:
    struct FDrawParameters : IRenderPassDrawParameters {
        cudaStream_t pCmd = nullptr; VqImage In{}, Out{};   // Out = blurred result, same size
    };
    explicit GaussianBlurPass(VQRenderer& r) : RenderPassBase(r) {}
    bool Initialize() override { return true; }
    void Destroy() override { OnDestroyWindowSizeDependentResources(); }
    void OnCreateWindowSizeDependentResources(unsigned W, unsigned H, const IRenderPassResourceCollection* = nullptr) override;
    void OnDestroyWindowSizeDependentResources() override;
    void RecordCommands(const IRenderPassDrawParameters* pDrawParameters = nullptr) override;   // X then Y through mTemp
private:
    FTexture2D mTemp;
};

class SinglePassDownsamplerPass : public RenderPassBase {   // FidelityFX SPD, AMDFidelityFX.hlsl:525-545
public:
    struct FDrawParameters : IRenderPassDrawParameters { cudaStream_t pCmd = nullptr; VqImage In{}; };
    explicit SinglePassDownsamplerPass(VQRenderer& r) : RenderPassBase(r) {}
    bool Initialize() override { return true; }
    void Destroy() override { OnDestroyWindowSizeDependentResources(); }
    void OnCreateWindowSizeDependentResources(unsigned W, unsigned H, const IRenderPassResourceCollection* = nullptr) override;
    void OnDestroyWindowSizeDependentResources() override { mMips.clear(); }
    void RecordCommands(const IRenderPassDrawParameters* pDrawParameters = nullptr) override;
    const std::vector<std::unique_ptr<FTexture2D>>& Mips() const { return mMips; }
private:
    std::vector<std::unique_ptr<FTexture2D>> mMips; VqSpdConstants mConstants{};
};

// ApplyReflectionsPass (Source/Renderer/Rendering/RenderPass/ApplyReflections.h:27-57): the one dispatch of the hot path that the
// reference itself wraps in an IRenderPass. FDrawParameters keeps its field names; SRV/UAV ids become image descriptors, the
// command list becomes a stream, pCBufferHeap disappears. SRVBoundingVolumes.ptr == nullptr == INVALID_ID selects the variant
// without COMPOSITE_BOUNDING_VOLUMES (ApplyReflections.cpp:52,62).
class ApplyReflectionsPass : public RenderPassBase {
public:
    struct FResourceCollection : IRenderPassResourceCollection {};
    struct FDrawParameters : IRenderPassDrawParameters {
        cudaStream_t pCmd = nullptr;
        VqImage SRVReflectionRadiance{};
        VqImage SRVBoundingVolumes{};
        VqImage UAVSceneRadiance{};
        int iSceneRTWidth = 0, iSceneRTHeight = 0;
    };
    explicit ApplyReflectionsPass(VQRenderer& r) : RenderPassBase(r) {}
    bool Initialize() override { return true; }
    void Destroy() override {}
    void OnCreateWindowSizeDependentResources(unsigned, unsigned, const IRenderPassResourceCollection* = nullptr) override {}
    void OnDestroyWindowSizeDependentResources() override {}
    void RecordCommands(const IRenderPassDrawParameters* pDrawParameters = nullptr) override;
};

// ---- the renderer front end ----
class VQRenderer {
public:
    VQRenderer() = default;
    ~VQRenderer() { Destroy(); }
    bool Initialize(int DeviceIndex = 0);                       // Renderer.cpp:Initialize (device + default queues)
    void Destroy();
    bool LoadDefaultResources();                                // BRDF integration LUT, 1024^2, 2048 samples (Renderer.cpp:912-974)
    bool OnWindowSizeChanged(int RenderW, int RenderH, int DisplayW, int DisplayH);   // window-size dependent targets

    // EnvironmentMapRendering.cpp:139-486: diffuse convolution -> per-face blur -> specular prefilter; BLOCKS like the engine
    bool PreFilterEnvironmentMap(FEnvironmentMapRenderingResources& env, float DiffuseIntegrationStep = 0.010f);

    bool RenderSceneColor(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                          const VqGBuffer& GBuffer, const FEnvironmentMapRenderingResources& env,
                          const FGraphicsSettings& GFXSettings, bool bHDR);
    // RenderSceneColor with PSMain run end to end from what the rasteriser interpolates and the scene's materials (one launch,
    // no G-buffer: vq_forward_lighting_from_materials); bAlphaMask selects the ENABLE_ALPHA_MASK variant. SceneColor must have
    // the size of the attribute planes.
    bool RenderSceneColorFromMaterials(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                       const VqSurfaceInputs& SurfaceInputs, const VqMaterialTable* MaterialTable,
                                       const FEnvironmentMapRenderingResources& env, const FGraphicsSettings& GFXSettings,
                                       bool bHDR, bool bAlphaMask = false);
    // The same two passes with the engine's shadow maps bound (ForwardLighting.hlsl:87-89, 321-377): vq_forward_lighting_shadowed
    // and vq_forward_lighting_shadowed_from_materials. The f2*ShadowMapDimensions constants are those of the bound maps.
    bool RenderSceneColor(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                          const VqGBuffer& GBuffer, const FEnvironmentMapRenderingResources& env,
                          const FGraphicsSettings& GFXSettings, bool bHDR, const VqShadowMaps& ShadowMaps);
    bool RenderSceneColorFromMaterials(cudaStream_t pCmd, const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                       const VqSurfaceInputs& SurfaceInputs, const VqMaterialTable* MaterialTable,
                                       const FEnvironmentMapRenderingResources& env, const FGraphicsSettings& GFXSettings,
                                       bool bHDR, const VqShadowMaps& ShadowMaps, bool bAlphaMask = false);
    const VqImage* RenderPostProcess(cudaStream_t pCmd, const FPostProcessParameters& PPParams, bool bHDR);
    // "Draw Environment Map" (SceneRendering.cpp:1821-1850, Skydome.hlsl): fills the pixels of SceneColor that no surface
    // covered (normal plane == 0) with the equirect HDRI seen through EnvironmentMapViewProj (row-major, row-vector
    // convention as XMMATRIX; SceneView.EnvironmentMapViewProj, Scene.cpp:573-584). Call after RenderSceneColor.
    bool RenderEnvironmentMap(cudaStream_t pCmd, const float EnvironmentMapViewProj[16], const VqGBuffer& GBuffer,
                              const FEnvironmentMapRenderingResources& env);
    // ApplyReflectionsPass::RecordCommands (ApplyReflections.hlsl:31-57): SceneColor.rgb += ReflectionRadiance.rgb
    bool ApplyReflections(cudaStream_t pCmd, const VqImage& ReflectionRadiance, const VqImage* BoundingVolumes = nullptr);
    // Image::SaveToDisk for .hdr (Image.cpp:192-220): returns the file image (empty on failure)
    std::vector<unsigned char> SaveToHDRFileImage(const VqImage& Image);

    VqContext* Context() const { return mCtx; }
    int Device() const { return mDevice; }
    const FTexture2D& SceneColor() const { return mSceneColor; }
    const FTexture2D& BRDFIntegrationLUT() const { return mBRDFLUT; }

private:
    friend class VQRendererGroup;   // binds each rank's targets and reuses the constant blocks and the post branch below
    void FillSceneConstants(const FSceneView& SceneView, const FPostProcessParameters& PPParams, const FEnvironmentMapRenderingResources& env,
                            const FGraphicsSettings& GFXSettings, bool bHDR, VqPerFrameData& PerFrame, VqPerViewLightingData& PerView) const;
    VqEnvironmentMaps EnvironmentMaps(const FEnvironmentMapRenderingResources& env) const;   // the IBL SRVs PSMain binds
    // RenderPostProcess's branch: the constant blocks of the passes that run (NULL: off) and the target they write
    struct FPostPlan { VqTonemapperParams Tonemapper; const uint32_t *CAS, *EASU, *RCAS; VqImage Output; };
    FPostPlan PlanPostProcess(const FPostProcessParameters& PPParams) const;
    VqContext* mCtx = nullptr;
    int mDevice = 0;
    FTexture2D mBRDFLUT;                                        // EProceduralTextures::IBL_BRDF_INTEGRATION_LUT
    FTexture2D mSceneColor, mBlurTemp, mBlurOut;
    FTexture2D mPostOut;                                        // RenderPostProcess's output without FSR (render size)
    FTexture2D mRCASOut;                                        // ... with FSR (display size)
    VqImage mLastOutput{};
};

// ---- the renderer front end over a device group (vqcuda_group.h): one frame strong-scaled over several GPUs of one process ----
// One VQRenderer per rank (its own context, BRDF LUT, scene colour and post targets, Rank(r)) and one non-blocking stream per rank
// (Stream(r)). Each method runs the engine call of the same name across the group with the band forms of the passes underneath:
// every rank computes its band and stores it into every rank's target, and the kernels' last CTAs meet (DESIGN.md §6), so every
// rank ends each method holding the whole LUT, cube or frame. Inputs that live on a device come one per rank, in rank order
// (G-buffers, surface inputs, material tables, shadow maps, environment resources, reflection radiance). The frame methods only
// enqueue on the ranks' streams; LoadDefaultResources and PreFilterEnvironmentMap block, like the engine's.
// Ranks may share a device (a simulated world: Initialize({0, 0})). Each rank's per-rank resources are made on its device:
// call cudaSetDevice(Rank(r).Device()) before allocating them (FEnvironmentMapRenderingResources does that itself).
class VQRendererGroup {
public:
    template <class T> using PerRank = std::vector<T>;
    VQRendererGroup() = default;
    ~VQRendererGroup() { Destroy(); }
    VQRendererGroup(const VQRendererGroup&) = delete; VQRendererGroup& operator=(const VQRendererGroup&) = delete;

    // one rank per entry of Devices (1..8); FlagArrays: nullptr -> the group allocates the flag words, else one caller-owned array
    // of NumRanks words per rank that every rank's device can reach, all holding FirstEpoch - 1 (zero for the default)
    bool Initialize(const std::vector<int>& Devices, uint32_t* const* FlagArrays = nullptr, uint32_t FirstEpoch = 1);
    void Destroy();
    int NumRanks() const { return (int)mRanks.size(); }
    VQRenderer& Rank(int r) { return *mRanks[r]; }
    cudaStream_t Stream(int r) const { return mStreams[r]; }
    const VqGroup* Group() const { return mGroup; }
    uint32_t Epoch() const { return mEpoch; }                  // the epoch the next signalled phase uses

    bool LoadDefaultResources();                               // BLOCKS; each rank computes its band of the LUT into every LUT
    // refused when a rank's scene band (even rows) or display band would be empty
    bool OnWindowSizeChanged(int RenderW, int RenderH, int DisplayW, int DisplayH);
    // BLOCKS. K2 band (epoch e) -> the cube blur locally -> K3 ranges (e + 1) -> vq_environment_prepare, on every rank; the frames
    // below accept only the maps (cubes and LUT, as descriptors) the last call registered on each rank
    bool PreFilterEnvironmentMap(const PerRank<FEnvironmentMapRenderingResources*>& envs, float DiffuseIntegrationStep = 0.010f);

    // VQRenderer's four scene-colour calls on each rank's scene band. EnvironmentMapViewProj (nullptr: no sky) draws the skydome
    // as the engine's RenderSceneColor does (SceneRendering.cpp:1821-1850): shading into the local frame, then the sky pass into
    // every frame. Without a sky the shading call stores into every frame itself.
    bool RenderSceneColor(const FSceneView& SceneView, const FPostProcessParameters& PPParams, const PerRank<VqGBuffer>& GBuffers,
                          const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                          bool bHDR, const float* EnvironmentMapViewProj);
    bool RenderSceneColorFromMaterials(const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                       const PerRank<VqSurfaceInputs>& SurfaceInputs, const PerRank<const VqMaterialTable*>& MaterialTables,
                                       const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                                       bool bHDR, const float* EnvironmentMapViewProj, bool bAlphaMask = false);
    bool RenderSceneColor(const FSceneView& SceneView, const FPostProcessParameters& PPParams, const PerRank<VqGBuffer>& GBuffers,
                          const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                          bool bHDR, const PerRank<VqShadowMaps>& ShadowMaps, const float* EnvironmentMapViewProj);
    bool RenderSceneColorFromMaterials(const FSceneView& SceneView, const FPostProcessParameters& PPParams,
                                       const PerRank<VqSurfaceInputs>& SurfaceInputs, const PerRank<const VqMaterialTable*>& MaterialTables,
                                       const PerRank<const FEnvironmentMapRenderingResources*>& envs, const FGraphicsSettings& GFXSettings,
                                       bool bHDR, const PerRank<VqShadowMaps>& ShadowMaps, const float* EnvironmentMapViewProj,
                                       bool bAlphaMask = false);
    bool ApplyReflections(const PerRank<VqImage>& ReflectionRadiance, const PerRank<VqImage>* BoundingVolumes = nullptr);
    // each rank's display frame (NumRanks() images, rank r at [r]); nullptr when refused. The Gaussian blur has no band form and
    // is refused.
    const VqImage* RenderPostProcess(const FPostProcessParameters& PPParams, bool bHDR);

    // ---- a step whose peer does not come back (vqcuda_rendezvous.h, DESIGN.md §6) ----
    // Registers a rendezvous deadline of Ns nanoseconds on every rank's context (1 ns..20 s; without one a wait that is never met
    // traps after 20 s). A rank whose wait gives up then ends its call normally and records the failure in its context's status.
    bool SetRendezvousDeadline(uint64_t Ns);
    // BLOCKS: synchronises every rank's stream and reads every rank's status. False, with LastError() naming each rank that saw a
    // failure and the ranks it missed, when a wait gave up since the last Resync(). LoadDefaultResources and
    // PreFilterEnvironmentMap check this themselves and return false. After a failure every signalled method refuses (returns
    // false, enqueues nothing) until Resync() succeeds: a late peer may still be storing an earlier step into a rank's targets.
    bool RendezvousOK();
    // BLOCKS: every rank clears its status and meets its peers at a fresh epoch (vq_group_barrier), then the statuses are read.
    // True once every rank met every peer: every store of the earlier steps, a late peer's included, has landed.
    bool Resync();

private:
    struct FSceneCall;
    bool RenderScene(const FSceneCall& call);
    // one signalled phase: issue(r) on every rank in order; if a rank refuses, the ranks from it on arrive at `epoch` in their
    // peers' flag arrays (vq_group_arrive), so that the ranks already enqueued finish instead of waiting for them
    template <class F> bool Phase(uint32_t epoch, F issue);
    bool Usable(const char* what) const;                        // initialized, and no rendezvous failure awaits a Resync()
    std::vector<VqImage> Targets(int r, const FTexture2D VQRenderer::* member) const;   // rank r's destinations in its rank order
    bool Prepared(const PerRank<const FEnvironmentMapRenderingResources*>& envs) const;

    std::vector<std::unique_ptr<VQRenderer>> mRanks;
    std::vector<cudaStream_t> mStreams;
    std::vector<VqEnvironmentMaps> mPrepared;                  // the maps vq_environment_prepare registered, per rank (ptr 0: none)
    std::vector<VqImage> mDisplay;
    VqGroup* mGroup = nullptr;
    uint32_t mEpoch = 1;
    bool mRendezvousFailed = false;                            // a wait gave up; the signalled methods refuse until Resync()
    std::vector<char> mShadowRecordsSized;                     // per rank: a PCF test has sized the records at this size (rule 3, DESIGN §6)
};

}  // namespace vq
