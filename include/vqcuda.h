/*
 * vqcuda.h — C-ABI of the H100 (sm_90a) headless shading backend.
 *
 * One entry point per GPU program the engine dispatches for its per-pixel passes.
 * The reference has no FFI of its own (SURVEY.md §8(b)); each function below names
 * the reference dispatch site + HLSL entry point it replaces. Conventions mirror the
 * engine's (SURVEY.md §8(b) "Conventions"):
 *   - resources are caller-owned (the engine passes integer IDs; here: device pointers
 *     described by {ptr, width, height, pitch}); the library never frees caller memory;
 *   - nothing throws across the boundary: every call returns 0 (VQ_OK) or a negative
 *     VqStatus; vq_last_error() gives a thread-local message;
 *   - calls that take `stream` only ENQUEUE work on it (== recording into a command list):
 *     they return without waiting for earlier work on `stream`, their kernels and copies
 *     read the inputs and write the outputs after that work, and nothing runs on another
 *     stream. One exception: a call that has to GROW context scratch (the first call at a
 *     larger size: the environment sampling copies of an unregistered environment, the PCF
 *     records of vq_forward_lighting_shadowed*, vq_image_resize's intermediate and tables,
 *     vq_depth_min_pyramid's pads, and vq_ctx_resize's host-call staging) first waits for
 *     the whole device (cudaDeviceSynchronize: an earlier launch on any stream may still
 *     read the old buffer), then enqueues. Pre-size with a first call at the largest size
 *     (or vq_ctx_resize) so that steady frames never wait;
 *   - they are thread-safe when callers use distinct streams (== per-thread command lists,
 *     SceneRendering.cpp:197-207): host-side context state is guarded by a lock, the error
 *     message is per thread, and every SPD or persistent launch takes its own ticket word
 *     from a ring of 128 (see below). EXCEPTIONS — calls whose DEVICE scratch is one
 *     buffer per context and which therefore must not be in flight concurrently on two
 *     streams of the same context (use one context per thread for these, or order them):
 *       vq_forward_lighting* with an environment that is NOT registered by
 *       vq_environment_prepare (the sampling copies are rebuilt into per-context scratch),
 *       vq_environment_prepare itself, vq_image_resize, vq_depth_min_pyramid,
 *       vq_forward_lighting_shadowed and vq_forward_lighting_shadowed_multi_signal (per-pixel PCF records),
 *       vq_forward_lighting_host.
 *     Ticket ring: the SPD kernels (vq_spd_downsample, vq_hdri_build_mips up to 4096^2) and
 *     the persistent or signalled kernels (K3, and every *_multi_signal / *_ranges call with
 *     a signal of n_ranks > 1) take words from one counter per context, 256 single words
 *     and 128 word pairs. Two launches running at the same time share a word if at least
 *     128 such calls on the context were made between them (e.g. a long prefilter on one
 *     stream while 128 SPD or K3 calls are issued on another): keep fewer in flight.
 *     Synchronisation is the caller's (cudaStreamSynchronize == fence wait), except the
 *     blocking calls below;
 *   - the BLOCKING calls (vq_forward_lighting_host, vq_hdr_load_host, vq_hdr_save_host,
 *     vq_material_table_create) wait for the whole device first, so they are ordered after
 *     all device work enqueued before them on ANY stream (legacy, blocking or non-blocking),
 *     and return with their own work complete. They do not wait for work enqueued later.
 *   - there is NO CPU fallback: without a CUDA device every device call fails with
 *     VQ_ERR_NO_DEVICE.
 *
 * All pixel data is linear fp32: RGBA32F (`float4`, 16 B) unless stated otherwise.
 * `stream` is a cudaStream_t passed as void* so that this header needs no CUDA headers.
 */
#ifndef VQCUDA_H
#define VQCUDA_H

#include "vq_shader_data.h"

#ifdef __cplusplus
extern "C" {
#endif

#if defined(_WIN32)
#  define VQ_API __declspec(dllexport)
#else
#  define VQ_API __attribute__((visibility("default")))
#endif

typedef enum VqStatus {
    VQ_OK               =  0,
    VQ_ERR_INVALID_ARG  = -1,
    VQ_ERR_CUDA         = -2,
    VQ_ERR_UNSUPPORTED  = -3,
    VQ_ERR_NO_DEVICE    = -4,
    VQ_ERR_OUT_OF_MEMORY= -5
} VqStatus;

/* ------------------------------------------------------------------------------------------
 * Resource descriptors (replace TextureID/SRV_ID/UAV_ID/RTV_ID, EnvironmentMapRendering.h:28-48)
 * ------------------------------------------------------------------------------------------ */

/* 2-D image of float4 texels (float2 where stated). pitch_bytes is a multiple of 16. */
typedef struct VqImage {
    void*   ptr;
    int32_t width, height;
    size_t  pitch_bytes;
} VqImage;

/* Cubemap with a mip chain, float4 texels, tightly packed, mip-major / face-minor:
 *   offset_texels(mip, face) = sum_{m<mip} 6*(res>>m)^2 + face*(res>>mip)^2
 * Face order = D3D / CubemapUtility.h:31-41: +X(RIGHT) -X(LEFT) +Y(UP) -Y(DOWN) +Z(FRONT) -Z(BACK). */
typedef struct VqCubemap {
    void*   ptr;
    int32_t res;   /* edge length of mip 0 */
    int32_t mips;
} VqCubemap;

/* Equirectangular HDRI with its CPU-style mip pyramid (TextureManager.cpp:714-727), float4,
 * tightly packed levels: level l is (width>>l) x (height>>l); levels <= vq_mip_level_count(). */
typedef struct VqPyramid {
    void*   ptr;
    int32_t width, height;
    int32_t levels;
} VqPyramid;

/* The surface record PSMain consumes after material-texture sampling (BRDF.hlsl:50-58,
 * ForwardLighting.hlsl:245-285) as three (optionally four) float4 planes:
 *   position_ao      = { P.xyz (world space), ao }   ao = fAmbientLightingFactor*localAO*SSAO
 *   normal_roughness = { N.xyz (unit, world space), roughness }
 *   albedo_metalness = { diffuseColor.rgb, metalness }
 *   emissive         = { emissiveColor.rgb, emissiveIntensity }   (ptr == NULL -> no emissive) */
typedef struct VqGBuffer {
    VqImage position_ao;
    VqImage normal_roughness;
    VqImage albedo_metalness;
    VqImage emissive;
} VqGBuffer;

/* The three IBL inputs PSMain binds (SceneRendering.cpp:1690-1717). brdf_lut holds float2 texels. */
typedef struct VqEnvironmentMaps {
    VqCubemap irradiance_diffuse;   /* blurred diffuse irradiance, 1 mip */
    VqCubemap irradiance_specular;  /* prefiltered specular, `mips` levels */
    VqImage   brdf_lut;             /* float2 (scale,bias), CubemapConvolution.hlsl:227-240 */
} VqEnvironmentMaps;

typedef struct VqContext VqContext;

/* ------------------------------------------------------------------------------------------
 * Lifetime  (IRenderPass::Initialize / Destroy / OnCreateWindowSizeDependentResources,
 *            RenderPass.h:44-59)
 * ------------------------------------------------------------------------------------------ */
VQ_API int  vq_ctx_create(int device, VqContext** out_ctx);
VQ_API int  vq_ctx_destroy(VqContext* ctx);
/* Pre-sizes internal scratch (SPD counters, host-call staging) for a render resolution. Optional. */
VQ_API int  vq_ctx_resize(VqContext* ctx, int width, int height);
VQ_API const char* vq_last_error(void);
VQ_API const char* vq_version(void);
/* Number of kernels this library has launched in this process (all contexts). */
VQ_API uint64_t vq_launch_count(void);

/* End-of-pass rendezvous of a multi-GPU step, run by the kernel itself (its last CTA): after all of this rank's stores
 * (local and peer) are ordered, it writes `epoch` into word `my_index` of every OTHER rank's flag array and then waits
 * until words j != my_index of its OWN array have reached `epoch` — i.e. until every peer has finished storing into this
 * rank's buffers. flags[0] = this rank's array, flags[1..n_ranks-1] = the peers' arrays mapped into this process
 * (n_ranks 32-bit words each, zero-initialised, e.g. in torch symmetric memory); epoch must increase from call to call.
 * Replaces a host-issued barrier per step: the step is ONE kernel. A peer that never arrives fails the kernel after 20 s (a trap)
 * unless the calling context registered a deadline (vqcuda_rendezvous.h): the wait then ends at the deadline or on a cancel and
 * is recorded in the context's status instead. */
typedef struct VqPeerSignal {
    uint32_t* flags[8];
    int32_t   n_ranks;
    int32_t   my_index;
    uint32_t  epoch;
} VqPeerSignal;

/* ------------------------------------------------------------------------------------------
 * K1  Forward PBR lighting.  Replaces VQRenderer::RenderSceneColor (SceneRendering.cpp:1619-1851)
 *     + PSMain (ForwardLighting.hlsl:222-391) over a G-buffer instead of rasterised draws.
 *     Shades rows [row_begin,row_end) of the image (row tiling for multi-GPU); out = {I.rgb, roughness}.
 *     This entry point binds no shadow maps: caster lists and a shadowing directional light are lit with shadow
 *     factor 1 (no occlusion) - which differs from PSMain whenever the engine has shadow maps bound; use
 *     vq_forward_lighting_shadowed (below) for the PCF-shadowed result.
 *     Where the shader text leaves the result undefined, K1 defines it (DESIGN.md §5):
 *       - a spot cosine that rounds outside [-1, 1] (on the spot's axis, or directly behind it) is clamped, so the pixel gets
 *         the on-axis (or opposite) intensity; HLSL's acos is unspecified there and the reference C++ gives NaN;
 *       - a pixel exactly at a point or spot light's position (squared distance 0) gets nothing from that light (its
 *         direction is undefined); the reference divides 0 by 0;
 *       - closer than 1e-13 to a light (squared distance < 1e-26) the light vector is scaled by 1/sqrt(d2 + 1e-30), so the
 *         light is dimmer than 1/d2 and stays finite where the reference overflows;
 *       - a pixel exactly at the camera position has no view direction and shades to NaN.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_forward_lighting(VqContext* ctx,
                               const VqPerFrameData* per_frame,
                               const VqPerViewLightingData* per_view,
                               const VqGBuffer* gbuffer,
                               const VqEnvironmentMaps* env,
                               VqImage out_color,
                               int row_begin, int row_end,
                               void* stream);

/* K1 fused with the gather of tiles (multi-GPU): shades rows [row_begin,row_end) of the local G-buffer tile and stores every
 * pixel to row (dst_row_offset + y) of EACH of the n_outs (<= 8) destination frames. Destinations other than the local
 * frame are peer-GPU buffers mapped into this process (CUDA IPC / torch symmetric memory): the stores travel over NVLink
 * while the SMs keep shading, so the all-gather of tiles overlaps the math instead of following it. The caller provides
 * the cross-rank barrier after the kernel (e.g. symmetric-memory barrier or a 1-element all-reduce). */
VQ_API int vq_forward_lighting_multi(VqContext* ctx,
                                     const VqPerFrameData* per_frame,
                                     const VqPerViewLightingData* per_view,
                                     const VqGBuffer* gbuffer,
                                     const VqEnvironmentMaps* env,
                                     const VqImage* out_frames, int n_outs, int dst_row_offset,
                                     int row_begin, int row_end,
                                     void* stream);
/* ... and with the cross-rank rendezvous run by the kernel's last CTA (VqPeerSignal above): shade + gather + barrier = ONE kernel. */
VQ_API int vq_forward_lighting_multi_signal(VqContext* ctx, const VqPerFrameData* per_frame, const VqPerViewLightingData* per_view,
                                            const VqGBuffer* gbuffer, const VqEnvironmentMaps* env, const VqImage* outs, int n_outs,
                                            int dst_row_offset, int row_begin, int row_end, const VqPeerSignal* signal, void* stream);
/* The other shading calls in the same multi-destination form. Into each of the n_outs (1..8) destinations, each call computes
 * what its single-destination call computes into its one output, bit for bit, at rows offset by dst_row_offset; rows outside
 * [row_begin,row_end) are not touched. With several destinations the pass runs as one kernel whose last CTA runs the rendezvous
 * when `signal` is given (NULL: no rendezvous). Refused with VQ_ERR_INVALID_ARG before
 * the device is touched, with vq_forward_lighting_multi_signal's messages: n_outs outside 1..8, a destination narrower or wider
 * than the source or without dst_row_offset + height rows, a negative offset, a signal with n_ranks > 1 and one destination or an
 * empty row range, and the shadow-map checks of vq_forward_lighting_shadowed.
 *   vq_forward_lighting_shadowed_multi_signal: vq_forward_lighting_shadowed (the PCF pre-pass, then the shadowed forward kernel
 *     with the multi-destination stores: two launches). The PCF records are context scratch, so calls on ONE context must be
 *     issued on one stream at a time, as for vq_forward_lighting_shadowed. The environment is checked after the PCF launch.
 *   vq_forward_lighting_from_materials_multi_signal: vq_forward_lighting_from_materials (shadow_maps NULL) or
 *     vq_forward_lighting_shadowed_from_materials, one launch and no context scratch; when no PCF test would run it is the
 *     unshadowed call. Pixels the alpha mask discards stay untouched in every destination. dst_row_offset must be even:
 *     the surface producer's quads sit on even rows of the attribute planes, and the texture LOD of a rank's band matches the
 *     whole frame's only if those rows are even rows of the frame too. A rank may pass the whole frame's attribute planes with its
 *     row range and offset 0, or planes holding just its band with rows [0, band) and offset = the band's first row (even); in
 *     the second form the SSAO plane wraps at the band's last row, not the frame's. */
struct VqShadowMaps; struct VqSurfaceInputs; struct VqMaterialTable;     /* defined below (SURVEY §8(f).1 and §8(f).4) */
VQ_API int vq_forward_lighting_shadowed_multi_signal(VqContext* ctx, const VqPerFrameData* per_frame,
                                                     const VqPerViewLightingData* per_view, const VqGBuffer* gbuffer,
                                                     const VqEnvironmentMaps* env, const struct VqShadowMaps* shadow_maps,
                                                     const VqImage* outs, int n_outs, int dst_row_offset, int row_begin, int row_end,
                                                     const VqPeerSignal* signal, void* stream);
VQ_API int vq_forward_lighting_from_materials_multi_signal(VqContext* ctx, const VqPerFrameData* per_frame,
                                                           const VqPerViewLightingData* per_view, const struct VqSurfaceInputs* in,
                                                           const struct VqMaterialTable* table, int alpha_mask,
                                                           const VqEnvironmentMaps* env, const struct VqShadowMaps* shadow_maps,
                                                           const VqImage* outs, int n_outs, int dst_row_offset, int row_begin,
                                                           int row_end, const VqPeerSignal* signal, void* stream);

/* The forward pass samples the IBL cubemaps from bordered copies (each face carries a 1-texel border of its
 * neighbours, so seamless bilinear taps never leave the face). vq_environment_prepare builds those copies once and
 * registers them in the context — the analogue of the RENDER_TARGET -> PIXEL_SHADER_RESOURCE barrier the engine
 * records after prefiltering (EnvironmentMapRendering.cpp:466-472). Call it again whenever the maps' contents
 * change, or vq_environment_invalidate to drop the registration. Without it vq_forward_lighting re-pads the cubes
 * into context scratch on every call (always correct; serialise such calls per context). */
VQ_API int vq_environment_prepare(VqContext* ctx, const VqEnvironmentMaps* env, void* stream);
VQ_API int vq_environment_invalidate(VqContext* ctx);

/* ------------------------------------------------------------------------------------------
 * K11 HDRI mip pyramid, 2x2 MIN filter, alpha = 1.  Replaces VQ_DXGI_UTILS::MipImage
 *     (DXGIUtils.cpp:289-317) called from TextureManager.cpp:714-727. Level 0 must be filled.
 *     MIN is the reference's std::min(a, b) = (b < a) ? b : a, nested min(s0, min(s1, min(s2, s3))) over the block's
 *     (0,0), (1,0), (0,1), (1,1) texels, for any float input: a NaN survives only in s0, a +0 / -0 tie keeps the earlier
 *     operand. Level sizes are floor-halved; an odd last row / column is not read.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_hdri_build_mips(VqContext* ctx, VqPyramid hdri, void* stream);

/* ------------------------------------------------------------------------------------------
 * K2  Diffuse irradiance convolution.  Replaces the per-face draws at
 *     EnvironmentMapRendering.cpp:221-240 + PSMain_DiffuseIrradiance (CubemapConvolution.hlsl:112-163).
 *     Two sampling modes:
 *       step  > 0 : the reference's float-accumulated (phi,theta) loops with that step
 *                   (INTEGRATION_STEP_DIFFUSE_IRRADIANCE; 0.010/0.025/0.050, PipelineStateObjects.cpp:1298-1306)
 *       step == 0 : an integer n_phi x n_theta grid, phi_i = i*(2pi/n_phi), theta_j = j*(pi/2/n_theta)
 *     Source level is HDRI mip `src_mip` (reference: 3). Computes texel rows [row_begin,row_end)
 *     of the flattened (face, row) space, face*res + row; out.mips must be 1.
 * ------------------------------------------------------------------------------------------ */
typedef struct VqDiffuseIrradianceParams {
    float   step;
    int32_t n_phi, n_theta;
    int32_t src_mip;
} VqDiffuseIrradianceParams;
VQ_API int vq_diffuse_irradiance(VqContext* ctx, const VqDiffuseIrradianceParams* params,
                                 VqPyramid hdri, VqCubemap out,
                                 int row_begin, int row_end, void* stream);
/* One rank's band of K2 into every rank's cube: vq_diffuse_irradiance_multi_signal (vqcuda_prefilter_multi.h). */

/* ------------------------------------------------------------------------------------------
 * K3  Specular prefilter (GGX importance sampling, 512 Hammersley samples, PDF-based source mip).
 *     Replaces the mip x face draw loop at EnvironmentMapRendering.cpp:413-465 +
 *     PSMain_SpecularIrradiance (CubemapConvolution.hlsl:168-223). For every mip m of `out`:
 *     Roughness = m/(mips-1), ViewDim = HDRI dims (EnvironmentMapRendering.cpp:432-434).
 *     Computes texel rows [row_begin,row_end) of the flattened (mip, face, row) space
 *     (vq_cubemap_row_count rows in total).
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_specular_prefilter(VqContext* ctx, VqPyramid hdri, VqCubemap out,
                                 int num_samples, int row_begin, int row_end, void* stream);
/* K3 fused with the gather of row blocks (multi-GPU strong scaling): every texel of rows [row_begin,row_end) is stored into
 * each of the n_outs (<= 8) cubemaps of identical shape — the local one first, then the other ranks' buffers mapped into
 * this process (CUDA IPC / torch symmetric memory). The stores travel over NVLink while the SMs keep integrating; the caller
 * provides the cross-rank barrier after the kernel(s). */
VQ_API int vq_specular_prefilter_multi(VqContext* ctx, VqPyramid hdri, const VqCubemap* outs, int n_outs,
                                       int num_samples, int row_begin, int row_end, void* stream);


/* K3 as ONE persistent launch over several row ranges (n_ranges pairs [begin,end), increasing and disjoint) of the
 * flattened (mip, face, row) space, stored into n_outs (<= 8) cubemaps, with the optional rendezvous above (NULL: none).
 * This is what one rank of the strong-scaled prefilter runs per step: its row block of every mip, the replicated tail
 * mips, the fused gather over NVLink and the cross-rank barrier, in one kernel. */
VQ_API int vq_specular_prefilter_ranges(VqContext* ctx, VqPyramid hdri, const VqCubemap* outs, int n_outs, int num_samples,
                                        const int* row_ranges, int n_ranges, const VqPeerSignal* signal, void* stream);

/* ------------------------------------------------------------------------------------------
 * K4  BRDF integration LUT (split-sum scale,bias).  Replaces ComputeBRDFIntegrationLUT
 *     (Renderer.cpp:871-909) + CSMain_BRDFIntegration (CubemapConvolution.hlsl:227-240).
 *     out holds float2 texels; NdotV = (x+.5)/W, roughness = (y+.5)/H; reference: 1024^2, 2048 samples.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_brdf_integration_lut(VqContext* ctx, VqImage out_rg, int num_samples,
                                   int row_begin, int row_end, void* stream);
/* One rank's band of K4 into every rank's LUT: vq_brdf_integration_lut_multi_signal (vqcuda_prefilter_multi.h). */

/* ------------------------------------------------------------------------------------------
 * K5  Separable 21-tap Gaussian blur, clamp-to-edge, alpha = 1.  Replaces the dispatches at
 *     EnvironmentMapRendering.cpp:341-372 / SceneRendering.cpp:2582-2638 + CSMain_X / CSMain_Y
 *     (GaussianBlur.hlsl:119-186).
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_gaussian_blur_x(VqContext* ctx, const VqBlurParams* params, VqImage in, VqImage out, void* stream);
VQ_API int vq_gaussian_blur_y(VqContext* ctx, const VqBlurParams* params, VqImage in, VqImage out, void* stream);
/* A whole one-mip cube, X then Y, in one launch: vq_gaussian_blur_cube (vqcuda_prefilter_multi.h). */
/* X then Y in one launch, and its band form for a multi-GPU frame: vq_gaussian_blur, vq_gaussian_blur_multi_signal (vqcuda_blur.h). */

/* ------------------------------------------------------------------------------------------
 * K6  Tonemapper.  Replaces the dispatch at SceneRendering.cpp:2640-2656 + CSMain (Tonemapper.hlsl:110-151).
 *     Domain limit of the sRGB curve: Reinhard c / (c + 1) divides with the fast reciprocal, so a channel whose finite
 *     c + 1 exceeds 2^126 in magnitude gives 0 (the shader's division gives 1). Inputs up to 2^126, which include the
 *     engine's whole RGBA16F range, match the shader to 1e-4; Inf and NaN give NaN as in the shader.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_tonemap(VqContext* ctx, const VqTonemapperParams* params, VqImage in, VqImage out, void* stream);

/* ------------------------------------------------------------------------------------------
 * K7  FidelityFX CAS, sharpen-only path.  Replaces SceneRendering.cpp:2658-2693 + CAS_CSMain
 *     (AMDFidelityFX.hlsl:122-174) -> CasFilter(noScaling) (CAS/ffx_cas.h:408-537).
 *     cas_const = the 8 words CasSetup wrote (FFFXCAS::CASConstantBlock, PostProcess.h:104-112).
 *     Reads outside the image return 0 (D3D Texture.Load). Output alpha is 1.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_cas(VqContext* ctx, const uint32_t cas_const[8], VqImage in, VqImage out, void* stream);

/* ------------------------------------------------------------------------------------------
 * K8  FSR1 EASU.  Replaces SceneRendering.cpp:2711-2734 + FSR_EASU_CSMain (AMDFidelityFX.hlsl:247-288)
 *     -> FsrEasuF (FSR1.0/ffx_fsr1.h:315-437). easu_const = FFSR1_EASU::EASUConstantBlock (16 words).
 *     Gathers use the engine's sampler addressing: VQ_ADDRESS_WRAP (RootSignatures.cpp:525) by default.
 *     con0 must have been built for these images (vq_fsr_easu_con with viewport <= input size, output = out's size).
 *     Before launching, the call evaluates the kernels' own texel positions floor(o * con0.xy + con0.zw) at the first and
 *     last output pixel of each axis (they bound all others) and returns VQ_ERR_INVALID_ARG, with nothing launched, when
 *       - any con0 value is not finite;
 *       - a tap (texels -1 .. +2 around those positions) leaves [-W, 2W) x [-H, 2H), W = max(in.width, 3),
 *         H = max(in.height, 3) (the range the WRAP fold handles), e.g. constants left over from before a resize;
 *       - on the upscaling path (0 < con0.x, con0.y <= 1) a 32 x 8 output tile would need more than 32 x 8 input texels.
 *     Every constant vq_fsr_easu_con builds for viewport <= input <= 8192 and output <= 16384 passes.
 * ------------------------------------------------------------------------------------------ */
enum { VQ_ADDRESS_WRAP = 0, VQ_ADDRESS_CLAMP = 1 };
VQ_API int vq_fsr_easu(VqContext* ctx, const uint32_t easu_const[16], int address_mode,
                       VqImage in, VqImage out, void* stream);

/* ------------------------------------------------------------------------------------------
 * K9  FSR1 RCAS.  Replaces SceneRendering.cpp:2735-2781 + FSR_RCAS_CSMain (AMDFidelityFX.hlsl:335-376)
 *     -> FsrRcasF (ffx_fsr1.h:684-769). rcas_const = FFSR1_RCAS::RCASConstantBlock (4 words).
 *     Subnormal channels: the hitMin reciprocal reads a subnormal 4*mx4 as 0 (rcp.approx.ftz). Where it does, the result is
 *     FsrRcasF of the input with that channel's subnormals flushed to zeros of their sign (D3D11 allows flushing); DESIGN §5.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_fsr_rcas(VqContext* ctx, const uint32_t rcas_const[4], VqImage in, VqImage out, void* stream);

/* ------------------------------------------------------------------------------------------
 * K6-K9 on a band of the output, into several frames: one rank's share of the post chain of a multi-GPU frame
 * (DESIGN.md §6). `in` is the pass's whole source image (the stencils read across band edges); rows [row_begin,row_end) are
 * rows of the pass's output; each of the n_outs (1..8) destinations has the output's size (the tonemapper's, CAS's and RCAS's
 * output is the size of `in`; EASU's is the size of outs[0]). Into each destination the call stores exactly the bits its
 * single-destination call (vq_tonemap, vq_cas, vq_fsr_easu, vq_fsr_rcas) stores on those rows, and touches no other row of any
 * destination. One launch per call, no context scratch: calls on several streams of one context are fine. With `signal`
 * (n_ranks > 1) the kernel's last CTA runs the rendezvous of VqPeerSignal after every store; NULL: no rendezvous. An empty row
 * range without a rendezvous launches nothing and returns VQ_OK.
 * Refused with VQ_ERR_INVALID_ARG before the device is touched (also with a NULL context): the single call's checks and messages
 * (null constants or params, size rules, `in` equal to any destination for CAS / EASU / RCAS, EASU's con0 checks above and an
 * unknown address mode), n_outs outside 1..8, rows outside the output or reversed, a signal with n_ranks > 1 and one
 * destination or an empty row range.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_tonemap_multi_signal(VqContext* ctx, const VqTonemapperParams* params, VqImage in, const VqImage* outs, int n_outs,
                                   int row_begin, int row_end, const VqPeerSignal* signal, void* stream);
VQ_API int vq_cas_multi_signal(VqContext* ctx, const uint32_t cas_const[8], VqImage in, const VqImage* outs, int n_outs,
                               int row_begin, int row_end, const VqPeerSignal* signal, void* stream);
VQ_API int vq_fsr_easu_multi_signal(VqContext* ctx, const uint32_t easu_const[16], int address_mode, VqImage in, const VqImage* outs,
                                    int n_outs, int row_begin, int row_end, const VqPeerSignal* signal, void* stream);
VQ_API int vq_fsr_rcas_multi_signal(VqContext* ctx, const uint32_t rcas_const[4], VqImage in, const VqImage* outs, int n_outs,
                                    int row_begin, int row_end, const VqPeerSignal* signal, void* stream);

/* ------------------------------------------------------------------------------------------
 * K6-K9 fused: RenderPostProcess in one launch (SceneRendering.cpp:2640-2781), from scene colour to display frame with no
 *     intermediate image in device memory. The tonemapper, then FSR1 EASU + RCAS when easu_const != NULL (rcas_const required),
 *     else CAS when cas_const != NULL, else the tonemapper alone (vq_tonemap's kernel). A NULL constant block turns its pass off;
 *     with FSR on, cas_const is ignored (the engine does not read CAS's output then). address_mode is EASU's (vq_fsr_easu).
 *     The display frame equals, bit for bit, vq_tonemap -> vq_fsr_easu -> vq_fsr_rcas, vq_tonemap -> vq_cas, or vq_tonemap.
 *     Output alpha: 1 with EASU/RCAS or CAS, the input's alpha otherwise. One launch per call, no context scratch: calls on
 *     several streams of one context are fine. The display is the size of scene_color without FSR, any size con0 was built for
 *     with it.
 *     Refused with VQ_ERR_INVALID_ARG before the device is touched (also with a NULL context): null params, bad descriptors,
 *     the size rules of vq_tonemap / vq_cas, scene_color equal to the display with EASU/RCAS or CAS, an unknown address mode,
 *     EASU's con0 checks (vq_fsr_easu) with the footprint bound of this kernel's tiles (on the upscaling path, a 30 x 14 display
 *     tile and its 1-pixel ring may need at most 32 x 16 input texels), con0 on EASU's downscaling path (neither the exact 2x
 *     nor 0 < con0.x, con0.y <= 1: run the three calls for those), and easu_const without rcas_const or the reverse.
 *   vq_post_process_multi_signal: one rank's band of the display frame into several frames, as the K6-K9 multi-destination
 *     calls above store theirs. Rows [row_begin,row_end) are rows of the DISPLAY frame; scene_color is the whole frame (the
 *     halo rows are read, not planned); each of the n_outs (1..8) destinations has the size of outs[0], the display size.
 *     Also refused: their destination, row and signal checks.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_post_process(VqContext* ctx, const VqTonemapperParams* tonemapper, const uint32_t cas_const[8],
                           const uint32_t easu_const[16], int address_mode, const uint32_t rcas_const[4],
                           VqImage scene_color, VqImage display, void* stream);
VQ_API int vq_post_process_multi_signal(VqContext* ctx, const VqTonemapperParams* tonemapper, const uint32_t cas_const[8],
                                        const uint32_t easu_const[16], int address_mode, const uint32_t rcas_const[4],
                                        VqImage scene_color, const VqImage* outs, int n_outs, int row_begin, int row_end,
                                        const VqPeerSignal* signal, void* stream);

/* ------------------------------------------------------------------------------------------
 * K10 FidelityFX SPD: the whole mip chain in one launch.  Replaces SPD_CSMain
 *     (AMDFidelityFX.hlsl:525-545) -> SpdDownsample (SPD/ffx_spd.h:811-835), reduction =
 *     (v0+v1+v2+v3)*0.25 (AMDFidelityFX.hlsl:463-466). `mips` are the destination levels
 *     1..constants->mips (mips[i] is level i+1, floor-halved sizes); src is level 0.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_spd_downsample(VqContext* ctx, const VqSpdConstants* constants,
                             VqImage src, const VqImage* mips, void* stream);

/* ------------------------------------------------------------------------------------------
 * Host-side constant setup == the FidelityFX `A_CPU` functions the engine calls
 * (PostProcess.cpp:39-99): bit-identical results.
 * ------------------------------------------------------------------------------------------ */
/* FsrEasuCon (ffx_fsr1.h:156-202) -> con[16] = con0|con1|con2|con3 */
VQ_API void vq_fsr_easu_con(uint32_t con[16],
                            float input_viewport_w, float input_viewport_h,
                            float input_size_w, float input_size_h,
                            float output_w, float output_h);
/* HOST. The rows of `in` that vq_fsr_easu reads for output rows [row_begin,row_end): up to two increasing, disjoint, non-adjacent
 * [begin,end) ranges in ranges[0..3]; returns their count (0 for an empty range) or VQ_ERR_INVALID_ARG (null pointers, unknown
 * address mode, heights < 1, rows outside the output or reversed, con0.y / con0.w not finite or putting taps outside [-H, 2H)).
 * The taps of output row y are the rows floor(y * con0.y + con0.w) - 1 .. + 2 folded by the address mode; under WRAP the first
 * and last bands of an upscale also read rows at the opposite edge, hence the second range. Exact whenever consecutive output
 * rows move at most 4 input rows (con0.y <= 4, every vq_fsr_easu_con with output >= input / 4); a covering superset otherwise. */
VQ_API int vq_fsr_easu_source_rows(const uint32_t easu_const[16], int address_mode, int in_height, int out_height,
                                   int row_begin, int row_end, int ranges[4]);
/* FsrRcasCon (ffx_fsr1.h:662-672) */
VQ_API void vq_fsr_rcas_con(uint32_t con[4], float sharpness_stops);
/* CasSetup (ffx_cas.h:375-394) -> con[8] = const0|const1 */
VQ_API void vq_cas_setup(uint32_t con[8], float sharpness,
                         float input_w, float input_h, float output_w, float output_h);
/* SpdSetup (ffx_spd.h:327-351); rect = {left, top, width, height}; mips < 0 -> derive from rect */
VQ_API void vq_spd_setup(uint32_t dispatch_xy[2], VqSpdConstants* constants,
                         const uint32_t rect[4], int mips);
/* Image::CalculateMipLevelCount (Libs/VQUtils/Source/Image.cpp:231-241) */
VQ_API int  vq_mip_level_count(uint64_t w, uint64_t h);

/* Layout helpers for the packed descriptors above (host-side arithmetic only). */
VQ_API uint64_t vq_cubemap_texel_count(int res, int mips);             /* total float4 texels */
VQ_API uint64_t vq_cubemap_offset(int res, int mip, int face);         /* texel offset of (mip,face) */
VQ_API int      vq_cubemap_row_count(int res, int mips);               /* rows in flattened (mip,face,row) */
VQ_API uint64_t vq_pyramid_texel_count(int width, int height, int levels);
VQ_API uint64_t vq_pyramid_offset(int width, int height, int level);   /* texel offset of a level */

/* ------------------------------------------------------------------------------------------
 * SURVEY §8(f).1  Surface producer: the part of PSMain BEFORE lighting (ForwardLighting.hlsl:226-283) —
 *     material-texture sampling, sRGB->linear, normal mapping, Has*Map selection — turned into a kernel
 *     that fills the G-buffer K1 consumes from what a rasteriser interpolates per covered pixel.
 * ------------------------------------------------------------------------------------------ */

/* Material texture: RGBA8 UNORM (what Image::LoadFromFile + TextureManager upload, 4 B/texel), with the CPU-built
 * box-filter mip chain (TextureManager.cpp:714-727 -> DXGIUtils.cpp:250-287), tightly packed levels, level l is
 * (width>>l) x (height>>l), levels <= vq_mip_level_count(); texel offsets as vq_pyramid_offset().
 * ptr == NULL is the engine's null SRV (Renderer_Resources.cpp:383-387): every read returns 0. */
typedef struct VqTexture2D {
    void*   ptr;
    int32_t width, height;
    int32_t levels;
} VqTexture2D;

/* the descriptor table of one material, in the order PSMain samples them (ForwardLighting.hlsl:87-94,229-235; texAlphaMask t3 is bound but never sampled) */
typedef struct VqMaterialTextures {
    VqTexture2D diffuse, normals, emissive, metalness, roughness, occl_rough_metal, local_ao;
} VqMaterialTextures;

/* PSInput as a rasteriser would deliver it (ForwardLighting.hlsl:42-53), one record per pixel in three float4 planes:
 *   position_u = { WorldSpacePosition.xyz, uv.x }
 *   normal_v   = { WorldSpaceNormal.xyz  (interpolated, not normalised), uv.y }
 *   tangent_m  = { WorldSpaceTangent.xyz (interpolated, not normalised), material index as an exact small float }
 *   ssao       = optional R32F plane, the texScreenSpaceAO the shader point-samples (NULL -> 1)
 * Domain: the material index converts toward zero with NaN -> 0 and saturation, then clamps to [0, count-1]. The floored
 * texel coordinate floor(u*W - 0.5) converts the same way and then wraps, so beyond 2^31 it reads the column of +-2^31 mod W.
 * A texel coordinate that is not finite gives a NaN sample (also when only one level of a trilinear pair overflows). */
typedef struct VqSurfaceInputs {
    VqImage position_u, normal_v, tangent_m;
    VqImage ssao;
} VqSurfaceInputs;

typedef struct VqMaterialTable VqMaterialTable;   /* device-resident copy of the scene's materials */

/* RGBA8 mip chain, per-channel (a+b+c+d)/4 truncating: VQ_DXGI_UTILS::MipImage, 4-byte branch (DXGIUtils.cpp:250-287).
 * Level 0 must be filled. Bit-exact. */
VQ_API int vq_texture_build_mips(VqContext* ctx, VqTexture2D tex, void* stream);

/* Uploads `count` materials (constants + texture descriptors, both HOST arrays; the texel pointers inside are DEVICE
 * pointers that must outlive the table). Material::GetCBufferData + the SRV table built at AssetLoader.cpp:406-420.
 * A material whose bound maps all have the same width, height and level count (>= 2 maps) also gets a SAMPLING COPY:
 * one 16-byte record per texel holding the bytes PSMain reads of every map, so a trilinear tap is one 128-bit load for
 * all maps (like the bordered cubemap copies of vq_environment_prepare). The copy is taken HERE, synchronously (the call
 * waits for the device first, so mip chains still being built on other streams are complete): fill the textures, mips
 * included, before creating the table, and re-create the table when texels change. Costs 16 B per texel of the shared
 * size; if that allocation fails, or with VQ_SURFACE_RECORDS=0 in the environment, the maps are sampled one by one.
 * textureConfig must lie in [0, 2^31) (it is converted with (int)); anything else, NaN included, is VQ_ERR_INVALID_ARG. */
VQ_API int vq_material_table_create(VqContext* ctx, const VqMaterialData* materials,
                                    const VqMaterialTextures* textures, int count, VqMaterialTable** out_table);
VQ_API int vq_material_table_destroy(VqContext* ctx, VqMaterialTable* table);

/* Fills rows [row_begin,row_end) of the G-buffer (emissive plane optional). `ambient_factor` = PerFrameData
 * fAmbientLightingFactor (ForwardLighting.hlsl:245). alpha_mask != 0 compiles in the ENABLE_ALPHA_MASK discard
 * (ForwardLighting.hlsl:237-240): such pixels are left untouched in the G-buffer. Texture LOD comes from the 2x2-quad
 * finite differences of uv, as the implicit-derivative Sample() of a pixel shader does (DESIGN.md §3.6). */
VQ_API int vq_gbuffer_from_materials(VqContext* ctx, const VqSurfaceInputs* in, const VqMaterialTable* table,
                                     float ambient_factor, int alpha_mask, const VqGBuffer* out,
                                     int row_begin, int row_end, void* stream);

/* PSMain end to end (ForwardLighting.hlsl:222-391) in ONE launch, from interpolants and materials to lit colour: computes
 * what vq_gbuffer_from_materials(ctx, in, table, per_frame->fAmbientLightingFactor, alpha_mask, &gb, ...) with an emissive
 * plane, followed by vq_forward_lighting(ctx, per_frame, per_view, &gb, env, out_color, ...), computes, bit for bit (with a
 * non-zero fHDRIOffsetInRadians a few pixels may differ in their last bits: the compiler contracts the yaw rotation of the
 * cube lookups differently in the two kernels), but the G-buffer never leaves the SM (no device memory is allocated or written for it). out_color has the size of the attribute
 * planes and receives {I.rgb, roughness}. Pixels the alpha mask discards are left untouched in out_color, as a discarded
 * fragment writes nothing. Rows [row_begin,row_end) follow vq_gbuffer_from_materials: quads are aligned to absolute even rows,
 * so row ranges tile the image. The defined deviations from the shader text are those of the two halves: the sampling rules
 * of vq_gbuffer_from_materials / VqSurfaceInputs and the K1 list at vq_forward_lighting. No shadow maps are bound (lit as
 * vq_forward_lighting lights them); vq_forward_lighting_shadowed_from_materials (SURVEY §8(f).4 below) is the same call with
 * the shadow maps bound. The arguments are checked before the device is touched.
 * Like vq_forward_lighting, it rebuilds the IBL sampling copies per call unless the environment is registered. */
VQ_API int vq_forward_lighting_from_materials(VqContext* ctx, const VqPerFrameData* per_frame,
                                              const VqPerViewLightingData* per_view, const VqSurfaceInputs* in,
                                              const VqMaterialTable* table, int alpha_mask, const VqEnvironmentMaps* env,
                                              VqImage out_color, int row_begin, int row_end, void* stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY §8(f).2  On-disk format at either end of the path: Radiance .hdr (RGBE).
 *     Load  = Image::LoadFromFile -> stbi_loadf(path, &x, &y, &n, 4) (Libs/VQUtils/Source/Image.cpp:119-121) with
 *             Image::CalculateMaxLuminance (Image.cpp:43-86) fused into the same pass; results are bit-identical to stb's.
 *     Save  = Image::SaveToDisk -> stbi_write_hdr(path, x, y, 4, data) (Image.cpp:210-213); files are byte-identical.
 *     The byte-serial work (header text, locating / emitting run lists) is host code; the per-texel work is kernels,
 *     so host<->device traffic is the file image (<= ~4 B/texel), not the fp32 image (16 B/texel).
 * ------------------------------------------------------------------------------------------ */
typedef struct VqHdrInfo {
    int32_t  width, height;
    uint64_t data_offset;   /* first byte after the resolution line (or where flat data starts) */
    int32_t  flat;          /* 1: 4 bytes per texel from data_offset on, no run-length encoding */
    int32_t  reserved;
} VqHdrInfo;
/* HOST. Parses the header of a .hdr file image. channel_offsets == NULL: header only (dims for allocation).
 * Otherwise (run-length encoded files: info->flat == 0 after the first call) it must hold 4*height+1 entries and
 * receives the file offset of every scanline's R,G,B,E run list (+ the end offset); the run headers are validated
 * (stb's "corrupt HDR" conditions -> VQ_ERR_INVALID_ARG; a stream that ends inside a scanline is an error, where stb
 * would spin on zero bytes; a resolution line with a zero dimension is rejected, where stb returns an image without texels).
 * A file whose scanlines turn out not to be run-length encoded flips info->flat to 1. */
VQ_API int vq_hdr_parse(const void* file, uint64_t size, VqHdrInfo* info, uint64_t* channel_offsets);
/* DEVICE. Expands the file image into `out` (width x height RGBA32F, alpha 1). dev_file: 16-byte aligned, allocation
 * padded to a multiple of 16 bytes. dev_channel_offsets: device copy of the index (NULL for flat files).
 * dev_max_luminance (optional): receives max over texels of 0.2126 r + 0.7152 g + 0.0722 b (Image::MaxLuminance). */
VQ_API int vq_hdr_decode(VqContext* ctx, const void* dev_file, uint64_t size, const VqHdrInfo* info,
                         const uint64_t* dev_channel_offsets, VqImage out, float* dev_max_luminance, void* stream);
/* Blocking: host file image -> device fp32 image (parse + upload + decode). Ordered after all earlier device work, on any
 * stream (the header's blocking calls): a kernel still reading `out` finishes before it is overwritten. */
VQ_API int vq_hdr_load_host(VqContext* ctx, const void* host_file, uint64_t size, VqImage out, float* max_luminance);
/* DEVICE. RGBA32F -> RGBE texels (4 bytes each, tightly packed rows), stbiw__linear_to_rgbe, for every float input:
 *   maxcomp = max(r, max(g, b)) with max(a, b) = a > b ? a : b, stb's nesting: a NaN in r or g is ignored
 *   (the comparison is false, so the other operand is taken), a NaN in b is not;
 *   maxcomp < 1e-32 (negative values, -0 and -Inf included) -> (0, 0, 0, 0);
 *   otherwise e = the frexp exponent of maxcomp (0 for +Inf and NaN), exponent byte = (e + 128) & 0xff, so maxcomp >= 2^127
 *   wraps it to 0 and the texel decodes as black (stb writes the same bytes and reads them back the same way);
 *   channel byte = the low byte of c * 2^(8 - e) truncated toward zero to int32 (a negative channel wraps, a NaN product
 *   gives 0: maxcomp = +Inf or NaN writes (0, 0, 0, 128); maxcomp = -Inf is below the cut-off and writes
 *   (0, 0, 0, 0)). */
VQ_API int vq_hdr_encode_rgbe(VqContext* ctx, VqImage in, void* dev_rgbe, void* stream);
/* HOST. RGBE texels -> the .hdr file image (text header + per-scanline run lists). file == NULL: size query. */
VQ_API int vq_hdr_pack_file(const void* host_rgbe, int width, int height, void* file, uint64_t capacity, uint64_t* size);
/* Blocking: device fp32 image -> host file image (encode + download + pack). Ordered after all earlier device work, on any
 * stream: a kernel still writing `in` finishes before it is encoded. */
VQ_API int vq_hdr_save_host(VqContext* ctx, VqImage in, void* host_file, uint64_t capacity, uint64_t* size);

/* Image::CreateResizedImage (Image.cpp:148-190) -> stbir_resize_float(in, w, h, 0, out, W, H, 0, 4): the downsize the engine
 * applies to a hi-res HDRI before saving the smaller .hdr (EnvironmentMap.cpp:142-209; 8k -> 4k/2k/1k). Separable
 * Mitchell-Netravali, edge clamp, weights normalised per output sample; bit-identical to the vendored stb_image_resize
 * v0.96. out.width <= in.width and out.height <= in.height (otherwise VQ_ERR_UNSUPPORTED). The intermediate image and the gather
 * tables live in the context (grow-only; tables are rebuilt when the size pair changes): serialise calls per context. */
VQ_API int vq_image_resize(VqContext* ctx, VqImage in, VqImage out, void* stream);
/* Non-finite inputs: stb adds a coefficient only where it is nonzero. The gather tables start and end every output's taps at
 * a nonzero weight, so +-Inf and NaN reach the same outputs as in stb, with one exception: at ratios where a Mitchell weight
 * rounds to exactly 0 between two taps of an output (|x| = 8/7; 7:5, for example), the kernels add 0 * Inf = NaN where stb
 * adds nothing. Finite inputs are bit-identical either way. */
/* HOST. The per-axis gather table vq_image_resize builds (first tap, tap count, normalised weights per output sample):
 * out[i] = sum_{t<count[i]} weights[i*capacity_taps + t] * in[clamp(start[i]+t, 0, in_size-1)], taps in increasing order.
 * start == NULL: only *max_taps is written. */
VQ_API int vq_resize_axis_table(int in_size, int out_size, int* start, int* count, float* weights, int capacity_taps, int* max_taps);

/* ------------------------------------------------------------------------------------------
 * SURVEY §8(f).3  The two streaming passes that complete a headless frame.
 *   Skydome: replaces the environment-map draw at SceneRendering.cpp:1821-1850 + PSMain (Skydome.hlsl:35-56).
 *     inv_view_proj = inverse of the matViewProj the engine uploads (SceneView.EnvironmentMapViewProj = skyCam.View *
 *     skyCam.Proj, Scene.cpp:573-584; row-vector convention), computed by the caller. The pass writes {rgb, 1} to
 *     rows [row_begin,row_end) of scene_color where no surface was shaded: pixels whose normal_mask texel has
 *     xyz == 0 (the G-buffer normal plane; the engine gets the same effect from the depth test), or every pixel when
 *     normal_mask is NULL. A ray that keeps no direction (its w rounds to 0, or |ray / w|^2 overflows fp32) is drawn black.
 *     Signed zeros follow atan2: the centre pixel of an axis-aligned camera looking along +-Y whose ray has x = -0 maps to
 *     u = 0 or 1 (the -X seam), not to u = 0.5.
 *   ApplyReflections: replaces CSMain (ApplyReflections.hlsl:31-57): scene.rgb += reflection.rgb, alpha kept;
 *     with a bounding_volumes layer (COMPOSITE_BOUNDING_VOLUMES) the sum is blended under it. In place.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_skydome(VqContext* ctx, const VqMatrix* inv_view_proj, VqPyramid hdri, const VqImage* normal_mask,
                      VqImage scene_color, int row_begin, int row_end, void* stream);
VQ_API int vq_apply_reflections(VqContext* ctx, VqImage scene_color, VqImage reflection_radiance,
                                const VqImage* bounding_volumes, void* stream);
/* Both passes on one rank's band of a multi-GPU frame, in the multi-destination form of the vq_*_multi_signal shading calls:
 * rows [row_begin,row_end) of the per-pixel inputs (normal_mask, reflection_radiance, bounding_volumes: the band only, or the whole
 * frame) are rows dst_row_offset + y of the frame. outs[0] is the rank's local frame, the source of the band and its first
 * destination; outs[1..n_outs-1] are the peers' frames mapped into this process. Every destination has the frame's size. One launch,
 * no context scratch; with a `signal` (n_ranks > 1) the kernel's last CTA runs the rendezvous of VqPeerSignal after every store.
 *   vq_skydome_multi_signal: afterwards rows dst_row_offset + [row_begin,row_end) of every destination hold, bit for bit, what
 *     outs[0] holds after vq_skydome on those frame rows with the mask at frame rows: where the mask's xyz is 0 (or everywhere when
 *     normal_mask is NULL) the sky along the ray through frame pixel (x, dst_row_offset + y); elsewhere what outs[0] already held,
 *     read back and copied to the peers. So one rank's scene-colour step is its shading call into outs[0] alone (no signal), then
 *     this call into every rank's frame: each pixel crosses NVLink once and has one writer. Where the alpha mask of a
 *     from-materials call discarded a pixel, outs[0]'s previous content is what is distributed. For from-materials frames the mask
 *     is the interpolants' normal_v plane (xyz 0 where nothing was rasterised).
 *   vq_apply_reflections_multi_signal: vq_apply_reflections in place on the band's rows of outs[0], the result stored into every
 *     destination. Run it after the sky's rendezvous, when every rank's frame is whole.
 * Refused with VQ_ERR_INVALID_ARG before the device is touched (also without a context): what the single call refuses; n_outs
 * outside 1..8, destinations of different sizes, a peer destination equal to outs[0], a negative offset, rows
 * dst_row_offset + [row_begin,row_end) outside the frame, a signal with n_ranks > 1 and one destination or an empty row range, a
 * bad signal; a mask, reflection or bounding-volume plane that is not as wide as the frame or has fewer than row_end rows. An empty
 * row range without a rendezvous launches nothing. */
VQ_API int vq_skydome_multi_signal(VqContext* ctx, const VqMatrix* inv_view_proj, VqPyramid hdri, const VqImage* normal_mask,
                                   const VqImage* outs, int n_outs, int dst_row_offset, int row_begin, int row_end,
                                   const VqPeerSignal* signal, void* stream);
VQ_API int vq_apply_reflections_multi_signal(VqContext* ctx, VqImage reflection_radiance, const VqImage* bounding_volumes,
                                             const VqImage* outs, int n_outs, int dst_row_offset, int row_begin, int row_end,
                                             const VqPeerSignal* signal, void* stream);

/* ------------------------------------------------------------------------------------------
 * SURVEY §8(f).4  Shadowed casters and the hierarchical MIN depth pyramid.
 *   vq_forward_lighting_shadowed: vq_forward_lighting with the shadow maps PSMain binds (ForwardLighting.hlsl:87-89):
 *     the caster lists are multiplied by OmnidirectionalShadowTestPCF / ShadowTestPCF and a shadowing directional light
 *     by ShadowTestPCF_Directional (Lighting.hlsl:79-272; ForwardLighting.hlsl:321-377). Maps are linear R32F, tightly
 *     packed, POINT-sampled with WRAP addressing (RootSignatures.cpp:148):
 *       point_cubes      [caster][face][y][x], value = distance / light range   (TextureCubeArray, t22)
 *       spot_maps        [caster][y][x],       value = light-space depth         (Texture2DArray, t16)
 *       directional_map  [y][x]                                                   (Texture2D, t13)
 *     A NULL map lights that light type unshadowed (factor 1). shadowViews / shadowViewDirectional and the
 *     f2*ShadowMapDimensions fields of per_frame are read as the shader reads them.
 *     Two launches: a PCF kernel that stores the shadowed-tap counts of every caster per pixel (8 B/pixel of scratch owned
 *     by the context), then the forward kernel, which weights the caster lights with them. Because of that scratch, calls
 *     on ONE context must be issued on one stream at a time (like vq_depth_min_pyramid).
 *   vq_depth_min_pyramid: replaces CSMain (DownsampleDepth.hlsl:85-119 = FidelityFX SPD with a MIN reduction): level 0 is
 *     a copy of the R32F depth image, level l = max(1, w>>l) x max(1, h>>l) holds the 2x2 minimum of the zero-padded
 *     level above; `levels` receives n_levels (<= vq_depth_pyramid_level_count = 1 + floor(log2(max(w,h))), at most 13)
 *     tightly packed levels, vq_depth_pyramid_texel_count() floats in total. The padded-domain levels ping-pong through scratch
 *     owned by the context (like vq_image_resize): calls on ONE context must be issued on one stream at a time.
 *     The minimum ignores NaN unless all four texels are NaN. Where the smallest value of a 2x2 block is a zero and zeros of
 *     both signs reach it (a +0 and a -0 depth, or a -0 next to the zero padding), the sign of the result is not specified,
 *     as D3D's min leaves it; every other result, denormals and infinities included, is exact.
 *   Parity: tests/test_shadow_gpu.py (15 tests against the oracle, itself pinned to the reference's shader text) and
 *     tests/test_frame_domain_gpu.py (every size edge, special depths, every n_levels, unaligned sources).
 * ------------------------------------------------------------------------------------------ */
typedef struct VqShadowMaps {
    const void* point_cubes;     int32_t point_res;
    const void* spot_maps;       int32_t spot_width, spot_height;
    const void* directional_map; int32_t directional_width, directional_height;
} VqShadowMaps;
VQ_API int vq_forward_lighting_shadowed(VqContext* ctx,
                                        const VqPerFrameData* per_frame,
                                        const VqPerViewLightingData* per_view,
                                        const VqGBuffer* gbuffer,
                                        const VqEnvironmentMaps* env,
                                        const VqShadowMaps* shadow_maps,
                                        VqImage out_color,
                                        int row_begin, int row_end,
                                        void* stream);
/* vq_forward_lighting_from_materials with the shadow maps bound: computes what vq_gbuffer_from_materials (with an emissive
 * plane) followed by vq_forward_lighting_shadowed(ctx, per_frame, per_view, &gb, env, shadow_maps, out_color, ...) computes,
 * bit for bit (with the same yaw caveat as vq_forward_lighting_from_materials), in ONE launch: the PCF tests run inside the
 * kernel on the positions and normals it has just produced, so neither the G-buffer nor the PCF records reach device memory
 * and the call uses no context scratch beyond the environment's sampling copies (the one-stream rule of
 * vq_forward_lighting_shadowed does not apply). Maps, caster lists and the f2*ShadowMapDimensions fields are read as
 * vq_forward_lighting_shadowed reads them; when no test runs (no map bound for any caster type present) the result is
 * vq_forward_lighting_from_materials's. Pixels the alpha mask discards are left untouched. Every argument is checked before
 * the device is touched. */
VQ_API int vq_forward_lighting_shadowed_from_materials(VqContext* ctx, const VqPerFrameData* per_frame,
                                                       const VqPerViewLightingData* per_view, const VqSurfaceInputs* in,
                                                       const VqMaterialTable* table, int alpha_mask, const VqEnvironmentMaps* env,
                                                       const VqShadowMaps* shadow_maps, VqImage out_color,
                                                       int row_begin, int row_end, void* stream);
VQ_API int      vq_depth_pyramid_level_count(int width, int height);
VQ_API uint64_t vq_depth_pyramid_texel_count(int width, int height, int levels);
VQ_API int vq_depth_min_pyramid(VqContext* ctx, VqImage depth_r32f, void* levels, int n_levels, void* stream);

/* ------------------------------------------------------------------------------------------
 * Blocking host-buffer entry points: the same passes called with HOST pointers (what an engine
 * integration that keeps its frame data in system memory would call). Each call uploads the
 * inputs, runs the kernel(s), downloads the result and returns when the result is in `out`.
 * Transfers are chunked by rows and overlapped with compute on internal streams.
 * ------------------------------------------------------------------------------------------ */
VQ_API int vq_forward_lighting_host(VqContext* ctx,
                                    const VqPerFrameData* per_frame,
                                    const VqPerViewLightingData* per_view,
                                    const VqGBuffer* host_gbuffer,
                                    const VqEnvironmentMaps* device_env,
                                    VqImage host_out_color);

#ifdef __cplusplus
}
#endif

/* The environment prefilter across GPUs: the band forms of K2 and K4 and the one-launch cube blur. */
#include "vqcuda_prefilter_multi.h"

/* The Gaussian blur of the post chain in one launch, and its band form. */
#include "vqcuda_blur.h"

#endif /* VQCUDA_H */
