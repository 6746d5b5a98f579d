/*
 * vqcuda_prefilter_multi.h — the environment-map prefilter (PreFilterEnvironmentMap, EnvironmentMapRendering.cpp:181-485)
 * across GPUs, part of the C-ABI of vqcuda.h (which includes this header; either may be included first). One rank's band of K2
 * (diffuse irradiance) and of K4 (BRDF LUT) into every rank's buffers with the in-kernel rendezvous of VqPeerSignal, and K5 on
 * the whole diffuse cube in one launch. With vq_specular_prefilter_ranges (vqcuda.h) a rank's environment step is four launches
 * and needs no collective library: the diffuse band (rendezvous, epoch e), vq_gaussian_blur_cube from the local diffuse cube
 * into the local blurred cube, the specular ranges (rendezvous, epoch e + 1), vq_environment_prepare. The blurred cube must not
 * be a peer destination: a peer's next diffuse stores may land while this rank still reads it (DESIGN.md §6).
 * Every call here follows vqcuda.h's conventions: it only enqueues on `stream`, grows no context scratch and is re-entrant.
 */
#ifndef VQCUDA_PREFILTER_MULTI_H
#define VQCUDA_PREFILTER_MULTI_H

#include "vqcuda.h"

#ifdef __cplusplus
extern "C" {
#endif

/* K2 on one rank's band, into several cubemaps: rows [row_begin,row_end) of the flattened (face, row) space are stored into each
 * of the n_outs (1..8) cubemaps of identical shape (res, 1 mip): the local one first, then the other ranks' buffers mapped into
 * this process. Into each it stores exactly the bits vq_diffuse_irradiance stores on those rows, and touches no other row. One
 * launch, no context scratch: calls on several streams of one context are fine. With `signal` (n_ranks > 1) the kernel's last
 * CTA runs the rendezvous of VqPeerSignal after every store; NULL: no rendezvous. An empty row range launches nothing.
 * Refused with VQ_ERR_INVALID_ARG before the device is touched (also with a NULL context): vq_diffuse_irradiance's checks and
 * messages on outs[0], a NULL list, n_outs outside 1..8, a destination of another shape or equal to outs[0], a signal with
 * n_ranks > 1 and one destination or an empty row range, and a bad signal descriptor. */
VQ_API int vq_diffuse_irradiance_multi_signal(VqContext* ctx, const VqDiffuseIrradianceParams* params, VqPyramid hdri,
                                              const VqCubemap* outs, int n_outs, int row_begin, int row_end,
                                              const VqPeerSignal* signal, void* stream);

/* K4 on one rank's band, into several LUTs: rows [row_begin,row_end) into each of the n_outs (1..8) float2 images of one size
 * (pitches may differ; the local one first), bit for bit what vq_brdf_integration_lut stores on those rows; no other row is
 * touched. One launch, no context scratch; `signal` and the empty range as for vq_diffuse_irradiance_multi_signal.
 * Refused with VQ_ERR_INVALID_ARG before the device is touched (also with a NULL context): bad descriptors, destinations of
 * another size or equal to outs[0], n_outs outside 1..8, num_samples outside 1..8192, rows outside the image or reversed, and
 * the signal rules above. */
VQ_API int vq_brdf_integration_lut_multi_signal(VqContext* ctx, const VqImage* outs, int n_outs, int num_samples,
                                                int row_begin, int row_end, const VqPeerSignal* signal, void* stream);

/* K5 on a whole one-mip cubemap in one launch: every face blurred X then Y, clamp-to-edge per face, alpha = 1, with no
 * intermediate image in device memory (a face's X pass stays in shared memory). Each face of `out` equals, bit for bit,
 * vq_gaussian_blur_x on the face into a temporary, then vq_gaussian_blur_y into `out` (EnvironmentMapRendering.cpp:341-372).
 * in == out (the same cube) is supported: each face is read completely before any of it is written. One launch, no context
 * scratch. Refused with VQ_ERR_INVALID_ARG before the device is touched (also with a NULL context): a null or misaligned
 * cubemap, mips != 1, a face edge outside 1..128 (the engine's diffuse cube is 64), in and out of different resolutions, and
 * cubes that overlap without being the same cube. */
VQ_API int vq_gaussian_blur_cube(VqContext* ctx, VqCubemap in, VqCubemap out, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VQCUDA_PREFILTER_MULTI_H */
