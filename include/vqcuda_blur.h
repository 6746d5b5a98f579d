/*
 * vqcuda_blur.h — K5, the 21-tap Gaussian blur of the post chain (GaussianBlur.hlsl:119-186), X then Y in one launch, and its
 * band form for one rank of a multi-GPU frame; part of the C-ABI of vqcuda.h (which includes this header; either may be included
 * first). Every call here follows vqcuda.h's conventions: it only enqueues on `stream`, grows no context scratch and is
 * re-entrant. A rank's blurred frame followed by its post chain band, and why that order is safe: DESIGN.md §6.
 */
#ifndef VQCUDA_BLUR_H
#define VQCUDA_BLUR_H

#include "vqcuda.h"

#ifdef __cplusplus
extern "C" {
#endif

/*   vq_gaussian_blur: X then Y in one launch, with no intermediate image and no context scratch (calls on several streams of one
 *     context are fine). `out` equals, bit for bit, vq_gaussian_blur_x(in -> tmp) followed by vq_gaussian_blur_y(tmp -> out), on
 *     every input including +-Inf, NaN and subnormals; pixels outside iImageSize are not touched. Refused with
 *     VQ_ERR_INVALID_ARG before the device is touched (also with a NULL context): the checks of vq_gaussian_blur_x with its
 *     messages (null params, bad descriptors, a non-positive iImageSize or one that exceeds either image, in == out).
 *   vq_gaussian_blur_multi_signal: one rank's band of vq_gaussian_blur into several frames, under the contract of the K6-K9
 *     multi-destination calls of vqcuda.h (vq_tonemap_multi_signal). `in` is the whole source frame: the call reads the band's 10-row
 *     halo itself. Rows [row_begin,row_end) are output rows within [0, iImageSizeY]; each of the n_outs (1..8) destinations has
 *     the size of outs[0]. Into each destination the call stores exactly the bits vq_gaussian_blur stores on those rows and
 *     touches no other row. Also refused: `in` equal to any destination, n_outs outside 1..8, rows outside [0, iImageSizeY] or
 *     reversed, and a signal with n_ranks > 1 and one destination or an empty row range. */
VQ_API int vq_gaussian_blur(VqContext* ctx, const VqBlurParams* params, VqImage in, VqImage out, void* stream);
VQ_API int vq_gaussian_blur_multi_signal(VqContext* ctx, const VqBlurParams* params, VqImage in, const VqImage* outs, int n_outs,
                                         int row_begin, int row_end, const VqPeerSignal* signal, void* stream);

#ifdef __cplusplus
}
#endif
#endif /* VQCUDA_BLUR_H */
