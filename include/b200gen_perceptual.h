/*
 * b200gen_perceptual.h — the perceptual-distance part of libb200gen.so's C-ABI (PerceptualLoss with
 * network_type="resnet50" of generative/losses/perceptual.py in the reference): the input preparation in front of the
 * ResNet-50 feature network and the distance between its features.  The network itself runs on b200gen.h's
 * convolution, pooling and BatchNorm-fold entry points.
 */
#ifndef B200GEN_PERCEPTUAL_H_
#define B200GEN_PERCEPTUAL_H_

#include "b200gen.h"

#ifdef __cplusplus
extern "C" {
#endif

/* ------------------------------------------------------------------------------------------------
 * The conventions of b200gen.h hold (return codes, no allocation, no synchronisation, work enqueued on `stream`).
 * ------------------------------------------------------------------------------------------------ */
#define B200_PERCEPTUAL_EPS 1e-10f

/* b200_perceptual_prep: both inputs of one perceptual call (x = input, y = target) to channels-last h16 images
 * [n_out][OH][OW][8] for the network, in one launch.  Source element (image q, channel c, row h, column w) of an input
 * is at  (q / S) * st[0] + c * st[1] + (q % S) * st[2] + h * st[3] + w * st[4]  (elements; host array st[5] per input,
 * any strides), in B200_DT_F32 / _F64 / _FP16 / _BF16.  S = 1 with st[2] = 0 reads 2-D images [N][C][H][W]; a 2.5-D
 * slice set along one spatial axis of [N][C][D0][D1][D2] puts that axis at st[2] and the remaining two, in order, at
 * st[3] (OH) and st[4] (OW) — the reference's permute(0, axis, 1, rest), so q = n * S + slice.
 * Output image b reads source image q = idx[b] (idx: device int64 [n_out], values in [0, N * S)), or q = b when idx is
 * NULL.  C is 1 or 3; with C == 1 the one channel is read for all three (the reference's repeat, which it applies only
 * when both inputs have one channel — the caller passes C == 1 only then).  Channel c of the output is
 *   h16( (fp32(v) - mean[c]) / std[c] ),  mean = {0.485f, 0.456f, 0.406f}, std = {0.229f, 0.224f, 0.225f},
 * fp32 subtraction and division, one rounding to h16 (torchvision's ImageNet z-score); channels 3..7 are +0.
 * out_x / out_y 16-byte aligned. */
int b200_perceptual_prep(const void* x, int32_t x_dtype, const int64_t* x_strides, const void* y, int32_t y_dtype,
                         const int64_t* y_strides, int32_t C, int32_t S, int32_t OH, int32_t OW, const int64_t* idx,
                         int32_t n_out, void* out_x, void* out_y, void* stream);

/* b200_perceptual_distance: per-image perceptual distance of two feature maps x, y, each [B][HW][pitch] in
 * B200_DT_F32 or B200_DT_H16 (the same for both), C channels (C <= pitch).  Per pixel p, in fp32:
 *   n_x = sqrt(sum_c x_c^2),  n_y likewise,
 *   pixel[b][p] = sum_c (x_c / (n_x + 1e-10f) - y_c / (n_y + 1e-10f))^2
 * in this direct form (two passes over the channels; not sum x^2 + sum y^2 - 2 sum xy, which cancels when x ~ y).
 * Each sum of squares is accumulated with fused multiply-adds over channels c = lane, lane + 32, ... of one warp in
 * order, then a butterfly over the 32 lanes, so every pixel's value is a fixed function of its two channel vectors.  Then per image, in fp64 and a fixed order without
 * atomics: image[b] = (sum_p pixel[b][p]) / HW, and image32[b] = fp32(image[b]) when image32 is not NULL.
 * Bitwise-equal x and y give exactly 0.  pixel: fp32 workspace [B][HW]. */
int b200_perceptual_distance(const void* x, const void* y, int32_t dtype, int32_t B, int32_t HW, int32_t C,
                             int32_t pitch, float* pixel, double* image, float* image32, void* stream);

/* b200_perceptual_mean: the loss from the per-image values of up to 3 groups stored one after another in image
 * (group g holds counts[g] >= 1 values; counts is a host array): means[g] = (sum of group g in index order) / counts[g],
 * means[n_groups] = sum_g means[g] in g order, all fp64; *loss = fp32(means[n_groups]).  One launch. */
int b200_perceptual_mean(const double* image, int32_t n_groups, const int32_t* counts, double* means, float* loss,
                         void* stream);

#ifdef __cplusplus
}
#endif
#endif /* B200GEN_PERCEPTUAL_H_ */
