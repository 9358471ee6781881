/* vf_b200_lpips.h — the LPIPS image metric of the reference's evaluators (utils/metrics.py:199-214 LPIPSMetric, models/utils.py:297-307:
 * lpips.LPIPS(net='vgg', version='0.1') on images in [0, 1]), in libvf_b200.so next to the entry points of vf_b200.h and under its
 * conventions (raw device pointers, plain sizes, vf_stream_t, 0 or a negative code with vf_last_error()).
 *
 * The 13 VGG16 convolutions run in fp32: the first (3 -> 64) here, the other 12 as exact split-fp16 vf_tc_gemm convolutions with the
 * VF_ACT_RELU epilogue.  Activations are NHWC; a batch holds the 2N images of N pairs, the first images of all pairs, then the second ones.
 *   vf_lpips_conv_in: y [N,H,W,Cout] = relu(conv3x3 pad 1 (s) + bias) of uint8 images x [N,H,W,3], where the conv input is
 *     s = (x * fp32(1/255) - shift[c]) / scale[c] per channel (tf.image.convert_image_dtype, then lpips' ScalingLayer), each operation
 *     rounded once in fp32; the padding is zero in s.  w_kn [27, Cout] fp32 (k = tap * 3 + c, tap = 3 (dy + 1) + dx + 1), Cout % 16 == 0,
 *     Cout <= 128; shift, scale [3].  (vf_conv3x3_small_cin's kernel.)
 *   vf_maxpool2x2_split: fp32 x [N,H,W,C] -> split fp16 [N, H/2, W/2, hi(C) | lo(C)] (sizes floored), the max of each 2x2 window taken in
 *     fp32 (a NaN in the window gives NaN) and split as vf_split_f16x2 does: the operand of the next exact convolution.  C % 4 == 0.
 *   vf_lpips_tap: one tap's term of every pair.  f [2N, H*W, C] fp32 (pair n: images n and n + N), lin [C]: for each pixel
 *     d = sum_c lin[c] (f0[c] / (|f0| + 1e-10) - f1[c] / (|f1| + 1e-10))^2 with |f| the channel L2 norm, all in fp32; then
 *     out[n] += (sum over pixels of d) / (H*W), summed in fp64 in a fixed order (no atomics: a repeated call gives the same bits).
 *     partial: fp64 scratch of N * ceil(H*W / 64) values.  C = 64, 128, 256 or 512.
 */
#ifndef VF_B200_LPIPS_H
#define VF_B200_LPIPS_H

#include "vf_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

int vf_lpips_conv_in(const uint8_t* x, const float* shift, const float* scale, const float* w_kn, const float* bias, int N, int H, int W,
                     int Cout, float* y, vf_stream_t s);
int vf_maxpool2x2_split(const float* x, int N, int H, int W, int C, void* out_f16, vf_stream_t s);
int vf_lpips_tap(const float* f, int N, int H, int W, int C, const float* lin, double* partial, double* out, vf_stream_t s);

#ifdef __cplusplus
}
#endif

#endif /* VF_B200_LPIPS_H */
