/* sessd_b200_lab.h -- C ABI of libsessd_b200_lab.so: the NON-DEFAULT BEV conv variants kept for cross-implementation tests
 * (csrc/bevconv_split.cu): fp32 NHWC input split inside the wgmma kernel, either into 3xTF32 (tf32 wgmma) or into two-term fp16
 * (fp16 wgmma).  Nothing in the product path (libsessd_b200.so, sessd_b200.engine) links or loads this library.  Same conventions as
 * sessd_b200.h. */
#ifndef SESSD_B200_LAB_H
#define SESSD_B200_LAB_H

#include "sessd_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* 3xTF32 BEV conv (tf32 wgmma, three products per MAC): same contract as sessd_bev_conv (in_stride 1 or 2, cin % 64 == 0, cout % 8 == 0).
 * d_weight_split [2 (hi|lo)][ntaps][cout_pad][cin]: hi = weights truncated to tf32, lo = w - hi; cout_pad is a multiple of the
 * N tile (128; 32 when cout <= 32).  d_scale nullable (identity). */
int sessd_bev_conv_tc(const float *d_in, const float *d_weight_split, int cout_pad, const float *d_scale,
                      const float *d_shift, const float *d_residual, float *d_out, const sessd_conv_desc *desc,
                      void *stream);

/* ConvTranspose2d(k3, s2, p1, op1) + BN + ReLU (+ residual) in one launch; d_weight_split [2][9][cout_pad][cin],
 * tap = ky*3+kx of W[cin][cout][ky][kx]; output [batch, 2*in_h, 2*in_w, cout] NHWC (rpn_v1.py:183-195). */
int sessd_bev_deconv_tc(const float *d_in, const float *d_weight_split, int cout_pad, const float *d_scale,
                        const float *d_shift, const float *d_residual, float *d_out, int batch, int in_h, int in_w,
                        int cin, int cout, int relu, void *stream);

/* fp16-split BEV conv from fp32 input (the split happens in shared memory): same contract as sessd_bev_conv_tc, in_stride 1 only
 * (a stride-2 patch and its fp32 staging copy do not fit in shared memory: SESSD_EINVAL).
 * d_weight_h2: __half [2 (hi|lo)][ntaps][cout_pad][cin] of 2^e[n]*w (per output channel n; max |2^e w| in [2^10, 2^11));
 * d_scale (required) = folded BN scale * 2^-e[n].
 * d_amax_in  (nullable): device scalar >= max|in| -- selects the activation scaling 2^s; NULL = no scaling (|in| must stay < 65504).
 * d_amax_out (nullable): device scalar, atomically raised to max|out| (the next layer's d_amax_in); zero it once per frame. */
int sessd_bev_conv_h2(const float *d_in, const void *d_weight_h2, int cout_pad, const float *d_scale,
                      const float *d_shift, const float *d_residual, float *d_out, const sessd_conv_desc *desc,
                      const float *d_amax_in, float *d_amax_out, void *stream);
int sessd_bev_deconv_h2(const float *d_in, const void *d_weight_h2, int cout_pad, const float *d_scale,
                        const float *d_shift, const float *d_residual, float *d_out, int batch, int in_h, int in_w,
                        int cin, int cout, int relu, const float *d_amax_in, float *d_amax_out, void *stream);

#ifdef __cplusplus
}
#endif
#endif
