/* sessd_b200_lab.h -- C ABI of libsessd_b200_lab.so (csrc/bevconv_split.cu): the BEV conv with its fp32 NHWC input split into two-term
 * fp16 inside the wgmma kernel and three separate products per MAC, the bitwise reference of the product kernel's folded wgmma
 * (tests/test_gpu_bev_p2_vs_h2.py); clock-counting and loader-only builds of the product's planes kernel for stall profiles; and the
 * launcher's plan, for the tests' restatement of it.  Nothing in the product path (libsessd_b200.so, sessd_b200.engine) links or
 * loads this library.  Same conventions as sessd_b200.h. */
#ifndef SESSD_B200_LAB_H
#define SESSD_B200_LAB_H

#include "sessd_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

/* fp16-split BEV conv from fp32 input (the split happens in shared memory): in_stride 1 or 2, cin % 64 == 0, cout % 8 == 0; a stride-2
 * 3x3 patch and its fp32 staging copy leave room for the weight ring only at cout_pad 32 (else SESSD_EINVAL).  cout_pad is a multiple of
 * the N tile (128; 32 when cout <= 32).
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

/* Stall profile of the product's planes conv / deconv (sessd_bev_conv_p2 / sessd_bev_deconv_p2, same arguments and results, d_prof
 * between d_segs and the stream): the kernel's clock counters are written to d_prof, int64 [grid][16] with grid = min(work items, SMs); word order in csrc/bevconv_p2.cuh
 * (P2Prof).  For measurement only: the counters cost clocks of their own. */
int sessd_bev_conv_p2_profile(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                              const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                              float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info,
                              const sessd_conv_desc *desc, const int *d_items, const int *d_segs, long long *d_prof, void *stream);
int sessd_bev_deconv_p2_profile(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                                const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                                float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info, int batch,
                                int in_h, int in_w, int cin, int cout, int relu, const int *d_items, const int *d_segs,
                                long long *d_prof, void *stream);

/* Loader-only probe of sessd_bev_conv_p2_profile's launch: the two TMA producer warps run unchanged, the consumers wait on the full
 * barriers and release them without issuing wgmma or an epilogue, so the launch's time is what the loads alone take (no output is
 * written; d_prof as above).  smem_a != 0 plans a stride-1 conv's patches as shared-memory A descriptors would need them, one copy
 * per tap shift along u, instead of the single copy the register-fed A reads: the traffic of these launches before and after. */
int sessd_bev_conv_p2_loads(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                            const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                            float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info,
                            const sessd_conv_desc *desc, const int *d_items, int smem_a, long long *d_prof, void *stream);
/* The same probe on a segment record of sessd_bev_skip_plan (d_segs, required; stride-1 conv): the patch layout of segment windows. */
int sessd_bev_conv_p2_seg_loads(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                                const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                                float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info,
                                const sessd_conv_desc *desc, const int *d_segs, long long *d_prof, void *stream);

/* The launch plan of the conv desc (deconv != 0: of the deconv of desc's batch, in_h, in_w, cin and cout) as sessd_bev_conv_p2 (split 0;
 * smem_a as for sessd_bev_conv_p2_loads) or sessd_bev_conv_h2 (split != 0) would launch it, without launching: plan[19] =
 * {u_is_x, n_tile, nblocks, tiles, total, ncopies, rows_v, pitch_u, npatch, bstages, dynamic shared memory bytes, taps of class 0-3,
 * class order 0-3} (0 past the launch's classes).  SESSD_EINVAL where the launcher refuses the launch.  Touches no device. */
int sessd_bev_p2_plan(const sessd_conv_desc *desc, int deconv, int cout_pad, int split, int smem_a, int *plan);

#ifdef __cplusplus
}
#endif
#endif
