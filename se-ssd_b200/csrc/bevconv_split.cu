// bevconv_split.cu -- the lab formats of the BEV conv / deconv (include/sessd_b200_lab.h): fp32 NHWC input split inside the wgmma kernel
// of bevconv_p2.cuh.  TMA stages the fp32 patch in shared memory and the consumer warpgroups split it there:
//   * sessd_bev_conv_tc / sessd_bev_deconv_tc: 3xTF32 -- x = tf32(x) + (x - tf32(x)), fp32 weights pre-split the same way (ops.pack_weight_tc);
//     three tf32 wgmma products per MAC (hi hi, hi lo, lo hi) over 16-channel stages;
//   * sessd_bev_conv_h2 / sessd_bev_deconv_h2: x * 2^s = fp16 hi + fp16 lo with 2^s from the input's abs-max, fp16 weights of
//     ops.pack_weight_h2; three fp16 wgmma products over 32-channel stages.
#include "bevconv_p2.cuh"

#include "../../include/sessd_b200_lab.h"

using namespace sessd;

extern "C" int sessd_bev_conv_tc(const float *d_in, const float *d_weight_split, int cout_pad, const float *d_scale, const float *d_shift,
                                 const float *d_residual, float *d_out, const sessd_conv_desc *desc, void *stream) {
    if (!d_in || !d_out) return SESSD_EINVAL;
    return p2_conv<kP2SplitTf32>(d_in, nullptr, d_weight_split, cout_pad, d_scale, d_shift, d_residual, nullptr, 0.f, 0.f, d_out, nullptr, nullptr,
                                 desc, stream);
}

extern "C" int sessd_bev_deconv_tc(const float *d_in, const float *d_weight_split, int cout_pad, const float *d_scale, const float *d_shift,
                                   const float *d_residual, float *d_out, int batch, int in_h, int in_w, int cin, int cout, int relu,
                                   void *stream) {
    if (!d_in || !d_out) return SESSD_EINVAL;
    return p2_deconv<kP2SplitTf32>(d_in, nullptr, d_weight_split, cout_pad, d_scale, d_shift, d_residual, nullptr, 0.f, 0.f, d_out, nullptr,
                                   nullptr, batch, in_h, in_w, cin, cout, relu, stream);
}

extern "C" int sessd_bev_conv_h2(const float *d_in, const void *d_weight_h2, int cout_pad, const float *d_scale, const float *d_shift,
                                 const float *d_residual, float *d_out, const sessd_conv_desc *desc, const float *d_amax_in,
                                 float *d_amax_out, void *stream) {
    if (!d_in || !d_out || !d_scale) return SESSD_EINVAL;
    return p2_conv<kP2SplitF16>(d_in, d_amax_in, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, nullptr, 0.f, 0.f, d_out, nullptr,
                                d_amax_out, desc, stream);
}

extern "C" int sessd_bev_deconv_h2(const float *d_in, const void *d_weight_h2, int cout_pad, const float *d_scale, const float *d_shift,
                                   const float *d_residual, float *d_out, int batch, int in_h, int in_w, int cin, int cout, int relu,
                                   const float *d_amax_in, float *d_amax_out, void *stream) {
    if (!d_in || !d_out || !d_scale) return SESSD_EINVAL;
    return p2_deconv<kP2SplitF16>(d_in, d_amax_in, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, nullptr, 0.f, 0.f, d_out, nullptr,
                                  d_amax_out, batch, in_h, in_w, cin, cout, relu, stream);
}
