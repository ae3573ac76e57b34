// bevconv_split.cu -- the lab library's builds of the wgmma kernel of bevconv_p2.cuh (include/sessd_b200_lab.h):
//   * sessd_bev_conv_h2 / sessd_bev_deconv_h2: fp32 NHWC input split inside the kernel -- TMA stages the fp32 patch in shared memory and
//     the consumer warpgroups split it there into x * 2^s = fp16 hi + fp16 lo (2^s from the input's abs-max); fp16 weights of
//     ops.pack_weight_h2; three separate fp16 wgmma products per MAC over 32-channel stages.  The product kernel's folded
//     a_hi x [b_lo ; b_hi] wgmma must sum the same products in the same order: this mode is its bitwise reference;
//   * the clock-counting and loader-only probes of the product's planes kernel (stall profiles);
//   * sessd_bev_p2_plan: the launcher's plan, host only (tests compare their restatement of it against this).
#include "bevconv_p2.cuh"

#include "../../include/sessd_b200_lab.h"

using namespace sessd;

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

// Stall profile of the product's planes kernel (scripts/p2_stall_profile.py): sessd_bev_conv_p2 / sessd_bev_deconv_p2 with the clock
// counters of the kP2ProbeClocks instantiation written to d_prof, [grid][kP2ProfWords] int64 (P2Prof, grid = min(work items, SMs)).
extern "C" int sessd_bev_conv_p2_profile(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                                         const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                                         float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info,
                                         const sessd_conv_desc *desc, const int *d_items, const int *d_segs, long long *d_prof,
                                         void *stream) {
    return p2_conv<kP2Planes, kP2ProbeClocks>(d_in_planes, d_in_info, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain,
                                              shift_max, d_out_f32, d_out_planes, d_out_info, desc, stream, d_items, d_prof, false, d_segs);
}

extern "C" int sessd_bev_deconv_p2_profile(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                                           const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                                           float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info, int batch,
                                           int in_h, int in_w, int cin, int cout, int relu, const int *d_items, const int *d_segs,
                                           long long *d_prof, void *stream) {
    return p2_deconv<kP2Planes, kP2ProbeClocks>(d_in_planes, d_in_info, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain,
                                                shift_max, d_out_f32, d_out_planes, d_out_info, batch, in_h, in_w, cin, cout, relu, stream,
                                                d_items, d_prof, d_segs);
}

// The loader-only probe: the launch of sessd_bev_conv_p2_profile with consumers that wait on the full barriers and release them,
// no wgmma and no epilogue (no output is written).  smem_a != 0 plans a stride-1 conv's patches as shared-memory A descriptors would
// need them (one copy per tap shift along u), the plan these launches had before A came from registers.
extern "C" int sessd_bev_conv_p2_loads(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                                       const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                                       float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info,
                                       const sessd_conv_desc *desc, const int *d_items, int smem_a, long long *d_prof, void *stream) {
    return p2_conv<kP2Planes, kP2ProbeLoads>(d_in_planes, d_in_info, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain,
                                             shift_max, d_out_f32, d_out_planes, d_out_info, desc, stream, d_items, d_prof, smem_a != 0);
}

// The loader-only probe on a segment record (d_segs, sessd_bev_skip_plan): the segment windows' patch layout of a stride-1 conv.
extern "C" int sessd_bev_conv_p2_seg_loads(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad,
                                           const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info,
                                           float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info,
                                           const sessd_conv_desc *desc, const int *d_segs, long long *d_prof, void *stream) {
    if (!d_segs) return SESSD_EINVAL;
    return p2_conv<kP2Planes, kP2ProbeLoads>(d_in_planes, d_in_info, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain,
                                             shift_max, d_out_f32, d_out_planes, d_out_info, desc, stream, nullptr, d_prof, false, d_segs);
}

// The plan p2_conv / p2_deconv would launch with (p2_plan), word order in sessd_b200_lab.h.  No device call.
extern "C" int sessd_bev_p2_plan(const sessd_conv_desc *desc, int deconv, int cout_pad, int split, int smem_a, int *plan) {
    if (!desc || !plan) return SESSD_EINVAL;
    const sessd_conv_desc &d = *desc;
    P2Params p;
    P2Taps cls[4];
    if (deconv) p2_deconv_params(d.batch, d.in_h, d.in_w, d.cin, d.cout, d.relu, p, cls);
    else if (p2_conv_params(d, p, cls[0])) return SESSD_EINVAL;
    const int mode = split ? kP2SplitF16 : kP2Planes;
    const bool reg_a = mode == kP2Planes && (deconv || (d.in_stride == 1 && !smem_a));
    int smem = 0;
    if (p2_plan(p, cls, deconv ? 4 : 1, deconv ? d.in_h : d.grid_h, deconv ? d.in_w : d.grid_w, cout_pad, mode, reg_a, &smem))
        return SESSD_EINVAL;
    const int rec[11] = {p.u_is_x, p.n_tile, p.nblocks, p.tiles, p.total, p.ncopies, p.rows_v, p.pitch_u, p.npatch, p.bstages, smem};
    for (int i = 0; i < 11; ++i) plan[i] = rec[i];
    for (int c = 0; c < 4; ++c) { plan[11 + c] = p.cls_ntaps[c]; plan[15 + c] = p.cls_order[c]; }      // 0 past the classes
    return 0;
}
