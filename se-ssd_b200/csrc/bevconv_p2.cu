// bevconv_p2.cu -- C ABI of the BEV conv / deconv from pre-split fp16 planes (kernel and launcher: bevconv_p2.cuh).
#include "bevconv_p2.cuh"

namespace sessd {

// fp32 rows [rows][C] -> fp16 (hi, lo) planes [2][rows][C] with the scale taken from info[0] (exact abs-max of the tensor); writes info[1]
__global__ void __launch_bounds__(256) bev_split_planes_kernel(const float4 *__restrict__ x, long long n4, float *__restrict__ info,
                                                               __half *__restrict__ planes, long long plane_stride) {
    const float s = pow2_scale_for_bound(__ldg(info));
    if (blockIdx.x == 0 && threadIdx.x == 0) info[1] = s;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(x + i);
        const float a[4] = {v.x * s, v.y * s, v.z * s, v.w * s};
        __align__(8) __half hi[4], lo[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) {
            hi[t] = __float2half_rn(a[t]);
            lo[t] = __float2half_rn(a[t] - __half2float(hi[t]));
        }
        *reinterpret_cast<uint2 *>(planes + 4 * i) = *reinterpret_cast<const uint2 *>(hi);
        *reinterpret_cast<uint2 *>(planes + plane_stride + 4 * i) = *reinterpret_cast<const uint2 *>(lo);
    }
}

}  // namespace sessd

using namespace sessd;

// Conv2d (stride 1 or 2, arbitrary tap list) + folded BN + ReLU (+ residual) from fp16 (hi, lo) planes.
//   d_in_planes  __half [2][batch][in_h][in_w][cin]; d_in_info [2] = {abs-max of the input, scale of its planes} (device);
//   d_weight_h2  __half [2 (hi|lo)][ntaps][cout_pad][cin] (ops.pack_weight_h2); d_scale = folded BN scale * 2^-e[n]; d_shift nullable;
//   d_residual   fp32 [batch][out_h][out_w][cout] added after the ReLU, with d_resid_info[0] = its abs-max;
//   gain, shift_max: |out| <= amax_in * gain + shift_max (+ amax_resid), see the header;
//   outputs: d_out_f32 (fp32 NHWC) and / or d_out_planes (__half [2][batch][out_h][out_w][cout], scale written to d_out_info[1]);
//   d_out_info[0] is atomically raised to max|out| (zero it once per frame).
//   d_items (nullable): a launch record of sessd_bev_skip_plan -- only the work items it lists run (same grid, same per-item work);
//   d_segs (nullable, stride 1 only, not with d_items): a launch's segment record of sessd_bev_skip_plan -- only its segments run.
extern "C" int sessd_bev_conv_p2(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                                 const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                                 float *d_out_f32, void *d_out_planes, float *d_out_info, const sessd_conv_desc *desc, const int *d_items,
                                 const int *d_segs, void *stream) {
    return p2_conv<kP2Planes>(d_in_planes, d_in_info, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain, shift_max,
                              d_out_f32, d_out_planes, d_out_info, desc, stream, d_items, nullptr, false, d_segs);
}

// ConvTranspose2d(k3, s2, p1, op1) + BN + ReLU (+ residual), four output-parity classes in one launch; weights [2][9][cout_pad][cin],
// tap = ky*3+kx of W[cin][cout][ky][kx]; output [batch, 2*in_h, 2*in_w, cout] (rpn_v1.py:183-195).
extern "C" int sessd_bev_deconv_p2(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                                   const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                                   float *d_out_f32, void *d_out_planes, float *d_out_info, int batch, int in_h, int in_w, int cin, int cout,
                                   int relu, const int *d_items, const int *d_segs, void *stream) {
    return p2_deconv<kP2Planes>(d_in_planes, d_in_info, d_weight_h2, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain, shift_max,
                                d_out_f32, d_out_planes, d_out_info, batch, in_h, in_w, cin, cout, relu, stream, d_items, nullptr, d_segs);
}

// fp32 [n] (n % 4 == 0, 16-byte aligned) -> planes [2][n] fp16 scaled by the power of two that maps d_info[0] (the tensor's abs-max,
// e.g. from sessd_absmax) into [2^14, 2^15); writes the scale to d_info[1]
extern "C" int sessd_bev_split_planes(const float *d_x, long long n, float *d_info, void *d_planes, void *stream) {
    if (!d_x || !d_info || !d_planes || n < 4 || (n & 3) || ((uintptr_t)d_x & 15)) return SESSD_EINVAL;
    SESSD_LAUNCH(bev_split_planes_kernel, persistent_grid(n / 4, 256), 256, 0, stream, reinterpret_cast<const float4 *>(d_x), n / 4, d_info,
                 (__half *)d_planes, n);
    return last_error();
}
