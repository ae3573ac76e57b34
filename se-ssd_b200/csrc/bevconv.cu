// bevconv.cu -- the SSFA attention-fusion tail (det3d/models/necks/rpn_v1.py:229-233) and the abs-max that scales the fp16 planes
// of tensors produced by kernels without an abs-max epilogue.  The neck's convs are in bevconv_p2.cu.
#include <cuda_fp16.h>

#include "common.cuh"

namespace sessd {

// SSFA tail (rpn_v1.py:229-233).  One warp per pixel; 128 channels = one float4 per lane.  Writes the result as fp16 (hi, lo) planes
// for the head GEMM (sessd_bev_conv_p2), and as fp32 when out is set: the output is a convex combination of x0 and x1, so
// max(amax0, amax1) bounds it exactly.
__global__ void __launch_bounds__(256) ssfa_fuse_kernel(const float *__restrict__ x0, const float *__restrict__ x1,
                                                        const float *__restrict__ w0, const float *__restrict__ w1, float s0, float t0,
                                                        float s1, float t1, int num_pixels, int C, float *__restrict__ out,
                                                        const float *__restrict__ info0, const float *__restrict__ info1,
                                                        float *__restrict__ out_info, __half *__restrict__ planes, long long plane_stride) {
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    const float am = fmaxf(__ldg(info0), __ldg(info1));
    const float sp = pow2_scale_for_bound(am);
    if (blockIdx.x == 0 && threadIdx.x == 0) { out_info[0] = am; out_info[1] = sp; }
    for (int p = blockIdx.x * warps_per_block + (threadIdx.x >> 5); p < num_pixels; p += gridDim.x * warps_per_block) {
        float d0 = 0.f, d1 = 0.f;
        for (int c = lane * 4; c < C; c += 128) {
            const float4 a = *reinterpret_cast<const float4 *>(x0 + (size_t)p * C + c);
            const float4 b = *reinterpret_cast<const float4 *>(x1 + (size_t)p * C + c);
            const float4 u = *reinterpret_cast<const float4 *>(w0 + c);
            const float4 v = *reinterpret_cast<const float4 *>(w1 + c);
            d0 += a.x * u.x + a.y * u.y + a.z * u.z + a.w * u.w;
            d1 += b.x * v.x + b.y * v.y + b.z * v.z + b.w * v.w;
        }
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) { d0 += __shfl_xor_sync(0xffffffffu, d0, o); d1 += __shfl_xor_sync(0xffffffffu, d1, o); }
        const float l0 = fmaf(d0, s0, t0), l1 = fmaf(d1, s1, t1);      // BN (no ReLU) on the 1-channel maps
        const float mx = fmaxf(l0, l1);
        const float e0 = expf(l0 - mx), e1 = expf(l1 - mx);            // softmax over the pair
        const float inv = 1.0f / (e0 + e1);
        const float a0 = e0 * inv, a1 = e1 * inv;
        for (int c = lane * 4; c < C; c += 128) {
            const float4 a = *reinterpret_cast<const float4 *>(x0 + (size_t)p * C + c);
            const float4 b = *reinterpret_cast<const float4 *>(x1 + (size_t)p * C + c);
            float4 r;
            r.x = a.x * a0 + b.x * a1; r.y = a.y * a0 + b.y * a1; r.z = a.z * a0 + b.z * a1; r.w = a.w * a0 + b.w * a1;
            if (out) *reinterpret_cast<float4 *>(out + (size_t)p * C + c) = r;
            const float q[4] = {r.x * sp, r.y * sp, r.z * sp, r.w * sp};
            __align__(8) __half hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                hi[e] = __float2half_rn(q[e]);
                lo[e] = __float2half_rn(q[e] - __half2float(hi[e]));
            }
            *reinterpret_cast<uint2 *>(planes + (size_t)p * C + c) = *reinterpret_cast<const uint2 *>(hi);
            *reinterpret_cast<uint2 *>(planes + plane_stride + (size_t)p * C + c) = *reinterpret_cast<const uint2 *>(lo);
        }
    }
}

// running abs-max of a tensor (feeds the activation scaling of the fp16 planes of tensors produced by other kernels)
__global__ void absmax_kernel(const float4 *__restrict__ x, long long n4, const float *__restrict__ tail, int ntail, float *__restrict__ amax) {
    float m = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(x + i);
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < ntail) m = fmaxf(m, fabsf(tail[threadIdx.x]));
    const unsigned w = __reduce_max_sync(0xFFFFFFFFu, __float_as_uint(m));
    __shared__ unsigned s_m[32];
    if ((threadIdx.x & 31) == 0) s_m[threadIdx.x >> 5] = w;
    __syncthreads();
    if (threadIdx.x < 32) {
        const unsigned v = threadIdx.x < (blockDim.x >> 5) ? s_m[threadIdx.x] : 0u;
        const unsigned r = __reduce_max_sync(0xFFFFFFFFu, v);
        if (threadIdx.x == 0 && r != 0u) atomicMax(reinterpret_cast<unsigned *>(amax), r);
    }
}

}  // namespace sessd

using namespace sessd;

// *d_amax = max(*d_amax, max |x[i]|); x 16-byte aligned
extern "C" int sessd_absmax(const float *d_x, long long n, float *d_amax, void *stream) {
    if (!d_x || !d_amax || n < 0 || ((uintptr_t)d_x & 15)) return SESSD_EINVAL;
    if (n == 0) return 0;
    const long long n4 = n / 4;
    const int blocks = (int)max(1LL, min((long long)kNumSMs * 8, (n4 + 255) / 256));
    absmax_kernel<<<blocks, 256, 0, (cudaStream_t)stream>>>(reinterpret_cast<const float4 *>(d_x), n4, d_x + n4 * 4, (int)(n - n4 * 4), d_amax);
    ++g_launches;
    return last_error();
}

// fused map as fp16 (hi, lo) planes [2][num_pixels][channels] + d_out_info = {bound, scale}, and as fp32 d_out (nullable);
// d_info0 / d_info1: [2] each, element 0 = abs-max of x0 / x1
extern "C" int sessd_ssfa_fuse_planes(const float *d_x0, const float *d_x1, const float *d_w0, const float *d_w1, float s0, float t0, float s1,
                                      float t1, int num_pixels, int channels, float *d_out, const float *d_info0, const float *d_info1,
                                      float *d_out_info, void *d_planes, void *stream) {
    if (!d_x0 || !d_x1 || !d_w0 || !d_w1 || !d_planes || !d_info0 || !d_info1 || !d_out_info || num_pixels < 1 || channels < 4 || channels % 4)
        return SESSD_EINVAL;
    SESSD_LAUNCH(ssfa_fuse_kernel, persistent_grid((long long)num_pixels * 32, 256), 256, 0, stream, d_x0, d_x1, d_w0, d_w1, s0, t0, s1, t1,
                 num_pixels, channels, d_out, d_info0, d_info1, d_out_info, (__half *)d_planes, (long long)num_pixels * channels);
    return last_error();
}
