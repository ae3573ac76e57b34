// bevconv.cu -- dense BEV neck/head convolutions as NHWC implicit GEMM with fused BatchNorm+ReLU(+residual) epilogue,
// and the SSFA attention-fusion tail.
//
// Replaces the cuDNN conv2d / conv_transpose2d + BatchNorm2d + ReLU triplets of det3d/models/necks/rpn_v1.py:135-210
// (13 convs + 15 BN + 13 ReLU launched separately, NCHW) and the four 1x1 head convs + permute copies of
// det3d/models/bbox_heads/mg_head_sessd.py:202-230.
//
// One "tap-list" kernel covers every layer shape of the neck:
//   out[b, oy*os+py, ox*os+px, :] = epi( sum_t  in[b, oy*is+dy_t, ox*is+dx_t, :] @ W[t] )
//   * conv3x3 s1/s2 : 9 taps, is = stride;   * conv1x1 : 1 tap;
//   * ConvTranspose2d(k3,s2,p1,op1) : four output-parity classes with 1/2/2/4 taps (no multiplications by the
//     zero-stuffed input that a naive "conv over the upsampled grid" would spend 75 % of its MACs on).
// GEMM view: M = B*grid_h*grid_w pixels, N = Cout, K = ntaps*Cin.  CTA tile 128x128, BK = 16, 256 threads with 8x8
// register micro-tiles, A rows gathered with zero-filling cp.async (3-stage pipeline), fp32 FMA accumulation.
// This SIMT version is the fp32 numerics baseline; the tensor-core versions read pre-split fp16 planes (bevconv_p2.cu).
// Algorithmic bytes per layer: 4 (M Cin [read once per CTA column] + M Cout) ; FLOPs 2 M N K.
#include <cuda_fp16.h>

#include "common.cuh"

namespace sessd {

__device__ __forceinline__ void cpa16(void *smem, const void *gmem, bool valid) {
    const unsigned int s = (unsigned int)__cvta_generic_to_shared(smem);
    const int sz = valid ? 16 : 0;
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}

constexpr int kBM = 128, kBN = 128, kBK = 16, kCvThreads = 256, kCvStages = 3;
constexpr int kAStr = kBK + 4;                       // floats per A row in smem
constexpr int kStageFloats = kBM * kAStr + kBK * kBN;
constexpr int kCvSmem = kCvStages * kStageFloats * 4 + kBM * 3 * 4;

__global__ void __launch_bounds__(kCvThreads, 2) bev_conv_kernel(const float *__restrict__ in, const float *__restrict__ wgt,
                                                                 const float *__restrict__ scale, const float *__restrict__ shift,
                                                                 const float *__restrict__ resid, float *__restrict__ out,
                                                                 sessd_conv_desc d) {
    extern __shared__ __align__(16) float smem[];
    int *s_pb = reinterpret_cast<int *>(smem + kCvStages * kStageFloats);   // [kBM] batch, oy, ox per tile row
    int *s_py = s_pb + kBM;
    int *s_px = s_py + kBM;

    const int tid = threadIdx.x;
    const int tn = tid & 15, tm = tid >> 4;
    const long long M = (long long)d.batch * d.grid_h * d.grid_w;
    const long long m0 = (long long)blockIdx.x * kBM;
    const int n0 = blockIdx.y * kBN;

    if (tid < kBM) {
        long long p = m0 + tid;
        int b = -1, oy = 0, ox = 0;
        if (p < M) {
            ox = (int)(p % d.grid_w); p /= d.grid_w;
            oy = (int)(p % d.grid_h); b = (int)(p / d.grid_h);
        }
        s_pb[tid] = b; s_py[tid] = oy; s_px[tid] = ox;
    }
    __syncthreads();

    const int kchunks = d.cin / kBK;
    const int steps = d.ntaps * kchunks;

    auto load_stage = [&](int st, int step) {
        float *sA = smem + st * kStageFloats;
        float *sB = sA + kBM * kAStr;
        const int t = step / kchunks, c0 = (step - t * kchunks) * kBK;
        const int dy = d.tap_dy[t], dx = d.tap_dx[t];
        // A: 128 rows x 4 chunks of 16 B
        for (int e = tid; e < kBM * (kBK / 4); e += kCvThreads) {
            const int r = e >> 2, c4 = e & 3;
            const int b = s_pb[r];
            const int iy = s_py[r] * d.in_stride + dy, ix = s_px[r] * d.in_stride + dx;
            const bool ok = (b >= 0) && iy >= 0 && iy < d.in_h && ix >= 0 && ix < d.in_w;
            const float *g = in + (ok ? ((((size_t)b * d.in_h + iy) * d.in_w + ix) * d.cin + c0 + c4 * 4) : 0);
            cpa16(sA + r * kAStr + c4 * 4, g, ok);
        }
        // B: 16 rows x 32 chunks
        const float *gw = wgt + ((size_t)t * d.cin + c0) * d.cout;
        for (int e = tid; e < kBK * (kBN / 4); e += kCvThreads) {
            const int r = e >> 5, c4 = e & 31;
            const int n = n0 + c4 * 4;
            const bool ok = n < d.cout;
            cpa16(sB + r * kBN + c4 * 4, gw + (size_t)r * d.cout + (ok ? n : 0), ok);
        }
        asm volatile("cp.async.commit_group;\n" ::);
    };

    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

    for (int s = 0; s < kCvStages - 1; ++s) {
        if (s < steps) load_stage(s, s);
        else asm volatile("cp.async.commit_group;\n" ::);
    }
    for (int step = 0; step < steps; ++step) {
        asm volatile("cp.async.wait_group %0;\n" ::"n"(kCvStages - 2));
        __syncthreads();
        // refill the stage consumed in the previous iteration
        const int nxt = step + kCvStages - 1;
        if (nxt < steps) load_stage(nxt % kCvStages, nxt);
        else asm volatile("cp.async.commit_group;\n" ::);
        const float *sA = smem + (step % kCvStages) * kStageFloats;
        const float *sB = sA + kBM * kAStr;
#pragma unroll
        for (int c = 0; c < kBK; c += 4) {
            float4 a[8];
#pragma unroll
            for (int i = 0; i < 8; ++i) a[i] = *reinterpret_cast<const float4 *>(sA + (i * 16 + tm) * kAStr + c);
#pragma unroll
            for (int kk = 0; kk < 4; ++kk) {
                const float4 b0 = *reinterpret_cast<const float4 *>(sB + (c + kk) * kBN + tn * 4);
                const float4 b1 = *reinterpret_cast<const float4 *>(sB + (c + kk) * kBN + 64 + tn * 4);
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                    const float av = kk == 0 ? a[i].x : kk == 1 ? a[i].y : kk == 2 ? a[i].z : a[i].w;
                    acc[i][0] = fmaf(av, b0.x, acc[i][0]); acc[i][1] = fmaf(av, b0.y, acc[i][1]);
                    acc[i][2] = fmaf(av, b0.z, acc[i][2]); acc[i][3] = fmaf(av, b0.w, acc[i][3]);
                    acc[i][4] = fmaf(av, b1.x, acc[i][4]); acc[i][5] = fmaf(av, b1.y, acc[i][5]);
                    acc[i][6] = fmaf(av, b1.z, acc[i][6]); acc[i][7] = fmaf(av, b1.w, acc[i][7]);
                }
            }
        }
    }
    asm volatile("cp.async.wait_group 0;\n" ::);

    // epilogue: BN(eval) scale/shift, ReLU, residual (added after the ReLU), float4 stores
#pragma unroll
    for (int h = 0; h < 2; ++h) {
        const int n = n0 + h * 64 + tn * 4;
        if (n >= d.cout) continue;
        float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
        if (scale) sc = *reinterpret_cast<const float4 *>(scale + n);
        if (shift) sh = *reinterpret_cast<const float4 *>(shift + n);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
            const int r = i * 16 + tm;
            const int b = s_pb[r];
            if (b < 0) continue;
            const int oy = s_py[r] * d.out_stride + d.out_off_y, ox = s_px[r] * d.out_stride + d.out_off_x;
            const size_t o = (((size_t)b * d.out_h + oy) * d.out_w + ox) * d.cout + n;
            float4 v;
            v.x = fmaf(acc[i][h * 4 + 0], sc.x, sh.x); v.y = fmaf(acc[i][h * 4 + 1], sc.y, sh.y);
            v.z = fmaf(acc[i][h * 4 + 2], sc.z, sh.z); v.w = fmaf(acc[i][h * 4 + 3], sc.w, sh.w);
            if (d.relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
            if (resid) {
                const float4 rr = *reinterpret_cast<const float4 *>(resid + o);
                v.x += rr.x; v.y += rr.y; v.z += rr.z; v.w += rr.w;
            }
            *reinterpret_cast<float4 *>(out + o) = v;
        }
    }
}

// SSFA tail (rpn_v1.py:229-233).  One warp per pixel; 128 channels = one float4 per lane.  Optionally also writes the result as
// fp16 (hi, lo) planes for the head GEMM (sessd_bev_conv_p2): the output is a convex combination of x0 and x1, so max(amax0, amax1)
// bounds it exactly.
__global__ void __launch_bounds__(256) ssfa_fuse_kernel(const float *__restrict__ x0, const float *__restrict__ x1,
                                                        const float *__restrict__ w0, const float *__restrict__ w1, float s0, float t0,
                                                        float s1, float t1, int num_pixels, int C, float *__restrict__ out,
                                                        const float *__restrict__ info0, const float *__restrict__ info1,
                                                        float *__restrict__ out_info, __half *__restrict__ planes, long long plane_stride) {
    const int lane = threadIdx.x & 31;
    const int warps_per_block = blockDim.x >> 5;
    float sp = 1.f;
    if (planes) {
        const float am = fmaxf(__ldg(info0), __ldg(info1));
        sp = pow2_scale_for_bound(am);
        if (blockIdx.x == 0 && threadIdx.x == 0) { out_info[0] = am; out_info[1] = sp; }
    }
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
            if (planes) {
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


extern "C" int sessd_bev_conv(const float *d_in, const float *d_weight, const float *d_scale, const float *d_shift,
                              const float *d_residual, float *d_out, const sessd_conv_desc *desc, void *stream) {
    if (!d_in || !d_weight || !d_out || !desc) return SESSD_EINVAL;
    const sessd_conv_desc &d = *desc;
    if (d.batch < 1 || d.cin < kBK || d.cin % kBK || d.cout < 4 || d.cout % 4 || d.ntaps < 1 || d.ntaps > 16 || d.in_stride < 1 ||
        d.out_stride < 1 || d.grid_h < 1 || d.grid_w < 1)
        return SESSD_EINVAL;
    if ((d.grid_h - 1) * d.out_stride + d.out_off_y >= d.out_h || (d.grid_w - 1) * d.out_stride + d.out_off_x >= d.out_w) return SESSD_EINVAL;
    static bool attr_done = false;
    if (!attr_done) {
        SESSD_CUDA_TRY(cudaFuncSetAttribute(bev_conv_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kCvSmem));
        attr_done = true;
    }
    const long long M = (long long)d.batch * d.grid_h * d.grid_w;
    dim3 grid(div_up(M, kBM), div_up(d.cout, kBN));
    SESSD_LAUNCH(bev_conv_kernel, grid, kCvThreads, kCvSmem, stream, d_in, d_weight, d_scale, d_shift, d_residual, d_out, d);
    return last_error();
}

extern "C" int sessd_ssfa_fuse(const float *d_x0, const float *d_x1, const float *d_w0, const float *d_w1, float s0, float t0, float s1,
                               float t1, int num_pixels, int channels, float *d_out, void *stream) {
    if (!d_x0 || !d_x1 || !d_w0 || !d_w1 || !d_out || num_pixels < 1 || channels < 4 || channels % 4) return SESSD_EINVAL;
    SESSD_LAUNCH(ssfa_fuse_kernel, persistent_grid((long long)num_pixels * 32, 256), 256, 0, stream, d_x0, d_x1, d_w0, d_w1, s0, t0, s1, t1,
                 num_pixels, channels, d_out, nullptr, nullptr, nullptr, nullptr, 0ll);
    return last_error();
}

// same, additionally (or only: d_out nullable) writing fp16 (hi, lo) planes [2][num_pixels][channels] + d_out_info = {bound, scale};
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
