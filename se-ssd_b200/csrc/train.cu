// train.cu -- optimiser-side kernels of the SE-SSD training step over FLAT parameter arenas (one launch per model, not per tensor).
//
// The reference walks the parameter list in Python for the teacher's exponential moving average
// (det3d/torchie/trainer/trainer_sessd.py:315-318: ema = alpha * ema + (1 - alpha) * param, ~300 tiny launches), flattens / unflattens
// the gradients around the all-reduce (det3d/core/utils/dist_utils.py:8-29) and steps a fastai-style Adam with decoupled weight decay
// (det3d/solver/fastai_optim.py).  Here every parameter of a model is a view into one contiguous fp32 buffer (sessd_b200/train.py:
// ParamArena), likewise its gradient, so each of these is ONE grid-stride kernel at the HBM roofline (8-28 bytes per element), and the
// all-reduce runs in place on the gradient arena (no flatten / unflatten copies).
#include "common.cuh"

namespace sessd {

// y = a * y + b * x    (EMA: a = alpha, b = 1 - alpha; gradient averaging: a = 1 / world, b = 0 with x = y)
__global__ void __launch_bounds__(256) axpby_kernel(float4 *__restrict__ y, const float4 *__restrict__ x, float a, float b, long long n4,
                                                    float *__restrict__ y_tail, const float *__restrict__ x_tail, int ntail) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n4; i += (long long)gridDim.x * blockDim.x) {
        float4 v = y[i];
        const float4 u = x ? __ldg(x + i) : make_float4(0.f, 0.f, 0.f, 0.f);
        v.x = fmaf(a, v.x, b * u.x); v.y = fmaf(a, v.y, b * u.y); v.z = fmaf(a, v.z, b * u.z); v.w = fmaf(a, v.w, b * u.w);
        y[i] = v;
    }
    if (blockIdx.x == 0 && (int)threadIdx.x < ntail) y_tail[threadIdx.x] = fmaf(a, y_tail[threadIdx.x], b * (x_tail ? x_tail[threadIdx.x] : 0.f));
}

// Adam with decoupled weight decay (torch.optim.AdamW semantics == fastai true_wd): p -= lr * wd * p; m, v updated; p -= step_size * m / (sqrt(v) / sqrt(bc2) + eps).
// Optional, both in the same pass: clip_coef (device scalar written by grad_norm_kernel) scales the gradient, g' = g * coef, and g' is stored back
// (torch's in-place clip_grad_norm_ leaves the same arena); ema (teacher arena) takes ema = ema_a * ema + ema_b * p_new, axpby_kernel's arithmetic.
__global__ void __launch_bounds__(256) adamw_kernel(float *__restrict__ p, float *__restrict__ g, float *__restrict__ m, float *__restrict__ v,
                                                    long long n, float lr, float beta1, float beta2, float eps, float wd, float bc1, float bc2_sqrt,
                                                    const float *__restrict__ clip_coef, float *__restrict__ ema, float ema_a, float ema_b) {
    const float step_size = lr / bc1;
    const float coef = clip_coef ? __ldg(clip_coef) : 1.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) {
        float gi = g[i];
        if (clip_coef) {
            gi *= coef;
            g[i] = gi;
        }
        float pi = p[i];
        pi *= 1.f - lr * wd;
        const float mi = m[i] + (1.f - beta1) * (gi - m[i]);          // torch: exp_avg.lerp_(grad, 1 - beta1)
        const float vi = beta2 * v[i] + (1.f - beta2) * gi * gi;
        m[i] = mi;
        v[i] = vi;
        const float denom = sqrtf(vi) / bc2_sqrt + eps;
        pi = pi - step_size * (mi / denom);
        p[i] = pi;
        if (ema) ema[i] = fmaf(ema_a, ema[i], ema_b * pi);
    }
}

// Squared L2 norm of a flat fp32 arena and the clip coefficient of torch.nn.utils.clip_grad_norm_, without a host round trip.  Bitwise
// deterministic, whatever the SM count: CTA c always owns elements [c * kNormChunk, (c + 1) * kNormChunk), each thread sums its squares in
// fp64 in a fixed order, each CTA reduces its threads in a fixed tree and writes one fp64 partial; the last CTA to finish (device counter,
// reset by that CTA) sums the partials in a fixed order and writes out[0] = total_norm = (float)sqrt(sum), out[1] = clip_coef.
constexpr int kNormThreads = 256;
constexpr int kNormChunk = kNormThreads * 4 * 16;                    // 16 float4 per thread

__device__ __forceinline__ double block_sum_fixed(double x, double *sh) {
    for (int o = 16; o > 0; o >>= 1) x += __shfl_down_sync(0xffffffffu, x, o);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = x;
    __syncthreads();
    double s = 0.0;
    if (threadIdx.x == 0)
        for (int w = 0; w < kNormThreads / 32; ++w) s += sh[w];
    return s;                                                         // valid in thread 0
}

__global__ void __launch_bounds__(kNormThreads) grad_norm_kernel(const float *__restrict__ x, long long n, float max_norm, float *__restrict__ out,
                                                                 unsigned int *__restrict__ counter, double *__restrict__ partials) {
    __shared__ double sh[kNormThreads / 32];
    __shared__ bool last;
    const long long base = (long long)blockIdx.x * kNormChunk;
    const long long len = n - base < kNormChunk ? n - base : kNormChunk;
    const int len4 = (int)(len > 0 ? len / 4 : 0);
    const float4 *x4 = reinterpret_cast<const float4 *>(x + base);
    double acc = 0.0;
    for (int j = threadIdx.x; j < len4; j += kNormThreads) {
        const float4 u = __ldg(x4 + j);
        acc = fma((double)u.x, (double)u.x, acc);
        acc = fma((double)u.y, (double)u.y, acc);
        acc = fma((double)u.z, (double)u.z, acc);
        acc = fma((double)u.w, (double)u.w, acc);
    }
    if ((int)threadIdx.x < (int)(len - (long long)len4 * 4)) {
        const double t = (double)x[base + (long long)len4 * 4 + threadIdx.x];
        acc = fma(t, t, acc);
    }
    const double s = block_sum_fixed(acc, sh);
    if (threadIdx.x == 0) {
        partials[blockIdx.x] = s;
        __threadfence();
        last = atomicAdd(counter, 1u) == gridDim.x - 1;
    }
    __syncthreads();
    if (!last) return;
    __threadfence();
    double tot = 0.0;
    for (unsigned int c = threadIdx.x; c < gridDim.x; c += kNormThreads) tot += __ldcg(partials + c);
    __syncthreads();                                                  // sh is reused
    tot = block_sum_fixed(tot, sh);
    if (threadIdx.x == 0) {
        const float total = (float)sqrt(tot);
        // torch: clip_coef = max_norm / (total_norm + 1e-6), which evaluates as (total_norm + 1e-6).reciprocal() * max_norm; clamp(max=1)
        const float c = (1.f / (total + 1e-6f)) * max_norm;
        out[0] = total;
        out[1] = c > 1.f ? 1.f : c;
        *counter = 0u;
    }
}

}  // namespace sessd

using namespace sessd;

// d_y[i] = a * d_y[i] + b * d_x[i]  (d_x nullable => b term dropped).  Teacher EMA of trainer_sessd.py:315-318 with a = alpha, b = 1 - alpha;
// gradient averaging after a SUM all-reduce with d_x = NULL, a = 1 / world_size.  Pointers 16-byte aligned.
extern "C" int sessd_axpby(float *d_y, const float *d_x, float a, float b, long long n, void *stream) {
    if (!d_y || n < 0 || ((uintptr_t)d_y & 15) || ((uintptr_t)d_x & 15)) return SESSD_EINVAL;
    if (n == 0) return 0;
    const long long n4 = n / 4;
    SESSD_LAUNCH(axpby_kernel, persistent_grid(n4 > 0 ? n4 : 1, 256), 256, 0, stream, reinterpret_cast<float4 *>(d_y), reinterpret_cast<const float4 *>(d_x),
                 a, b, n4, d_y + n4 * 4, d_x ? d_x + n4 * 4 : nullptr, (int)(n - n4 * 4));
    return last_error();
}

static long long norm_chunks(long long n) { return n > 0 ? (n + kNormChunk - 1) / kNormChunk : 1; }

extern "C" size_t sessd_grad_sqnorm_workspace_bytes(long long n) { return 16 + sizeof(double) * (size_t)norm_chunks(n < 0 ? 0 : n); }

// d_out[0] = ||d_x||_2 (fp32), d_out[1] = min(1, max_norm / (d_out[0] + 1e-6)).  d_x 16-byte aligned.  d_workspace holds the completion
// counter and the per-chunk partials: sessd_grad_sqnorm_workspace_bytes(n) bytes, zero-filled once before its first use (the kernel leaves
// the counter at zero); one workspace serves one stream at a time.
extern "C" int sessd_grad_sqnorm(const float *d_x, long long n, float max_norm, float *d_out, void *d_workspace, void *stream) {
    if (!d_x || !d_out || !d_workspace || n < 0 || ((uintptr_t)d_x & 15) || ((uintptr_t)d_workspace & 15)) return SESSD_EINVAL;
    const long long chunks = norm_chunks(n);
    if (chunks > 0x7fffffffLL) return SESSD_EINVAL;
    char *ws = static_cast<char *>(d_workspace);
    SESSD_LAUNCH(grad_norm_kernel, (int)chunks, kNormThreads, 0, stream, d_x, n, max_norm, d_out, reinterpret_cast<unsigned int *>(ws),
                 reinterpret_cast<double *>(ws + 16));
    return last_error();
}

static int adamw_launch(float *d_param, float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, long long n, float lr, float beta1, float beta2,
                        float eps, float weight_decay, int step, const float *d_clip_coef, float *d_ema, double ema_alpha, void *stream) {
    if (n == 0) return 0;
    const double bc1 = 1.0 - pow((double)beta1, (double)step), bc2 = 1.0 - pow((double)beta2, (double)step);
    SESSD_LAUNCH(adamw_kernel, persistent_grid(n, 256), 256, 0, stream, d_param, d_grad, d_exp_avg, d_exp_avg_sq, n, lr, beta1, beta2, eps,
                 weight_decay, (float)bc1, (float)sqrt(bc2), d_clip_coef, d_ema, (float)ema_alpha, (float)(1.0 - ema_alpha));
    return last_error();
}

// One AdamW step over flat fp32 arenas (parameters, gradients, first / second moments); step = 1, 2, ... (bias corrections computed on the host).
extern "C" int sessd_adamw_step(float *d_param, const float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, long long n, float lr, float beta1,
                                float beta2, float eps, float weight_decay, int step, void *stream) {
    if (!d_param || !d_grad || !d_exp_avg || !d_exp_avg_sq || n < 0 || step < 1) return SESSD_EINVAL;
    return adamw_launch(d_param, const_cast<float *>(d_grad), d_exp_avg, d_exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, nullptr,
                        nullptr, 0.0, stream);                        // without a clip coefficient the kernel never writes d_grad
}

// The same step with the gradient scaled by *d_clip_coef (and written back) and the teacher arena d_ema updated from the new parameters,
// ema = (float)ema_alpha * ema + (float)(1 - ema_alpha) * p; either may be NULL.
extern "C" int sessd_adamw_clip_ema_step(float *d_param, float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, long long n, float lr, float beta1,
                                         float beta2, float eps, float weight_decay, int step, const float *d_clip_coef, float *d_ema,
                                         double ema_alpha, void *stream) {
    if (!d_param || !d_grad || !d_exp_avg || !d_exp_avg_sq || n < 0 || step < 1) return SESSD_EINVAL;
    return adamw_launch(d_param, d_grad, d_exp_avg, d_exp_avg_sq, n, lr, beta1, beta2, eps, weight_decay, step, d_clip_coef, d_ema, ema_alpha,
                        stream);
}
