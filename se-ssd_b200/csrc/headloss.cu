// headloss.cu -- supervised SSD-head loss terms of SE-SSD, forward AND gradient in one pass on the device (SURVEY.md 8(f) row 1, first
// slice of the training step: targets come from sessd_assign_targets, predictions from the fused head GEMM).
//
// Replaces, for the terms that do not involve the teacher (det3d/models/bbox_heads/mg_head_sessd.py:706-760):
//   * prepare_loss_weights, NormByNumPositives            mg_head_sessd.py:525-572 (config.py:71)
//   * SigmoidFocalLoss(alpha=0.25, gamma=2)               det3d/models/losses/losses.py:345-420
//   * add_sin_difference + WeightedSmoothL1Loss(sigma=3)  mg_head_sessd.py:39-44, losses.py:147-204   (logged as loc_loss; not part of the
//                                                         reference's total, which uses the ODIoU loss instead -- weight w_loc lets the caller choose)
//   * get_direction_target + WeightedSoftmaxClassificationLoss   mg_head_sessd.py:62-76, losses.py:489-531
// The reference builds ~25 full-size [B, 70400, *] temporaries with ~40 elementwise launches and autograd replays them backwards; here
// one thread per anchor reads its 11 head outputs + label + 7 targets once (the head tensor is NHWC [B, H*W, stride] with the layout of
// postproc.cu: box 2x7 | cls 2 | dir 2x2 | iou 2), evaluates the three terms and their analytic derivatives and writes the gradient
// w.r.t. the head tensor in place of the autograd graph.  Per-frame sums are reduced in a fixed order (block partials -> one block per
// frame): bitwise run-to-run deterministic.  Algorithmic bytes: (44 + 4 + 28) read + 44 written per anchor = 8.4 MB / frame.
#include "common.cuh"

namespace sessd {

constexpr int kHlThreads = 256;
constexpr int kHlTerms = 6;      // cls, loc, dir, cls_pos, cls_neg, (unused)

__global__ void __launch_bounds__(kHlThreads) headloss_count_kernel(const int *__restrict__ labels, int num_anchors, int *__restrict__ counts) {
    __shared__ int s[40];
    const int b = blockIdx.y;
    int pos = 0, neg = 0;
    for (int a = blockIdx.x * kHlThreads + threadIdx.x; a < num_anchors; a += gridDim.x * kHlThreads) {
        const int l = labels[(size_t)b * num_anchors + a];
        pos += l > 0;
        neg += l == 0;
    }
    int tp, tn;
    block_excl_scan(pos, s, &tp);
    block_excl_scan(neg, s, &tn);
    if (threadIdx.x == 0) { atomicAdd(&counts[2 * b], tp); atomicAdd(&counts[2 * b + 1], tn); }
}

struct HlCfg {
    int batch, num_anchors, apl, head_stride;
    float alpha, sigma, dir_offset, pos_cls_weight, neg_cls_weight, w_cls, w_loc, w_dir;
};

__global__ void __launch_bounds__(kHlThreads) headloss_kernel(const float *__restrict__ head, const float *__restrict__ anchors,
                                                              const int *__restrict__ labels, const float *__restrict__ reg_targets, HlCfg c,
                                                              const int *__restrict__ counts, float *__restrict__ partial /*[B][gridDim.x][6]*/,
                                                              float *__restrict__ grad_head) {
    __shared__ float s_red[kHlTerms][kHlThreads / 32];
    const int b = blockIdx.y;
    const int A = c.num_anchors, apl = c.apl;
    const float pos_norm = fmaxf((float)counts[2 * b], 1.f);
    const float inv_b = 1.f / (float)c.batch;
    float acc[kHlTerms] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    for (int a = blockIdx.x * kHlThreads + threadIdx.x; a < A; a += gridDim.x * kHlThreads) {
        const int pix = a / apl, r = a - pix * apl;
        const size_t hb = ((size_t)b * (A / apl) + pix) * c.head_stride;
        const float *h = head + hb;
        const int label = labels[(size_t)b * A + a];
        const bool pos = label > 0, neg = label == 0;
        // ---- classification: sigmoid focal loss (gamma = 2), weights = cls_weight / num_pos
        const float x = h[7 * apl + r];
        const float t = pos ? 1.f : 0.f;
        const float w = (pos ? c.pos_cls_weight : (neg ? c.neg_cls_weight : 0.f)) / pos_norm;
        const float p = 1.f / (1.f + expf(-x));
        const float ce = fmaxf(x, 0.f) - x * t + log1pf(expf(-fabsf(x)));
        const float pt = t * p + (1.f - t) * (1.f - p);
        const float om = 1.f - pt;
        const float aw = t * c.alpha + (1.f - t) * (1.f - c.alpha);
        const float cls = om * om * aw * ce * w;
        acc[0] += cls;
        if (pos) acc[3] += cls;
        if (neg) acc[4] += cls;
        // d/dx: mod' ce + mod ce',  mod = (1 - pt)^2,  dpt/dx = (2t - 1) p (1 - p),  ce' = p - t
        const float g_cls = w * aw * (-2.f * om * (2.f * t - 1.f) * p * (1.f - p) * ce + om * om * (p - t));
        float g_box[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, g_dir[2] = {0.f, 0.f};
        if (pos) {
            const float rw = 1.f / pos_norm;
            const float *tg = reg_targets + ((size_t)b * A + a) * 7;
            const float inv_s2 = 1.f / (c.sigma * c.sigma);
            float loc = 0.f;
#pragma unroll
            for (int j = 0; j < 7; ++j) {
                const float bp = h[7 * r + j];
                float d, chain = 1.f;
                if (j < 6) d = bp - tg[j];
                else {      // sin(a) cos(b) - cos(a) sin(b)  (evaluated like the reference, not as sin(a - b))
                    const float sa = sinf(bp), ca = cosf(bp), sb = sinf(tg[6]), cb = cosf(tg[6]);
                    d = sa * cb - ca * sb;
                    chain = ca * cb + sa * sb;
                }
                const float ad = fabsf(d);
                const bool small = ad <= inv_s2;
                const float sd = ad * c.sigma;
                loc += (small ? 0.5f * sd * sd : ad - 0.5f * inv_s2) * rw;
                g_box[j] = (small ? c.sigma * c.sigma * d : (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f))) * chain * rw;
            }
            acc[1] += loc;
            // ---- direction: 2-way softmax CE, target = (rot_gt - offset > 0), rot_gt = target residual + anchor yaw
            const float rot_gt = tg[6] + anchors[(size_t)a * 7 + 6];
            const int cls_t = (rot_gt - c.dir_offset) > 0.f ? 1 : 0;
            const float l0 = h[7 * apl + apl + 2 * r], l1 = h[7 * apl + apl + 2 * r + 1];
            const float m = fmaxf(l0, l1);
            const float e0 = expf(l0 - m), e1 = expf(l1 - m);
            const float lse = m + logf(e0 + e1);
            acc[2] += (lse - (cls_t ? l1 : l0)) * rw;
            const float s0 = e0 / (e0 + e1), s1 = e1 / (e0 + e1);
            g_dir[0] = (s0 - (cls_t ? 0.f : 1.f)) * rw;
            g_dir[1] = (s1 - (cls_t ? 1.f : 0.f)) * rw;
        }
        if (grad_head) {
            float *g = grad_head + hb;
#pragma unroll
            for (int j = 0; j < 7; ++j) g[7 * r + j] = g_box[j] * c.w_loc * inv_b;
            g[7 * apl + r] = g_cls * c.w_cls * inv_b;
            g[7 * apl + apl + 2 * r] = g_dir[0] * c.w_dir * inv_b;
            g[7 * apl + apl + 2 * r + 1] = g_dir[1] * c.w_dir * inv_b;
            g[7 * apl + apl + 2 * apl + r] = 0.f;                                       // iou head: no supervised term here
            if (r == 0) for (int j = 7 * apl + apl + 3 * apl; j < c.head_stride; ++j) g[j] = 0.f;
        }
    }
    // fixed-order block reduction: warp shuffle tree, then warp 0 sums the warp results in order
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int k = 0; k < kHlTerms; ++k) {
        float v = acc[k];
#pragma unroll
        for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(0xffffffffu, v, d);
        if (lane == 0) s_red[k][warp] = v;
    }
    __syncthreads();
    if (threadIdx.x < kHlTerms) {
        float v = 0.f;
        for (int i = 0; i < kHlThreads / 32; ++i) v += s_red[threadIdx.x][i];
        partial[((size_t)b * gridDim.x + blockIdx.x) * kHlTerms + threadIdx.x] = v;
    }
}

__global__ void __launch_bounds__(32) headloss_finish_kernel(const float *__restrict__ partial, int nblocks, const int *__restrict__ counts,
                                                             float *__restrict__ losses /*[B][8]*/) {
    const int b = blockIdx.x, k = threadIdx.x;
    if (k < kHlTerms) {
        float v = 0.f;
        for (int i = 0; i < nblocks; ++i) v += partial[((size_t)b * nblocks + i) * kHlTerms + k];
        losses[b * 8 + k] = v;
    }
    if (k == 6) losses[b * 8 + 6] = (float)counts[2 * b];
    if (k == 7) losses[b * 8 + 7] = (float)counts[2 * b + 1];
}

constexpr int kHlBlocks = 74;      // per frame; x batch >= 1 wave on the 132 SMs of an H100 from batch 2

}  // namespace sessd

using namespace sessd;

extern "C" size_t sessd_head_loss_workspace_bytes(int batch) {
    if (batch < 1) return 0;
    return sizeof(int) * 2 * (size_t)batch + 256 + sizeof(float) * (size_t)batch * kHlBlocks * kHlTerms;
}

extern "C" int sessd_head_loss(const float *d_head, const float *d_anchors, const int *d_labels, const float *d_reg_targets, int batch,
                               int num_anchors, int anchors_per_loc, int head_stride, float alpha, float sigma, float dir_offset,
                               float pos_cls_weight, float neg_cls_weight, float w_cls, float w_loc, float w_dir, float *d_losses,
                               float *d_grad_head, void *workspace, size_t workspace_bytes, void *stream) {
    if (!d_head || !d_anchors || !d_labels || !d_reg_targets || !d_losses || batch < 1 || num_anchors < 1 || anchors_per_loc != 2 ||
        head_stride < 22 || (num_anchors % anchors_per_loc) || !(sigma > 0.f))
        return SESSD_EINVAL;
    if (!workspace || workspace_bytes < sessd_head_loss_workspace_bytes(batch)) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    int *counts = (int *)workspace;
    float *partial = (float *)((char *)workspace + ((sizeof(int) * 2 * (size_t)batch + 255) & ~(size_t)255));
    SESSD_CUDA_TRY(cudaMemsetAsync(counts, 0, sizeof(int) * 2 * (size_t)batch, st));
    dim3 grid(kHlBlocks, batch);
    SESSD_LAUNCH(headloss_count_kernel, grid, kHlThreads, 0, st, d_labels, num_anchors, counts);
    HlCfg c{batch, num_anchors, anchors_per_loc, head_stride, alpha, sigma, dir_offset, pos_cls_weight, neg_cls_weight, w_cls, w_loc, w_dir};
    SESSD_LAUNCH(headloss_kernel, grid, kHlThreads, 0, st, d_head, d_anchors, d_labels, d_reg_targets, c, counts, partial, d_grad_head);
    SESSD_LAUNCH(headloss_finish_kernel, batch, 32, 0, st, partial, kHlBlocks, counts, d_losses);
    return last_error();
}
