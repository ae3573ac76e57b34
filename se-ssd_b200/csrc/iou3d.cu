// iou3d.cu -- the iou3d_cuda operator family on the GPU: rotated BEV overlap / IoU / 3-D IoU matrices and the three
// NMS variants with the greedy reduction done ON DEVICE.
//
// Replaces det3d/core/iou3d/src/iou3d.cpp:34-281 and iou3d_kernel.cu:270-365,425-530.  Differences by design:
//   * explicit stream, no cudaMalloc / blocking cudaMemcpy inside (the reference allocates the N x N/64 mask and
//     copies it to the host on the legacy stream, iou3d.cpp:131-142);
//   * only the upper block-triangle of the suppression mask is computed (the reference's host loop never reads
//     the rest, iou3d.cpp:152-156);
//   * greedy scan: 64 rows at a time -- one thread resolves the diagonal word chain, the CTA ORs the kept rows.
// Compiled with -fmad=false (see rotbox.cuh).
#include "common.cuh"
#include "rotbox.cuh"

namespace sessd {

// mode: 0 overlap, 1 iou bev, 2 iou 3d
template <int MODE>
__global__ void __launch_bounds__(256) box_matrix_kernel(const float *__restrict__ a, int n, const float *__restrict__ b, int m,
                                                         float *__restrict__ out) {
    constexpr int W = (MODE == 2) ? 7 : 5;
    const long long total = (long long)n * m;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(t / m), j = (int)(t - (long long)i * m);
        float ba[W], bb[W];
#pragma unroll
        for (int k = 0; k < W; ++k) { ba[k] = a[(size_t)i * W + k]; bb[k] = b[(size_t)j * W + k]; }
        float v;
        if (MODE == 0) v = rot_overlap5(ba, bb);
        else if (MODE == 1) v = rot_iou_bev(ba, bb);
        else v = rot_iou_3d(ba, bb);
        out[t] = v;
    }
}

__global__ void __launch_bounds__(256) box_aligned_overlap_kernel(const float *__restrict__ a, const float *__restrict__ b, int n,
                                                                  float *__restrict__ out) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        float ba[5], bb[5];
#pragma unroll
        for (int k = 0; k < 5; ++k) { ba[k] = a[(size_t)i * 5 + k]; bb[k] = b[(size_t)i * 5 + k]; }
        out[i] = rot_overlap5(ba, bb);
    }
}

// suppression mask, upper block triangle.  mode 0 rot-bev, 1 3d, 2 axis-aligned.  bit (i, j) iff iou > thresh.
template <int MODE>
__global__ void __launch_bounds__(64) nms_mask_kernel(const float *__restrict__ boxes, int n, float thresh,
                                                      unsigned long long *__restrict__ mask) {
    constexpr int W = (MODE == 1) ? 7 : 5;
    const int rb = blockIdx.y, cb = blockIdx.x;
    if (cb < rb) return;
    const int col_blocks = (n + 63) / 64;
    __shared__ float sb[64 * W];
    const int ncol = min(n - cb * 64, 64);
    if ((int)threadIdx.x < ncol)
        for (int k = 0; k < W; ++k) sb[threadIdx.x * W + k] = boxes[(size_t)(cb * 64 + threadIdx.x) * W + k];
    __syncthreads();
    const int i = rb * 64 + threadIdx.x;
    if (i >= n) return;
    float me[W];
#pragma unroll
    for (int k = 0; k < W; ++k) me[k] = boxes[(size_t)i * W + k];
    unsigned long long bits = 0;
    const int start = (rb == cb) ? threadIdx.x + 1 : 0;
    for (int j = start; j < ncol; ++j) {
        float v;
        if (MODE == 0) v = rot_iou_bev(me, sb + j * W);
        else if (MODE == 1) v = rot_iou_3d(me, sb + j * W);
        else v = axis_iou(me, sb + j * W);
        if (v > thresh) bits |= 1ull << j;
    }
    mask[(size_t)i * col_blocks + cb] = bits;
}

// greedy reduction over a (row-major, upper-triangular) mask; keeps at most max_keep rows.
// One CTA.  remv lives in dynamic shared memory (col_blocks words).
__global__ void __launch_bounds__(256) nms_reduce_kernel(const unsigned long long *__restrict__ mask, int n, int max_keep,
                                                         long long *__restrict__ keep, int *__restrict__ num_keep) {
    extern __shared__ unsigned long long remv[];
    __shared__ unsigned long long diag[64];
    __shared__ unsigned long long s_keepbits;
    __shared__ int s_nkeep;
    const int col_blocks = (n + 63) / 64;
    for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) remv[j] = 0;
    if (threadIdx.x == 0) s_nkeep = 0;
    __syncthreads();
    for (int b = 0; b < col_blocks; ++b) {
        const int rows = min(64, n - b * 64);
        if ((int)threadIdx.x < rows) diag[threadIdx.x] = mask[(size_t)(b * 64 + threadIdx.x) * col_blocks + b];
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long cur = remv[b], kb = 0;
            int nk = s_nkeep;
            for (int t = 0; t < rows && nk < max_keep; ++t) {
                if (!((cur >> t) & 1ull)) {
                    keep[nk++] = b * 64 + t;
                    kb |= 1ull << t;
                    cur |= diag[t];
                }
            }
            s_keepbits = kb;
            s_nkeep = nk;
        }
        __syncthreads();
        const unsigned long long kb = s_keepbits;
        if (s_nkeep >= max_keep) break;
        for (int j = b + 1 + threadIdx.x; j < col_blocks; j += blockDim.x) {
            unsigned long long acc = remv[j];
            unsigned long long bits = kb;
            while (bits) {
                const int t = __ffsll((long long)bits) - 1;
                bits &= bits - 1;
                acc |= mask[(size_t)(b * 64 + t) * col_blocks + j];
            }
            remv[j] = acc;
        }
        __syncthreads();
    }
    if (threadIdx.x == 0) *num_keep = s_nkeep;
}


// ---------------------------------------------------------------------------------------------------------------------------------
// IoU-prediction loss of the SE-SSD head (training; det3d/models/bbox_heads/mg_head_sessd.py:755-768): for every positive anchor decode
// the predicted and the target box (det3d/core/bbox/box_torch_ops.py:81-147), take their ALIGNED rotated 3-D IoU
// (det3d/core/iou3d/iou3d_utils.py:197-252: bev overlap x height overlap / clamp(vol_a + vol_b - overlap, 1e-7)) as a constant target
// 2 IoU - 1 and apply WeightedSmoothL1Loss(sigma = 3) to the head's iou output with weight 1 / num_pos.  One thread per anchor (only the
// positives work), fixed-order reduction.  Lives in this file because the polygon arithmetic must be compiled without FMA contraction.
constexpr int kIpThreads = 256;
constexpr int kIpBlocks = 74;

__global__ void __launch_bounds__(kIpThreads) iou_pred_loss_kernel(const float *__restrict__ head, const float *__restrict__ anchors,
                                                                   const int *__restrict__ labels, const float *__restrict__ reg_targets,
                                                                   int batch, int A, int apl, int stride, float sigma, float w_iou,
                                                                   const float *__restrict__ losses, float *__restrict__ partial,
                                                                   float *__restrict__ grad_head) {
    __shared__ float s_red[kIpThreads / 32];
    const int b = blockIdx.y;
    const float rw = 1.f / fmaxf(losses[b * 8 + 6], 1.f);            // 1 / num_pos (written by sessd_head_loss)
    const float inv_s2 = 1.f / (sigma * sigma);
    float acc = 0.f;
    for (int a = blockIdx.x * kIpThreads + threadIdx.x; a < A; a += gridDim.x * kIpThreads) {
        if (labels[(size_t)b * A + a] <= 0) continue;
        const int pix = a / apl, r = a - pix * apl;
        const size_t hb = ((size_t)b * (A / apl) + pix) * stride;
        const float *h = head + hb;
        const float *an = anchors + (size_t)a * 7;
        const float *tg = reg_targets + ((size_t)b * A + a) * 7;
        const float diag = sqrtf(an[4] * an[4] + an[3] * an[3]);
        float q[7], g[7];
        {
            const float *e = h + 7 * r;
            q[0] = e[0] * diag + an[0]; q[1] = e[1] * diag + an[1]; q[2] = e[2] * an[5] + an[2];
            q[3] = expf(e[3]) * an[3]; q[4] = expf(e[4]) * an[4]; q[5] = expf(e[5]) * an[5]; q[6] = e[6] + an[6];
            g[0] = tg[0] * diag + an[0]; g[1] = tg[1] * diag + an[1]; g[2] = tg[2] * an[5] + an[2];
            g[3] = expf(tg[3]) * an[3]; g[4] = expf(tg[4]) * an[4]; g[5] = expf(tg[5]) * an[5]; g[6] = tg[6] + an[6];
        }
        const float ov_bev = rot_overlap(q[0] - q[3] / 2.f, q[1] - q[4] / 2.f, q[0] + q[3] / 2.f, q[1] + q[4] / 2.f, q[6],
                                         g[0] - g[3] / 2.f, g[1] - g[4] / 2.f, g[0] + g[3] / 2.f, g[1] + g[4] / 2.f, g[6]);
        const float lo = fmaxf(q[2] - q[5] / 2.f, g[2] - g[5] / 2.f), hi = fminf(q[2] + q[5] / 2.f, g[2] + g[5] / 2.f);
        const float ov3 = ov_bev * fmaxf(hi - lo, 0.f);
        const float iou = ov3 / fmaxf(q[3] * q[4] * q[5] + g[3] * g[4] * g[5] - ov3, 1e-7f);
        const float target = 2.f * iou - 1.f;
        const int ch = 7 * apl + apl + 2 * apl + r;
        const float d = h[ch] - target;
        const float ad = fabsf(d);
        const bool small = ad <= inv_s2;
        const float sd = ad * sigma;
        acc += (small ? 0.5f * sd * sd : ad - 0.5f * inv_s2) * rw;
        if (grad_head) grad_head[hb + ch] = (small ? sigma * sigma * d : (d > 0.f ? 1.f : (d < 0.f ? -1.f : 0.f))) * rw * w_iou / (float)batch;
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, d);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float v = 0.f;
        for (int i = 0; i < kIpThreads / 32; ++i) v += s_red[i];
        partial[(size_t)b * gridDim.x + blockIdx.x] = v;
    }
}

__global__ void iou_pred_finish_kernel(const float *__restrict__ partial, int nblocks, float *__restrict__ losses) {
    const int b = blockIdx.x;
    if (threadIdx.x == 0) {
        float v = 0.f;
        for (int i = 0; i < nblocks; ++i) v += partial[(size_t)b * nblocks + i];
        losses[b * 8 + 5] = v;
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" int sessd_boxes_overlap_bev(const float *d_a, int n, const float *d_b, int m, float *d_out, void *stream) {
    if (n < 0 || m < 0) return SESSD_EINVAL;
    if (n == 0 || m == 0) return SESSD_OK;
    SESSD_LAUNCH((box_matrix_kernel<0>), persistent_grid((long long)n * m, 256), 256, 0, stream, d_a, n, d_b, m, d_out);
    return last_error();
}

extern "C" int sessd_boxes_iou_bev(const float *d_a, int n, const float *d_b, int m, float *d_out, void *stream) {
    if (n < 0 || m < 0) return SESSD_EINVAL;
    if (n == 0 || m == 0) return SESSD_OK;
    SESSD_LAUNCH((box_matrix_kernel<1>), persistent_grid((long long)n * m, 256), 256, 0, stream, d_a, n, d_b, m, d_out);
    return last_error();
}

extern "C" int sessd_boxes_iou3d(const float *d_a, int n, const float *d_b, int m, float *d_out, void *stream) {
    if (n < 0 || m < 0) return SESSD_EINVAL;
    if (n == 0 || m == 0) return SESSD_OK;
    SESSD_LAUNCH((box_matrix_kernel<2>), persistent_grid((long long)n * m, 256), 256, 0, stream, d_a, n, d_b, m, d_out);
    return last_error();
}

extern "C" int sessd_boxes_aligned_overlap_bev(const float *d_a, const float *d_b, int n, float *d_out, void *stream) {
    if (n < 0) return SESSD_EINVAL;
    if (n == 0) return SESSD_OK;
    SESSD_LAUNCH(box_aligned_overlap_kernel, persistent_grid(n, 256), 256, 0, stream, d_a, d_b, n, d_out);
    return last_error();
}

extern "C" size_t sessd_nms_workspace_bytes(int n) {
    if (n < 0) return 0;
    const size_t cb = (size_t)(n + 63) / 64;
    return sizeof(unsigned long long) * ((size_t)n * cb + 64);
}

extern "C" int sessd_nms_sorted(const float *d_boxes, int n, float thresh, int mode, long long *d_keep, int *d_num_keep,
                                void *workspace, size_t workspace_bytes, void *stream) {
    if (n < 0 || mode < 0 || mode > 2 || !d_num_keep) return SESSD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    if (n == 0) { SESSD_CUDA_TRY(cudaMemsetAsync(d_num_keep, 0, sizeof(int), st)); return SESSD_OK; }
    if (workspace_bytes < sessd_nms_workspace_bytes(n) || !workspace) return SESSD_EWORKSPACE;
    const int cb = (n + 63) / 64;
    if ((size_t)cb * 8 > 200 * 1024) return SESSD_ECAPACITY;   // remv[] must fit in shared memory
    unsigned long long *mask = (unsigned long long *)workspace;
    dim3 grid(cb, cb);
    if (mode == 0) SESSD_LAUNCH((nms_mask_kernel<0>), grid, 64, 0, st, d_boxes, n, thresh, mask);
    else if (mode == 1) SESSD_LAUNCH((nms_mask_kernel<1>), grid, 64, 0, st, d_boxes, n, thresh, mask);
    else SESSD_LAUNCH((nms_mask_kernel<2>), grid, 64, 0, st, d_boxes, n, thresh, mask);
    const size_t sm = sizeof(unsigned long long) * cb;
    if (sm > 48 * 1024)
        SESSD_CUDA_TRY(cudaFuncSetAttribute(nms_reduce_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    SESSD_LAUNCH(nms_reduce_kernel, 1, 256, sm, st, mask, n, n, d_keep, d_num_keep);
    return last_error();
}

extern "C" size_t sessd_iou_pred_loss_workspace_bytes(int batch) { return batch < 1 ? 0 : sizeof(float) * (size_t)batch * kIpBlocks; }

// Must run after sessd_head_loss on the same stream: reads num_pos from d_losses[b][6], writes the per-frame sum to d_losses[b][5] and the
// gradient of  w_iou * sum / batch  into the iou channels of d_grad_head (which sessd_head_loss zeroed).
extern "C" int sessd_iou_pred_loss(const float *d_head, const float *d_anchors, const int *d_labels, const float *d_reg_targets, int batch,
                                   int num_anchors, int anchors_per_loc, int head_stride, float sigma, float w_iou, float *d_losses,
                                   float *d_grad_head, void *workspace, size_t workspace_bytes, void *stream) {
    if (!d_head || !d_anchors || !d_labels || !d_reg_targets || !d_losses || batch < 1 || num_anchors < 1 || anchors_per_loc != 2 ||
        head_stride < 22 || !(sigma > 0.f))
        return SESSD_EINVAL;
    if (!workspace || workspace_bytes < sessd_iou_pred_loss_workspace_bytes(batch)) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(kIpBlocks, batch);
    SESSD_LAUNCH(iou_pred_loss_kernel, grid, kIpThreads, 0, st, d_head, d_anchors, d_labels, d_reg_targets, batch, num_anchors, anchors_per_loc,
                 head_stride, sigma, w_iou, d_losses, (float *)workspace, d_grad_head);
    SESSD_LAUNCH(iou_pred_finish_kernel, batch, 32, 0, st, (const float *)workspace, kIpBlocks, d_losses);
    return last_error();
}
