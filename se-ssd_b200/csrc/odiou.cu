// odiou.cu -- ODIoU box-regression loss of the SE-SSD head on the device, value and gradient (SURVEY.md 8(f) row 1; the reference's largest
// CPU stall: det3d/models/losses/odious.py runs per-box numpy loops with hand-written Jacobians inside the training step,
// det3d/models/bbox_heads/mg_head_sessd.py:770-778).  One thread per positive anchor decodes the predicted and the target box
// (det3d/core/bbox/box_torch_ops.py:81-147) and evaluates odiou_pair<Dual<7>> (odiou.cuh): the value and its exact gradient w.r.t. the
// predicted box by forward-mode differentiation; the decode Jacobian is diagonal, so the gradient w.r.t. the head's box outputs is one more
// multiply.  Per-frame sums are reduced in a fixed order.  Compiled without FMA contraction like the other geometry files.
#include "odiou.cuh"

namespace sessd {

constexpr int kOdThreads = 128;
constexpr int kOdBlocks = kNumSMs;

__global__ void __launch_bounds__(kOdThreads) odiou_loss_kernel(const float *__restrict__ head, const float *__restrict__ anchors,
                                                                const int *__restrict__ labels, const float *__restrict__ reg_targets, int batch,
                                                                int A, int apl, int stride, float w_odiou, const float *__restrict__ losses,
                                                                float *__restrict__ partial, float *__restrict__ grad_head) {
    __shared__ float s_red[kOdThreads / 32];
    const int b = blockIdx.y;
    const float rw = 1.f / fmaxf(losses[b * 8 + 6], 1.f);            // 1 / num_pos (written by sessd_head_loss)
    float acc = 0.f;
    for (int a = blockIdx.x * kOdThreads + threadIdx.x; a < A; a += gridDim.x * kOdThreads) {
        if (labels[(size_t)b * A + a] <= 0) continue;
        const int pix = a / apl, r = a - pix * apl;
        const size_t hb = ((size_t)b * (A / apl) + pix) * stride;
        const float *e = head + hb + 7 * r;
        const float *an = anchors + (size_t)a * 7;
        const float *tg = reg_targets + ((size_t)b * A + a) * 7;
        const float diag = sqrtf(an[4] * an[4] + an[3] * an[3]);
        float g[7], qv[7], jac[7];
        g[0] = tg[0] * diag + an[0]; g[1] = tg[1] * diag + an[1]; g[2] = tg[2] * an[5] + an[2];
        g[3] = expf(tg[3]) * an[3]; g[4] = expf(tg[4]) * an[4]; g[5] = expf(tg[5]) * an[5]; g[6] = tg[6] + an[6];
        qv[0] = e[0] * diag + an[0]; qv[1] = e[1] * diag + an[1]; qv[2] = e[2] * an[5] + an[2];
        qv[3] = expf(e[3]) * an[3]; qv[4] = expf(e[4]) * an[4]; qv[5] = expf(e[5]) * an[5]; qv[6] = e[6] + an[6];
        jac[0] = diag; jac[1] = diag; jac[2] = an[5]; jac[3] = qv[3]; jac[4] = qv[4]; jac[5] = qv[5]; jac[6] = 1.f;
        Dual<7> q[7];
#pragma unroll
        for (int j = 0; j < 7; ++j) q[j] = dual_var<7>(qv[j], j);
        const Dual<7> od = odiou_pair<Dual<7>>(g, q);
        acc += od.v * rw;
        if (grad_head) {
            float *gh = grad_head + hb + 7 * r;
#pragma unroll
            for (int j = 0; j < 7; ++j) gh[j] += od.d[j] * jac[j] * rw * w_odiou / (float)batch;
        }
    }
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_down_sync(0xffffffffu, acc, d);
    if (lane == 0) s_red[warp] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        float v = 0.f;
        for (int i = 0; i < kOdThreads / 32; ++i) v += s_red[i];
        partial[(size_t)b * gridDim.x + blockIdx.x] = v;
    }
}

__global__ void odiou_finish_kernel(const float *__restrict__ partial, int nblocks, float *__restrict__ out) {
    const int b = blockIdx.x;
    if (threadIdx.x == 0) {
        float v = 0.f;
        for (int i = 0; i < nblocks; ++i) v += partial[(size_t)b * nblocks + i];
        out[b] = v;
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" size_t sessd_odiou_loss_workspace_bytes(int batch) { return batch < 1 ? 0 : sizeof(float) * (size_t)batch * kOdBlocks; }

// Run AFTER sessd_head_loss on the same stream (reads num_pos from d_losses[b][6]; ADDS w_odiou * d(sum_b odiou_sum[b]) / batch to the box
// channels of d_grad_head).  d_odiou_sum [batch] = per-frame sum of odiou / num_pos over the positives (the reference's ious_loss is
// 2.0 * batch total / batch_size, mg_head_sessd.py:778 / odious.py:899: pass w_odiou = 2.0).
extern "C" int sessd_odiou_loss(const float *d_head, const float *d_anchors, const int *d_labels, const float *d_reg_targets, int batch,
                                int num_anchors, int anchors_per_loc, int head_stride, float w_odiou, const float *d_losses,
                                float *d_odiou_sum, float *d_grad_head, void *workspace, size_t workspace_bytes, void *stream) {
    if (!d_head || !d_anchors || !d_labels || !d_reg_targets || !d_losses || !d_odiou_sum || batch < 1 || num_anchors < 1 ||
        anchors_per_loc != 2 || head_stride < 22)
        return SESSD_EINVAL;
    if (!workspace || workspace_bytes < sessd_odiou_loss_workspace_bytes(batch)) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    dim3 grid(kOdBlocks, batch);
    SESSD_LAUNCH(odiou_loss_kernel, grid, kOdThreads, 0, st, d_head, d_anchors, d_labels, d_reg_targets, batch, num_anchors, anchors_per_loc,
                 head_stride, w_odiou, d_losses, (float *)workspace, d_grad_head);
    SESSD_LAUNCH(odiou_finish_kernel, batch, 32, 0, st, (const float *)workspace, kOdBlocks, d_odiou_sum);
    return last_error();
}

// HOST evaluation of the same template (no GPU involved): odiou value and d(odiou)/d(q) of n (target, prediction) box pairs
// (x, y, z, w, l, h, r).  It exists so that the arithmetic of the device kernel can be checked on the CPU against the reference's own
// odiou_3D (tests/golden/odiou_case.npz) -- it is not a fallback of the device path.
extern "C" int sessd_odiou_pairs_host(const float *h_gboxes, const float *h_qboxes, int n, float *h_odiou, float *h_grad_q) {
    if (n < 0 || (n > 0 && (!h_gboxes || !h_qboxes || !h_odiou))) return SESSD_EINVAL;
    for (int i = 0; i < n; ++i) {
        Dual<7> q[7];
        for (int j = 0; j < 7; ++j) q[j] = dual_var<7>(h_qboxes[(size_t)i * 7 + j], j);
        const Dual<7> od = odiou_pair<Dual<7>>(h_gboxes + (size_t)i * 7, q);
        h_odiou[i] = od.v;
        if (h_grad_q)
            for (int j = 0; j < 7; ++j) h_grad_q[(size_t)i * 7 + j] = od.d[j];
    }
    return SESSD_OK;
}
