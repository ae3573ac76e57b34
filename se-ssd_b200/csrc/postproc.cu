// postproc.cu -- device-resident detection post-processing: score -> threshold -> top-k -> decode -> rotated NMS
// -> frustum filter -> direction fix -> range mask, with zero host round trips.
//
// Replaces MultiGroupHead.predict / get_task_detections (det3d/models/bbox_heads/mg_head_sessd.py:893-1057),
// second_box_decode (det3d/core/bbox/box_torch_ops.py:81-147), rotate_nms (:527-548), rotate_nms_cc
// (det3d/ops/nms/nms_cpu.py:37-48) and rotate_non_max_suppression_cpu (det3d/ops/nms/nms_cpu.h:72-168).
// The reference syncs to the host twice per frame (box_torch_ops.py:536, mg_head_sessd.py:1026) and runs the
// O(n^2) polygon clipping on one CPU thread.
//
// Stages (per frame, all frames of the batch in the same launches):
//   1. score    : one thread per anchor; sigmoid(cls) >= thr  -> candidate key (rectified score, anchor) appended
//                 with a warp-aggregated atomic.                               [HBM: reads 4 of 22 head floats]
//   2. select   : rank-by-counting top-k (k = nms_pre_max): rank_i = #{j : key_j > key_i}; exact, deterministic
//                 tie-break (lower anchor index first), no multi-pass radix logic; O(n^2) compares from smem.
//   3. prepare  : decode the <= k selected boxes only (the reference decodes all 70400), build the NMS geometry:
//                 [x-w/2, y-l/2, x+w/2, y+l/2, r] and the stand-up AABB of the rotated corners
//                 (box_np_ops.py:512-532, corner_to_standup_nd).
//   4. mask     : upper-triangular 64x64-tile suppression bitmask; a pair is skipped when the stand-up IoU
//                 (iou_jit eps=0, box_np_ops.py:1007-1046) is <= 0 (nms_cpu.h:104-105) and suppressed when the rotated
//                 IoU >= thr (nms_cpu.h:155; '>' selectable for iou3d nms_gpu semantics).
//   5. finalize : greedy scan (stops at nms_post_max), frustum planes, direction flip (mg_head_sessd.py:1035-1037),
//                 post-centre range mask (:1040-1045), ordered compaction into the fixed-size outputs.
// DI-NMS (cfg.nms_mode 1, mg_head_sessd.py:999-1018 -> box_torch_ops.py:552-621 -> nms_cpu.h:173-384) replaces 4 and the scan of 5:
//   4'. overlap : the dense k x k BEV IoU matrix of each frame, on the 32x32 upper-triangle tiles of stage 4.
//   4''. cluster: one CTA per frame: the centerness softmax, then one pick per iteration (block argmax, a pass over the pick's
//                 matrix row, block reductions); emitted clusters feed the frustum / flip / range / compaction of stage 5.
// Tasks (cfg.num_tasks = T > 1, MultiGroupHead with one class per task): every stage runs over B*T slots s = b*T + t in the same
// launches.  Slot (b, t) reads head floats at pix*head_stride + t*task_stride and anchors at d_anchors + t*A*7, frame b's frustum, and its
// own candidate / top-k / mask workspace, so top-k, NMS and nms_post_max are per task (no suppression across classes).  The finalize
// stage compacts each slot into a staging area and post_merge_kernel concatenates the tasks of a frame in task order with label t.
// Compiled with -fmad=false (rotbox.cuh).
#include "common.cuh"
#include "rotbox.cuh"

namespace sessd {

// head layout per pixel and task: [box 2x7 | cls 2 | dir 2x2 | iou 2] = 22 floats at t*task_stride, row stride cfg.head_stride

// tasks of a post-processing config (num_tasks 0 means one) and the head floats between them
__host__ __device__ __forceinline__ int post_tasks(const sessd_post_cfg &c) { return c.num_tasks > 1 ? c.num_tasks : 1; }
__host__ __device__ __forceinline__ int post_task_stride(const sessd_post_cfg &c) { return c.num_tasks > 1 ? c.task_stride : 0; }

struct PostWs {
    unsigned long long *cand;      // [B, A] candidate keys
    int *ncand;                    // [B]
    unsigned long long *sel;       // [B, K] sorted keys
    float *sbox;                   // [B, K, 7] decoded boxes
    float *sbev;                   // [B, K, 5]
    float *ssu;                    // [B, K, 4] stand-up AABB
    RotBox *srot;                  // [B, K] corners + trig precomputed once per box
    float *sscore;                 // [B, K]
    int *sdir;                     // [B, K]
    unsigned long long *mask;      // [B, K, K/64]
    // DI-NMS only (null in rotate_nms mode, which carves exactly the buffers above)
    float *iou;                    // [B, K, K] BEV IoU matrix
    float *sq;                     // [B, K] rectified IoU prediction q = (iou + 1) / 2
    int *slab;                     // [B, K] labels: stand-alone entry only (null on the head path: one class, label 0)
    float *obox;                   // [B, K, 7] emitted clusters (head path): averaged box
    float *oscore;                 // [B, K]
    int *odir;                     // [B, K]
    int *osel;                     // [B, K] anchor index of the pick
    int *ostat;                    // [B, 2] emitted clusters, picks
    // several tasks only: each slot's compacted detections before post_merge_kernel concatenates a frame's tasks
    float *fbox;                   // [B, P, 7]
    float *fscore;                 // [B, P]
    int *fanchor;                  // [B, P] anchor index into the concatenated anchors (t*A + a)
    int *fcount;                   // [B]
    size_t bytes;
};

static inline size_t al(size_t x) { return (x + 255) & ~(size_t)255; }

// batch: slots (frames x tasks); dinms: carve the DI-NMS buffers; labels: also the per-candidate labels, which only the stand-alone entry
// fills; stage_p > 0: the staging rows of several tasks, stage_p per slot
static PostWs post_carve(void *base, int batch, int anchors, int k, bool dinms = false, bool labels = false, int stage_p = 0) {
    PostWs w;
    char *p = (char *)base;
    size_t o = 0;
    auto take = [&](size_t bytes) { char *r = p ? p + o : nullptr; o += al(bytes); return (void *)r; };
    const int cb = (k + 63) / 64;
    w.cand = (unsigned long long *)take(sizeof(unsigned long long) * (size_t)batch * anchors);
    w.ncand = (int *)take(sizeof(int) * batch);
    w.sel = (unsigned long long *)take(sizeof(unsigned long long) * (size_t)batch * k);
    w.sbox = (float *)take(sizeof(float) * (size_t)batch * k * 7);
    w.sbev = (float *)take(sizeof(float) * (size_t)batch * k * 5);
    w.ssu = (float *)take(sizeof(float) * (size_t)batch * k * 4);
    w.srot = (RotBox *)take(sizeof(RotBox) * (size_t)batch * k);
    w.sscore = (float *)take(sizeof(float) * (size_t)batch * k);
    w.sdir = (int *)take(sizeof(int) * (size_t)batch * k);
    w.mask = (unsigned long long *)take(sizeof(unsigned long long) * (size_t)batch * k * cb);
    w.iou = dinms ? (float *)take(sizeof(float) * (size_t)batch * k * k) : nullptr;
    w.sq = dinms ? (float *)take(sizeof(float) * (size_t)batch * k) : nullptr;
    w.slab = (dinms && labels) ? (int *)take(sizeof(int) * (size_t)batch * k) : nullptr;
    w.obox = dinms ? (float *)take(sizeof(float) * (size_t)batch * k * 7) : nullptr;
    w.oscore = dinms ? (float *)take(sizeof(float) * (size_t)batch * k) : nullptr;
    w.odir = dinms ? (int *)take(sizeof(int) * (size_t)batch * k) : nullptr;
    w.osel = dinms ? (int *)take(sizeof(int) * (size_t)batch * k) : nullptr;
    w.ostat = dinms ? (int *)take(sizeof(int) * (size_t)batch * 2) : nullptr;
    const bool st = stage_p > 0;
    w.fbox = st ? (float *)take(sizeof(float) * (size_t)batch * stage_p * 7) : nullptr;
    w.fscore = st ? (float *)take(sizeof(float) * (size_t)batch * stage_p) : nullptr;
    w.fanchor = st ? (int *)take(sizeof(int) * (size_t)batch * stage_p) : nullptr;
    w.fcount = st ? (int *)take(sizeof(int) * (size_t)batch) : nullptr;
    w.bytes = o;
    return w;
}

__device__ __forceinline__ unsigned long long make_key(float score, int idx) {
    // score >= 0 (or +inf); larger key == better; ties broken towards the lower index
    unsigned int sb = __float_as_uint(score);
    if (sb & 0x80000000u) sb = 0;   // -0 / negative garbage sorts last
    return ((unsigned long long)sb << 32) | (unsigned int)(0xFFFFFFFFu - (unsigned int)idx);
}
// stand-alone NMS: scores of any sign (raw logits, say). The high word is the float's bits mapped monotonically onto unsigned:
// non-negative floats set the sign bit, negative ones flip every bit; -0 counts as +0 so that the two tie and fall back to index
// order. Order-preserving over all finite floats; NaN / Inf scores are out of scope. key_score() does not apply to these keys.
__device__ __forceinline__ unsigned long long make_key_signed(float score, int idx) {
    unsigned int sb = __float_as_uint(score);
    if (sb == 0x80000000u) sb = 0u;
    sb = (sb & 0x80000000u) ? ~sb : (sb | 0x80000000u);
    return ((unsigned long long)sb << 32) | (unsigned int)(0xFFFFFFFFu - (unsigned int)idx);
}
__device__ __forceinline__ int key_index(unsigned long long k) { return (int)(0xFFFFFFFFu - (unsigned int)(k & 0xFFFFFFFFull)); }
__device__ __forceinline__ float key_score(unsigned long long k) { return __uint_as_float((unsigned int)(k >> 32)); }

__device__ __forceinline__ void append_key(unsigned long long *list, int *count, bool pred, unsigned long long key) {
    // warp-aggregated atomic append
    const unsigned int ballot = __ballot_sync(0xffffffffu, pred);
    if (!ballot) return;
    const int lane = threadIdx.x & 31;
    const int leader = __ffs(ballot) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(count, __popc(ballot));
    base = __shfl_sync(0xffffffffu, base, leader);
    if (pred) list[base + __popc(ballot & ((1u << lane) - 1))] = key;
}

// 1. score ---------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) post_score_kernel(const float *__restrict__ head, sessd_post_cfg cfg,
                                                         unsigned long long *__restrict__ cand, int *__restrict__ ncand) {
    const int s = blockIdx.y, T = post_tasks(cfg);                   // slot = frame * T + task
    const int b = s / T, toff = (s - b * T) * post_task_stride(cfg);
    const int apl = cfg.anchors_per_loc;
    const int A = cfg.num_anchors;
    const int a_pad = (A + 31) & ~31;   // keep whole warps in the loop for the ballot
    for (int a = blockIdx.x * blockDim.x + threadIdx.x; a < a_pad; a += gridDim.x * blockDim.x) {
        bool keep = false;
        unsigned long long key = 0;
        if (a < A) {
            const int pix = a / apl, r = a - pix * apl;
            const float *h = head + ((size_t)b * (A / apl) + pix) * cfg.head_stride + toff;
            const float logit = h[7 * apl + r];
            const float s = 1.0f / (1.0f + expf(-logit));          // torch.sigmoid
            keep = s >= cfg.score_thresh;                          // mg_head_sessd.py:965-969
            if (keep) {
                const float q = (h[7 * apl + apl + 2 * apl + r] + 1.0f) * 0.5f;   // (iou + 1) * 0.5   (:971)
                const float q2 = q * q;
                key = make_key(s * (q2 * q2), a);                  // score * pow(q, 4)              (:972)
            }
        }
        append_key(cand + (size_t)s * A, ncand + s, keep, key);
    }
}

// stand-alone variant: keys from a score vector
__global__ void __launch_bounds__(256) keys_from_scores_kernel(const float *__restrict__ scores, const int *__restrict__ d_n,
                                                               int max_n, unsigned long long *__restrict__ cand, int *__restrict__ ncand) {
    const int n = min(*d_n, max_n);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) cand[i] = make_key_signed(scores[i], i);
    if (blockIdx.x == 0 && threadIdx.x == 0) *ncand = n;
}

// 2. select --------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) post_select_kernel(const unsigned long long *__restrict__ cand, const int *__restrict__ ncand,
                                                          int stride, int k, unsigned long long *__restrict__ sel) {
    __shared__ unsigned long long tile[1024];
    const int b = blockIdx.y;
    const int n = ncand[b];
    const unsigned long long *c = cand + (size_t)b * stride;
    // all CTAs whose first candidate is beyond n leave together (n is uniform per frame)
    for (int base = blockIdx.x * blockDim.x; base < n; base += gridDim.x * blockDim.x) {
        const int i = base + threadIdx.x;
        const unsigned long long me = (i < n) ? c[i] : 0ull;
        int rank = 0;
        for (int t0 = 0; t0 < n; t0 += 1024) {
            const int cnt = min(1024, n - t0);
            __syncthreads();
            for (int t = threadIdx.x; t < cnt; t += blockDim.x) tile[t] = c[t0 + t];
            __syncthreads();
            if (i < n && rank < k) {
#pragma unroll 8
                for (int t = 0; t < cnt; ++t) rank += (tile[t] > me) ? 1 : 0;
            }
        }
        if (i < n && rank < k) sel[(size_t)b * k + rank] = me;
    }
}

// 3. prepare -------------------------------------------------------------------------------------------------
__device__ __forceinline__ void nms_geometry(const float *box7, float *bev, float *su) {
    const float x = box7[0], y = box7[1], w = box7[3], l = box7[4], r = box7[6];
    const float hw = w / 2.0f, hl = l / 2.0f;                      // iou3d/utils.py:88-95
    bev[0] = x - hw; bev[1] = y - hl; bev[2] = x + hw; bev[3] = y + hl; bev[4] = r;
    const float s = sinf(r), c = cosf(r);
    const float nx[4] = {-0.5f, -0.5f, 0.5f, 0.5f};
    const float ny[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
    float xmin = 0, ymin = 0, xmax = 0, ymax = 0;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const float px = w * nx[k], py = l * ny[k];
        float rx = px * c + py * s;                                 // rotation_2d (box_np_ops.py:433-446)
        float ry = px * (-s) + py * c;
        rx += x; ry += y;
        if (k == 0) { xmin = xmax = rx; ymin = ymax = ry; }
        else { xmin = fminf(xmin, rx); xmax = fmaxf(xmax, rx); ymin = fminf(ymin, ry); ymax = fmaxf(ymax, ry); }
    }
    su[0] = xmin; su[1] = ymin; su[2] = xmax; su[3] = ymax;
}

__global__ void __launch_bounds__(128) post_prepare_kernel(const float *__restrict__ head, const float *__restrict__ anchors,
                                                           sessd_post_cfg cfg, PostWs w) {
    const int s = blockIdx.y, T = post_tasks(cfg);                   // slot = frame * T + task
    const int b = s / T, t_ = s - b * T;
    const int K = cfg.nms_pre_max;
    const int m = min(w.ncand[s], K);
    const int apl = cfg.anchors_per_loc;
    anchors += (size_t)t_ * cfg.num_anchors * 7;
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const unsigned long long key = w.sel[(size_t)s * K + i];
        const int a = key_index(key);
        const int pix = a / apl, r = a - pix * apl;
        const float *h = head + ((size_t)b * (cfg.num_anchors / apl) + pix) * cfg.head_stride + t_ * post_task_stride(cfg);
        const float *t = h + 7 * r;
        const float *an = anchors + (size_t)a * 7;
        float box[7];
        const float diag = sqrtf(an[4] * an[4] + an[3] * an[3]);   // sqrt(la^2 + wa^2)  (box_torch_ops.py:113)
        box[0] = t[0] * diag + an[0];
        box[1] = t[1] * diag + an[1];
        box[2] = t[2] * an[5] + an[2];
        box[3] = expf(t[3]) * an[3];
        box[4] = expf(t[4]) * an[4];
        box[5] = expf(t[5]) * an[5];
        box[6] = t[6] + an[6];
        const size_t o = (size_t)s * K + i;
#pragma unroll
        for (int j = 0; j < 7; ++j) w.sbox[o * 7 + j] = box[j];
        nms_geometry(box, w.sbev + o * 5, w.ssu + o * 4);
        w.srot[o] = rot_prepare(w.sbev[o * 5], w.sbev[o * 5 + 1], w.sbev[o * 5 + 2], w.sbev[o * 5 + 3], w.sbev[o * 5 + 4]);
        w.sscore[o] = key_score(key);
        const float *d = h + 7 * apl + apl + 2 * r;
        w.sdir[o] = (d[1] > d[0]) ? 1 : 0;                           // torch.max(dim=-1)[1]: first max wins
        if (w.sq) w.sq[o] = (h[7 * apl + apl + 2 * apl + r] + 1.0f) * 0.5f;   // DI-NMS: (iou + 1) * 0.5 (:971)
    }
}

__global__ void __launch_bounds__(128) nms_prepare_kernel(const float *__restrict__ boxes5, int K, PostWs w) {
    const int m = min(w.ncand[0], K);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const int src = key_index(w.sel[i]);
        const float *q = boxes5 + (size_t)src * 5;
        float box[7] = {q[0], q[1], 0.f, q[2], q[3], 0.f, q[4]};
        nms_geometry(box, w.sbev + (size_t)i * 5, w.ssu + (size_t)i * 4);
        const float *bv = w.sbev + (size_t)i * 5;
        w.srot[i] = rot_prepare(bv[0], bv[1], bv[2], bv[3], bv[4]);
    }
}

// 4. mask ----------------------------------------------------------------------------------------------------
__device__ __forceinline__ float standup_iou_pos(const float *bn, const float *qk) {
    // iou_jit(eps=0) value for the pair (row box bn, query box qk); 0 when disjoint
    const float box_area = (qk[2] - qk[0]) * (qk[3] - qk[1]);
    const float iw = fminf(bn[2], qk[2]) - fmaxf(bn[0], qk[0]);
    if (iw > 0) {
        const float ih = fminf(bn[3], qk[3]) - fmaxf(bn[1], qk[1]);
        if (ih > 0) {
            const float ua = (bn[2] - bn[0]) * (bn[3] - bn[1]) + box_area - iw * ih;
            return iw * ih / ua;
        }
    }
    return 0.f;
}

// one CTA per 32x32 tile of the upper triangle (a frame's ~400 candidates = 91 tiles: one wave; 64x64 tiles gave 28 CTAs with eight serial
// polygon clips per thread, 40 us); 256 threads = 8 rows x 32 columns per pass, one warp = one row: its ballot is a 32-bit half of the row's
// 64-bit mask word
constexpr int kMaskThreads = 256, kMaskTile = 32;
__global__ void __launch_bounds__(kMaskThreads) post_mask_kernel(PostWs w, int K, float thresh, int ge) {
    const int b = blockIdx.z;
    const int rb = blockIdx.y, cb = blockIdx.x;
    const int m = min(w.ncand[b], K);
    if (rb * kMaskTile >= m || cb * kMaskTile >= m) return;
    const int col_blocks = (K + 63) / 64;
    if (cb < rb) {
        // below the diagonal nothing is read -- except the low half of the 64-bit diagonal word of the rows in the upper half of a 64-row
        // block (the scan loads whole words): zero it
        if ((rb & 1) && cb == rb - 1) {
            const int r = threadIdx.x;
            if (r < kMaskTile && rb * kMaskTile + r < m)
                reinterpret_cast<unsigned int *>(w.mask + ((size_t)b * K + rb * kMaskTile + r) * col_blocks + (cb >> 1))[0] = 0u;
        }
        return;
    }
    __shared__ RotBox s_col[kMaskTile];
    __shared__ RotBox s_row[kMaskTile];
    __shared__ float s_csu[kMaskTile * 4];
    __shared__ float s_rsu[kMaskTile * 4];
    const int ncol = min(m - cb * kMaskTile, kMaskTile), nrow = min(m - rb * kMaskTile, kMaskTile);
    const size_t fb = (size_t)b * K;
    if ((int)threadIdx.x < kMaskTile) {
        const int t = threadIdx.x;
        if (t < ncol) {
            s_col[t] = w.srot[fb + cb * kMaskTile + t];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_csu[t * 4 + k] = w.ssu[(fb + cb * kMaskTile + t) * 4 + k];
        }
    } else if (threadIdx.x < 2 * kMaskTile) {
        const int t = threadIdx.x - kMaskTile;
        if (t < nrow) {
            s_row[t] = w.srot[fb + rb * kMaskTile + t];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_rsu[t * 4 + k] = w.ssu[(fb + rb * kMaskTile + t) * 4 + k];
        }
    }
    __syncthreads();
    const int j = threadIdx.x & 31;           // column within the tile
    for (int r0 = 0; r0 < kMaskTile; r0 += kMaskThreads / 32) {
        const int r = r0 + (threadIdx.x >> 5);
        bool hit = false;
        if (r < nrow && j < ncol && (rb != cb || j > r)) {
            if (standup_iou_pos(s_rsu + r * 4, s_csu + j * 4) > 0.0f) {            // nms_cpu.h:104-105
                const float v = rot_iou_bev_pre(s_row[r], s_col[j]);
                hit = ge ? (v >= thresh) : (v > thresh);
            }
        }
        const unsigned int bits = __ballot_sync(0xffffffffu, hit);
        if (j == 0 && r < nrow)
            reinterpret_cast<unsigned int *>(w.mask + (fb + rb * kMaskTile + r) * col_blocks + (cb >> 1))[cb & 1] = bits;
    }
}

// 4'. overlap (DI-NMS) --------------------------------------------------------------------------------------------
// The loop reads the pick's whole row, every box of the frame included (nms_cpu.h:244-320 clips the pick against all j), so each frame
// gets a dense k x k matrix.  Same tiles and polygon clips as post_mask_kernel: a tile of the upper triangle computes its pairs once and
// writes them twice, the mirrored block through a shared-memory transpose, so the matrix is exactly symmetric like the reference's
// (boost clips (i, j) and (j, i) to the same polygon).  A pair whose stand-up boxes do not overlap gets 0 without a clip.
// Identical rectangles (the diagonal, duplicate candidates) get exactly 1, as boost's intersection of a ring with itself gives: the
// clip is not asked to decide that degenerate case.
__device__ __forceinline__ bool same_rect(const RotBox &a, const RotBox &b) {
    return a.x1 == b.x1 && a.y1 == b.y1 && a.x2 == b.x2 && a.y2 == b.y2 && a.c == b.c && a.s == b.s;
}

__global__ void __launch_bounds__(kMaskThreads) dinms_iou_kernel(PostWs w, int K) {
    const int b = blockIdx.z;
    const int rb = blockIdx.y, cb = blockIdx.x;
    const int m = min(w.ncand[b], K);
    if (cb < rb || rb * kMaskTile >= m || cb * kMaskTile >= m) return;
    __shared__ RotBox s_col[kMaskTile];
    __shared__ RotBox s_row[kMaskTile];
    __shared__ float s_csu[kMaskTile * 4];
    __shared__ float s_rsu[kMaskTile * 4];
    __shared__ float s_t[kMaskTile][kMaskTile + 1];
    const int ncol = min(m - cb * kMaskTile, kMaskTile), nrow = min(m - rb * kMaskTile, kMaskTile);
    const size_t fb = (size_t)b * K;
    if ((int)threadIdx.x < kMaskTile) {
        const int t = threadIdx.x;
        if (t < ncol) {
            s_col[t] = w.srot[fb + cb * kMaskTile + t];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_csu[t * 4 + k] = w.ssu[(fb + cb * kMaskTile + t) * 4 + k];
        }
    } else if (threadIdx.x < 2 * kMaskTile) {
        const int t = threadIdx.x - kMaskTile;
        if (t < nrow) {
            s_row[t] = w.srot[fb + rb * kMaskTile + t];
#pragma unroll
            for (int k = 0; k < 4; ++k) s_rsu[t * 4 + k] = w.ssu[(fb + rb * kMaskTile + t) * 4 + k];
        }
    }
    __syncthreads();
    float *mat = w.iou + fb * K;
    const int lane = threadIdx.x & 31;
    for (int r0 = 0; r0 < kMaskTile; r0 += kMaskThreads / 32) {
        const int r = r0 + (threadIdx.x >> 5), j = lane;
        if (r < nrow && j < ncol && (rb != cb || j >= r)) {
            float v = 0.f;
            if ((rb == cb && j == r) || same_rect(s_row[r], s_col[j])) v = 1.f;
            else if (standup_iou_pos(s_rsu + r * 4, s_csu + j * 4) > 0.0f) v = rot_iou_bev_pre(s_row[r], s_col[j]);
            mat[(size_t)(rb * kMaskTile + r) * K + cb * kMaskTile + j] = v;
            s_t[r][j] = v;
        }
    }
    __syncthreads();
    // mirrored block: element (row c, column r) = s_t[r][c]; one warp per mirrored row, lanes along its columns
    for (int c0 = 0; c0 < kMaskTile; c0 += kMaskThreads / 32) {
        const int c = c0 + (threadIdx.x >> 5), r = lane;
        if (c < ncol && r < nrow && (rb != cb || c > r)) mat[(size_t)(cb * kMaskTile + c) * K + rb * kMaskTile + r] = s_t[r][c];
    }
}

// 4''. cluster loop (DI-NMS) ---------------------------------------------------------------------------------------
// One CTA per frame; candidate j (top-k position) is owned by thread j % kClusterThreads for the whole kernel, so its state needs no
// barrier between the pass that writes it and the next pass.  Shared memory: adjusted score, q, label and state of every candidate;
// state -1 = live, -2 = picked (suppressed for good), it >= 0 = suppressed by pick `it` (its recover list, nms_cpu.h:308-313, 357-360).
// Per pick: one pass over the pick's matrix row and one block reduction of cnt, wsum, avg[7], score_box and two argmax keys (best live
// box, best box of this pick's recover list), so the next pick is known without another pass.  The only serial term is the pick count.
constexpr int kClusterThreads = 512;

struct DinmsOut {
    float *box;       // [B, K, 7]
    float *score;     // [B, K]
    int *label;       // [B, K] nullable
    int *dir;         // [B, K]
    int *pos;         // [B, K] nullable: top-k position of the pick
    int *sel;         // [B, K] anchor / input index of the pick
    int *stat;        // [B, 2] emitted clusters, picks
};

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ unsigned long long warp_max_u64(unsigned long long v) {
#pragma unroll
    for (int o = 16; o; o >>= 1) {
        const unsigned long long u = __shfl_xor_sync(0xffffffffu, v, o);
        v = u > v ? u : v;
    }
    return v;
}
// block-wide sum or max of one float (all threads get the result); s_tmp: [kClusterThreads / 32 + 1] floats
__device__ __forceinline__ float block_reduce(float v, bool is_max, float *s_tmp) {
    constexpr int NW = kClusterThreads / 32;
    v = is_max ? warp_max(v) : warp_sum(v);
    if ((threadIdx.x & 31) == 0) s_tmp[threadIdx.x >> 5] = v;
    __syncthreads();
    if (threadIdx.x < 32) {
        float u = (threadIdx.x < NW) ? s_tmp[threadIdx.x] : (is_max ? -INFINITY : 0.f);
        u = is_max ? warp_max(u) : warp_sum(u);
        if (threadIdx.x == 0) s_tmp[NW] = u;
    }
    __syncthreads();
    const float r = s_tmp[NW];
    __syncthreads();
    return r;
}

// anchors: slot b reads anchors + (b % tasks) * task_anchors * 7 (its task's anchors)
__global__ void __launch_bounds__(kClusterThreads) dinms_cluster_kernel(PostWs w, int K, const float *__restrict__ anchors, int tasks,
                                                                         int task_anchors, sessd_dinms_cfg c, DinmsOut o) {
    constexpr int NW = kClusterThreads / 32;
    extern __shared__ float cdyn[];
    float *s_adj = cdyn;
    float *s_q = s_adj + K;
    int *s_lab = (int *)(s_q + K);
    int *s_state = s_lab + K;
    __shared__ float s_tmp[NW + 1];
    __shared__ float s_red[NW][10];
    __shared__ unsigned long long s_key[NW][2];
    __shared__ unsigned long long s_next;
    __shared__ int s_kept;
    const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int m = min(w.ncand[b], K);
    const size_t fb = (size_t)b * K;
    const float *sbox = w.sbox + fb * 7;
    if (anchors) anchors += (size_t)(b % tasks) * task_anchors * 7;

    // centerness (box_torch_ops.py:584-588): d = |centre - anchor centre|, m = softmax(d) over the k candidates,
    // score *= (1 - m)^pow; d is parked in s_adj until the softmax is known
    float dmax = -INFINITY;
    for (int i = tid; i < m; i += kClusterThreads) {
        const float *an = anchors ? anchors + (size_t)key_index(w.sel[fb + i]) * 7 : nullptr;
        float d = 0.f;
        if (c.centerness) {
            const float dx = fabsf(sbox[i * 7] - an[0]), dy = fabsf(sbox[i * 7 + 1] - an[1]);
            d = sqrtf(dx * dx + dy * dy);
        }
        s_adj[i] = d;
        dmax = fmaxf(dmax, d);
    }
    dmax = block_reduce(dmax, true, s_tmp);
    float se = 0.f;
    if (c.centerness)
        for (int i = tid; i < m; i += kClusterThreads) se += expf(s_adj[i] - dmax);
    se = block_reduce(se, false, s_tmp);
    float smax = -INFINITY;
    unsigned long long best = 0;
    for (int i = tid; i < m; i += kClusterThreads) {
        float s = w.sscore[fb + i];
        if (c.centerness) {
            const float t = 1.0f - expf(s_adj[i] - dmax) / se;
            s *= (c.centerness_pow == 2.0f) ? t * t : powf(t, c.centerness_pow);   // torch.pow(x, 2) is x * x
        }
        s_adj[i] = s;
        s_q[i] = w.sq[fb + i];
        s_lab[i] = w.slab ? w.slab[fb + i] : 0;
        s_state[i] = -1;
        smax = fmaxf(smax, s);
        const unsigned long long key = make_key(s, i);
        best = key > best ? key : best;
    }
    smax = block_reduce(smax, true, s_tmp);          // score_max4norm (nms_cpu.h:226-235)
    best = warp_max_u64(best);
    if (lane == 0) s_key[wid][0] = best;
    __syncthreads();
    if (tid < 32) {
        unsigned long long u = tid < NW ? s_key[tid][0] : 0ull;
        u = warp_max_u64(u);
        if (tid == 0) s_next = u;
    }
    __syncthreads();

    int nout = 0, picks = 0;
    for (int it = 0;; ++it) {
        const unsigned long long next = s_next;
        if (next == 0ull) break;                      // every candidate suppressed
        const int idx = key_index(next);             // argmax of the adjusted score, strict '>': the first position wins a tie
        // sigma^2 band of the pick's distance to the origin (sqrt of the fp64 sum, stored as fp32, nms_cpu.h:255)
        const float px = sbox[idx * 7], py = sbox[idx * 7 + 1];
        const float dist = (float)sqrt((double)px * (double)px + (double)py * (double)py);
        float s2 = 0.f;
        bool band = false;
#pragma unroll
        for (int k = 0; k < 3; ++k)
            if (dist >= c.dist_edge[k] && dist < c.dist_edge[k + 1]) { s2 = c.sigma2[k]; band = true; }
        const float *row = w.iou + (fb + idx) * K;
        const int li = s_lab[idx];
        float cnt = 0.f, wsum = 0.f, sb = -1.f, av[7];
#pragma unroll
        for (int k = 0; k < 7; ++k) av[k] = 0.f;
        unsigned long long best_live = 0, best_rec = 0;
        for (int j = tid; j < m; j += kClusterThreads) {
            const float ov = row[j];
            int st = (j == idx) ? -2 : s_state[j];
            if (s_lab[j] == li) {
                const float qj = s_q[j];
                if (ov > 0.f) cnt += ov * qj;
                if (ov > c.suppressed_thresh) {                                 // member (nms_cpu.h:284-301)
                    sb = fmaxf(sb, s_adj[j] / smax);
                    // no band (distance >= the last edge): weight 0, so wsum = 0 and a kept cluster's box is NaN, as in the reference
                    const float wt = band ? (float)exp(-((double)(1.f - ov) * (double)(1.f - ov)) / (double)s2) : 0.f;
                    const float wq = wt * qj;
#pragma unroll
                    for (int k = 0; k < 7; ++k) av[k] += wq * sbox[j * 7 + k];
                    wsum += wq;
                }
            }
            // suppression (nms_cpu.h:303-309) also requires overlapping stand-up boxes; IoU >= thr > 0 implies that, so it is not tested
            if (st == -1 && ov >= c.suppressed_thresh) st = it;
            s_state[j] = st;
            const unsigned long long key = make_key(s_adj[j], j);
            if (st == -1) best_live = key > best_live ? key : best_live;
            else if (st == it) best_rec = key > best_rec ? key : best_rec;
        }
        cnt = warp_sum(cnt);
        wsum = warp_sum(wsum);
        sb = warp_max(sb);
#pragma unroll
        for (int k = 0; k < 7; ++k) av[k] = warp_sum(av[k]);
        best_live = warp_max_u64(best_live);
        best_rec = warp_max_u64(best_rec);
        if (lane == 0) {
            s_red[wid][0] = cnt; s_red[wid][1] = wsum; s_red[wid][2] = sb;
#pragma unroll
            for (int k = 0; k < 7; ++k) s_red[wid][3 + k] = av[k];
            s_key[wid][0] = best_live; s_key[wid][1] = best_rec;
        }
        __syncthreads();
        if (tid < 32) {
            float v[10];
#pragma unroll
            for (int k = 0; k < 10; ++k) v[k] = tid < NW ? s_red[tid][k] : (k == 2 ? -1.f : 0.f);
            unsigned long long kl = tid < NW ? s_key[tid][0] : 0ull, kr = tid < NW ? s_key[tid][1] : 0ull;
            v[0] = warp_sum(v[0]);
            v[1] = warp_sum(v[1]);
            v[2] = warp_max(v[2]);
#pragma unroll
            for (int k = 3; k < 10; ++k) v[k] = warp_sum(v[k]);
            kl = warp_max_u64(kl);
            kr = warp_max_u64(kr);
            if (tid == 0) {
                ++picks;
                const bool kept = v[0] > c.cnt_thresh;
                if (kept) {
                    const size_t r = fb + nout;
#pragma unroll
                    for (int k = 0; k < 7; ++k) o.box[r * 7 + k] = v[3 + k] / v[1];
                    o.score[r] = v[2] * smax;
                    o.dir[r] = w.sdir[fb + idx];
                    if (o.label) o.label[r] = li;
                    if (o.pos) o.pos[r] = idx;
                    o.sel[r] = key_index(w.sel[fb + idx]);
                    ++nout;
                }
                s_kept = kept;
                s_next = kept ? kl : (kl > kr ? kl : kr);
            }
        }
        __syncthreads();
        if (!s_kept)                                  // recover this pick's list (nms_cpu.h:357-360)
            for (int j = tid; j < m; j += kClusterThreads)
                if (s_state[j] == it) s_state[j] = -1;
    }
    if (tid == 0) {
        o.stat[2 * b] = nout;
        o.stat[2 * b + 1] = picks;
    }
}

// 5. finalize ------------------------------------------------------------------------------------------------
// greedy scan shared by the detection path and the stand-alone NMS; returns kept positions (into the sorted list)
// in s_keep[0..nkeep).  One CTA (256 threads) per frame.
__device__ int greedy_scan(const unsigned long long *__restrict__ mask, int m, int col_blocks, int max_keep,
                           unsigned long long *remv /*[col_blocks] smem*/, unsigned long long *diag /*[64] smem*/,
                           int *s_keep /*[max_keep] smem*/, int *s_misc /*[4] smem*/, unsigned long long *s_kb /*[1] smem*/) {
    const int nblk = (m + 63) / 64;
    for (int j = threadIdx.x; j < col_blocks; j += blockDim.x) remv[j] = 0;
    if (threadIdx.x == 0) s_misc[0] = 0;
    // the diagonal word of row (64 b + t) is fetched one block ahead, so its L2 round trip overlaps the previous block's scan
    unsigned long long dcur = 0;
    if ((int)threadIdx.x < min(64, m)) dcur = mask[(size_t)threadIdx.x * col_blocks];
    __syncthreads();
    for (int b = 0; b < nblk; ++b) {
        const int rows = min(64, m - b * 64);
        if ((int)threadIdx.x < rows) diag[threadIdx.x] = dcur;
        if (b + 1 < nblk && (int)threadIdx.x < min(64, m - (b + 1) * 64)) dcur = mask[(size_t)((b + 1) * 64 + threadIdx.x) * col_blocks + b + 1];
        __syncthreads();
        if (threadIdx.x == 0) {
            unsigned long long cur = remv[b], kb = 0;
            int nk = s_misc[0];
            for (int t = 0; t < rows && nk < max_keep; ++t)
                if (!((cur >> t) & 1ull)) { s_keep[nk++] = b * 64 + t; kb |= 1ull << t; cur |= diag[t]; }
            s_misc[0] = nk;
            *s_kb = kb;
        }
        __syncthreads();
        const unsigned long long kb = *s_kb;
        if (s_misc[0] >= max_keep) break;
        for (int j = b + 1 + threadIdx.x; j < nblk; j += blockDim.x) {
            // predicated, unrolled: the loads of all kept rows are in flight together (one L2 round trip per block, not one per kept row)
            unsigned long long acc = remv[j];
            const unsigned long long *col = mask + (size_t)(b * 64) * col_blocks + j;
#pragma unroll 16
            for (int t = 0; t < 64; ++t)
                if ((kb >> t) & 1ull) acc |= col[(size_t)t * col_blocks];
            remv[j] = acc;
        }
        __syncthreads();
    }
    __syncthreads();
    return s_misc[0];
}

// optional packed copy of the results for ONE device->host transfer per batch (FrameEngine): packed [B, P, 8] = box 7 | score,
// meta [B, 8 + P] = count, candidates, pre-NMS count, NMS-selected count, voxels of the frame, capacity status, 0, 0,
// then the anchor index of every returned detection (-1 beyond count)
struct PostPack {
    float *packed;
    int *meta;
    const int *num_voxels;     // [B] nullable
    const int *status;         // [1] nullable
};

// kDI: the rows come from the DI-NMS cluster loop (w.obox / oscore / odir / osel, w.ostat) instead of the greedy scan over the mask,
// and the capacity P is nms_pre_max.  One CTA per slot (frame b, task t).  One task: the CTA writes the frame's outputs.  Several
// tasks: d_sel_anchor and d_aux are written per slot ([B, T*P] with task t's block at t*P, and [B*T, 4]); the compacted rows go to the
// slot's staging rows (w.fbox / fscore / fanchor / fcount), which post_merge_kernel concatenates.
template <bool kDI>
__global__ void __launch_bounds__(256) post_finalize_kernel(PostWs w, sessd_post_cfg cfg, const float *__restrict__ frustum,
                                                            float *__restrict__ out_boxes, float *__restrict__ out_scores,
                                                            int *__restrict__ out_labels, int *__restrict__ out_count,
                                                            int *__restrict__ out_aux, int *__restrict__ out_sel_anchor, PostPack pk) {
    extern __shared__ unsigned long long dyn[];
    const int K = cfg.nms_pre_max, P = kDI ? cfg.nms_pre_max : cfg.nms_post_max;
    const int col_blocks = (K + 63) / 64;
    unsigned long long *remv = dyn;
    unsigned long long *diag = dyn + col_blocks;
    int *s_keep = (int *)(diag + 64);
    int *s_flag = s_keep + P;
    __shared__ int s_misc[4];
    __shared__ unsigned long long s_kb;
    const int slot = blockIdx.x, T = post_tasks(cfg);
    const int b = slot / T, task = slot - b * T;
    const bool staged = T > 1;
    const int n = w.ncand[slot];
    const int m = min(n, K);
    const size_t fb = (size_t)slot * K;
    const int abase = task * cfg.num_anchors;                        // index into the concatenated anchors [T, A, 7]
    int nk;
    if constexpr (kDI) nk = w.ostat[2 * slot];
    else nk = greedy_scan(w.mask + fb * col_blocks, m, col_blocks, P, remv, diag, s_keep, s_misc, &s_kb);
    // row t of the kept list: its box, score, direction label and anchor index
    auto row_box = [&](int t) -> const float * { return kDI ? w.obox + (fb + t) * 7 : w.sbox + (fb + s_keep[t]) * 7; };
    auto row_score = [&](int t) { return kDI ? w.oscore[fb + t] : w.sscore[fb + s_keep[t]]; };
    auto row_dir = [&](int t) { return kDI ? w.odir[fb + t] : w.sdir[fb + s_keep[t]]; };
    auto row_anchor = [&](int t) { return abase + (kDI ? w.osel[fb + t] : key_index(w.sel[fb + s_keep[t]])); };
    int *sel_out = out_sel_anchor + ((size_t)b * T + task) * P;
    // per kept box: frustum test + range mask (the direction fix happens before the range test but only touches r)
    for (int t = threadIdx.x; t < P; t += blockDim.x) {
        int ok = 0;
        if (t < nk) {
            const float *bx = row_box(t);
            ok = 1;
            if (cfg.use_frustum && frustum) {
                const float *pl = frustum + (size_t)b * 24;
                for (int s = 0; s < 6; ++s) {
                    const float sign = bx[0] * pl[4 * s] + bx[1] * pl[4 * s + 1] + bx[2] * pl[4 * s + 2] + pl[4 * s + 3];
                    if (sign >= 0.f) ok = 0;                        // geometry.py:262-275
                }
            }
            for (int j = 0; j < 3; ++j)
                if (!(bx[j] >= cfg.post_range[j] && bx[j] <= cfg.post_range[3 + j])) ok = 0;
            sel_out[t] = row_anchor(t);
        } else {
            sel_out[t] = -1;
        }
        s_flag[t] = ok;
    }
    __syncthreads();
    // ordered compaction (P <= a few hundred: serial prefix by one thread is cheapest)
    if (threadIdx.x == 0) {
        int c = 0;
        for (int t = 0; t < P; ++t) { int f = s_flag[t]; s_flag[t] = f ? c : -1; c += f; }
        out_aux[slot * 4 + 0] = n;
        out_aux[slot * 4 + 1] = m;
        out_aux[slot * 4 + 2] = nk;
        out_aux[slot * 4 + 3] = kDI ? w.ostat[2 * slot + 1] : 0;
        if (staged) w.fcount[slot] = c;
        else out_count[b] = c;
        s_misc[1] = c;
        if (pk.meta && !staged) {
            int *mt = pk.meta + (size_t)b * (8 + P);
            mt[0] = c; mt[1] = n; mt[2] = m; mt[3] = nk;
            mt[4] = pk.num_voxels ? pk.num_voxels[b] : 0;
            mt[5] = pk.status ? *pk.status : 0;
            mt[6] = 0; mt[7] = 0;
        }
    }
    __syncthreads();
    const int total = s_misc[1];
    for (int t = threadIdx.x; t < P; t += blockDim.x) {
        const int dst = s_flag[t];
        if (dst >= 0) {
            const float *bx = row_box(t);
            float *ob = (staged ? w.fbox : out_boxes) + ((size_t)slot * P + dst) * 7;
#pragma unroll
            for (int j = 0; j < 6; ++j) ob[j] = bx[j];
            float r = bx[6];
            const bool opp = ((r - cfg.direction_offset) > 0.f) != (row_dir(t) == 1);   // :1035-1037
            if (opp) r += 3.14159265358979323846f;   // torch.tensor(np.pi).type_as(fp32)
            ob[6] = r;
            const float sc = row_score(t);
            if (staged) {
                w.fscore[(size_t)slot * P + dst] = sc;
                w.fanchor[(size_t)slot * P + dst] = row_anchor(t);
                continue;
            }
            out_scores[(size_t)b * P + dst] = sc;
            out_labels[(size_t)b * P + dst] = task;
            if (pk.packed) {
                float *pp = pk.packed + ((size_t)b * P + dst) * 8;
#pragma unroll
                for (int j = 0; j < 6; ++j) pp[j] = ob[j];
                pp[6] = r;
                pp[7] = sc;
                pk.meta[(size_t)b * (8 + P) + 8 + dst] = row_anchor(t);
            }
        }
    }
    if (staged) return;
    for (int t = total + threadIdx.x; t < P; t += blockDim.x) {
        float *ob = out_boxes + ((size_t)b * P + t) * 7;
        for (int j = 0; j < 7; ++j) ob[j] = 0.f;
        out_scores[(size_t)b * P + t] = 0.f;
        out_labels[(size_t)b * P + t] = -1;
        if (pk.packed) {
            float *pp = pk.packed + ((size_t)b * P + t) * 8;
            for (int j = 0; j < 8; ++j) pp[j] = 0.f;
            pk.meta[(size_t)b * (8 + P) + 8 + t] = -1;
        }
    }
}

// several tasks: one CTA per frame concatenates its slots' staged detections in task order into the [B, T*P] outputs, label = task,
// count = the frame total, the packed block's meta header summed over the tasks; rows beyond the total as in post_finalize_kernel
__global__ void __launch_bounds__(256) post_merge_kernel(PostWs w, sessd_post_cfg cfg, int P, float *__restrict__ out_boxes,
                                                         float *__restrict__ out_scores, int *__restrict__ out_labels,
                                                         int *__restrict__ out_count, const int *__restrict__ out_aux, PostPack pk) {
    const int b = blockIdx.x, T = post_tasks(cfg), TP = T * P;
    const size_t ob0 = (size_t)b * TP;
    int off = 0;
    for (int t = 0; t < T; ++t) {
        const int slot = b * T + t, c = w.fcount[slot];
        for (int i = threadIdx.x; i < c; i += blockDim.x) {
            const size_t src = (size_t)slot * P + i, dst = ob0 + off + i;
            const float *bx = w.fbox + src * 7;
            float *o = out_boxes + dst * 7;
#pragma unroll
            for (int j = 0; j < 7; ++j) o[j] = bx[j];
            out_scores[dst] = w.fscore[src];
            out_labels[dst] = t;
            if (pk.packed) {
                float *pp = pk.packed + dst * 8;
#pragma unroll
                for (int j = 0; j < 7; ++j) pp[j] = bx[j];
                pp[7] = w.fscore[src];
                pk.meta[(size_t)b * (8 + TP) + 8 + off + i] = w.fanchor[src];
            }
        }
        off += c;
    }
    for (int t = off + threadIdx.x; t < TP; t += blockDim.x) {
        float *o = out_boxes + (ob0 + t) * 7;
        for (int j = 0; j < 7; ++j) o[j] = 0.f;
        out_scores[ob0 + t] = 0.f;
        out_labels[ob0 + t] = -1;
        if (pk.packed) {
            float *pp = pk.packed + (ob0 + t) * 8;
            for (int j = 0; j < 8; ++j) pp[j] = 0.f;
            pk.meta[(size_t)b * (8 + TP) + 8 + t] = -1;
        }
    }
    if (threadIdx.x == 0) {
        out_count[b] = off;
        if (pk.meta) {
            int sum[3] = {0, 0, 0};
            for (int t = 0; t < T; ++t)
                for (int j = 0; j < 3; ++j) sum[j] += out_aux[(b * T + t) * 4 + j];
            int *mt = pk.meta + (size_t)b * (8 + TP);
            mt[0] = off; mt[1] = sum[0]; mt[2] = sum[1]; mt[3] = sum[2];
            mt[4] = pk.num_voxels ? pk.num_voxels[b] : 0;
            mt[5] = pk.status ? *pk.status : 0;
            mt[6] = 0; mt[7] = 0;
        }
    }
}

__global__ void __launch_bounds__(256) nms_finalize_kernel(PostWs w, int K, int P, int *__restrict__ keep, int *__restrict__ num_keep) {
    extern __shared__ unsigned long long dyn[];
    const int col_blocks = (K + 63) / 64;
    unsigned long long *remv = dyn;
    unsigned long long *diag = dyn + col_blocks;
    int *s_keep = (int *)(diag + 64);
    __shared__ int s_misc[4];
    __shared__ unsigned long long s_kb;
    const int m = min(w.ncand[0], K);
    const int nk = greedy_scan(w.mask, m, col_blocks, P, remv, diag, s_keep, s_misc, &s_kb);
    for (int t = threadIdx.x; t < P; t += blockDim.x) keep[t] = (t < nk) ? key_index(w.sel[s_keep[t]]) : -1;
    if (threadIdx.x == 0) *num_keep = nk;
}

}  // namespace sessd

using namespace sessd;

// per-frame capacity of one task: nms_post_max, nms_pre_max under DI-NMS
static int post_slot_capacity(const sessd_post_cfg &c) { return c.nms_mode == 1 ? c.nms_pre_max : c.nms_post_max; }

// the workspace of a config: slots = frames x tasks, plus the staging rows when there are several tasks
static PostWs post_carve_cfg(void *base, const sessd_post_cfg &c) {
    const int T = post_tasks(c);
    return post_carve(base, c.batch * T, c.num_anchors, c.nms_pre_max, c.nms_mode == 1, false, T > 1 ? post_slot_capacity(c) : 0);
}

extern "C" size_t sessd_postprocess_workspace_bytes(const sessd_post_cfg *cfg) {
    if (!cfg) return 0;
    return post_carve_cfg(nullptr, *cfg).bytes;
}

static bool dinms_cfg_ok(const sessd_dinms_cfg &c) {
    return c.suppressed_thresh > 0.f && c.sigma2[0] > 0.f && c.sigma2[1] > 0.f && c.sigma2[2] > 0.f;
}

static size_t cluster_smem(int K) { return (sizeof(float) * 2 + sizeof(int) * 2) * (size_t)K; }

// overlap matrix + cluster loop of B frames whose candidates stage 3 (or dinms_prepare_kernel) has laid out in w
// B: slots; slot b reads the anchors of task b % tasks (task_anchors rows each)
static int dinms_launch(PostWs w, int B, int K, const float *d_anchors, int tasks, int task_anchors, const sessd_dinms_cfg &c, DinmsOut o,
                        cudaStream_t st) {
    const int cb = (K + kMaskTile - 1) / kMaskTile;
    dim3 g(cb, cb, B);
    SESSD_LAUNCH(dinms_iou_kernel, g, kMaskThreads, 0, st, w, K);
    const size_t sm = cluster_smem(K);
    if (sm > 48 * 1024) SESSD_CUDA_TRY(cudaFuncSetAttribute(dinms_cluster_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    SESSD_LAUNCH(dinms_cluster_kernel, B, kClusterThreads, sm, st, w, K, d_anchors, tasks, task_anchors, c, o);
    return 0;
}

static size_t finalize_smem(int K, int P) {
    const int cb = (K + 63) / 64;
    return sizeof(unsigned long long) * (cb + 64) + sizeof(int) * (2 * (size_t)P + 8);
}

static int postprocess_impl(const float *d_head, const float *d_anchors, const float *d_frustum,
                            const sessd_post_cfg *cfg, float *d_boxes, float *d_scores, int *d_labels, int *d_count,
                            int *d_aux, int *d_sel_anchor, PostPack pk, void *workspace, size_t workspace_bytes, void *stream) {
    if (!cfg || !d_head || !d_anchors || !d_boxes || !d_scores || !d_labels || !d_count || !d_aux || !d_sel_anchor)
        return SESSD_EINVAL;
    if (cfg->batch < 1 || cfg->num_anchors < 1 || cfg->anchors_per_loc < 1 || cfg->num_anchors % cfg->anchors_per_loc ||
        cfg->nms_pre_max < 1 || cfg->nms_post_max < 1 || cfg->nms_post_max > 4096 || cfg->nms_pre_max > 16384)
        return SESSD_EINVAL;
    if (cfg->anchors_per_loc != 2 || cfg->head_stride < 22) return SESSD_EINVAL;   // head layout is fixed at 22 channels
    if (cfg->nms_mode != 0 && cfg->nms_mode != 1) return SESSD_EINVAL;
    // several tasks: each one's 22 floats at t * task_stride inside the pixel row
    if (cfg->num_tasks < 0 || cfg->num_tasks > SESSD_POST_MAX_TASKS) return SESSD_EINVAL;
    const int T = post_tasks(*cfg);
    if (T > 1 && (cfg->task_stride < 22 || (long long)(T - 1) * cfg->task_stride + 22 > cfg->head_stride)) return SESSD_EINVAL;
    const bool dinms = cfg->nms_mode == 1;
    if (dinms && (cfg->nms_pre_max > SESSD_DINMS_MAX_PRE || !dinms_cfg_ok(cfg->dinms))) return SESSD_EINVAL;
    PostWs w = post_carve_cfg(workspace, *cfg);
    if (!workspace || w.bytes > workspace_bytes) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    // B: slots (frame b, task t) = b * T + t; every stage below runs over all of them
    const int B = cfg->batch * T, A = cfg->num_anchors, K = cfg->nms_pre_max, P = post_slot_capacity(*cfg);
    SESSD_CUDA_TRY(cudaMemsetAsync(w.ncand, 0, sizeof(int) * B, st));
    dim3 g1(div_up(A, 256), B);
    SESSD_LAUNCH(post_score_kernel, g1, 256, 0, st, d_head, *cfg, w.cand, w.ncand);
    dim3 g2(div_up(A, 256), B);
    SESSD_LAUNCH(post_select_kernel, g2, 256, 0, st, w.cand, w.ncand, A, K, w.sel);
    dim3 g3(div_up(K, 128), B);
    SESSD_LAUNCH(post_prepare_kernel, g3, 128, 0, st, d_head, d_anchors, *cfg, w);
    const size_t sm = finalize_smem(K, P);
    if (dinms) {
        DinmsOut o = {w.obox, w.oscore, nullptr, w.odir, nullptr, w.osel, w.ostat};
        const int rc = dinms_launch(w, B, K, d_anchors, T, A, cfg->dinms, o, st);
        if (rc) return rc;
        if (sm > 48 * 1024)
            SESSD_CUDA_TRY(cudaFuncSetAttribute(post_finalize_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        SESSD_LAUNCH(post_finalize_kernel<true>, B, 256, sm, st, w, *cfg, d_frustum, d_boxes, d_scores, d_labels, d_count, d_aux,
                     d_sel_anchor, pk);
        if (T > 1) SESSD_LAUNCH(post_merge_kernel, cfg->batch, 256, 0, st, w, *cfg, P, d_boxes, d_scores, d_labels, d_count, d_aux, pk);
        return last_error();
    }
    const int cb = (K + kMaskTile - 1) / kMaskTile;
    dim3 g4(cb, cb, B);
    SESSD_LAUNCH(post_mask_kernel, g4, kMaskThreads, 0, st, w, K, cfg->nms_iou_thresh, cfg->nms_ge);
    if (sm > 48 * 1024) SESSD_CUDA_TRY(cudaFuncSetAttribute(post_finalize_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    SESSD_LAUNCH(post_finalize_kernel<false>, B, 256, sm, st, w, *cfg, d_frustum, d_boxes, d_scores, d_labels, d_count, d_aux, d_sel_anchor, pk);
    if (T > 1) SESSD_LAUNCH(post_merge_kernel, cfg->batch, 256, 0, st, w, *cfg, P, d_boxes, d_scores, d_labels, d_count, d_aux, pk);
    return last_error();
}

extern "C" int sessd_postprocess(const float *d_head, const float *d_anchors, const float *d_frustum,
                                 const sessd_post_cfg *cfg, float *d_boxes, float *d_scores, int *d_labels, int *d_count,
                                 int *d_aux, int *d_sel_anchor, void *workspace, size_t workspace_bytes, void *stream) {
    PostPack pk = {nullptr, nullptr, nullptr, nullptr};
    return postprocess_impl(d_head, d_anchors, d_frustum, cfg, d_boxes, d_scores, d_labels, d_count, d_aux, d_sel_anchor, pk, workspace,
                            workspace_bytes, stream);
}

extern "C" int sessd_postprocess_packed(const float *d_head, const float *d_anchors, const float *d_frustum,
                                        const sessd_post_cfg *cfg, float *d_boxes, float *d_scores, int *d_labels, int *d_count,
                                        int *d_aux, int *d_sel_anchor, float *d_packed, int *d_meta, const int *d_num_voxels,
                                        const int *d_status, void *workspace, size_t workspace_bytes, void *stream) {
    if (!d_packed || !d_meta) return SESSD_EINVAL;
    PostPack pk = {d_packed, d_meta, d_num_voxels, d_status};
    return postprocess_impl(d_head, d_anchors, d_frustum, cfg, d_boxes, d_scores, d_labels, d_count, d_aux, d_sel_anchor, pk, workspace,
                            workspace_bytes, stream);
}

extern "C" size_t sessd_rotate_nms_workspace_bytes(int max_boxes, int pre_max) {
    if (max_boxes < 1 || pre_max < 1) return 0;
    return post_carve(nullptr, 1, max_boxes, pre_max).bytes;
}

extern "C" int sessd_rotate_nms(const float *d_boxes5, const float *d_scores, const int *d_n, int max_boxes, int pre_max,
                                int post_max, float iou_thresh, int ge, int *d_keep, int *d_num_keep, void *workspace,
                                size_t workspace_bytes, void *stream) {
    if (!d_boxes5 || !d_scores || !d_n || !d_keep || !d_num_keep || max_boxes < 1 || pre_max < 1 || post_max < 1 ||
        pre_max > 16384 || post_max > 4096)
        return SESSD_EINVAL;
    PostWs w = post_carve(workspace, 1, max_boxes, pre_max);
    if (!workspace || w.bytes > workspace_bytes) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    SESSD_LAUNCH(keys_from_scores_kernel, persistent_grid(max_boxes, 256), 256, 0, st, d_scores, d_n, max_boxes, w.cand, w.ncand);
    dim3 g2(div_up(max_boxes, 256), 1);
    SESSD_LAUNCH(post_select_kernel, g2, 256, 0, st, w.cand, w.ncand, max_boxes, pre_max, w.sel);
    SESSD_LAUNCH(nms_prepare_kernel, div_up(pre_max, 128), 128, 0, st, d_boxes5, pre_max, w);
    const int cb = (pre_max + kMaskTile - 1) / kMaskTile;
    dim3 g4(cb, cb, 1);
    SESSD_LAUNCH(post_mask_kernel, g4, kMaskThreads, 0, st, w, pre_max, iou_thresh, ge);
    const size_t sm = finalize_smem(pre_max, post_max);
    if (sm > 48 * 1024) SESSD_CUDA_TRY(cudaFuncSetAttribute(nms_finalize_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
    SESSD_LAUNCH(nms_finalize_kernel, 1, 256, sm, st, w, pre_max, post_max, d_keep, d_num_keep);
    return last_error();
}

// ---------------------------------------------------------------------------------------------------------------- stand-alone DI-NMS
// gather the top-k rows of the caller's arrays into the layout the overlap stage and the cluster loop read
__global__ void __launch_bounds__(128) dinms_prepare_kernel(const float *__restrict__ boxes7, const float *__restrict__ boxes5,
                                                            const float *__restrict__ scores, const float *__restrict__ iou_preds,
                                                            const int *__restrict__ labels, const int *__restrict__ dirs, int K, PostWs w) {
    const int m = min(w.ncand[0], K);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < m; i += gridDim.x * blockDim.x) {
        const int src = key_index(w.sel[i]);
        const float *q = boxes5 + (size_t)src * 5;
        float box[7] = {q[0], q[1], 0.f, q[2], q[3], 0.f, q[4]};
        nms_geometry(box, w.sbev + (size_t)i * 5, w.ssu + (size_t)i * 4);
        const float *bv = w.sbev + (size_t)i * 5;
        w.srot[i] = rot_prepare(bv[0], bv[1], bv[2], bv[3], bv[4]);
#pragma unroll
        for (int j = 0; j < 7; ++j) w.sbox[(size_t)i * 7 + j] = boxes7[(size_t)src * 7 + j];
        w.sscore[i] = scores[src];
        w.sq[i] = iou_preds[src];
        w.slab[i] = labels[src];
        w.sdir[i] = dirs[src];
    }
}

extern "C" size_t sessd_rotate_weighted_nms_workspace_bytes(int max_boxes, int pre_max) {
    if (max_boxes < 1 || pre_max < 1) return 0;
    return post_carve(nullptr, 1, max_boxes, pre_max, true, true).bytes;
}

extern "C" int sessd_rotate_weighted_nms(const float *d_boxes7, const float *d_boxes5, const float *d_scores, const float *d_iou_preds,
                                         const int *d_labels, const int *d_dirs, const float *d_anchors, const int *d_n, int max_boxes,
                                         int pre_max, const sessd_dinms_cfg *cfg, float *d_out_boxes, float *d_out_scores,
                                         int *d_out_labels, int *d_out_dirs, int *d_keep, int *d_selected, int *d_count, void *workspace,
                                         size_t workspace_bytes, void *stream) {
    if (!d_boxes7 || !d_boxes5 || !d_scores || !d_iou_preds || !d_labels || !d_dirs || !d_n || !cfg || !d_out_boxes || !d_out_scores ||
        !d_out_labels || !d_out_dirs || !d_keep || !d_selected || !d_count || max_boxes < 1 || pre_max < 1 ||
        pre_max > SESSD_DINMS_MAX_PRE || !dinms_cfg_ok(*cfg) || (cfg->centerness && !d_anchors))
        return SESSD_EINVAL;
    PostWs w = post_carve(workspace, 1, max_boxes, pre_max, true, true);
    if (!workspace || w.bytes > workspace_bytes) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    SESSD_LAUNCH(keys_from_scores_kernel, persistent_grid(max_boxes, 256), 256, 0, st, d_scores, d_n, max_boxes, w.cand, w.ncand);
    dim3 g2(div_up(max_boxes, 256), 1);
    SESSD_LAUNCH(post_select_kernel, g2, 256, 0, st, w.cand, w.ncand, max_boxes, pre_max, w.sel);
    SESSD_LAUNCH(dinms_prepare_kernel, div_up(pre_max, 128), 128, 0, st, d_boxes7, d_boxes5, d_scores, d_iou_preds, d_labels, d_dirs,
                 pre_max, w);
    DinmsOut o = {d_out_boxes, d_out_scores, d_out_labels, d_out_dirs, d_keep, d_selected, d_count};
    const int rc = dinms_launch(w, 1, pre_max, d_anchors, 1, max_boxes, *cfg, o, st);
    if (rc) return rc;
    return last_error();
}
