// augment.cu -- SE-SSD's training augmentation on the GPU: per-object box noise with collision tests, the points' and boxes' per-object
// transform, the teacher's un-augmented twin, global flip / rotation / scaling, the shuffle, and the box bookkeeping before assignment.
//
// Replaces the numba loops of det3d/core/sampler/preprocess.py and the array code of Preprocess.__call__
// (det3d/datasets/pipelines/preprocess.py:68-175) without GT-AUG and SA-DA:
//   box_collision_test (:944-1027)  -- BEV corner-set collision: standup pre-test, 4x4 segment crossing, containment both ways;
//   noise_per_box      (:579-611)   -- box i (valid only, index order) takes the first of its tries whose rotated-and-shifted corners
//                                      collide with no other box's CURRENT corners (earlier boxes that moved count at their new place;
//                                      invalid boxes block but never move); no free try -> -1;
//   the corner set of noise_per_object_v4_ (:618-640): boxes (x, y, w + ctx, l + ctx, ry), box2d_to_corner_jit (box_np_ops.py:536-565);
//   points_transform_ / box3d_transform_ (:545-569), random_flip_v2 / global_rotation_v3 / global_scaling_v3 (:896-941), the shuffle,
//   and filter_gt_box_outside_range / limit_period of Voxelization / AssignTarget (pipelines/preprocess.py:200-205, :290-330).
// The random draws are inputs (made on the host by a numpy RandomState, sessd_b200/augment.py): the kernels are pure functions.
//
// Precision (traced through the reference; oracle/augment_ref.py restates the same arithmetic): `gt_boxes[:, [0, 1, 3, 4, 6]] + offset`
// adds a Python list, which numpy promotes to float64, so the corners, the draws and the whole collision predicate are evaluated in fp64.
// The rotations are BLAS gemm calls, which on x86-64 evaluate sum_j a_j r_jk as fma(a2, r2k, fma(a1, r1k, a0 r0k)): restated with
// __fma_rn / __fmaf_rn (fp64 for the 2x2 corner rotations, fp32 for the points and boxes).  Every other operation is individually rounded
// (the file is compiled with -fmad=false).  sin / cos of the draws are CUDA's fp64 functions (within 2 ulp of glibc's): a collision
// outcome depending on that last bit needs a predicate within ~1e-16 of a tie, and an fp32 value rounded from them differs only when the
// fp64 value lies within 2^-51 of an fp32 rounding boundary.  The global stages' fp32 cos / sin / scale / angle come from the host,
// rounded as the reference rounds them.
//
// noise_per_box_kernel: one CTA per frame; the frame's current corners live in shared memory; boxes are visited in order (the
// dependency on earlier boxes is real), and for each valid box all tries x all boxes are tested by the whole CTA, then the smallest
// collision-free try is taken (a shared-memory atomicMin: exactly the reference's first `break`).
// augment_points_kernel: one thread per student row (frame = blockIdx.y): reads the permuted source point, finds the first valid box
// holding it (box-frame test in fp64 against the frame's boxes in shared memory), applies the selected transform (writes the twin), then
// the global stages.  augment_boxes_kernel: one CTA per frame, one thread per box.
// The collision predicate and the membership frame live in augment.cuh (shared with gtaug.cu); sessd_gtaug_select_host runs the same
// predicate on the host (this file's host code is compiled with -ffp-contract=off, so it evaluates operation for operation like the device).
#include "augment.cuh"

namespace sessd {

constexpr int kAugThreads = 256;
constexpr int kAugMaxGt = 256;     // SESSD_AUGMENT_MAX_GT
constexpr int kAugMaxTry = 128;    // SESSD_AUGMENT_MAX_TRY

// box2d_to_corner_jit of one (x, y, w, l, r): corners_norm (-.5,-.5) (-.5,.5) (.5,.5) (.5,-.5) times (w, l), rotated, plus the centre
__device__ __forceinline__ Quad box_corners(double x, double y, double w, double l, double r) {
    const double s = sin(r), c = cos(r);
    const double nx[4] = {-0.5, -0.5, 0.5, 0.5}, ny[4] = {-0.5, 0.5, 0.5, -0.5};
    Quad q;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const double cx = __dmul_rn(w, nx[k]), cy = __dmul_rn(l, ny[k]);
        q.x[k] = __dadd_rn(__fma_rn(cy, s, __dmul_rn(cx, c)), x);      // rot_mat_T = [[c, -s], [s, c]]
        q.y[k] = __dadd_rn(__fma_rn(cy, c, __dmul_rn(cx, -s)), y);
    }
    return q;
}

__global__ void __launch_bounds__(kAugThreads) box_collision_kernel(const double *__restrict__ boxes, int n, const double *__restrict__ qboxes,
                                                                    int k, uint8_t *__restrict__ out) {
    const long long total = (long long)n * k;
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int i = (int)(t / k), j = (int)(t % k);
        out[t] = quads_collide(load_quad(boxes + 8 * (size_t)i), load_quad(qboxes + 8 * (size_t)j)) ? 1 : 0;
    }
}

__global__ void __launch_bounds__(kAugThreads) noise_per_box_kernel(const float *__restrict__ gt_boxes, const int *__restrict__ num_gt,
                                                                    const uint8_t *__restrict__ valid, int max_gt,
                                                                    const double *__restrict__ loc_noise, const double *__restrict__ rot_noise,
                                                                    int num_try, double ctx, int *__restrict__ selected) {
    __shared__ Quad s_cur[kAugMaxGt];
    __shared__ Quad s_try[kAugMaxTry];
    __shared__ unsigned char s_coll[kAugMaxTry];
    __shared__ int s_first;
    const int b = blockIdx.x;
    const int n = min(max(num_gt[b], 0), max_gt);
    const float *bx = gt_boxes + (size_t)b * max_gt * 7;
    const uint8_t *vb = valid + (size_t)b * max_gt;
    int *sel = selected + (size_t)b * max_gt;
    for (int i = threadIdx.x; i < max_gt; i += blockDim.x) sel[i] = -1;
    // `+ offset`: [0, 0, ctx, ctx, 0] in fp64 (the reference adds zeros when data_aug_with_context <= 0)
    const double add = ctx > 0.0 ? ctx : 0.0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float *p = bx + 7 * i;
        s_cur[i] = box_corners((double)p[0], (double)p[1], __dadd_rn((double)p[3], add), __dadd_rn((double)p[4], add), (double)p[6]);
    }
    __syncthreads();
    for (int i = 0; i < n; ++i) {
        if (!vb[i]) continue;                                 // uniform across the CTA
        const float *p = bx + 7 * i;
        const double cx = (double)p[0], cy = (double)p[1];
        const double *ln = loc_noise + (((size_t)b * max_gt + i) * num_try) * 3;
        const double *rn = rot_noise + ((size_t)b * max_gt + i) * num_try;
        for (int j = threadIdx.x; j < num_try; j += blockDim.x) {
            // current_corners = box_corners[i] - boxes[i, :2]; @ rot(rot_noise); += boxes[i, :2] + loc_noise[:2]
            const double s = sin(rn[j]), c = cos(rn[j]);
            const double tx = __dadd_rn(cx, ln[3 * j]), ty = __dadd_rn(cy, ln[3 * j + 1]);
            Quad q;
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const double ux = __dsub_rn(s_cur[i].x[k], cx), uy = __dsub_rn(s_cur[i].y[k], cy);
                q.x[k] = __dadd_rn(__fma_rn(uy, s, __dmul_rn(ux, c)), tx);
                q.y[k] = __dadd_rn(__fma_rn(uy, c, __dmul_rn(ux, -s)), ty);
            }
            s_try[j] = q;
            s_coll[j] = 0;
        }
        if (threadIdx.x == 0) s_first = num_try;
        __syncthreads();
        for (int t = threadIdx.x; t < num_try * n; t += blockDim.x) {
            const int j = t / n, k = t % n;
            if (k != i && !s_coll[j] && quads_collide(s_try[j], s_cur[k])) s_coll[j] = 1;
        }
        __syncthreads();
        for (int j = threadIdx.x; j < num_try; j += blockDim.x)
            if (!s_coll[j]) atomicMin(&s_first, j);
        __syncthreads();
        const int f = s_first;
        if (f < num_try) {
            if (threadIdx.x == 0) { sel[i] = f; s_cur[i] = s_try[f]; }
        }
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ points and boxes
// Per-box constants of the point pass: the membership frame of the pre-noise box and the selected try's transform (zero when the try
// is -1: the reference still applies -c, R(0), +c, +0 to the points it holds).
struct AugBox {
    MemberFrame<float> m;             // its centre is also the fp32 centre points_transform_ subtracts and adds
    float rc, rs;              // fp32(cos / sin) of the selected try's angle (rot_mat_T of _rotation_matrix_3d_)
    int valid;
    double lx, ly, lz;         // selected try's translation (fp64, added before the fp32 store)
};

// random_flip_v2 -> global_rotation_v3 -> global_scaling_v3 on one point: g = {cos, sin, scale, flip, angle} (fp32, from the host)
__device__ __forceinline__ void global32(float &x, float &y, float &z, const float *g) {
    if (g[3] != 0.f) y = -y;
    rot32(x, y, z, g[0], g[1]);
    x = __fmul_rn(x, g[2]); y = __fmul_rn(y, g[2]); z = __fmul_rn(z, g[2]);
}

__global__ void __launch_bounds__(kAugThreads) augment_points_kernel(
    const float *__restrict__ points, const int *__restrict__ frame_off, const float *__restrict__ gt_boxes, const int *__restrict__ num_gt,
    const uint8_t *__restrict__ valid, int max_gt, const double *__restrict__ loc_noise, const double *__restrict__ rot_noise, int num_try,
    const int *__restrict__ selected, double ctx, const float *__restrict__ global, const int *__restrict__ perm,
    const uint8_t *__restrict__ labeled, float *__restrict__ points_raw, float *__restrict__ points_out) {
    __shared__ AugBox s_box[kAugMaxGt];
    const int b = blockIdx.y;
    const bool lab = labeled == nullptr || labeled[b] != 0;
    const int off = frame_off[b], np = frame_off[b + 1] - off;
    const int n = lab ? min(max(num_gt[b], 0), max_gt) : 0;
    const double add = ctx > 0.0 ? ctx : 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) {
        const size_t bj = (size_t)b * max_gt + j;
        const float *p = gt_boxes + bj * 7;
        AugBox a;
        a.m = member_frame(p, add);
        a.valid = valid[bj];
        const int t = a.valid ? selected[bj] : -1;
        double rot = 0.0;
        a.lx = a.ly = a.lz = 0.0;
        if (t >= 0) {
            const double *l = loc_noise + (bj * num_try + t) * 3;
            a.lx = l[0]; a.ly = l[1]; a.lz = l[2];
            rot = rot_noise[bj * num_try + t];
        }
        a.rc = (float)cos(rot); a.rs = (float)sin(rot);
        s_box[j] = a;
    }
    __syncthreads();
    const float *g = global + 5 * (size_t)b;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x) {
        const int src = perm[off + k];
        if ((unsigned)src >= (unsigned)np) continue;   // not a frame-local permutation: the row is left unwritten (header contract)
        const float4 q = reinterpret_cast<const float4 *>(points)[off + src];
        float x = q.x, y = q.y, z = q.z;
        if (lab) {
            int owner = -1;
            for (int j = 0; j < n; ++j)            // the first VALID box that holds the point (pre-noise boxes)
                if (s_box[j].valid && in_frame(x, y, z, s_box[j].m)) { owner = j; break; }
            if (owner >= 0) {
                const AugBox &a = s_box[owner];
                const float cx = a.m.cx, cy = a.m.cy, cz = a.m.cz;
                x = __fsub_rn(x, cx); y = __fsub_rn(y, cy); z = __fsub_rn(z, cz);
                rot32(x, y, z, a.rc, a.rs);
                x = __fadd_rn(x, cx); y = __fadd_rn(y, cy); z = __fadd_rn(z, cz);
                x = (float)__dadd_rn((double)x, a.lx); y = (float)__dadd_rn((double)y, a.ly); z = (float)__dadd_rn((double)z, a.lz);
            }
            if (points_raw) reinterpret_cast<float4 *>(points_raw)[off + src] = make_float4(x, y, z, q.w);
        }
        global32(x, y, z, g);
        reinterpret_cast<float4 *>(points_out)[off + k] = make_float4(x, y, z, q.w);
    }
}

// points_in_rbbox / points_in_convex_polygon_3d_jit as a mask: d_mask[i, j] = point i lies inside box j (membership frame above)
__global__ void __launch_bounds__(kAugThreads) points_in_boxes_kernel(const float *__restrict__ points, int n, int stride,
                                                                      const float *__restrict__ boxes, int m, double add,
                                                                      uint8_t *__restrict__ mask) {
    for (long long t = blockIdx.x * (long long)blockDim.x + threadIdx.x; t < (long long)n * m; t += (long long)gridDim.x * blockDim.x) {
        const long long i = t / m;
        const int j = (int)(t % m);
        const float *p = points + i * stride;
        mask[t] = in_frame(p[0], p[1], p[2], member_frame(boxes + 7 * (size_t)j, add)) ? 1 : 0;
    }
}

// box3d_transform_ (valid boxes), the valid-box selection and the raw copy, the global stages, then the bookkeeping of
// Voxelization / AssignTarget: the student's boxes lose those with no BEV corner strictly inside range[4] (filter_gt_box_outside_range,
// fp32 corners as the host mirror forms them); both sets keep the target-class boxes, get limit_period(r, 0.5, 2 pi) and are compacted.
// boxes_global (optional): every valid box after the global stages, compacted before the range filter and limit_period (SA-DA's boxes).
__global__ void __launch_bounds__(kAugMaxGt) augment_boxes_kernel(
    const float *__restrict__ gt_boxes, const int *__restrict__ num_gt, const uint8_t *__restrict__ valid, const uint8_t *__restrict__ target,
    int max_gt, const double *__restrict__ loc_noise, const double *__restrict__ rot_noise, int num_try, const int *__restrict__ selected,
    const float *__restrict__ global, float rx0, float ry0, float rx1, float ry1, float *__restrict__ boxes_raw, int *__restrict__ num_raw,
    float *__restrict__ boxes_out, int *__restrict__ num_out, float *__restrict__ boxes_global, int *__restrict__ num_global) {
    __shared__ unsigned char s_keep_raw[kAugMaxGt], s_keep_out[kAugMaxGt], s_keep_glob[kAugMaxGt];
    const int b = blockIdx.x, j = threadIdx.x;
    const int n = min(max(num_gt[b], 0), max_gt);
    const size_t bj = (size_t)b * max_gt + j;
    float v[7] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f}, w[7];
    bool keep_raw = false, keep_out = false;
    const bool keep_glob = j < n && valid[bj];
    if (j < n) {
#pragma unroll
        for (int c = 0; c < 7; ++c) v[c] = gt_boxes[bj * 7 + c];
        if (valid[bj]) {
            box_noise(v, loc_noise, rot_noise, num_try, bj, selected[bj]);
            keep_raw = target == nullptr || target[bj] != 0;
        }
    }
#pragma unroll
    for (int c = 0; c < 7; ++c) w[c] = v[c];
    const float *g = global + 5 * (size_t)b;
    box_global(w, g);
    if (keep_raw) {
        const float s = sinf(w[6]), c = cosf(w[6]);
        const float nx[4] = {-0.5f, -0.5f, 0.5f, 0.5f}, ny[4] = {-0.5f, 0.5f, 0.5f, -0.5f};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float cx = __fmul_rn(w[3], nx[k]), cy = __fmul_rn(w[4], ny[k]);
            const float x = __fadd_rn(__fadd_rn(__fmul_rn(cx, c), __fmul_rn(cy, s)), w[0]);
            const float y = __fadd_rn(__fadd_rn(__fmul_rn(-cx, s), __fmul_rn(cy, c)), w[1]);
            keep_out |= x > rx0 && x < rx1 && y > ry0 && y < ry1;
        }
    }
    s_keep_raw[j] = keep_raw; s_keep_out[j] = keep_out; s_keep_glob[j] = keep_glob;
    __syncthreads();
    int pos_raw = 0, pos_out = 0, pos_glob = 0, tot_raw = 0, tot_out = 0, tot_glob = 0;
    for (int i = 0; i < max_gt; ++i) {
        pos_raw += (i < j) & s_keep_raw[i]; pos_out += (i < j) & s_keep_out[i]; pos_glob += (i < j) & s_keep_glob[i];
        tot_raw += s_keep_raw[i]; tot_out += s_keep_out[i]; tot_glob += s_keep_glob[i];
    }
    if (boxes_global) {                                       // an invalid box's w is its unnoised global box: the padding is zeros
        float *glob = boxes_global + (size_t)b * max_gt * 7;
#pragma unroll
        for (int c = 0; c < 7; ++c) {
            if (keep_glob) glob[pos_glob * 7 + c] = w[c];
            if (j >= tot_glob) glob[j * 7 + c] = 0.f;
        }
        if (j == 0) num_global[b] = tot_glob;
    }
    // limit_period(r, 0.5, 2 pi) in fp32 (the period is a Python float: numpy keeps the fp32 array's type)
    const float kTwoPi = 6.28318548202514648f;
    v[6] = __fsub_rn(v[6], __fmul_rn(floorf(__fadd_rn(__fdiv_rn(v[6], kTwoPi), 0.5f)), kTwoPi));
    w[6] = __fsub_rn(w[6], __fmul_rn(floorf(__fadd_rn(__fdiv_rn(w[6], kTwoPi), 0.5f)), kTwoPi));
    float *raw = boxes_raw + (size_t)b * max_gt * 7, *out = boxes_out + (size_t)b * max_gt * 7;
    if (keep_raw) {
#pragma unroll
        for (int c = 0; c < 7; ++c) raw[pos_raw * 7 + c] = v[c];
    }
    if (keep_out) {
#pragma unroll
        for (int c = 0; c < 7; ++c) out[pos_out * 7 + c] = w[c];
    }
    if (j >= tot_raw) {
#pragma unroll
        for (int c = 0; c < 7; ++c) raw[j * 7 + c] = 0.f;
    }
    if (j >= tot_out) {
#pragma unroll
        for (int c = 0; c < 7; ++c) out[j * 7 + c] = 0.f;
    }
    if (j == 0) { num_raw[b] = tot_raw; num_out[b] = tot_out; }
}

}  // namespace sessd

using namespace sessd;

extern "C" int sessd_box_collision(const double *d_boxes, int n, const double *d_qboxes, int k, uint8_t *d_out, void *stream) {
    if (n < 0 || k < 0 || !d_boxes || !d_qboxes || !d_out) return SESSD_EINVAL;
    if ((long long)n * k == 0) return SESSD_OK;
    const long long total = (long long)n * k;
    const int blocks = (int)std::min<long long>(div_up(total, (long long)kAugThreads), 4096);
    SESSD_LAUNCH(box_collision_kernel, blocks, kAugThreads, 0, (cudaStream_t)stream, d_boxes, n, d_qboxes, k, d_out);
    return last_error();
}

// sample_class_v2's acceptance loop (sample_ops_v2.py:253-276) on the host: candidate i is rejected when its corner set collides with
// any box, any accepted earlier candidate or any later candidate (coll_mat[i].any() over the full row, the diagonal and the rows /
// columns of rejected candidates cleared); a rejected candidate blocks nothing afterwards.  Pairs are evaluated only where needed.
extern "C" int sessd_gtaug_select_host(const double *h_corners, int num_boxes, int num_cand, uint8_t *h_accepted) {
    if (!h_corners || !h_accepted || num_boxes < 0 || num_cand < 0) return SESSD_EINVAL;
    const int n = num_boxes + num_cand;
    int accepted = 0;
    for (int c = 0; c < num_cand; ++c) h_accepted[c] = 1;       // undecided candidates still block (their column is set)
    for (int c = 0; c < num_cand; ++c) {
        const int i = num_boxes + c;
        const Quad qi = load_quad(h_corners + 8 * (size_t)i);
        bool hit = false;
        for (int j = 0; j < n && !hit; ++j) {
            if (j == i || (j >= num_boxes && !h_accepted[j - num_boxes])) continue;
            hit = quads_collide(qi, load_quad(h_corners + 8 * (size_t)j));
        }
        h_accepted[c] = hit ? 0 : 1;
        accepted += hit ? 0 : 1;
    }
    return accepted;
}

extern "C" int sessd_noise_per_box(const float *d_gt_boxes, const int *d_num_gt, const uint8_t *d_valid, int batch, int max_gt,
                                   const double *d_loc_noise, const double *d_rot_noise, int num_try, double context, int *d_selected,
                                   void *stream) {
    if (batch <= 0 || max_gt < 0 || num_try <= 0) return SESSD_EINVAL;
    if (!d_num_gt || !d_selected) return SESSD_EINVAL;
    if (max_gt > 0 && (!d_gt_boxes || !d_valid || !d_loc_noise || !d_rot_noise)) return SESSD_EINVAL;
    if (max_gt > kAugMaxGt || num_try > kAugMaxTry) return SESSD_ECAPACITY;
    if (max_gt == 0) return SESSD_OK;
    SESSD_LAUNCH(noise_per_box_kernel, batch, kAugThreads, 0, (cudaStream_t)stream, d_gt_boxes, d_num_gt, d_valid, max_gt, d_loc_noise,
                 d_rot_noise, num_try, context, d_selected);
    return last_error();
}

extern "C" int sessd_points_in_boxes(const float *d_points, int n, int point_stride, const float *d_boxes, int m, double context,
                                     uint8_t *d_mask, void *stream) {
    if (n < 0 || m < 0 || point_stride < 3 || !d_points || !d_boxes || !d_mask) return SESSD_EINVAL;
    if ((long long)n * m == 0) return SESSD_OK;
    const int blocks = (int)std::min<long long>(div_up((long long)n * m, (long long)kAugThreads), 8192);
    SESSD_LAUNCH(points_in_boxes_kernel, blocks, kAugThreads, 0, (cudaStream_t)stream, d_points, n, point_stride, d_boxes, m,
                 context > 0.0 ? context : 0.0, d_mask);
    return last_error();
}

extern "C" int sessd_augment_points(const float *d_points, const int *d_frame_off, int batch, int max_frame_points, const float *d_gt_boxes,
                                    const int *d_num_gt, const uint8_t *d_valid, int max_gt, const double *d_loc_noise,
                                    const double *d_rot_noise, int num_try, const int *d_selected, double context, const float *d_global,
                                    const int *d_perm, const uint8_t *d_labeled, float *d_points_raw, float *d_points_out, void *stream) {
    if (batch <= 0 || max_frame_points < 0 || max_gt < 0 || num_try <= 0) return SESSD_EINVAL;
    if (!d_points || !d_frame_off || !d_num_gt || !d_global || !d_perm || !d_points_out) return SESSD_EINVAL;
    if ((((uintptr_t)d_points) | ((uintptr_t)d_points_out) | ((uintptr_t)d_points_raw)) & 15) return SESSD_EINVAL;   // float4 rows
    if (max_gt > 0 && (!d_gt_boxes || !d_valid || !d_loc_noise || !d_rot_noise || !d_selected)) return SESSD_EINVAL;
    if (max_gt > kAugMaxGt || num_try > kAugMaxTry) return SESSD_ECAPACITY;
    if (max_frame_points == 0) return SESSD_OK;
    dim3 grid(std::min(div_up(max_frame_points, kAugThreads), 1024), batch);
    SESSD_LAUNCH(augment_points_kernel, grid, kAugThreads, 0, (cudaStream_t)stream, d_points, d_frame_off, d_gt_boxes, d_num_gt, d_valid,
                 max_gt, d_loc_noise, d_rot_noise, num_try, d_selected, context, d_global, d_perm, d_labeled, d_points_raw, d_points_out);
    return last_error();
}

extern "C" int sessd_augment_boxes(const float *d_gt_boxes, const int *d_num_gt, const uint8_t *d_valid, const uint8_t *d_target, int batch,
                                   int max_gt, const double *d_loc_noise, const double *d_rot_noise, int num_try, const int *d_selected,
                                   const float *d_global, const float *range_bev, float *d_boxes_raw, int *d_num_raw, float *d_boxes_out,
                                   int *d_num_out, float *d_boxes_global, int *d_num_global, void *stream) {
    if (batch <= 0 || max_gt < 0 || num_try <= 0) return SESSD_EINVAL;
    if (!d_num_gt || !d_global || !range_bev || !d_num_raw || !d_num_out) return SESSD_EINVAL;
    if (d_boxes_global && !d_num_global) return SESSD_EINVAL;
    if (max_gt > 0 && (!d_gt_boxes || !d_valid || !d_loc_noise || !d_rot_noise || !d_selected || !d_boxes_raw || !d_boxes_out ||
                       (d_num_global && !d_boxes_global)))
        return SESSD_EINVAL;
    if (max_gt > kAugMaxGt || num_try > kAugMaxTry) return SESSD_ECAPACITY;
    cudaStream_t st = (cudaStream_t)stream;
    if (max_gt == 0) {
        SESSD_CUDA_TRY(cudaMemsetAsync(d_num_raw, 0, sizeof(int) * batch, st));
        SESSD_CUDA_TRY(cudaMemsetAsync(d_num_out, 0, sizeof(int) * batch, st));
        if (d_num_global) SESSD_CUDA_TRY(cudaMemsetAsync(d_num_global, 0, sizeof(int) * batch, st));
        return SESSD_OK;
    }
    SESSD_LAUNCH(augment_boxes_kernel, batch, max_gt, 0, st, d_gt_boxes, d_num_gt, d_valid, d_target, max_gt, d_loc_noise, d_rot_noise,
                 num_try, d_selected, d_global, range_bev[0], range_bev[1], range_bev[2], range_bev[3], d_boxes_raw, d_num_raw, d_boxes_out,
                 d_num_out, d_boxes_global, d_num_global);
    return last_error();
}
