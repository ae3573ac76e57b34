// kitti_prep.cu -- KITTI data preparation on the GPU: the image-frustum point clouds (velodyne_reduced), the point counts of the label boxes
// (num_points_in_gt) and the GT database's object points.
//
// Replaces the numba membership of det3d/core/bbox/geometry.py:_points_in_convex_polygon_3d_jit as the reference's data preparation uses
// it: remove_outside_points (box_np_ops.py:981-992) inside _create_reduced_point_cloud and _calculate_num_points_in_gt
// (kitti_common.py:62-92, 154-185), and points_in_rbbox (box_np_ops.py:1152-1157) inside _calculate_num_points_in_gt and
// create_groundtruth_database (create_gt_database.py:86-95).  Every plane is computed on the host (sessd_b200/kitti_prep.py, the
// arithmetic of surface_equ_3d_jitv2); the device only evaluates the sign tests and moves points.
//
// Precision: a point is inside a polyhedron when (((x*a) + (y*b)) + (z*c)) + d < 0 for each of its six planes, x y z the fp32 coordinates
// widened to fp64 and every operation rounded on its own (the __d*_rn intrinsics; this file is also compiled with -fmad=false).  A sign
// >= 0 is outside, so a point exactly on a plane is outside; a NaN sign is not >= 0 and keeps the point, as in the reference.  The
// database rows are fp32(double(p) - centre) for x y z: the reference's `gt_points[:, :3] -= gt_boxes[i, :3]` on an fp32 array.
//
// Launch shape: frustum compaction is flag (one thread per point) -> device_scan (common.cuh) -> offsets -> scatter, as the GT-AUG
// removal; the box count and the object gather run one CTA per box over its frame's points in 256-point tiles (the gather with a
// block-level ordered compaction per tile), so no CTA holds a whole frame and the output order is the frame order.
#include "common.cuh"

namespace sessd {

constexpr int kPrepThreads = 256;

// the sign test of one convex polyhedron of six planes [6][4] (a, b, c, d); the planes stay in fp64 registers of the caller
__device__ __forceinline__ bool prep_inside(float px, float py, float pz, const double *__restrict__ pl) {
    const double x = (double)px, y = (double)py, z = (double)pz;
#pragma unroll
    for (int k = 0; k < 6; ++k) {
        const double *q = pl + 4 * k;
        const double s = __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(x, q[0]), __dmul_rn(y, q[1])), __dmul_rn(z, q[2])), q[3]);
        if (s >= 0.0) return false;
    }
    return true;
}

struct CompactWs {
    int *rank;       // [num_points + 1]: kept points before each point, then their total
    int *scan;       // device_scan scratch
    uint8_t *keep;   // [num_points]
};

static size_t compact_layout(int num_points, char *base, CompactWs *ws) {
    size_t off = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + off : nullptr; off += (bytes + 15) & ~(size_t)15; return p; };
    CompactWs w;
    w.rank = (int *)take(sizeof(int) * ((size_t)num_points + 1));
    w.scan = (int *)take(scan_scratch_bytes(num_points));
    w.keep = (uint8_t *)take((size_t)num_points);
    if (ws) *ws = w;
    return off;
}

__global__ void __launch_bounds__(kPrepThreads) frustum_flag_kernel(const float *__restrict__ points, int num_points,
                                                                     const int *__restrict__ frame_off, int batch,
                                                                     const double *__restrict__ planes, CompactWs ws) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_points) return;
    const int b = find_frame(frame_off, batch, i);
    const float4 p = reinterpret_cast<const float4 *>(points)[i];
    // a row outside every frame (before frame_off[0] or from frame_off[batch] on) is dropped
    const bool owned = i >= frame_off[0] && i < frame_off[batch];
    ws.keep[i] = owned && prep_inside(p.x, p.y, p.z, planes + 24 * (size_t)b);
}

struct PrepKeepFlag {
    const uint8_t *keep;
    __device__ __forceinline__ int operator()(long long i) const { return keep[i]; }
};
struct PrepRank {
    int *rank;
    __device__ __forceinline__ void operator()(long long i, int ex, int) const { rank[i] = ex; }
};

// new frame offsets: the kept points before each frame boundary
__global__ void __launch_bounds__(kPrepThreads) frustum_offsets_kernel(int num_points, const int *__restrict__ frame_off, int batch,
                                                                        CompactWs ws, int *__restrict__ frame_off_out) {
    for (int b = blockIdx.x * blockDim.x + threadIdx.x; b <= batch; b += gridDim.x * blockDim.x)
        frame_off_out[b] = ws.rank[min(max(frame_off[b], 0), num_points)];
}

__global__ void __launch_bounds__(kPrepThreads) frustum_scatter_kernel(const float *__restrict__ points, int num_points, CompactWs ws,
                                                                        float *__restrict__ out, int capacity) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_points || !ws.keep[i]) return;
    const int row = ws.rank[i];
    if (row < capacity) reinterpret_cast<float4 *>(out)[row] = reinterpret_cast<const float4 *>(points)[i];
}

// the point range [lo, hi) of box k's frame, clamped to [0, num_points)
__device__ __forceinline__ void box_frame_range(const int *__restrict__ box_off, const int *__restrict__ frame_off, int batch, int num_points,
                                                int k, int *lo, int *hi) {
    const int b = find_frame(box_off, batch, k);
    *lo = min(max(frame_off[b], 0), num_points);
    *hi = min(max(frame_off[b + 1], *lo), num_points);
}

// one CTA per box: the number of its frame's points inside it
__global__ void __launch_bounds__(kPrepThreads) box_count_kernel(const float *__restrict__ points, int num_points,
                                                                  const int *__restrict__ frame_off, int batch, const double *__restrict__ planes,
                                                                  const int *__restrict__ box_off, int *__restrict__ counts) {
    __shared__ double s_pl[24];
    __shared__ int s_scan[40];
    const int k = blockIdx.x;
    if (threadIdx.x < 24) s_pl[threadIdx.x] = planes[24 * (size_t)k + threadIdx.x];
    int lo, hi;
    box_frame_range(box_off, frame_off, batch, num_points, k, &lo, &hi);
    __syncthreads();
    int n = 0;
    for (int i = lo + threadIdx.x; i < hi; i += kPrepThreads) {
        const float4 p = reinterpret_cast<const float4 *>(points)[i];
        n += prep_inside(p.x, p.y, p.z, s_pl);
    }
    int tot;
    block_excl_scan(n, s_scan, &tot);
    if (threadIdx.x == 0) counts[k] = tot;
}

struct GatherWs {
    int *scan;   // device_scan scratch
};

static size_t gather_layout(int num_boxes, char *base, GatherWs *ws) {
    size_t off = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + off : nullptr; off += (bytes + 15) & ~(size_t)15; return p; };
    GatherWs w;
    w.scan = (int *)take(scan_scratch_bytes(num_boxes));
    if (ws) *ws = w;
    return off;
}

struct CountLoad {
    const int *counts;
    __device__ __forceinline__ int operator()(long long i) const { return max(counts[i], 0); }
};
struct OffsetStore {
    int *off;
    __device__ __forceinline__ void operator()(long long i, int ex, int) const { off[i] = ex; }
};

// one CTA per box: its frame's points inside it, in frame order, relative to the fp64 centre, from row obj_off[k] on (never past
// obj_off[k + 1] nor the capacity)
__global__ void __launch_bounds__(kPrepThreads) box_gather_kernel(const float *__restrict__ points, int num_points,
                                                                   const int *__restrict__ frame_off, int batch, const double *__restrict__ planes,
                                                                   const double *__restrict__ centres, const int *__restrict__ box_off,
                                                                   const int *__restrict__ obj_off, float *__restrict__ out, int capacity) {
    __shared__ double s_pl[24];
    __shared__ int s_scan[40];
    const int k = blockIdx.x;
    if (threadIdx.x < 24) s_pl[threadIdx.x] = planes[24 * (size_t)k + threadIdx.x];
    int lo, hi;
    box_frame_range(box_off, frame_off, batch, num_points, k, &lo, &hi);
    const double cx = centres[3 * (size_t)k], cy = centres[3 * (size_t)k + 1], cz = centres[3 * (size_t)k + 2];
    const int r0 = obj_off[k], r1 = min(obj_off[k + 1], capacity);
    __syncthreads();
    int carry = 0;
    for (int base = lo; base < hi; base += kPrepThreads) {   // uniform trip count across the CTA: block_excl_scan syncs
        const int i = base + threadIdx.x;
        float4 p = make_float4(0.f, 0.f, 0.f, 0.f);
        bool in = false;
        if (i < hi) {
            p = reinterpret_cast<const float4 *>(points)[i];
            in = prep_inside(p.x, p.y, p.z, s_pl);
        }
        int tot;
        const int ex = block_excl_scan(in ? 1 : 0, s_scan, &tot);
        const int row = r0 + carry + ex;
        if (in && row < r1)
            reinterpret_cast<float4 *>(out)[row] =
                make_float4((float)__dsub_rn((double)p.x, cx), (float)__dsub_rn((double)p.y, cy), (float)__dsub_rn((double)p.z, cz), p.w);
        carry += tot;
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" size_t sessd_prep_frustum_compact_workspace_bytes(int num_points) {
    if (num_points < 0) return 0;
    return compact_layout(num_points, nullptr, nullptr);
}

extern "C" int sessd_prep_frustum_compact(const float *d_points, const int *d_frame_off, int batch, int num_points, const double *d_planes,
                                          void *d_workspace, size_t workspace_bytes, float *d_points_out, int capacity, int *d_frame_off_out,
                                          void *stream) {
    if (batch <= 0 || num_points < 0 || capacity < 0) return SESSD_EINVAL;
    if (!d_frame_off || !d_planes || !d_workspace || !d_frame_off_out) return SESSD_EINVAL;
    if (num_points > 0 && (!d_points || !d_points_out)) return SESSD_EINVAL;
    if ((((uintptr_t)d_points) | ((uintptr_t)d_points_out)) & 15) return SESSD_EINVAL;   // float4 rows
    if (workspace_bytes < compact_layout(num_points, nullptr, nullptr)) return SESSD_EWORKSPACE;
    if (capacity < num_points) return SESSD_ECAPACITY;
    CompactWs ws;
    compact_layout(num_points, (char *)d_workspace, &ws);
    cudaStream_t st = (cudaStream_t)stream;
    const int blocks = div_up(num_points, kPrepThreads);
    if (blocks > 0)
        SESSD_LAUNCH(frustum_flag_kernel, blocks, kPrepThreads, 0, st, d_points, num_points, d_frame_off, batch, d_planes, ws);
    device_scan(PrepKeepFlag{ws.keep}, PrepRank{ws.rank}, nullptr, num_points, num_points, ws.scan, ws.rank + num_points, st);
    SESSD_LAUNCH(frustum_offsets_kernel, div_up(batch + 1, kPrepThreads), kPrepThreads, 0, st, num_points, d_frame_off, batch, ws,
                 d_frame_off_out);
    if (blocks > 0) SESSD_LAUNCH(frustum_scatter_kernel, blocks, kPrepThreads, 0, st, d_points, num_points, ws, d_points_out, capacity);
    return last_error();
}

extern "C" int sessd_prep_box_count(const float *d_points, const int *d_frame_off, int batch, int num_points, const double *d_box_planes,
                                    const int *d_box_off, int num_boxes, int *d_counts, void *stream) {
    if (batch <= 0 || num_points < 0 || num_boxes < 0) return SESSD_EINVAL;
    if (!d_frame_off || !d_box_off) return SESSD_EINVAL;
    if (num_points > 0 && !d_points) return SESSD_EINVAL;
    if (num_boxes > 0 && (!d_box_planes || !d_counts)) return SESSD_EINVAL;
    if (((uintptr_t)d_points) & 15) return SESSD_EINVAL;
    if (num_boxes > 0)
        SESSD_LAUNCH(box_count_kernel, num_boxes, kPrepThreads, 0, (cudaStream_t)stream, d_points, num_points, d_frame_off, batch, d_box_planes,
                     d_box_off, d_counts);
    return last_error();
}

extern "C" size_t sessd_prep_box_gather_workspace_bytes(int num_boxes) {
    if (num_boxes < 0) return 0;
    return gather_layout(num_boxes, nullptr, nullptr);
}

extern "C" int sessd_prep_box_gather(const float *d_points, const int *d_frame_off, int batch, int num_points, const double *d_box_planes,
                                     const double *d_centres, const int *d_box_off, int num_boxes, const int *d_counts, int num_rows,
                                     void *d_workspace, size_t workspace_bytes, float *d_rows_out, int capacity, int *d_obj_off, void *stream) {
    if (batch <= 0 || num_points < 0 || num_boxes < 0 || num_rows < 0 || capacity < 0) return SESSD_EINVAL;
    if (!d_frame_off || !d_box_off || !d_obj_off || !d_workspace) return SESSD_EINVAL;
    if (num_points > 0 && !d_points) return SESSD_EINVAL;
    if (num_boxes > 0 && (!d_box_planes || !d_centres || !d_counts)) return SESSD_EINVAL;
    if (num_rows > 0 && !d_rows_out) return SESSD_EINVAL;
    if ((((uintptr_t)d_points) | ((uintptr_t)d_rows_out)) & 15) return SESSD_EINVAL;
    if (workspace_bytes < gather_layout(num_boxes, nullptr, nullptr)) return SESSD_EWORKSPACE;
    if (capacity < num_rows) return SESSD_ECAPACITY;
    GatherWs ws;
    gather_layout(num_boxes, (char *)d_workspace, &ws);
    cudaStream_t st = (cudaStream_t)stream;
    device_scan(CountLoad{d_counts}, OffsetStore{d_obj_off}, nullptr, num_boxes, num_boxes, ws.scan, d_obj_off + num_boxes, st);
    if (num_boxes > 0)
        SESSD_LAUNCH(box_gather_kernel, num_boxes, kPrepThreads, 0, st, d_points, num_points, d_frame_off, batch, d_box_planes, d_centres,
                     d_box_off, d_obj_off, d_rows_out, capacity);
    return last_error();
}
