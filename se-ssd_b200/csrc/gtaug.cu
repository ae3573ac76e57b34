// gtaug.cu -- GT-database sampling (GT-AUG) on the GPU: the accepted database objects are pasted into a batch of frames, and the scene
// points inside the pasted boxes are removed.
//
// Replaces the point half of DataBaseSamplerV2.sample_all (det3d/core/sampler/sample_ops_v2.py:133-150, `np.fromfile` +
// `s_points[:, :3] += info["box3d_lidar"][:3]` per object) and Preprocess.__call__'s paste (det3d/datasets/pipelines/preprocess.py:96-110:
// remove_points_after_sample through points_in_rbbox, then `concatenate([sampled_points, points])`).  Which objects a frame takes is
// decided on the host (sessd_gtaug_select_host in augment.cu; the draws and the sampler's resets depend on every earlier frame).
//
// Precision (traced through the reference): box3d_lidar is float64 -- box_camera_to_lidar (box_np_ops.py:937-970) multiplies the fp32
// label by an fp64 matrix and concatenates, and create_gt_database.py:60-110 stores those rows.  The database file holds fp32
// `points - box3d_lidar[:3]`; sample_all adds the fp64 centre in place into the fp32 array, so each coordinate is
// fp32(double(rel) + centre): one fp64 add, rounded once (this file is compiled with -fmad=false).  points_in_rbbox runs on the fp64
// sampled boxes: the membership frame of augment.cuh with an fp64 centre.
//
// Launch shape: removal_kernel tests each scene point against its frame's pasted boxes and flags the survivors (one thread per point);
// device_scan (common.cuh) turns the flags into each point's survivor rank; plan_kernel (one CTA) reads each frame's survivor prefix off
// the ranks and finds the new frame offsets and each object's first output row; scatter_kernel copies each survivor to its row (one
// thread per point); gather_kernel writes one object per CTA.  No CTA holds a whole frame.
#include "augment.cuh"

namespace sessd {

constexpr int kPasteThreads = 256;
constexpr int kPlanThreads = 1024;

struct PasteWs {
    MemberFrame<double> *mf;       // [num_obj]
    int *rank;                     // [num_points + 1]: survivors before each point, then their total
    int *scan;                     // device_scan scratch
    int *surv;                     // [batch + 1]: survivors before frame_off[b] (global prefix)
    int *paste;                    // [batch]: pasted rows per frame
    int *obj_row;                  // [num_obj]: first output row of each object (-1: bad id)
    uint8_t *keep;                 // [num_points]
};

// the arrays in order of decreasing alignment, so each one starts aligned without padding
static size_t paste_layout(int batch, int num_points, int num_obj, char *base, PasteWs *ws) {
    size_t off = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + off : nullptr; off += bytes; return p; };
    PasteWs w;
    w.mf = (MemberFrame<double> *)take(sizeof(MemberFrame<double>) * (size_t)num_obj);
    w.rank = (int *)take(sizeof(int) * ((size_t)num_points + 1));
    w.scan = (int *)take(scan_scratch_bytes(num_points));
    w.surv = (int *)take(sizeof(int) * ((size_t)batch + 1));
    w.paste = (int *)take(sizeof(int) * (size_t)batch);
    w.obj_row = (int *)take(sizeof(int) * (size_t)num_obj);
    w.keep = (uint8_t *)take((size_t)num_points);
    if (ws) *ws = w;
    return off;
}

// the membership frame of each accepted object's fp64 box; a bad id gets an empty frame (it removes nothing)
__global__ void __launch_bounds__(kPasteThreads) frames_kernel(const int *__restrict__ obj_ids, int num_obj, const double *__restrict__ db_boxes,
                                                               int db_size, PasteWs ws) {
    const int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k >= num_obj) return;
    const int id = obj_ids[k];
    if ((unsigned)id < (unsigned)db_size) {
        ws.mf[k] = member_frame(db_boxes + 7 * (size_t)id, 0.0);
    } else {
        MemberFrame<double> f = {0.0, 0.0, 0.0, 1.0, 0.0, -1.0, -1.0, -1.0};
        ws.mf[k] = f;
    }
}

__global__ void __launch_bounds__(kPasteThreads) removal_kernel(const float *__restrict__ points, int num_points,
                                                                const int *__restrict__ frame_off, int batch, const int *__restrict__ obj_off,
                                                                PasteWs ws) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_points) return;
    const int b = find_frame(frame_off, batch, i);
    const float4 p = reinterpret_cast<const float4 *>(points)[i];
    bool keep = true;
    for (int k = obj_off[b], e = obj_off[b + 1]; k < e && keep; ++k) keep = !in_frame(p.x, p.y, p.z, ws.mf[k]);
    ws.keep[i] = keep;
}

struct KeepFlag {
    const uint8_t *keep;
    __device__ __forceinline__ int operator()(long long i) const { return keep[i]; }
};
struct SurvivorRank {
    int *rank;
    __device__ __forceinline__ void operator()(long long i, int ex, int) const { rank[i] = ex; }
};

__global__ void __launch_bounds__(kPlanThreads) plan_kernel(int num_points, const int *__restrict__ frame_off, int batch,
                                                            const int *__restrict__ obj_off, const int *__restrict__ obj_ids, int db_size,
                                                            const int *__restrict__ db_count, PasteWs ws, int *__restrict__ frame_off_out) {
    __shared__ int s_scan[40];
    // survivors before each frame boundary (rank[num_points] is the total)
    for (int b = threadIdx.x; b <= batch; b += kPlanThreads) ws.surv[b] = ws.rank[min(max(frame_off[b], 0), num_points)];
    // rows per object (0 for a bad id), their first row inside the frame's pasted block, and the pasted rows per frame
    for (int b = threadIdx.x; b < batch; b += kPlanThreads) {
        int rows = 0;
        for (int k = obj_off[b], e = obj_off[b + 1]; k < e; ++k) {
            const int id = obj_ids[k];
            const bool ok = (unsigned)id < (unsigned)db_size;
            ws.obj_row[k] = ok ? rows : -1;
            rows += ok ? db_count[id] : 0;
        }
        ws.paste[b] = rows;
    }
    __syncthreads();
    // new frame offsets: the exclusive scan of [pasted rows, surviving rows] per frame
    int carry = 0;
    for (int c = 0; c < batch; c += kPlanThreads) {
        const int b = c + threadIdx.x;
        const int rows = b < batch ? ws.paste[b] + ws.surv[b + 1] - ws.surv[b] : 0;
        int tot;
        const int ex = block_excl_scan(rows, s_scan, &tot);
        if (b < batch) frame_off_out[b] = carry + ex;
        carry += tot;
    }
    if (threadIdx.x == 0) frame_off_out[batch] = carry;
}

// each survivor to its frame's block: after the frame's pasted rows, in order
__global__ void __launch_bounds__(kPasteThreads) scatter_kernel(const float *__restrict__ points, int num_points, const int *__restrict__ frame_off,
                                                                int batch, PasteWs ws, const int *__restrict__ frame_off_out,
                                                                float *__restrict__ out, int capacity) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= num_points || !ws.keep[i]) return;
    const int b = find_frame(frame_off, batch, i);
    const int row = frame_off_out[b] + ws.paste[b] + (ws.rank[i] - ws.surv[b]);
    if (row < capacity) reinterpret_cast<float4 *>(out)[row] = reinterpret_cast<const float4 *>(points)[i];
}

// one CTA per accepted object: fp32(double(rel) + centre) for x y z, the intensity copied
__global__ void __launch_bounds__(kPasteThreads) gather_kernel(const int *__restrict__ obj_off, int batch, const int *__restrict__ obj_ids,
                                                               const float *__restrict__ db_points, const int *__restrict__ db_off,
                                                               const int *__restrict__ db_count, const double *__restrict__ db_boxes,
                                                               PasteWs ws, const int *__restrict__ frame_off_out, float *__restrict__ out,
                                                               int capacity) {
    const int k = blockIdx.x;
    const int r0 = ws.obj_row[k];
    if (r0 < 0) return;                                         // bad id: no rows
    const int id = obj_ids[k];
    // the object's frame: obj_off is non-decreasing, the frame is the last b with obj_off[b] <= k
    const int b = find_frame(obj_off, batch, k);
    const double *c = db_boxes + 7 * (size_t)id;
    const double cx = c[0], cy = c[1], cz = c[2];
    const int n = db_count[id], src = db_off[id], dst = frame_off_out[b] + r0;
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const float4 q = reinterpret_cast<const float4 *>(db_points)[src + i];
        const float4 v = make_float4((float)((double)q.x + cx), (float)((double)q.y + cy), (float)((double)q.z + cz), q.w);
        if (dst + i < capacity) reinterpret_cast<float4 *>(out)[dst + i] = v;
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" size_t sessd_gtaug_paste_workspace_bytes(int batch, int num_points, int num_objects) {
    if (batch <= 0 || num_points < 0 || num_objects < 0) return 0;
    return paste_layout(batch, num_points, num_objects, nullptr, nullptr);
}

extern "C" int sessd_gtaug_paste(const float *d_points, const int *d_frame_off, int batch, int num_points, const int *d_obj_off,
                                 const int *d_obj_ids, int num_objects, int max_paste_points, const float *d_db_points,
                                 const int *d_db_off, const int *d_db_count, const double *d_db_boxes, int db_size, void *d_workspace,
                                 size_t workspace_bytes, float *d_points_out, int capacity, int *d_frame_off_out, void *stream) {
    if (batch <= 0 || num_points < 0 || num_objects < 0 || max_paste_points < 0 || db_size < 0 || capacity < 0) return SESSD_EINVAL;
    if (!d_frame_off || !d_obj_off || !d_frame_off_out || !d_workspace || !d_points_out) return SESSD_EINVAL;
    if (num_points > 0 && !d_points) return SESSD_EINVAL;
    if (num_objects > 0 && (!d_obj_ids || !d_db_points || !d_db_off || !d_db_count || !d_db_boxes)) return SESSD_EINVAL;
    if ((((uintptr_t)d_points) | ((uintptr_t)d_points_out) | ((uintptr_t)d_db_points)) & 15) return SESSD_EINVAL;   // float4 rows
    if (workspace_bytes < paste_layout(batch, num_points, num_objects, nullptr, nullptr)) return SESSD_EWORKSPACE;
    if ((long long)capacity < (long long)num_points + max_paste_points) return SESSD_ECAPACITY;
    PasteWs ws;
    paste_layout(batch, num_points, num_objects, (char *)d_workspace, &ws);
    cudaStream_t st = (cudaStream_t)stream;
    const int blocks = div_up(num_points, kPasteThreads);
    if (num_objects > 0)
        SESSD_LAUNCH(frames_kernel, div_up(num_objects, kPasteThreads), kPasteThreads, 0, st, d_obj_ids, num_objects, d_db_boxes, db_size, ws);
    if (blocks > 0) SESSD_LAUNCH(removal_kernel, blocks, kPasteThreads, 0, st, d_points, num_points, d_frame_off, batch, d_obj_off, ws);
    device_scan(KeepFlag{ws.keep}, SurvivorRank{ws.rank}, nullptr, num_points, num_points, ws.scan, ws.rank + num_points, st);
    SESSD_LAUNCH(plan_kernel, 1, kPlanThreads, 0, st, num_points, d_frame_off, batch, d_obj_off, d_obj_ids, db_size, d_db_count, ws,
                 d_frame_off_out);
    if (blocks > 0)
        SESSD_LAUNCH(scatter_kernel, blocks, kPasteThreads, 0, st, d_points, num_points, d_frame_off, batch, ws, d_frame_off_out, d_points_out,
                     capacity);
    if (num_objects > 0)
        SESSD_LAUNCH(gather_kernel, num_objects, kPasteThreads, 0, st, d_obj_off, batch, d_obj_ids, d_db_points, d_db_off, d_db_count,
                     d_db_boxes, ws, d_frame_off_out, d_points_out, capacity);
    return last_error();
}
