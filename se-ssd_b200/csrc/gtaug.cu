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
// Launch shape: the batch's scene points are cut into tiles of kTile rows.  keep_kernel tests each point against its frame's pasted
// boxes and counts the survivors per tile; plan_kernel (one CTA) scans the tile counts, finds each frame's survivor prefix, the new
// frame offsets and each object's first output row; scatter_kernel writes the survivors in order (a block scan per 256-row round);
// gather_kernel writes one object per CTA.  No CTA holds a whole frame.
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "augment.cuh"

namespace sessd {

constexpr int kPasteThreads = 256;
constexpr int kPasteRounds = 8;
constexpr int kTile = kPasteThreads * kPasteRounds;    // scene rows per tile
constexpr int kPlanThreads = 1024;

struct PasteWs {
    uint8_t *keep;                 // [num_points]
    int *tile;                     // [tiles + 1]: survivors per tile, then their exclusive prefix
    int *surv;                     // [batch + 1]: survivors before frame_off[b] (global prefix)
    int *paste;                    // [batch]: pasted rows per frame
    int *obj_row;                  // [num_obj]: first output row of each object (-1: bad id)
    MemberFrame<double> *mf;       // [num_obj]
};

static size_t align16(size_t v) { return (v + 15) & ~(size_t)15; }

static size_t paste_layout(int batch, int num_points, int num_obj, char *base, PasteWs *ws) {
    const size_t tiles = (size_t)div_up(num_points, kTile) + 1;
    size_t off = 0;
    auto take = [&](size_t bytes) { char *p = base ? base + off : nullptr; off += align16(bytes); return p; };
    PasteWs w;
    w.mf = (MemberFrame<double> *)take(sizeof(MemberFrame<double>) * (size_t)num_obj);
    w.keep = (uint8_t *)take((size_t)num_points);
    w.tile = (int *)take(sizeof(int) * tiles);
    w.surv = (int *)take(sizeof(int) * ((size_t)batch + 1));
    w.paste = (int *)take(sizeof(int) * (size_t)batch);
    w.obj_row = (int *)take(sizeof(int) * (size_t)num_obj);
    if (ws) *ws = w;
    return off;
}

__device__ __forceinline__ int frame_of(const int *frame_off, int batch, int i) {   // largest b with frame_off[b] <= i
    int lo = 0, hi = batch - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (frame_off[mid] <= i) lo = mid; else hi = mid - 1;
    }
    return lo;
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

__global__ void __launch_bounds__(kPasteThreads) keep_kernel(const float *__restrict__ points, int num_points, const int *__restrict__ frame_off,
                                                             int batch, const int *__restrict__ obj_off, PasteWs ws) {
    using Reduce = cub::BlockReduce<int, kPasteThreads>;
    __shared__ typename Reduce::TempStorage s_red;
    const int base = blockIdx.x * kTile;
    int kept = 0;
#pragma unroll 1
    for (int r = 0; r < kPasteRounds; ++r) {
        const int i = base + r * kPasteThreads + threadIdx.x;
        if (i >= num_points) break;
        const int b = frame_of(frame_off, batch, i);
        const float4 p = reinterpret_cast<const float4 *>(points)[i];
        bool keep = true;
        for (int k = obj_off[b], e = obj_off[b + 1]; k < e && keep; ++k) keep = !in_frame(p.x, p.y, p.z, ws.mf[k]);
        ws.keep[i] = keep;
        kept += keep;
    }
    const int total = Reduce(s_red).Sum(kept);
    if (threadIdx.x == 0) ws.tile[blockIdx.x] = total;
}

// exclusive block-wide scan of a[0, n) in place (one CTA), returns the total
__device__ int block_scan_inplace(int *a, int n) {
    using Scan = cub::BlockScan<int, kPlanThreads>;
    __shared__ typename Scan::TempStorage s_scan;
    __shared__ int s_carry;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int c = 0; c < n; c += kPlanThreads) {
        const int i = c + threadIdx.x;
        const int v = i < n ? a[i] : 0;
        int x, tot;
        Scan(s_scan).ExclusiveSum(v, x, tot);
        const int carry = s_carry;
        if (i < n) a[i] = carry + x;
        __syncthreads();
        if (threadIdx.x == 0) s_carry = carry + tot;
        __syncthreads();
    }
    return s_carry;
}

__global__ void __launch_bounds__(kPlanThreads) plan_kernel(int num_points, const int *__restrict__ frame_off, int batch,
                                                            const int *__restrict__ obj_off, const int *__restrict__ obj_ids, int db_size,
                                                            const int *__restrict__ db_count, int tiles, PasteWs ws,
                                                            int *__restrict__ frame_off_out) {
    if (threadIdx.x == 0) ws.tile[tiles] = 0;                  // the end sentinel: the prefix at tiles is the survivor total
    __syncthreads();
    block_scan_inplace(ws.tile, tiles + 1);
    // survivors before each frame boundary: the tile prefix plus the tile's own flags up to the boundary (one warp per boundary)
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int b = warp; b <= batch; b += kPlanThreads / 32) {
        const int i = min(max(frame_off[b], 0), num_points);
        const int t = i / kTile;
        int s = 0;
        for (int j = t * kTile + lane; j < i; j += 32) s += ws.keep[j];
#pragma unroll
        for (int o = 16; o; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
        if (lane == 0) ws.surv[b] = ws.tile[t] + s;
    }
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
    // new frame offsets: [pasted rows, surviving rows] per frame
    for (int b = threadIdx.x; b < batch; b += kPlanThreads) frame_off_out[b] = ws.paste[b] + ws.surv[b + 1] - ws.surv[b];
    __syncthreads();
    const int total = block_scan_inplace(frame_off_out, batch);
    if (threadIdx.x == 0) frame_off_out[batch] = total;
}

__global__ void __launch_bounds__(kPasteThreads) scatter_kernel(const float *__restrict__ points, int num_points, const int *__restrict__ frame_off,
                                                                int batch, PasteWs ws, const int *__restrict__ frame_off_out,
                                                                float *__restrict__ out, int capacity) {
    using Scan = cub::BlockScan<int, kPasteThreads>;
    __shared__ typename Scan::TempStorage s_scan;
    const int base = blockIdx.x * kTile;
    int carry = ws.tile[blockIdx.x];
#pragma unroll 1
    for (int r = 0; r < kPasteRounds; ++r) {
        const int i = base + r * kPasteThreads + threadIdx.x;
        const int keep = i < num_points ? ws.keep[i] : 0;
        int pos, tot;
        Scan(s_scan).ExclusiveSum(keep, pos, tot);
        if (keep) {
            const int b = frame_of(frame_off, batch, i);
            const int row = frame_off_out[b] + ws.paste[b] + (carry + pos - ws.surv[b]);
            if (row < capacity) reinterpret_cast<float4 *>(out)[row] = reinterpret_cast<const float4 *>(points)[i];
        }
        carry += tot;
        __syncthreads();
    }
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
    const int b = frame_of(obj_off, batch, k);
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
    const int tiles = div_up(num_points, kTile);
    if (num_objects > 0)
        SESSD_LAUNCH(frames_kernel, div_up(num_objects, kPasteThreads), kPasteThreads, 0, st, d_obj_ids, num_objects, d_db_boxes, db_size, ws);
    if (tiles > 0) SESSD_LAUNCH(keep_kernel, tiles, kPasteThreads, 0, st, d_points, num_points, d_frame_off, batch, d_obj_off, ws);
    SESSD_LAUNCH(plan_kernel, 1, kPlanThreads, 0, st, num_points, d_frame_off, batch, d_obj_off, d_obj_ids, db_size, d_db_count, tiles, ws,
                 d_frame_off_out);
    if (tiles > 0)
        SESSD_LAUNCH(scatter_kernel, tiles, kPasteThreads, 0, st, d_points, num_points, d_frame_off, batch, ws, d_frame_off_out, d_points_out,
                     capacity);
    if (num_objects > 0)
        SESSD_LAUNCH(gather_kernel, num_objects, kPasteThreads, 0, st, d_obj_off, batch, d_obj_ids, d_db_points, d_db_off, d_db_count,
                     d_db_boxes, ws, d_frame_off_out, d_points_out, capacity);
    return last_error();
}
