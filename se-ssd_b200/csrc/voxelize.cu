// voxelize.cu -- order-preserving hash-grid voxeliser with fused per-voxel mean (sm_90a).
//
// Replaces the sequential numba loop of det3d/ops/point_cloud/point_cloud_ops_v2.py:9-62 (called through
// det3d/core/input/voxel_generator.py:24-32) and VoxelFeatureExtractorV3 (det3d/models/readers/voxel_encoder.py
// :205-210).  The reference semantics are inherently sequential:
//   * voxel id        = rank of the voxel's FIRST point in input order,
//   * kept points     = the first `max_points` points of the cell, in input order,
//   * max_voxels cut  = the loop breaks at the first point that would open voxel #max_voxels, dropping every
//                       later point of the frame (even those of existing voxels).
// Parallel formulation (all integer-exact, no floating point on the control path except the cell index):
//   1. insert   : cell -> slot of a 64-bit hash (key<<24 | point index), atomicMin keeps the first point;
//   2. scan     : exclusive scan of "is first point of its cell" flags in input order  => voxel rank;
//   3. assign   : first points with rank < max_voxels publish slot -> voxel id and the voxel's coordinates;
//                 the first point with rank == max_voxels publishes the frame's cut index;
//   4. collect  : every surviving point (index < cut) bubbles its index into the voxel's sorted list of the
//                 `max_points` smallest indices with a chain of atomicMin (order independent, exact);
//   5. gather   : one warp-lane group per voxel copies the points, zero-pads, writes counts and the mean.
// Cell index arithmetic uses IEEE fp32 subtract / divide / floor exactly like the reference (:38): reciprocal
// multiplication or fp64 would move ~1e-5 of the points into a neighbouring cell (SURVEY.md Appendix A.4).
//
// HBM traffic per frame: 16 N read (+8 N for the per-point scratch) and 112 M written -- the kernel family is
// latency / atomic bound at KITTI sizes and bandwidth bound in the 200k-point stress configuration.
#include "common.cuh"

namespace sessd {

long long g_launches = 0;

struct VoxParams {
    float vs[3], lo[3];
    int grid[3];
    int max_points, max_voxels, nfeat, batch;
    int cap_mask;
};

__device__ __forceinline__ int find_frame(const int *__restrict__ off, int batch, int i) {
    int lo = 0, hi = batch;   // off[lo] <= i < off[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (i >= off[mid]) lo = mid; else hi = mid;
    }
    return lo;
}

// 1. insert ------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vox_insert_kernel(const float *__restrict__ pts, const int *__restrict__ off,
                                                         VoxParams p, unsigned long long *tbl, int *__restrict__ slot_of) {
    extern __shared__ int s_off[];
    for (int t = threadIdx.x; t <= p.batch; t += blockDim.x) s_off[t] = off[t];
    __syncthreads();
    const int n = s_off[p.batch];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float *q = pts + (size_t)i * p.nfeat;
        int c[3];
        bool ok = true;
#pragma unroll
        for (int j = 0; j < 3; ++j) {
            float cf = floorf(__fdiv_rn(__fsub_rn(q[j], p.lo[j]), p.vs[j]));
            ok = ok && (cf >= 0.f) && (cf < (float)p.grid[j]);   // NaN fails both => rejected
            c[j] = (int)cf;
        }
        int slot = -1;
        if (ok) {
            const int f = find_frame(s_off, p.batch, i);
            unsigned long long key = (((unsigned long long)f * p.grid[2] + c[2]) * p.grid[1] + c[1]) * p.grid[0] + c[0];
            slot = hash_insert_min(tbl, p.cap_mask, key, (unsigned int)i);
        }
        slot_of[i] = slot;
    }
}

// 2. scan functors -------------------------------------------------------------------------------------
struct FirstFlagLoad {
    const unsigned long long *tbl;
    const int *slot_of;
    __device__ __forceinline__ int operator()(long long i) const {
        int s = slot_of[i];
        return (s >= 0 && (int)(tbl[s] & kHashValMask) == (int)i) ? 1 : 0;
    }
};
struct RankStore {
    int *rank;   // exclusive count of first points before i (global over the batch); -1-encoded flag folded in sign
    __device__ __forceinline__ void operator()(long long i, int ex, int v) const { rank[i] = v ? ex : ~ex; }
};

// frame meta: per-frame number of distinct cells, voxel counts and compact output bases ----------------
__global__ void vox_meta_kernel(const int *__restrict__ off, const int *__restrict__ rank, const int *__restrict__ d_total,
                                VoxParams p, int *__restrict__ frame_first /*[B+1] global rank at frame start*/,
                                int *__restrict__ vbase /*[B+1]*/, int *__restrict__ num_voxels /*[B+1]*/,
                                int *__restrict__ cut /*[B]*/) {
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    const int n = off[p.batch];
    int base = 0;
    for (int f = 0; f <= p.batch; ++f) {
        int start = off[f];
        int r;
        if (start >= n) r = *d_total;
        else { int v = rank[start]; r = v >= 0 ? v : ~v; }
        frame_first[f] = r;
    }
    for (int f = 0; f < p.batch; ++f) {
        int cells = frame_first[f + 1] - frame_first[f];
        int nv = cells < p.max_voxels ? cells : p.max_voxels;
        vbase[f] = base;
        num_voxels[f] = nv;
        cut[f] = off[f + 1];          // default: no cut
        base += nv;
    }
    vbase[p.batch] = base;
    num_voxels[p.batch] = base;
}

// 3. assign --------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vox_assign_kernel(const float *__restrict__ pts, const int *__restrict__ off,
                                                         VoxParams p, const int *__restrict__ slot_of,
                                                         const int *__restrict__ rank, const int *__restrict__ frame_first,
                                                         const int *__restrict__ vbase, int *__restrict__ slot_vid,
                                                         int *__restrict__ coors, int *__restrict__ cut) {
    extern __shared__ int s_off[];
    for (int t = threadIdx.x; t <= p.batch; t += blockDim.x) s_off[t] = off[t];
    __syncthreads();
    const int n = s_off[p.batch];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int r = rank[i];
        if (r < 0) continue;                       // not the first point of its cell
        const int f = find_frame(s_off, p.batch, i);
        const int local = r - frame_first[f];
        const int slot = slot_of[i];
        if (local < p.max_voxels) {
            const int vid = vbase[f] + local;
            slot_vid[slot] = vid;
            const float *q = pts + (size_t)i * p.nfeat;
            int c[3];
#pragma unroll
            for (int j = 0; j < 3; ++j) c[j] = (int)floorf(__fdiv_rn(__fsub_rn(q[j], p.lo[j]), p.vs[j]));
            reinterpret_cast<int4 *>(coors)[vid] = make_int4(f, c[2], c[1], c[0]);
        } else {
            slot_vid[slot] = -1;
            if (local == p.max_voxels) cut[f] = i;   // the reference loop breaks exactly here
        }
    }
}

// 4. collect -------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) vox_collect_kernel(const int *__restrict__ off, VoxParams p,
                                                          const int *__restrict__ slot_of, const int *__restrict__ slot_vid,
                                                          const int *__restrict__ cut, int *__restrict__ lists,
                                                          int *__restrict__ counts) {
    extern __shared__ int s_off[];
    for (int t = threadIdx.x; t <= p.batch; t += blockDim.x) s_off[t] = off[t];
    __syncthreads();
    const int n = s_off[p.batch];
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int slot = slot_of[i];
        if (slot < 0) continue;
        const int vid = slot_vid[slot];
        if (vid < 0) continue;
        const int f = find_frame(s_off, p.batch, i);
        if (i >= cut[f]) continue;
        atomicAdd(&counts[vid], 1);
        // concurrent sorted insertion: position k ends up holding the (k+1)-th smallest index
        int v = i;
        int *lst = lists + (size_t)vid * p.max_points;
        for (int k = 0; k < p.max_points; ++k) {
            int old = atomicMin(&lst[k], v);
            v = old > v ? old : v;
            if (v >= 0x7f7f7f7f) break;
        }
    }
}

// 5. gather --------------------------------------------------------------------------------------------
// 4-feature KITTI layout (MP = max_points known at compile time, 5 in the config): one thread per voxel loads its <= MP points as
// float4 (independent loads), writes the zero-padded [MP][4] block and num_points, and forms the VoxelFeatureExtractorV3 mean from the
// registers in the reference's order (voxel_encoder.py:209: sum over the point axis k = 0..MP-1, then divide by the count) -- no
// 64-bit divisions, no second gather for the mean (ncu at the stress shape: the per-(voxel, slot) version was ALU-bound, sm 70 %).
template <int MP>
__global__ void __launch_bounds__(256) vox_gather4_kernel(const float4 *__restrict__ pts, const int *__restrict__ num_voxels, int batch,
                                                          const int *__restrict__ lists, const int *__restrict__ counts,
                                                          float4 *__restrict__ voxels, int *__restrict__ num_points,
                                                          float4 *__restrict__ mean) {
    const int total = num_voxels[batch];
    for (int vid = blockIdx.x * blockDim.x + threadIdx.x; vid < total; vid += gridDim.x * blockDim.x) {
        int cnt = counts[vid];
        cnt = cnt < MP ? cnt : MP;
        float4 v[MP];
#pragma unroll
        for (int k = 0; k < MP; ++k) {
            v[k] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (k < cnt) v[k] = __ldg(&pts[lists[(size_t)vid * MP + k]]);
        }
        float4 s = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int k = 0; k < MP; ++k) {
            voxels[(size_t)vid * MP + k] = v[k];
            if (k < cnt) { s.x = __fadd_rn(s.x, v[k].x); s.y = __fadd_rn(s.y, v[k].y); s.z = __fadd_rn(s.z, v[k].z); s.w = __fadd_rn(s.w, v[k].w); }
        }
        num_points[vid] = cnt;
        if (mean) {
            const float c = (float)cnt;
            mean[vid] = make_float4(__fdiv_rn(s.x, c), __fdiv_rn(s.y, c), __fdiv_rn(s.z, c), __fdiv_rn(s.w, c));
        }
    }
}

// generic layout: one thread per (voxel, slot-in-voxel)
__global__ void __launch_bounds__(256) vox_gather_kernel(const float *__restrict__ pts, VoxParams p,
                                                         const int *__restrict__ num_voxels, const int *__restrict__ lists,
                                                         const int *__restrict__ counts, float *__restrict__ voxels,
                                                         int *__restrict__ num_points, float *__restrict__ mean) {
    const int total = num_voxels[p.batch];
    const long long work = (long long)total * p.max_points;
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < work; w += (long long)gridDim.x * blockDim.x) {
        const int vid = (int)(w / p.max_points);
        const int k = (int)(w - (long long)vid * p.max_points);
        int cnt = counts[vid];
        cnt = cnt < p.max_points ? cnt : p.max_points;
        float *dst = voxels + ((size_t)vid * p.max_points + k) * p.nfeat;
        if (k < cnt) {
            const float *src = pts + (size_t)lists[(size_t)vid * p.max_points + k] * p.nfeat;
            for (int j = 0; j < p.nfeat; ++j) dst[j] = src[j];
        } else {
            for (int j = 0; j < p.nfeat; ++j) dst[j] = 0.f;
        }
        if (k == 0) {
            num_points[vid] = cnt;
            if (mean) {
                // voxel_encoder.py:209: sum over the (zero padded) point axis, then divide by the count
                for (int j = 0; j < p.nfeat; ++j) {
                    float s = 0.f;
                    for (int q = 0; q < cnt; ++q)
                        s = __fadd_rn(s, pts[(size_t)lists[(size_t)vid * p.max_points + q] * p.nfeat + j]);
                    mean[(size_t)vid * p.nfeat + j] = __fdiv_rn(s, (float)cnt);
                }
            }
        }
    }
}

// workspace carve-up -------------------------------------------------------------------------------------
struct VoxWs {
    unsigned long long *tbl;
    int *slot_of, *rank, *slot_vid, *lists, *counts, *scan, *frame_first, *vbase, *cut, *total;
    int capacity;
    size_t bytes;
};

static inline size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

static VoxWs carve(void *base, int max_total_points, int batch, const sessd_voxel_cfg *cfg) {
    VoxWs w;
    int cap = 1024;
    while (cap < 2 * max_total_points) cap <<= 1;
    w.capacity = cap;
    char *p = (char *)base;
    size_t o = 0;
    auto take = [&](size_t bytes) { char *r = p ? p + o : nullptr; o += align_up(bytes); return (void *)r; };
    const size_t nv = (size_t)batch * cfg->max_voxels;
    w.tbl = (unsigned long long *)take(sizeof(unsigned long long) * cap);
    w.slot_vid = (int *)take(sizeof(int) * cap);
    w.slot_of = (int *)take(sizeof(int) * (size_t)max_total_points);
    w.rank = (int *)take(sizeof(int) * ((size_t)max_total_points + 1));
    w.lists = (int *)take(sizeof(int) * nv * cfg->max_points);
    w.counts = (int *)take(sizeof(int) * nv);
    w.scan = (int *)take(scan_scratch_bytes(max_total_points));
    w.frame_first = (int *)take(sizeof(int) * (batch + 2));
    w.vbase = (int *)take(sizeof(int) * (batch + 2));
    w.cut = (int *)take(sizeof(int) * (batch + 2));
    w.total = (int *)take(sizeof(int) * 4);
    w.bytes = o;
    return w;
}

}  // namespace sessd

using namespace sessd;

extern "C" const char *sessd_version(void) { return "sessd_b200 0.1 (sm_90a)"; }
extern "C" long long sessd_launch_count(void) { return g_launches; }

extern "C" size_t sessd_voxelize_workspace_bytes(int max_total_points, int batch, const sessd_voxel_cfg *cfg) {
    if (!cfg || max_total_points < 0 || batch < 1) return 0;
    return carve(nullptr, max_total_points > 0 ? max_total_points : 1, batch, cfg).bytes;
}

extern "C" int sessd_voxelize(const float *d_points, const int *d_frame_off, int batch, int max_total_points,
                              const sessd_voxel_cfg *cfg, float *d_voxels, int *d_coors, int *d_num_points,
                              float *d_mean, int *d_num_voxels, void *workspace, size_t workspace_bytes, void *stream) {
    if (!cfg || !d_frame_off || !d_voxels || !d_coors || !d_num_points || !d_num_voxels || !workspace) return SESSD_EINVAL;
    if (batch < 1 || batch > 4096 || max_total_points < 1 || cfg->max_points < 1 || cfg->max_voxels < 1 || cfg->num_feat < 3)
        return SESSD_EINVAL;
    if ((long long)max_total_points >= (1ll << kHashValBits)) return SESSD_ECAPACITY;
    VoxWs w = carve(workspace, max_total_points, batch, cfg);
    if (w.bytes > workspace_bytes) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    VoxParams p;
    for (int j = 0; j < 3; ++j) { p.vs[j] = cfg->voxel_size[j]; p.lo[j] = cfg->range_min[j]; p.grid[j] = cfg->grid[j]; }
    p.max_points = cfg->max_points; p.max_voxels = cfg->max_voxels; p.nfeat = cfg->num_feat; p.batch = batch;
    p.cap_mask = w.capacity - 1;
    const size_t nv = (size_t)batch * cfg->max_voxels;
    SESSD_CUDA_TRY(cudaMemsetAsync(w.tbl, 0xff, sizeof(unsigned long long) * w.capacity, st));
    SESSD_CUDA_TRY(cudaMemsetAsync(w.lists, 0x7f, sizeof(int) * nv * cfg->max_points, st));
    SESSD_CUDA_TRY(cudaMemsetAsync(w.counts, 0, sizeof(int) * nv, st));
    const int grid = persistent_grid(max_total_points, 256);
    const size_t sm = sizeof(int) * (batch + 1);
    SESSD_LAUNCH(vox_insert_kernel, grid, 256, sm, st, d_points, d_frame_off, p, w.tbl, w.slot_of);
    // scan the first-point flags over all points of the batch (count read from d_frame_off[batch])
    FirstFlagLoad ld{w.tbl, w.slot_of};
    RankStore stf{w.rank};
    device_scan(ld, stf, d_frame_off + batch, 1, max_total_points, w.scan, w.total, st);
    SESSD_LAUNCH(vox_meta_kernel, 1, 32, 0, st, d_frame_off, w.rank, w.total, p, w.frame_first, w.vbase, d_num_voxels, w.cut);
    SESSD_LAUNCH(vox_assign_kernel, grid, 256, sm, st, d_points, d_frame_off, p, w.slot_of, w.rank, w.frame_first,
                 w.vbase, w.slot_vid, d_coors, w.cut);
    SESSD_LAUNCH(vox_collect_kernel, grid, 256, sm, st, d_frame_off, p, w.slot_of, w.slot_vid, w.cut, w.lists, w.counts);
    if (cfg->num_feat == 4 && cfg->max_points == 5) {
        SESSD_LAUNCH((vox_gather4_kernel<5>), persistent_grid((long long)nv, 256), 256, 0, st, (const float4 *)d_points, d_num_voxels, batch,
                     w.lists, w.counts, (float4 *)d_voxels, d_num_points, (float4 *)d_mean);
    } else {
        const int ggrid = persistent_grid((long long)nv * cfg->max_points, 256);
        SESSD_LAUNCH(vox_gather_kernel, ggrid, 256, 0, st, d_points, p, d_num_voxels, w.lists, w.counts, d_voxels,
                     d_num_points, d_mean);
    }
    return last_error();
}

extern "C" int sessd_voxelize_host(const float *h_points, int num_points, const sessd_voxel_cfg *cfg, float *h_voxels,
                                   int *h_coors_zyx, int *h_num_points) {
    if (!cfg || num_points < 0 || (num_points > 0 && !h_points)) return SESSD_EINVAL;
    const int cap = num_points > 0 ? num_points : 1;
    const size_t ws_bytes = sessd_voxelize_workspace_bytes(cap, 1, cfg);
    const size_t nv = (size_t)cfg->max_voxels;
    float *d_pts = nullptr, *d_vox = nullptr;
    int *d_off = nullptr, *d_coors = nullptr, *d_num = nullptr, *d_nv = nullptr;
    void *d_ws = nullptr;
    int rc = 0, count = 0;
    cudaStream_t st = nullptr;
#define HTRY(e) do { cudaError_t _e = (e); if (_e != cudaSuccess) { rc = (int)_e; goto done; } } while (0)
    HTRY(cudaStreamCreateWithFlags(&st, cudaStreamNonBlocking));
    HTRY(cudaMalloc(&d_pts, sizeof(float) * (size_t)cap * cfg->num_feat));
    HTRY(cudaMalloc(&d_off, sizeof(int) * 2));
    HTRY(cudaMalloc(&d_vox, sizeof(float) * nv * cfg->max_points * cfg->num_feat));
    HTRY(cudaMalloc(&d_coors, sizeof(int) * nv * 4));
    HTRY(cudaMalloc(&d_num, sizeof(int) * nv));
    HTRY(cudaMalloc(&d_nv, sizeof(int) * 2));
    HTRY(cudaMalloc(&d_ws, ws_bytes));
    {
        int off[2] = {0, num_points};
        HTRY(cudaMemcpyAsync(d_off, off, sizeof(off), cudaMemcpyHostToDevice, st));
        if (num_points > 0)
            HTRY(cudaMemcpyAsync(d_pts, h_points, sizeof(float) * (size_t)num_points * cfg->num_feat, cudaMemcpyHostToDevice, st));
        rc = sessd_voxelize(d_pts, d_off, 1, cap, cfg, d_vox, d_coors, d_num, nullptr, d_nv, d_ws, ws_bytes, st);
        if (rc) goto done;
        HTRY(cudaMemcpyAsync(&count, d_nv, sizeof(int), cudaMemcpyDeviceToHost, st));
        HTRY(cudaStreamSynchronize(st));
        if (count > 0) {
            HTRY(cudaMemcpyAsync(h_voxels, d_vox, sizeof(float) * (size_t)count * cfg->max_points * cfg->num_feat,
                                 cudaMemcpyDeviceToHost, st));
            HTRY(cudaMemcpyAsync(h_num_points, d_num, sizeof(int) * (size_t)count, cudaMemcpyDeviceToHost, st));
            int *tmp = (int *)malloc(sizeof(int) * 4 * (size_t)count);
            cudaError_t e = cudaMemcpyAsync(tmp, d_coors, sizeof(int) * 4 * (size_t)count, cudaMemcpyDeviceToHost, st);
            if (e == cudaSuccess) e = cudaStreamSynchronize(st);
            if (e == cudaSuccess)
                for (int i = 0; i < count; ++i) {
                    h_coors_zyx[3 * i] = tmp[4 * i + 1]; h_coors_zyx[3 * i + 1] = tmp[4 * i + 2]; h_coors_zyx[3 * i + 2] = tmp[4 * i + 3];
                }
            free(tmp);
            HTRY(e);
        }
    }
done:
#undef HTRY
    cudaFree(d_pts); cudaFree(d_off); cudaFree(d_vox); cudaFree(d_coors); cudaFree(d_num); cudaFree(d_nv); cudaFree(d_ws);
    if (st) cudaStreamDestroy(st);
    return rc ? (rc > 0 ? -rc - 1000 : rc) : count;
}
