// kitti_eval.cu -- KITTI object evaluation on the device: detection -> camera annotation conversion, per-frame overlap blocks (2D,
// BEV, 3D), the two matching passes, the threshold choice and the precision / AOS curves with their R11 / R40 averages.
// Compiled with -fmad=false (build.py NO_FMA): every fp32 / fp64 expression below rounds once per operation, in the order written.
//
// Precision of each step, worked out from the reference's types (det3d/datasets/kitti/kitti.py, det3d/datasets/utils/eval.py,
// det3d/datasets/kitti/eval.py, det3d/ops/nms/nms_gpu.py):
//   conversion   lidar box fp32: limit_period and centre-z -> bottom-z in fp32 (numpy keeps the fp32 array type against Python
//                scalars); lidar -> camera with M = R0_rect . Tr_velo_to_cam (fp64, the host forms M with numpy as the reference does)
//                in fp64; corners with origin (0.5, 1.0, 0.5) and cos / sin of ry in fp64; projection through P2 with a ZERO fourth
//                homogeneous coordinate (project_to_image concatenates zeros, so P2's last column never contributes); alpha =
//                fp64(-atan2(-y, x) rounded to fp32) + ry_cam (np.arctan2 of two fp32 scalars is fp32).
//   2D overlap   image_box_overlap in fp64 (criterion -1; criterion 0 for the DontCare test).
//   BEV overlap  rotate_iou_gpu_eval: boxes rounded to fp32; corners, inside tests, crossings, the sort and each triangle's
//                cross product in fp32; each triangle area widened to fp64 by its `/ 2.0`, the fan summed in fp64 (`area_val = 0.0`);
//                area1 + area2 in fp32, the union and quotient in fp64; the kernel stores into an fp32 array, and
//                `iou.astype(boxes.dtype)` is fp32 because `boxes` was rebound to its fp32 copy -- so every BEV overlap is an fp32
//                value (widened to fp64 by calculate_iou_partly).
//   3D overlap   the criterion-2 BEV intersection above (fp32), then box3d_overlap_kernel in fp64 on the fp64 annotations, stored
//                back into that fp32 array: every 3D overlap is fp32 too.
//   matching     fp64 overlaps, scores (fp32 widened) and alphas; tp / fp are exact integers; the AOS similarity is an fp64 sum in
//                ground-truth order within a frame, then over frames in frame order.
//   thresholds   get_thresholds' recall arithmetic in fp64, exactly as written.
// cos / sin of a box angle are taken in fp64 and rounded to fp32, i.e. correctly rounded, where the reference's numba kernel calls
// the fp32 library functions: those may differ from the exact value by an ulp, and a pair with a corner on the other box's edge
// turns such an ulp into a 1e-4 change of IoU.  Rounding exactly makes the value independent of the math library.  alpha's atan2 is
// likewise taken in fp64 and rounded to fp32.
// The reference's vertex buffer holds 8 points (16 floats), and its sort buffer 16 floats; the geometric maximum is 8 inside
// corners plus 16 crossings, so both buffers here hold 24 points.  Identical boxes give 8 points (each corner twice, every corner
// is inside the other box and no crossing passes the strict orientation tests) and IoU 1 up to fp32 rounding; axis-aligned boxes
// that share an edge keep the 4 corners on that edge (the inside test is inclusive) and a fan of area 0, so IoU 0.
#include <cub/cub.cuh>
#include <math.h>

#include "common.cuh"

namespace {
using namespace sessd;

constexpr int kRec = SESSD_KITTI_REC;        // doubles per box record
constexpr int kPts = 41;                      // sample points of the precision curve
constexpr int kMaxDt = 1024;                  // detections per frame: 32 lanes x 32 mask bits
constexpr int kNoDet = -10000000;             // compute_statistics_jit's NO_DETECTION
constexpr int kCar = 0, kPedestrian = 1, kPersonSitting = SESSD_KITTI_PERSON_SITTING, kVan = SESSD_KITTI_VAN;

// ------------------------------------------------------------------------------------------------ rotated-box intersection
// (the eval kernel's RRPN clip; not rotbox.cuh, whose inside test and crossing rule differ)
__device__ __forceinline__ double tri_area(float ax, float ay, float bx, float by, float cx, float cy) {
    const float t = (ax - cx) * (by - cy) - (ay - cy) * (bx - cx);
    return (double)t / 2.0;
}

__device__ __forceinline__ void corners_of(const float *r, float *c) {
    const float ca = (float)cos((double)r[4]), sa = (float)sin((double)r[4]);   // correctly rounded: see the header
    const float hx = r[2] / 2.f, hy = r[3] / 2.f;
    const float cx[4] = {-hx, -hx, hx, hx}, cy[4] = {-hy, hy, hy, -hy};
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        c[2 * i] = ca * cx[i] + sa * cy[i] + r[0];
        c[2 * i + 1] = -sa * cx[i] + ca * cy[i] + r[1];
    }
}

__device__ __forceinline__ bool inside_quad(float px, float py, const float *q) {
    const float ab0 = q[2] - q[0], ab1 = q[3] - q[1];
    const float ad0 = q[6] - q[0], ad1 = q[7] - q[1];
    const float ap0 = px - q[0], ap1 = py - q[1];
    const float abab = ab0 * ab0 + ab1 * ab1, abap = ab0 * ap0 + ab1 * ap1;
    const float adad = ad0 * ad0 + ad1 * ad1, adap = ad0 * ap0 + ad1 * ap1;
    return abab >= abap && abap >= 0.f && adad >= adap && adap >= 0.f;
}

__device__ __forceinline__ bool crossing(const float *p1, const float *p2, int i, int j, float &ox, float &oy) {
    const float A0 = p1[2 * i], A1 = p1[2 * i + 1];
    const float B0 = p1[2 * ((i + 1) & 3)], B1 = p1[2 * ((i + 1) & 3) + 1];
    const float C0 = p2[2 * j], C1 = p2[2 * j + 1];
    const float D0 = p2[2 * ((j + 1) & 3)], D1 = p2[2 * ((j + 1) & 3) + 1];
    const float BA0 = B0 - A0, BA1 = B1 - A1, DA0 = D0 - A0, CA0 = C0 - A0, DA1 = D1 - A1, CA1 = C1 - A1;
    const bool acd = DA1 * CA0 > CA1 * DA0;
    const bool bcd = (D1 - B1) * (C0 - B0) > (C1 - B1) * (D0 - B0);
    if (acd == bcd) return false;
    const bool abc = CA1 * BA0 > BA1 * CA0;
    const bool abd = DA1 * BA0 > BA1 * DA0;
    if (abc == abd) return false;
    const float DC0 = D0 - C0, DC1 = D1 - C1;
    const float ABBA = A0 * B1 - B0 * A1, CDDC = C0 * D1 - D0 * C1;
    const float DH = BA1 * DC0 - BA0 * DC1;
    const float Dx = ABBA * DC0 - BA0 * CDDC, Dy = ABBA * DC1 - BA1 * CDDC;
    ox = Dx / DH;
    oy = Dy / DH;
    return true;
}

// intersection area of rbox1 = (x, y, dx, dy, angle) and rbox2, fp64 as numba types `area`
__device__ double rbox_inter(const float *r1, const float *r2) {
    float c1[8], c2[8], px[24], py[24], vs[24];
    corners_of(r1, c1);
    corners_of(r2, c2);
    int n = 0;
    for (int i = 0; i < 4; ++i) {
        if (inside_quad(c1[2 * i], c1[2 * i + 1], c2)) { px[n] = c1[2 * i]; py[n] = c1[2 * i + 1]; ++n; }
        if (inside_quad(c2[2 * i], c2[2 * i + 1], c1)) { px[n] = c2[2 * i]; py[n] = c2[2 * i + 1]; ++n; }
    }
    for (int i = 0; i < 4; ++i)
        for (int j = 0; j < 4; ++j) {
            float x, y;
            if (crossing(c1, c2, i, j, x, y)) { px[n] = x; py[n] = y; ++n; }
        }
    if (n > 0) {
        float sx = 0.f, sy = 0.f;
        for (int i = 0; i < n; ++i) { sx += px[i]; sy += py[i]; }
        sx = (float)((double)sx / (double)n);          // fp32 /= int32 promotes to fp64, stored back to fp32
        sy = (float)((double)sy / (double)n);
        for (int i = 0; i < n; ++i) {
            float v0 = px[i] - sx, v1 = py[i] - sy;
            const float d = sqrtf(v0 * v0 + v1 * v1);
            v0 = v0 / d;
            v1 = v1 / d;
            if (v1 < 0.f) v0 = -2.f - v0;
            vs[i] = v0;
        }
        for (int i = 1; i < n; ++i) {
            if (vs[i - 1] > vs[i]) {
                const float t = vs[i], tx = px[i], ty = py[i];
                int j = i;
                while (j > 0 && vs[j - 1] > t) { vs[j] = vs[j - 1]; px[j] = px[j - 1]; py[j] = py[j - 1]; --j; }
                vs[j] = t; px[j] = tx; py[j] = ty;
            }
        }
    }
    double a = 0.0;
    for (int i = 0; i < n - 2; ++i) a += fabs(tri_area(px[0], py[0], px[i + 1], py[i + 1], px[i + 2], py[i + 2]));
    return a;
}

// ------------------------------------------------------------------------------------------------ overlaps
__device__ __forceinline__ double pymin(double a, double b) { return b < a ? b : a; }
__device__ __forceinline__ double pymax(double a, double b) { return b > a ? b : a; }

// np.min / np.max of a corner set: a NaN propagates (fmin / fmax would drop it)
__device__ __forceinline__ double npmin(double a, double b) { return a != a ? a : (b != b ? b : (b < a ? b : a)); }
__device__ __forceinline__ double npmax(double a, double b) { return a != a ? a : (b != b ? b : (b > a ? b : a)); }

// image_box_overlap(dt, gt, criterion) for one pair; criterion -1 (IoU) or 0 (over the first box's area)
__device__ __forceinline__ double box2d_overlap(const double *b, const double *q, int criterion) {
    const double qa = (q[2] - q[0]) * (q[3] - q[1]);
    const double iw = pymin(b[2], q[2]) - pymax(b[0], q[0]);
    if (!(iw > 0)) return 0.0;
    const double ih = pymin(b[3], q[3]) - pymax(b[1], q[1]);
    if (!(ih > 0)) return 0.0;
    const double ba = (b[2] - b[0]) * (b[3] - b[1]);
    const double ua = criterion == -1 ? ba + qa - iw * ih : ba;
    return iw * ih / ua;
}

// BEV box of a record on the two axes that are not z_axis: (loc a, loc b, dim a, dim b, ry), rounded to fp32
__device__ __forceinline__ void bev_of(const double *r, int z_axis, float *o) {
    const int a = z_axis == 0 ? 1 : 0, b = z_axis == 2 ? 1 : 2;
    o[0] = (float)r[5 + a]; o[1] = (float)r[5 + b]; o[2] = (float)r[8 + a]; o[3] = (float)r[8 + b]; o[4] = (float)r[11];
}

__device__ double pair_overlap(int metric, const double *dt, const double *gt, int z_axis, double z_center) {
    if (metric == 0) return box2d_overlap(dt, gt, -1);
    float bg[5], bd[5];
    bev_of(gt, z_axis, bg);
    bev_of(dt, z_axis, bd);
    const double inter = rbox_inter(bg, bd);                 // rbox1 = GT, rbox2 = detection (calculate_iou_partly swaps its operands)
    if (metric == 1) {
        const float area1 = bg[2] * bg[3], area2 = bd[2] * bd[3];
        return (double)(float)(inter / ((double)(area1 + area2) - inter));
    }
    const float rinc = (float)inter;
    if (!(rinc > 0.f)) return (double)rinc;
    const double *bl = dt + 5, *bd3 = dt + 8, *ql = gt + 5, *qd3 = gt + 8;   // boxes = detections, qboxes = GT
    const double up = 1 - z_center;
    const double min_z = pymin(bl[z_axis] + bd3[z_axis] * up, ql[z_axis] + qd3[z_axis] * up);
    const double max_z = pymax(bl[z_axis] - bd3[z_axis] * z_center, ql[z_axis] - qd3[z_axis] * z_center);
    const double iw = min_z - max_z;
    if (!(iw > 0)) return 0.0;
    const double v1 = bd3[0] * bd3[1] * bd3[2], v2 = qd3[0] * qd3[1] * qd3[2];
    const double inc = iw * (double)rinc;
    return (double)(float)(inc / (v1 + v2 - inc));
}

// one block per frame; block [n_dt_f, n_gt_f] at ov_off[f], row stride n_gt_f
__global__ void overlaps_kernel(SessdKittiFrames fr, int metric, int z_axis, double z_center, double *ov) {
    const int f = blockIdx.x;
    const int g0 = fr.gt_off[f], ng = fr.gt_off[f + 1] - g0;
    const int d0 = fr.dt_off[f], nd = fr.dt_cnt[f];
    double *o = ov + fr.ov_off[f];
    for (int p = threadIdx.x; p < nd * ng; p += blockDim.x) {
        const int j = p / ng, i = p - j * ng;
        o[p] = pair_overlap(metric, fr.dt + (size_t)(d0 + j) * kRec, fr.gt + (size_t)(g0 + i) * kRec, z_axis, z_center);
    }
}

// ------------------------------------------------------------------------------------------------ matching (compute_statistics_jit)
__constant__ int kMinHeight[3] = {40, 25, 25};
__constant__ int kMaxOcclusion[3] = {0, 1, 2};
__constant__ double kMaxTruncation[3] = {0.15, 0.3, 0.5};

__device__ __forceinline__ int ignored_gt(const SessdKittiFrames &fr, int g, int cls, int diff) {
    const int code = fr.gt_code[g];
    const double *r = fr.gt + (size_t)g * kRec;
    int valid = -1;
    if (code == cls) valid = 1;
    else if ((cls == kPedestrian && code == kPersonSitting) || (cls == kCar && code == kVan)) valid = 0;
    const double h = r[3] - r[1];
    const bool ign = fr.gt_occluded[g] > kMaxOcclusion[diff] || r[12] > kMaxTruncation[diff] || h <= (double)kMinHeight[diff];
    if (valid == 1 && !ign) return 0;
    if (valid == 0 || (ign && valid == 1)) return 1;
    return -1;
}

struct Pick { int rank; double key; int j; };

// a beats b: higher rank; then (rank 2: larger overlap, pass 1: larger score) ; then the smaller index (the first in scan order)
__device__ __forceinline__ bool beats(const Pick &a, const Pick &b) {
    if (a.rank != b.rank) return a.rank > b.rank;
    if (a.rank == 0) return false;
    if (a.key != b.key && (a.rank == 2)) return a.key > b.key;
    return a.j < b.j;
}

__device__ __forceinline__ Pick warp_best(Pick p) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        Pick q;
        q.rank = __shfl_xor_sync(0xffffffffu, p.rank, o);
        q.key = __shfl_xor_sync(0xffffffffu, p.key, o);
        q.j = __shfl_xor_sync(0xffffffffu, p.j, o);
        if (beats(q, p)) p = q;
    }
    return p;
}

struct FrameStats { int tp, fp; double sim; };

// one warp runs compute_statistics_jit for one frame.  Lane l owns detections j = 32 b + l; bit b of each mask is detection j.
// FP = false: pass 1 (compute_fp=False, thresh=0), TP scores go to `tp_scores` in ground-truth order.
template <bool FP>
__device__ FrameStats match_frame(const SessdKittiFrames &fr, int f, const double *ov, int metric, int cls, int diff,
                                  double min_ov, double thresh, bool aos, double *tp_scores) {
    const int lane = threadIdx.x & 31;
    const int g0 = fr.gt_off[f], ng = fr.gt_off[f + 1] - g0;
    const int d0 = fr.dt_off[f], nd = fr.dt_cnt[f];
    const int nb = (nd + 31) >> 5;
    unsigned neg = 0, one = 0, thr = 0, asg = 0;
    for (int b = 0; b < nb; ++b) {
        const int j = 32 * b + lane;
        if (j >= nd) { neg |= 1u << b; continue; }
        const double *r = fr.dt + (size_t)(d0 + j) * kRec;
        if (fabs(r[3] - r[1]) < (double)kMinHeight[diff]) one |= 1u << b;
        else if (fr.dt_code[d0 + j] != cls) neg |= 1u << b;
        if (FP && r[12] < thresh) thr |= 1u << b;
    }
    FrameStats s{0, 0, 0.0};
    for (int i = 0; i < ng; ++i) {
        const int ig = ignored_gt(fr, g0 + i, cls, diff);
        if (ig == -1) continue;
        Pick p{0, 0.0, 0x7fffffff};
        for (int b = 0; b < nb; ++b) {
            const unsigned bit = 1u << b;
            if ((neg | asg | thr) & bit) continue;
            const int j = 32 * b + lane;
            const double o = ov[(size_t)j * ng + i];
            if (!(o > min_ov)) continue;
            Pick c;
            if (!FP) {
                const double sc = fr.dt[(size_t)(d0 + j) * kRec + 12];
                if (!(sc > (double)kNoDet)) continue;
                c = Pick{1, sc, j};
                if (p.rank == 0 || sc > p.key) p = c;
            } else {
                c = (one & bit) ? Pick{1, 0.0, j} : Pick{2, o, j};
                if (beats(c, p)) p = c;
            }
        }
        if (!FP) {
            // pass 1 orders by score, then index: reuse beats() with rank 2 semantics
            if (p.rank) p.rank = 2;
        }
        p = warp_best(p);
        if (p.rank == 0) continue;                                       // no detection: fn (unused)
        const int j = p.j;
        const bool det_one = (__shfl_sync(0xffffffffu, one, j & 31) >> (j >> 5)) & 1u;
        if (!(ig == 1 || det_one)) {
            if (!FP) {
                if (lane == 0) tp_scores[g0 + s.tp] = fr.dt[(size_t)(d0 + j) * kRec + 12];
            } else if (aos) {
                const double delta = fr.gt[(size_t)(g0 + i) * kRec + 4] - fr.dt[(size_t)(d0 + j) * kRec + 4];
                s.sim += (1.0 + cos(delta)) / 2.0;
            }
            ++s.tp;
        }
        if (lane == (j & 31)) asg |= 1u << (j >> 5);
    }
    if (!FP) return s;
    unsigned fpm = ~(asg | neg | one | thr);
    if (nb < 32) fpm &= (1u << nb) - 1u;
    int fp = __reduce_add_sync(0xffffffffu, __popc(fpm));
    if (metric == 0) {
        const int c0 = fr.dc_off[f], nc = fr.dc_off[f + 1] - c0;
        int nstuff = 0;
        for (int c = 0; c < nc; ++c) {
            const double *dc = fr.dc + (size_t)(c0 + c) * 4;
            for (int b = 0; b < nb; ++b) {
                const unsigned bit = 1u << b;
                if ((asg | neg | one | thr) & bit) continue;
                const int j = 32 * b + lane;
                if (box2d_overlap(fr.dt + (size_t)(d0 + j) * kRec, dc, 0) > min_ov) { asg |= bit; ++nstuff; }
            }
        }
        fp -= __reduce_add_sync(0xffffffffu, nstuff);
    }
    s.fp = fp;
    return s;
}

__global__ void fill_kernel(double *p, long long n, double v) {
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x) p[i] = v;
}

__global__ void segments_kernel(int *seg, int ncfg, int total_gt) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c <= ncfg) seg[c] = c * total_gt;
}

// pass 1: warp per (config, frame)
__global__ void pass1_kernel(SessdKittiFrames fr, const double *ov, int metric, int ncfg, const int *cfg, const double *min_ov,
                             int total_gt, double *scores, int *n_tp, int *n_valid) {
    const long long items = (long long)ncfg * fr.num_frames;
    const int lane = threadIdx.x & 31;
    for (long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; w < items;
         w += ((long long)gridDim.x * blockDim.x) >> 5) {
        const int c = (int)(w / fr.num_frames), f = (int)(w - (long long)c * fr.num_frames);
        const int cls = cfg[2 * c], diff = cfg[2 * c + 1];
        FrameStats s = match_frame<false>(fr, f, ov + fr.ov_off[f], metric, cls, diff, min_ov[c], 0.0, false,
                                          scores + (size_t)c * total_gt);
        int nv = 0;
        const int g0 = fr.gt_off[f], ng = fr.gt_off[f + 1] - g0;
        for (int i = lane; i < ng; i += 32) nv += ignored_gt(fr, g0 + i, cls, diff) == 0;
        nv = __reduce_add_sync(0xffffffffu, nv);
        if (lane == 0) {
            if (s.tp) atomicAdd(&n_tp[c], s.tp);
            if (nv) atomicAdd(&n_valid[c], nv);
        }
    }
}

// get_thresholds on the descending TP scores of each config (one thread per config; fp64 recall arithmetic as written)
__global__ void thresholds_kernel(int ncfg, int total_gt, const double *sorted, const int *n_tp, const int *n_valid, double *thr,
                                  int *n_thr) {
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (c >= ncfg) return;
    const double *s = sorted + (size_t)c * total_gt;
    const int n = n_tp[c];
    const double num_gt = (double)n_valid[c];
    double cur = 0.0;
    int k = 0;
    for (int i = 0; i < n; ++i) {
        const double l = (double)(i + 1) / num_gt;
        const double r = i < n - 1 ? (double)(i + 2) / num_gt : l;
        if ((r - cur) < (cur - l) && i < n - 1) continue;
        if (k < kPts) thr[(size_t)c * kPts + k] = s[i];
        ++k;
        cur += 1.0 / (kPts - 1.0);
    }
    n_thr[c] = k < kPts ? k : kPts;
    for (int t = k; t < kPts; ++t) thr[(size_t)c * kPts + t] = 0.0;
}

// pass 2: warp per (config, frame), every threshold of the config
__global__ void pass2_kernel(SessdKittiFrames fr, const double *ov, int metric, int ncfg, const int *cfg, const double *min_ov,
                             const double *thr, const int *n_thr, int aos, int *tpfp, double *sim) {
    const int F = fr.num_frames;
    const long long items = (long long)ncfg * F;
    const int lane = threadIdx.x & 31;
    for (long long w = (blockIdx.x * (long long)blockDim.x + threadIdx.x) >> 5; w < items;
         w += ((long long)gridDim.x * blockDim.x) >> 5) {
        const int c = (int)(w / F), f = (int)(w - (long long)c * F);
        const int cls = cfg[2 * c], diff = cfg[2 * c + 1];
        for (int t = 0; t < n_thr[c]; ++t) {
            FrameStats s = match_frame<true>(fr, f, ov + fr.ov_off[f], metric, cls, diff, min_ov[c], thr[(size_t)c * kPts + t],
                                             aos != 0, nullptr);
            if (lane == 0) {
                if (s.tp) atomicAdd(&tpfp[((size_t)c * kPts + t) * 2], s.tp);
                if (s.fp) atomicAdd(&tpfp[((size_t)c * kPts + t) * 2 + 1], s.fp);
                if (aos) sim[((size_t)c * kPts + t) * F + f] = (s.tp > 0 || s.fp > 0) ? s.sim : 0.0;
            }
        }
    }
}

// block per config: frame-ordered similarity sums (the pass-2 workspace keeps one fp64 similarity per (config, threshold, frame),
// ncfg * 41 * F doubles: 133 MB for 108 configs over 3769 frames; it is only allocated when AOS is computed), precision / AOS, suffix max (np.max: NaN wins), R11 and R40 averages
__global__ void finish_kernel(int ncfg, int F, const int *n_thr, const int *tpfp, const double *sim, int aos, double *prec,
                              double *orient, double *map) {
    const int c = blockIdx.x, t = threadIdx.x;
    __shared__ double sp[kPts], sa[kPts];
    if (t < kPts) {
        double p = 0.0, a = 0.0;
        if (t < n_thr[c]) {
            const double tp = tpfp[((size_t)c * kPts + t) * 2], fp = tpfp[((size_t)c * kPts + t) * 2 + 1];
            p = tp / (tp + fp);
            if (aos) {
                const double *s = sim + ((size_t)c * kPts + t) * F;
                double acc = 0.0;
                for (int f = 0; f < F; ++f) acc += s[f];
                a = acc / (tp + fp);
            }
        }
        sp[t] = p;
        sa[t] = a;
    }
    __syncthreads();
    if (t == 0) {
        const int n = n_thr[c];
        for (int pass = 0; pass < 2; ++pass) {
            double *v = pass ? sa : sp;
            for (int i = n - 2; i >= 0; --i) {
                const double m = v[i + 1];                          // max of v[i+1:], already final
                if (isnan(v[i]) || isnan(m)) v[i] = NAN;
                else if (m > v[i]) v[i] = m;
            }
        }
        // get_mAP: sums = 0 + p[0] + p[4] + ... + p[40], / 11 * 100; get_mAP_v2: p[1] + ... + p[40], / 40 * 100
        double r11 = 0.0, r40 = 0.0, a11 = 0.0, a40 = 0.0;
        for (int i = 0; i < kPts; i += 4) { r11 = r11 + sp[i]; a11 = a11 + sa[i]; }
        for (int i = 1; i < kPts; ++i) { r40 = r40 + sp[i]; a40 = a40 + sa[i]; }
        map[4 * c + 0] = r11 / 11 * 100;
        map[4 * c + 1] = r40 / 40 * 100;
        map[4 * c + 2] = a11 / 11 * 100;
        map[4 * c + 3] = a40 / 40 * 100;
    }
    __syncthreads();
    if (t < kPts) {
        prec[(size_t)c * kPts + t] = sp[t];
        orient[(size_t)c * kPts + t] = sa[t];
    }
}

// ------------------------------------------------------------------------------------------------ detection -> camera annotation
__global__ void convert_kernel(const float *boxes, const float *scores, const int *labels, const int *off, int F, const double *calib,
                               const int *image_hw, double *rec, int *keep) {
    const int f = blockIdx.x;
    const int d0 = off[f], nd = off[f + 1] - d0;
    const double *M = calib + (size_t)f * 24, *P = M + 12;
    const double H = image_hw[2 * f], W = image_hw[2 * f + 1];
    for (int k = threadIdx.x; k < nd; k += blockDim.x) {
        const int j = d0 + k;
        const float *b = boxes + (size_t)j * 7;
        const float P2f = (float)(2.0 * M_PI);
        const float ry = b[6] - floorf(b[6] / P2f + 0.5f) * P2f;
        const float zb = b[2] - b[5] / 2.f;
        const double x = b[0], y = b[1], z = zb;
        double cam[3];
        for (int r = 0; r < 3; ++r) cam[r] = x * M[4 * r] + y * M[4 * r + 1] + z * M[4 * r + 2] + 1.0 * M[4 * r + 3];
        const double dl = b[4], dh = b[5], dw = b[3];     // camera dims (l, h, w)
        const double rc = cos((double)ry), rs = sin((double)ry);
        double u0 = INFINITY, v0 = INFINITY, u1 = -INFINITY, v1 = -INFINITY;
        for (int q = 0; q < 8; ++q) {
            const int o = q ^ ((q >> 1) & 1);                // corners_nd's order 0 1 3 2 4 5 7 6
            const double nx = (double)((o >> 2) & 1) - 0.5, ny = (double)((o >> 1) & 1) - 1.0, nz = (double)(o & 1) - 0.5;
            const double px = dl * nx, py = dh * ny, pz = dw * nz;
            const double X = px * rc + py * 0.0 + pz * rs + cam[0];
            const double Y = px * 0.0 + py * 1.0 + pz * 0.0 + cam[1];
            const double Z = px * -rs + py * 0.0 + pz * rc + cam[2];
            const double U = X * P[0] + Y * P[1] + Z * P[2] + 0.0 * P[3];
            const double V = X * P[4] + Y * P[5] + Z * P[6] + 0.0 * P[7];
            const double Wd = X * P[8] + Y * P[9] + Z * P[10] + 0.0 * P[11];
            const double u = U / Wd, v = V / Wd;
            u0 = npmin(u0, u); v0 = npmin(v0, v); u1 = npmax(u1, u); v1 = npmax(v1, v);
        }
        const bool ok = !(u0 > W || v0 > H) && !(u1 < 0 || v1 < 0);
        keep[j] = ok;
        double *o = rec + (size_t)j * kRec;
        o[0] = pymax(u0, 0.0); o[1] = pymax(v0, 0.0); o[2] = pymin(u1, W); o[3] = pymin(v1, H);
        o[4] = (double)(-(float)atan2(-(double)b[1], (double)b[0])) + (double)ry;
        o[5] = cam[0]; o[6] = cam[1]; o[7] = cam[2];
        o[8] = dl; o[9] = dh; o[10] = dw;
        o[11] = (double)ry;
        o[12] = (double)scores[j];
    }
}

// stable per-frame compaction of the kept records (block per frame, input order kept)
__global__ void compact_kernel(const int *off, const int *keep, const double *rec, const int *labels, const int *label_code,
                               int num_labels, double *out, int *out_label, int *out_code, int *cnt) {
    typedef cub::BlockScan<int, 128> Scan;
    __shared__ typename Scan::TempStorage ts;
    __shared__ int base;
    const int f = blockIdx.x;
    const int d0 = off[f], nd = off[f + 1] - d0;
    if (threadIdx.x == 0) base = 0;
    __syncthreads();
    for (int k0 = 0; k0 < nd; k0 += 128) {
        const int k = k0 + threadIdx.x;
        const int kp = k < nd ? keep[d0 + k] : 0;
        int pos, tot;
        Scan(ts).ExclusiveSum(kp, pos, tot);
        if (kp) {
            const int dst = d0 + base + pos;
            for (int e = 0; e < kRec; ++e) out[(size_t)dst * kRec + e] = rec[(size_t)(d0 + k) * kRec + e];
            const int lab = labels[d0 + k];
            out_label[dst] = lab;
            out_code[dst] = lab >= 0 && lab < num_labels ? label_code[lab] : -1;
        }
        __syncthreads();
        if (threadIdx.x == 0) base += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0) cnt[f] = base;
}

struct EvalWs {
    double *ov, *scores, *sorted, *sim;
    int *seg, *n_tp, *n_valid, *tpfp;
    void *cub_tmp;
    size_t cub_bytes, bytes;
};

size_t align_up(size_t x) { return (x + 255) & ~(size_t)255; }

EvalWs eval_carve(void *base, int F, long long total_gt, long long ov_elems, int ncfg) {
    EvalWs w{};
    size_t nsc = (size_t)ncfg * (size_t)(total_gt > 0 ? total_gt : 1);
    cub::DeviceSegmentedRadixSort::SortKeysDescending((void *)nullptr, w.cub_bytes, (const double *)nullptr, (double *)nullptr,
                                                      (int)nsc, ncfg, (const int *)nullptr, (const int *)nullptr);
    char *p = (char *)base;
    size_t o = 0;
    auto take = [&](size_t b) { char *r = p + o; o += align_up(b); return (void *)r; };
    w.ov = (double *)take(sizeof(double) * (size_t)(ov_elems > 0 ? ov_elems : 1));
    w.scores = (double *)take(sizeof(double) * nsc);
    w.sorted = (double *)take(sizeof(double) * nsc);
    w.sim = (double *)take(sizeof(double) * (size_t)ncfg * kPts * (size_t)F);
    w.seg = (int *)take(sizeof(int) * (size_t)(ncfg + 1));
    w.n_tp = (int *)take(sizeof(int) * (size_t)ncfg * 2);
    w.n_valid = w.n_tp + ncfg;
    w.tpfp = (int *)take(sizeof(int) * (size_t)ncfg * kPts * 2);
    w.cub_tmp = take(w.cub_bytes > 0 ? w.cub_bytes : 1);
    w.bytes = o;
    return w;
}

bool frames_ok(const SessdKittiFrames *fr) {
    return fr && fr->num_frames > 0 && fr->gt_off && fr->gt && fr->gt_code && fr->gt_occluded && fr->dc_off && fr->dt_off &&
           fr->dt_cnt && fr->dt && fr->dt_code && fr->ov_off;
}

}  // namespace

size_t convert_ws_bytes(long long cap) { return align_up(sizeof(double) * kRec * (size_t)cap) + align_up(sizeof(int) * (size_t)cap); }

extern "C" size_t sessd_kitti_convert_workspace_bytes(long long capacity) { return capacity < 1 ? 0 : convert_ws_bytes(capacity); }

extern "C" int sessd_kitti_convert_detections(const float *d_boxes7, const float *d_scores, const int *d_labels, const int *d_off,
                                              int num_frames, long long capacity, const double *d_calib, const int *d_image_hw,
                                              const int *d_label_code, int num_labels, double *d_rec, int *d_label, int *d_code,
                                              int *d_cnt, void *workspace, size_t workspace_bytes, void *stream) {
    if (!d_boxes7 || !d_scores || !d_labels || !d_off || num_frames < 1 || capacity < 1 || !d_calib || !d_image_hw ||
        !d_label_code || num_labels < 1 || !d_rec || !d_label || !d_code || !d_cnt)
        return SESSD_EINVAL;
    if (!workspace || workspace_bytes < convert_ws_bytes(capacity)) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    double *stage = (double *)workspace;
    int *keep = (int *)((char *)workspace + align_up(sizeof(double) * kRec * (size_t)capacity));
    SESSD_LAUNCH(convert_kernel, num_frames, 128, 0, st, d_boxes7, d_scores, d_labels, d_off, num_frames, d_calib, d_image_hw,
                 stage, keep);
    SESSD_LAUNCH(compact_kernel, num_frames, 128, 0, st, d_off, keep, stage, d_labels, d_label_code, num_labels, d_rec, d_label,
                 d_code, d_cnt);
    return last_error();
}

extern "C" int sessd_kitti_overlaps(const SessdKittiFrames *frames, int metric, int z_axis, double z_center, double *d_overlaps,
                                    void *stream) {
    if (!frames_ok(frames) || metric < 0 || metric > 2 || z_axis < 0 || z_axis > 2 || !d_overlaps) return SESSD_EINVAL;
    SESSD_LAUNCH(overlaps_kernel, frames->num_frames, 128, 0, (cudaStream_t)stream, *frames, metric, z_axis, z_center, d_overlaps);
    return last_error();
}

extern "C" size_t sessd_kitti_eval_workspace_bytes(int num_frames, long long total_gt, long long overlap_elems, int num_configs,
                                                   int compute_aos) {
    if (num_frames < 1 || total_gt < 0 || overlap_elems < 0 || num_configs < 1) return 0;
    return eval_carve(nullptr, compute_aos ? num_frames : 0, total_gt, overlap_elems, num_configs).bytes;
}

extern "C" int sessd_kitti_eval(const SessdKittiFrames *frames, int max_frame_dt, int metric, int z_axis, double z_center, int num_configs,
                                const int *d_cfg, const double *d_min_overlap, int compute_aos, long long total_gt,
                                long long overlap_elems, double *d_thresholds, int *d_num_thresholds, double *d_precision,
                                double *d_aos, double *d_map, void *workspace, size_t workspace_bytes, void *stream) {
    if (!frames_ok(frames) || metric < 0 || metric > 2 || z_axis < 0 || z_axis > 2 || num_configs < 1 || !d_cfg || !d_min_overlap ||
        total_gt < 0 || total_gt > 0x7fffffff / num_configs || overlap_elems < 0 || !d_thresholds || !d_num_thresholds ||
        !d_precision || !d_aos || !d_map)
        return SESSD_EINVAL;
    if (max_frame_dt > kMaxDt) return SESSD_ECAPACITY;
    const int F = frames->num_frames;
    EvalWs w = eval_carve(workspace, compute_aos ? F : 0, total_gt, overlap_elems, num_configs);
    if (!workspace || workspace_bytes < w.bytes) return SESSD_EWORKSPACE;
    cudaStream_t st = (cudaStream_t)stream;
    const int ng = (int)(total_gt > 0 ? total_gt : 1);
    const long long nsc = (long long)num_configs * ng;
    SESSD_CUDA_TRY(cudaMemsetAsync(w.n_tp, 0, sizeof(int) * 2 * (size_t)num_configs, st));
    SESSD_CUDA_TRY(cudaMemsetAsync(w.tpfp, 0, sizeof(int) * 2 * kPts * (size_t)num_configs, st));
    SESSD_LAUNCH(overlaps_kernel, F, 128, 0, st, *frames, metric, z_axis, z_center, w.ov);
    SESSD_LAUNCH(fill_kernel, persistent_grid(nsc, 256), 256, 0, st, w.scores, nsc, -INFINITY);
    SESSD_LAUNCH(segments_kernel, div_up(num_configs + 1, 128), 128, 0, st, w.seg, num_configs, ng);
    const long long warps = (long long)num_configs * F;
    SESSD_LAUNCH(pass1_kernel, persistent_grid(warps * 32, 128, 16), 128, 0, st, *frames, w.ov, metric, num_configs, d_cfg,
                 d_min_overlap, ng, w.scores, w.n_tp, w.n_valid);
    size_t cb = w.cub_bytes;
    SESSD_CUDA_TRY(cub::DeviceSegmentedRadixSort::SortKeysDescending(w.cub_tmp, cb, w.scores, w.sorted, (int)nsc, num_configs, w.seg,
                                                                     w.seg + 1, 0, (int)(sizeof(double) * 8), st));
    ++::sessd::g_launches;
    SESSD_LAUNCH(thresholds_kernel, div_up(num_configs, 64), 64, 0, st, num_configs, ng, w.sorted, w.n_tp, w.n_valid, d_thresholds,
                 d_num_thresholds);
    SESSD_LAUNCH(pass2_kernel, persistent_grid(warps * 32, 128, 16), 128, 0, st, *frames, w.ov, metric, num_configs, d_cfg,
                 d_min_overlap, d_thresholds, d_num_thresholds, compute_aos, w.tpfp, w.sim);
    SESSD_LAUNCH(finish_kernel, num_configs, 64, 0, st, num_configs, F, d_num_thresholds, w.tpfp, w.sim, compute_aos, d_precision,
                 d_aos, d_map);
    return last_error();
}
