// augment.cuh -- the geometry that augment.cu (per-object noise, point pass) and gtaug.cu (GT-database sampling) share: the BEV corner-set
// collision predicate of box_collision_test and the fp64 box-frame membership test of points_in_rbbox.
//
// quads_collide / quad_contains are __host__ __device__: the device runs them in the noise selection and sessd_box_collision, the host in
// sessd_gtaug_select_host (GT-AUG's acceptance loop).  They are written with plain fp64 operators; every file that includes this header
// is compiled with -fmad=false for the device and -ffp-contract=off for the host (se-ssd_b200/build.py), so each operation is
// individually rounded on both sides and the two evaluate the same predicate bit for bit.
#pragma once
#include <math.h>

#include "common.cuh"

namespace sessd {

struct Quad { double x[4], y[4]; };

__host__ __device__ __forceinline__ Quad load_quad(const double *p) {   // [4][2] (x, y)
    Quad q;
#pragma unroll
    for (int k = 0; k < 4; ++k) { q.x[k] = p[2 * k]; q.y[k] = p[2 * k + 1]; }
    return q;
}

// the containment loop of box_collision_test: vec = -(a[k] - a[k+1]) (clockwise); cross = vec.y (a[k].x - p.x) - vec.x (a[k].y - p.y);
// a corner with cross >= 0 is not inside
__host__ __device__ __forceinline__ bool quad_contains(const Quad &a, const Quad &p) {
#pragma unroll
    for (int l = 0; l < 4; ++l)
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int k1 = (k + 1) & 3;
            const double vx = -(a.x[k] - a.x[k1]), vy = -(a.y[k] - a.y[k1]);
            double cross = vy * (a.x[k] - p.x[l]);
            cross = cross - vx * (a.y[k] - p.y[l]);
            if (cross >= 0.0) return false;
        }
    return true;
}

// box_collision_test for one (box, qbox) pair, clockwise = True, operation for operation
__host__ __device__ inline bool quads_collide(const Quad &b, const Quad &q) {
    double bx0 = b.x[0], bx1 = b.x[0], by0 = b.y[0], by1 = b.y[0], qx0 = q.x[0], qx1 = q.x[0], qy0 = q.y[0], qy1 = q.y[0];
#pragma unroll
    for (int k = 1; k < 4; ++k) {
        bx0 = fmin(bx0, b.x[k]); bx1 = fmax(bx1, b.x[k]); by0 = fmin(by0, b.y[k]); by1 = fmax(by1, b.y[k]);
        qx0 = fmin(qx0, q.x[k]); qx1 = fmax(qx1, q.x[k]); qy0 = fmin(qy0, q.y[k]); qy1 = fmax(qy1, q.y[k]);
    }
    const double iw = fmin(bx1, qx1) - fmax(bx0, qx0);
    if (!(iw > 0.0)) return false;
    const double ih = fmin(by1, qy1) - fmax(by0, qy0);
    if (!(ih > 0.0)) return false;
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const int k1 = (k + 1) & 3;
        const double ax = b.x[k], ay = b.y[k], bbx = b.x[k1], bby = b.y[k1];
#pragma unroll
        for (int l = 0; l < 4; ++l) {
            const int l1 = (l + 1) & 3;
            const double cx = q.x[l], cy = q.y[l], dx = q.x[l1], dy = q.y[l1];
            const bool acd = (dy - ay) * (cx - ax) > (cy - ay) * (dx - ax);
            const bool bcd = (dy - bby) * (cx - bbx) > (cy - bby) * (dx - bbx);
            if (acd != bcd) {
                const bool abc = (cy - ay) * (bbx - ax) > (bby - ay) * (cx - ax);
                const bool abd = (dy - ay) * (bbx - ax) > (bby - ay) * (dx - ax);
                if (abc != abd) return true;
            }
        }
    }
    // box contains qbox, then qbox contains box (each corner of one strictly on the inner side of every edge of the other)
    return quad_contains(b, q) || quad_contains(q, b);
}

// The membership frame of one box: points_in_convex_polygon_3d_jit over the faces of center_to_corner_box3d(origin 0.5) holds the same
// points as |R^T (p - c)| < dims / 2 everywhere except within rounding of a face; evaluated in fp64 from the box, w and l enlarged by
// the context (noise_per_object_v4_'s offset[2:5]).  T is the box's own type: fp32 for the frame's boxes (point pass,
// sessd_points_in_boxes), fp64 for GT-AUG's database boxes (points_in_rbbox of the sampled box3d_lidar, sessd_gtaug_paste).
template <typename T>
struct MemberFrame {
    T cx, cy, cz;
    double mc, ms;             // cos / sin of the box angle
    double hx, hy, hz;         // half extents
};

template <typename T>
__device__ __forceinline__ MemberFrame<T> member_frame(const T *p, double add) {
    MemberFrame<T> f;
    f.cx = p[0]; f.cy = p[1]; f.cz = p[2];
    const double r = (double)p[6];
    f.mc = cos(r); f.ms = sin(r);
    f.hx = __dmul_rn(__dadd_rn((double)p[3], add), 0.5); f.hy = __dmul_rn(__dadd_rn((double)p[4], add), 0.5);
    f.hz = __dmul_rn((double)p[5], 0.5);
    return f;
}

template <typename T>
__device__ __forceinline__ bool in_frame(float x, float y, float z, const MemberFrame<T> &f) {
    const double dx = __dsub_rn((double)x, (double)f.cx), dy = __dsub_rn((double)y, (double)f.cy);
    const double dz = __dsub_rn((double)z, (double)f.cz);
    const double lx = __dsub_rn(__dmul_rn(dx, f.mc), __dmul_rn(dy, f.ms));
    const double ly = __dadd_rn(__dmul_rn(dx, f.ms), __dmul_rn(dy, f.mc));
    return fabs(lx) < f.hx && fabs(ly) < f.hy && fabs(dz) < f.hz;
}

// the fp32 BLAS chain of `p @ [[c, -s, 0], [s, c, 0], [0, 0, 1]]` (1x3 @ 3x3 and N x 3 @ 3x3 gemm, see oracle/augment_ref.py)
__device__ __forceinline__ void rot32(float &x, float &y, float &z, float c, float s) {
    const float x0 = x, y0 = y, z0 = z;
    x = __fmaf_rn(z0, 0.f, __fmaf_rn(y0, s, __fmul_rn(x0, c)));
    y = __fmaf_rn(z0, 0.f, __fmaf_rn(y0, c, __fmul_rn(x0, -s)));
    z = __fmaf_rn(z0, 1.f, __fmaf_rn(y0, 0.f, __fmul_rn(x0, 0.f)));
}

// box3d_transform_ of one valid box v [7] (fp32) by its selected try t (-1: unmoved): centre and angle plus the fp64 noise, rounded once
__device__ __forceinline__ void box_noise(float *v, const double *loc_noise, const double *rot_noise, int num_try, size_t bj, int t) {
    if (t < 0) return;
    const double *l = loc_noise + (bj * num_try + t) * 3;
    v[0] = (float)__dadd_rn((double)v[0], l[0]); v[1] = (float)__dadd_rn((double)v[1], l[1]);
    v[2] = (float)__dadd_rn((double)v[2], l[2]);
    v[6] = (float)__dadd_rn((double)v[6], rot_noise[bj * num_try + t]);
}

// random_flip_v2 -> global_rotation_v3 -> global_scaling_v3 on one box w [7]: g = {cos, sin, scale, flip, angle} (fp32, from the host)
__device__ __forceinline__ void box_global(float *w, const float *g) {
    const float kPi = 3.14159274101257324f;                  // float32(np.pi)
    if (g[3] != 0.f) { w[1] = -w[1]; w[6] = __fadd_rn(-w[6], kPi); }
    rot32(w[0], w[1], w[2], g[0], g[1]);
    w[6] = __fadd_rn(w[6], g[4]);
#pragma unroll
    for (int c = 0; c < 6; ++c) w[c] = __fmul_rn(w[c], g[2]);
}

}  // namespace sessd
