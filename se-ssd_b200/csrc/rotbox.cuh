// rotbox.cuh -- rotated-rectangle BEV overlap / IoU device functions (sm_90a).
//
// Same algorithm and fp32 operation order as the reference's box_overlap / iou_bev / iou_3d
// (det3d/core/iou3d/src/iou3d_kernel.cu:125-268, CPU twin iou3d_cpu.cpp:126-254): rotate the four corners of each
// box clockwise about its centre, collect the proper edge-edge crossings and the corners of one box lying inside
// the other (margin 1e-5), order the vertices by polar angle about their centroid and apply the shoelace fan.
// Files including this header are compiled with -fmad=false so that products and sums round exactly like the
// CPU twin (the oracle); the only remaining difference is CUDA's cosf/sinf/atan2f vs glibc's (<= 2 ulp).
// Implementation differences from the reference (results identical): polar angles are computed once per vertex
// instead of inside the sort comparator, and vertices live in a fixed 24-slot array (8 crossings + 8 corners
// is the geometric maximum; degenerate inputs are clamped instead of overrunning a 16-slot array).
#pragma once
#include <cuda_runtime.h>

namespace sessd {

constexpr float kRotEps = 1e-8f;

struct P2 { float x, y; };

__device__ __forceinline__ float rb_cross3(P2 p1, P2 p2, P2 p0) {
    return (p1.x - p0.x) * (p2.y - p0.y) - (p2.x - p0.x) * (p1.y - p0.y);
}

__device__ __forceinline__ P2 rb_spin(P2 c, float ca, float sa, P2 p) {
    P2 r;
    r.x = (p.x - c.x) * ca + (p.y - c.y) * sa + c.x;
    r.y = -(p.x - c.x) * sa + (p.y - c.y) * ca + c.y;
    return r;
}

__device__ __forceinline__ bool rb_seg_cross(P2 p1, P2 p0, P2 q1, P2 q0, P2 &out) {
    if (!(fminf(p0.x, p1.x) <= fmaxf(q0.x, q1.x) && fminf(q0.x, q1.x) <= fmaxf(p0.x, p1.x) &&
          fminf(p0.y, p1.y) <= fmaxf(q0.y, q1.y) && fminf(q0.y, q1.y) <= fmaxf(p0.y, p1.y)))
        return false;
    const float s1 = rb_cross3(q0, p1, p0);
    const float s2 = rb_cross3(p1, q1, p0);
    const float s3 = rb_cross3(p0, q1, q0);
    const float s4 = rb_cross3(q1, p1, q0);
    if (!(s1 * s2 > 0 && s3 * s4 > 0)) return false;
    const float s5 = rb_cross3(q1, p1, p0);
    if (fabsf(s5 - s1) > kRotEps) {
        out.x = (s5 * q0.x - s1 * q1.x) / (s5 - s1);
        out.y = (s5 * q0.y - s1 * q1.y) / (s5 - s1);
    } else {
        const float a0 = p0.y - p1.y, b0 = p1.x - p0.x, c0 = p0.x * p1.y - p1.x * p0.y;
        const float a1 = q0.y - q1.y, b1 = q1.x - q0.x, c1 = q0.x * q1.y - q1.x * q0.y;
        const float D = a0 * b1 - a1 * b0;
        out.x = (b0 * c1 - b1 * c0) / D;
        out.y = (a1 * c0 - a0 * c1) / D;
    }
    return true;
}

// box = [x1, y1, x2, y2] + angle; (cneg, sneg) = cos/sin of -angle
__device__ __forceinline__ bool rb_inside(float x1, float y1, float x2, float y2, float cneg, float sneg, P2 p) {
    const float margin = 1e-5f;
    const float cx = (x1 + x2) / 2, cy = (y1 + y2) / 2;
    const float rx = (p.x - cx) * cneg + (p.y - cy) * sneg + cx;
    const float ry = -(p.x - cx) * sneg + (p.y - cy) * cneg + cy;
    return rx > x1 - margin && rx < x2 + margin && ry > y1 - margin && ry < y2 + margin;
}

// overlap area of two rotated rectangles given as (x1, y1, x2, y2, angle)
__device__ inline float rot_overlap(float ax1, float ay1, float ax2, float ay2, float aang,
                                    float bx1, float by1, float bx2, float by2, float bang) {
    const P2 ca = {(ax1 + ax2) / 2, (ay1 + ay2) / 2};
    const P2 cb = {(bx1 + bx2) / 2, (by1 + by2) / 2};
    P2 A[5] = {{ax1, ay1}, {ax2, ay1}, {ax2, ay2}, {ax1, ay2}, {0, 0}};
    P2 B[5] = {{bx1, by1}, {bx2, by1}, {bx2, by2}, {bx1, by2}, {0, 0}};
    const float cosa = cosf(aang), sina = sinf(aang);
    const float cosb = cosf(bang), sinb = sinf(bang);
#pragma unroll
    for (int k = 0; k < 4; ++k) { A[k] = rb_spin(ca, cosa, sina, A[k]); B[k] = rb_spin(cb, cosb, sinb, B[k]); }
    A[4] = A[0]; B[4] = B[0];

    P2 poly[24];
    float ang[24];
    P2 ctr = {0.f, 0.f};
    int cnt = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            P2 x;
            if (rb_seg_cross(A[i + 1], A[i], B[j + 1], B[j], x)) {
                ctr.x = ctr.x + x.x; ctr.y = ctr.y + x.y;
                if (cnt < 24) poly[cnt++] = x;
            }
        }
    const float cna = cosf(-aang), sna = sinf(-aang);
    const float cnb = cosf(-bang), snb = sinf(-bang);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (rb_inside(ax1, ay1, ax2, ay2, cna, sna, B[k])) {
            ctr.x = ctr.x + B[k].x; ctr.y = ctr.y + B[k].y;
            if (cnt < 24) poly[cnt++] = B[k];
        }
        if (rb_inside(bx1, by1, bx2, by2, cnb, snb, A[k])) {
            ctr.x = ctr.x + A[k].x; ctr.y = ctr.y + A[k].y;
            if (cnt < 24) poly[cnt++] = A[k];
        }
    }
    if (cnt < 3) return 0.f;   // fewer than three vertices: the reference's fan sum is exactly 0 as well
    ctr.x /= cnt; ctr.y /= cnt;
    for (int k = 0; k < cnt; ++k) ang[k] = atan2f(poly[k].y - ctr.y, poly[k].x - ctr.x);
    // same bubble sort as the reference (:221-229): stable w.r.t. ties, so the vertex order is identical
    for (int j = 0; j < cnt - 1; ++j)
        for (int i = 0; i < cnt - j - 1; ++i)
            if (ang[i] > ang[i + 1]) {
                P2 t = poly[i]; poly[i] = poly[i + 1]; poly[i + 1] = t;
                float ta = ang[i]; ang[i] = ang[i + 1]; ang[i + 1] = ta;
            }
    float area = 0.f;
    for (int k = 0; k < cnt - 1; ++k) {
        const float ux = poly[k].x - poly[0].x, uy = poly[k].y - poly[0].y;
        const float vx = poly[k + 1].x - poly[0].x, vy = poly[k + 1].y - poly[0].y;
        area += ux * vy - uy * vx;
    }
    return fabsf(area) / 2.0f;
}

// ---- precomputed form: corners + trig evaluated once per box (bit-identical to rot_overlap: same expressions; uses
// cosf(-x) == cosf(x) and sinf(-x) == -sinf(x), which hold exactly for CUDA's implementations) ----------------------------
struct RotBox {
    float x1, y1, x2, y2;
    float c, s;          // cos / sin of the angle
    P2 corner[4];        // rotated corners, same order as the reference
};

__device__ __forceinline__ RotBox rot_prepare(float x1, float y1, float x2, float y2, float ang) {
    RotBox b;
    b.x1 = x1; b.y1 = y1; b.x2 = x2; b.y2 = y2;
    b.c = cosf(ang); b.s = sinf(ang);
    const P2 ctr = {(x1 + x2) / 2, (y1 + y2) / 2};
    const P2 raw[4] = {{x1, y1}, {x2, y1}, {x2, y2}, {x1, y2}};
#pragma unroll
    for (int k = 0; k < 4; ++k) b.corner[k] = rb_spin(ctr, b.c, b.s, raw[k]);
    return b;
}

__device__ inline float rot_overlap_pre(const RotBox &a, const RotBox &b) {
    P2 A[5], B[5];
#pragma unroll
    for (int k = 0; k < 4; ++k) { A[k] = a.corner[k]; B[k] = b.corner[k]; }
    A[4] = A[0]; B[4] = B[0];
    P2 poly[24];
    float ang[24];
    P2 ctr = {0.f, 0.f};
    int cnt = 0;
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            P2 x;
            if (rb_seg_cross(A[i + 1], A[i], B[j + 1], B[j], x)) {
                ctr.x = ctr.x + x.x; ctr.y = ctr.y + x.y;
                if (cnt < 24) poly[cnt++] = x;
            }
        }
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (rb_inside(a.x1, a.y1, a.x2, a.y2, a.c, -a.s, B[k])) {
            ctr.x = ctr.x + B[k].x; ctr.y = ctr.y + B[k].y;
            if (cnt < 24) poly[cnt++] = B[k];
        }
        if (rb_inside(b.x1, b.y1, b.x2, b.y2, b.c, -b.s, A[k])) {
            ctr.x = ctr.x + A[k].x; ctr.y = ctr.y + A[k].y;
            if (cnt < 24) poly[cnt++] = A[k];
        }
    }
    if (cnt < 3) return 0.f;
    ctr.x /= cnt; ctr.y /= cnt;
    for (int k = 0; k < cnt; ++k) ang[k] = atan2f(poly[k].y - ctr.y, poly[k].x - ctr.x);
    for (int j = 0; j < cnt - 1; ++j)
        for (int i = 0; i < cnt - j - 1; ++i)
            if (ang[i] > ang[i + 1]) {
                P2 t = poly[i]; poly[i] = poly[i + 1]; poly[i + 1] = t;
                float ta = ang[i]; ang[i] = ang[i + 1]; ang[i + 1] = ta;
            }
    float area = 0.f;
    for (int k = 0; k < cnt - 1; ++k) {
        const float ux = poly[k].x - poly[0].x, uy = poly[k].y - poly[0].y;
        const float vx = poly[k + 1].x - poly[0].x, vy = poly[k + 1].y - poly[0].y;
        area += ux * vy - uy * vx;
    }
    return fabsf(area) / 2.0f;
}

__device__ __forceinline__ float rot_iou_bev_pre(const RotBox &a, const RotBox &b) {
    const float sa = (a.x2 - a.x1) * (a.y2 - a.y1);
    const float sb = (b.x2 - b.x1) * (b.y2 - b.y1);
    const float so = rot_overlap_pre(a, b);
    return so / fmaxf(sa + sb - so, kRotEps);
}

__device__ __forceinline__ float rot_overlap5(const float *a, const float *b) {
    return rot_overlap(a[0], a[1], a[2], a[3], a[4], b[0], b[1], b[2], b[3], b[4]);
}

__device__ __forceinline__ float rot_iou_bev(const float *a, const float *b) {
    const float sa = (a[2] - a[0]) * (a[3] - a[1]);
    const float sb = (b[2] - b[0]) * (b[3] - b[1]);
    const float so = rot_overlap5(a, b);
    return so / fmaxf(sa + sb - so, kRotEps);
}

// boxes [x1,y1,z1,x2,y2,z2,angle]  (iou3d_kernel.cu:256-268)
__device__ __forceinline__ float rot_iou_3d(const float *a, const float *b) {
    const float va = (a[3] - a[0]) * (a[4] - a[1]) * (a[5] - a[2]);
    const float vb = (b[3] - b[0]) * (b[4] - b[1]) * (b[5] - b[2]);
    const float lo = fmaxf(a[2], b[2]);
    const float hi = fminf(a[5], b[5]);
    const float dh = fmaxf(hi - lo, kRotEps);
    if (dh == kRotEps) return 0.f;
    const float vo = rot_overlap(a[0], a[1], a[3], a[4], a[6], b[0], b[1], b[3], b[4], b[6]) * dh;
    return vo / fmaxf(va + vb - vo, kRotEps);
}

// axis-aligned IoU on [x1,y1,x2,y2,*]  (iou3d_kernel.cu:413-423)
__device__ __forceinline__ float axis_iou(const float *a, const float *b) {
    const float left = fmaxf(a[0], b[0]), right = fminf(a[2], b[2]);
    const float top = fmaxf(a[1], b[1]), bottom = fminf(a[3], b[3]);
    const float w = fmaxf(right - left, 0.f), h = fmaxf(bottom - top, 0.f);
    const float inter = w * h;
    const float sa = (a[2] - a[0]) * (a[3] - a[1]);
    const float sb = (b[2] - b[0]) * (b[3] - b[1]);
    return inter / fmaxf(sa + sb - inter, kRotEps);
}

}  // namespace sessd
