// sada.cu -- shape-aware data augmentation (SA-DA) of SE-SSD's training frames on the GPU: pyramid dropout, farthest-point sparsify and
// pyramid swap of one frame (reference: det3d/datasets/utils/sa_da_v2.py, pyramid_augment_v0, get_pyramids, points_in_pyramids_mask).
//
// Every random draw is made on the host (sessd_b200/sada.py); the kernels are pure functions of the points, the pyramids and the lists of
// pyramids each stage acts on (the boxes pyramid_augment_v0 receives come from sessd_augment_boxes).  The building blocks:
//   pyramids_kernel      -- get_pyramids (apex = box centre, base = one face of center_to_corner_box3d(origin 0.5)) and the 5 face planes
//                           of each pyramid as surface_equ_3d_jitv2 computes them, once per pyramid.
//   member_kernel        -- per point, a bit set over a list of pyramid ids (points_in_convex_polygon_3d_jit: sign >= 0 is outside) and
//                           the count of each listed pyramid.
//   sessd_sada_compact   -- order-preserving removal of the points inside the listed pyramids whose count passes a threshold: one
//                           device_scan (common.cuh) of the kept flags whose store writes each kept row.
//   fps_kernel           -- one CTA per listed pyramid that passes the threshold: its points in row order, exact farthest-point sampling
//                           (start at row 0, fp64 distances, ties to the lowest row), the picks written in pick order after the kept rows.
//   swap_kernel          -- one CTA per pair: get_points_ratio / recover_points_by_ratio and the min / max intensity transform.
//   shuffle_kernel       -- the batch's point shuffle after SA-DA.
//
// Precision: the boxes are fp32, so is every pyramid, plane and ratio; each operation is individually rounded (the file is compiled with
// -fmad=false) in the reference's order: numpy reduces 3-element sums left to right, einsum's rotation is c0 cos + c1 sin.  The fp32
// sin / cos of a box angle are the correctly rounded values (fp32 of CUDA's fp64 functions); numpy's SIMD float32 sin / cos can differ by
// an ulp (see DESIGN §7).
#include <cub/block/block_reduce.cuh>
#include <cub/block/block_scan.cuh>

#include "augment.cuh"

namespace sessd {

constexpr int kSadaThreads = 256;
constexpr int kSadaMaxBoxes = 256;             // SESSD_AUGMENT_MAX_GT
constexpr int kSadaMaxIds = 6 * kSadaMaxBoxes;  // SESSD_SADA_MAX_IDS
constexpr int kFpsThreads = 512;
constexpr int kFpsSmemPoints = 4096;           // points a CTA gathers into shared memory (20 B each); larger pyramids stay in global

// ------------------------------------------------------------------------------------------------ pyramids
// get_pyramids' face orders: corners of center_to_corner_box3d (0 (-,-,-) 1 (-,-,+) 2 (-,+,+) 3 (-,+,-) 4 (+,-,-) 5 (+,-,+) 6 (+,+,+)
// 7 (+,+,-) in (w, l, h)); points_in_pyramids_mask's surfaces over the 5 pyramid points (0 = apex) are (1 2 0) (2 3 0) (3 4 0) (4 1 0)
// (4 3 2)
__constant__ int c_face[6][4] = {{0, 1, 5, 4}, {4, 5, 6, 7}, {7, 6, 2, 3}, {3, 2, 1, 0}, {1, 2, 6, 5}, {0, 4, 7, 3}};

// surface_equ_3d_jitv2 of the surface (A, B, C): normal (A - B) x (B - C), offset -A . normal (left to right)
__device__ __forceinline__ void face_plane(const float *A, const float *B, const float *C, float *pl) {
    const float u0 = __fsub_rn(A[0], B[0]), u1 = __fsub_rn(A[1], B[1]), u2 = __fsub_rn(A[2], B[2]);
    const float v0 = __fsub_rn(B[0], C[0]), v1 = __fsub_rn(B[1], C[1]), v2 = __fsub_rn(B[2], C[2]);
    const float n0 = __fsub_rn(__fmul_rn(u1, v2), __fmul_rn(u2, v1));
    const float n1 = __fsub_rn(__fmul_rn(u2, v0), __fmul_rn(u0, v2));
    const float n2 = __fsub_rn(__fmul_rn(u0, v1), __fmul_rn(u1, v0));
    pl[0] = n0; pl[1] = n1; pl[2] = n2;
    pl[3] = __fsub_rn(__fsub_rn(__fmul_rn(-A[0], n0), __fmul_rn(A[1], n1)), __fmul_rn(A[2], n2));
}

__global__ void __launch_bounds__(kSadaThreads) pyramids_kernel(const float *__restrict__ boxes, int num_boxes, float *__restrict__ pyramids,
                                                                float *__restrict__ planes) {
    const int t = blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= num_boxes * 6) return;
    const int i = t / 6, f = t % 6;
    const float *bx = boxes + 7 * (size_t)i;
    const double a = (double)bx[6];
    const float s = (float)sin(a), c = (float)cos(a);
    float P[5][3];
    P[0][0] = bx[0]; P[0][1] = bx[1]; P[0][2] = bx[2];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
        const int k = c_face[f][q];
        const float sx = k >= 4 ? 0.5f : -0.5f, sy = (k & 3) == 2 || (k & 3) == 3 ? 0.5f : -0.5f, sz = k == 1 || k == 2 || k == 5 || k == 6 ? 0.5f : -0.5f;
        const float cx = __fmul_rn(bx[3], sx), cy = __fmul_rn(bx[4], sy), cz = __fmul_rn(bx[5], sz);
        P[q + 1][0] = __fadd_rn(__fadd_rn(__fmul_rn(cx, c), __fmul_rn(cy, s)), bx[0]);
        P[q + 1][1] = __fadd_rn(__fadd_rn(__fmul_rn(cx, -s), __fmul_rn(cy, c)), bx[1]);
        P[q + 1][2] = __fadd_rn(cz, bx[2]);
    }
    float *pyr = pyramids + 15 * (size_t)t;
#pragma unroll
    for (int q = 0; q < 5; ++q) { pyr[3 * q] = P[q][0]; pyr[3 * q + 1] = P[q][1]; pyr[3 * q + 2] = P[q][2]; }
    float *pl = planes + 20 * (size_t)t;
    face_plane(P[1], P[2], P[0], pl);
    face_plane(P[2], P[3], P[0], pl + 4);
    face_plane(P[3], P[4], P[0], pl + 8);
    face_plane(P[4], P[1], P[0], pl + 12);
    face_plane(P[4], P[3], P[2], pl + 16);
}

// ------------------------------------------------------------------------------------------------ membership
__device__ __forceinline__ bool in_pyramid(float x, float y, float z, const float *__restrict__ pl) {
#pragma unroll
    for (int k = 0; k < 5; ++k) {
        const float sgn = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(x, pl[4 * k]), __fmul_rn(y, pl[4 * k + 1])), __fmul_rn(z, pl[4 * k + 2])),
                                    pl[4 * k + 3]);
        if (sgn >= 0.f) return false;
    }
    return true;
}

// the rows a stage reads: *d_n (a count left on the device by the stage before) clamped to the buffer's n, or n
__device__ __forceinline__ int rows_of(int n, const int *d_n) { return d_n ? min(max(*d_n, 0), n) : n; }

// bits [n][words] (optional) and counts [num_ids]; an id outside [0, num_pyramids) holds no point
__global__ void __launch_bounds__(kSadaThreads) member_kernel(const float *__restrict__ points, int n, const int *__restrict__ d_n,
                                                              const float *__restrict__ planes,
                                                              int num_pyramids, const int *__restrict__ ids, int num_ids, int words,
                                                              uint32_t *__restrict__ bits, int *__restrict__ counts) {
    extern __shared__ int s_count[];
    n = rows_of(n, d_n);
    for (int a = threadIdx.x; a < num_ids; a += blockDim.x) s_count[a] = 0;
    __syncthreads();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const float4 p = reinterpret_cast<const float4 *>(points)[i];
        for (int w = 0; w < words; ++w) {
            uint32_t word = 0;
            for (int a = 32 * w; a < min(num_ids, 32 * w + 32); ++a) {
                const int id = ids[a];
                if ((unsigned)id < (unsigned)num_pyramids && in_pyramid(p.x, p.y, p.z, planes + 20 * (size_t)id)) {
                    word |= 1u << (a & 31);
                    atomicAdd(&s_count[a], 1);
                }
            }
            if (bits) bits[(size_t)i * words + w] = word;
        }
    }
    __syncthreads();
    for (int a = threadIdx.x; a < num_ids; a += blockDim.x)
        if (s_count[a]) atomicAdd(&counts[a], s_count[a]);
}

// the listed pyramids that act: count > min_count (min_count < 0: every listed pyramid)
__device__ __forceinline__ bool removed(const uint32_t *__restrict__ bits, size_t i, int words, int num_ids, const int *__restrict__ counts,
                                        int min_count) {
    for (int w = 0; w < words; ++w) {
        uint32_t word = bits[i * words + w];
        while (word) {
            const int a = 32 * w + __ffs(word) - 1;
            word &= word - 1;
            if (a < num_ids && counts[a] > min_count) return true;
        }
    }
    return false;
}

// sessd_sada_compact as a device_scan: the flag of a row is "not removed", the store writes each kept row to its rank
struct NotRemoved {
    const uint32_t *bits;
    int words, num_ids, min_count;
    const int *counts;
    __device__ __forceinline__ int operator()(long long i) const { return !removed(bits, (size_t)i, words, num_ids, counts, min_count); }
};
struct StoreKept {
    const float *points;
    float *out;
    int capacity;
    __device__ __forceinline__ void operator()(long long i, int ex, int v) const {
        if (v && ex < capacity) reinterpret_cast<float4 *>(out)[ex] = reinterpret_cast<const float4 *>(points)[i];
    }
};

// ------------------------------------------------------------------------------------------------ members of one listed pyramid, in row order
// Calls f(rank, row) for every point whose bit a is set, rank = its position among them.  One CTA walks the frame in blockDim rounds.
template <int kThreads, class F>
__device__ __forceinline__ void for_members(const uint32_t *__restrict__ bits, int n, int words, int a, F f) {
    using Scan = cub::BlockScan<int, kThreads>;
    __shared__ typename Scan::TempStorage s_scan;
    int carry = 0;
    for (int c = 0; c < n; c += kThreads) {
        const int i = c + threadIdx.x;
        const int in = i < n ? (int)((bits[(size_t)i * words + (a >> 5)] >> (a & 31)) & 1u) : 0;
        int pos, tot;
        Scan(s_scan).ExclusiveSum(in, pos, tot);
        if (in) f(carry + pos, i);
        carry += tot;
        __syncthreads();
    }
}

// ------------------------------------------------------------------------------------------------ farthest-point sampling
struct Best { double d; int i; };

__device__ __forceinline__ Best better(Best x, Best y) { return (y.d > x.d || (y.d == x.d && y.i < x.i)) ? y : x; }

__global__ void __launch_bounds__(kFpsThreads, 1) fps_kernel(const float *__restrict__ points, int n, const int *__restrict__ d_n, const uint32_t *__restrict__ bits,
                                                          int words, int num_ids, const int *__restrict__ counts, int min_count, int k,
                                                          float *__restrict__ g_xyz, double *__restrict__ g_dist, int *__restrict__ g_row,
                                                          float *__restrict__ out, int capacity, int *__restrict__ num) {
    extern __shared__ __align__(16) unsigned char s_raw[];
    __shared__ Best s_best[kFpsThreads / 32];
    __shared__ int s_pick;
    const int a = blockIdx.x;
    const int m = counts[a];
    const int cap = n;                                              // the workspace holds n rows per listed pyramid
    n = rows_of(n, d_n);
    if (m <= min_count) return;
    int rank = 0;                                                   // valid pyramids before this one: its block of k output rows
    for (int q = 0; q < a; ++q) rank += counts[q] > min_count;
    const int base = num[0] + rank * k;
    const bool smem = m <= kFpsSmemPoints;
    if (m > cap) return;                                            // counts not made over these rows
    double *dist = smem ? reinterpret_cast<double *>(s_raw) : g_dist + (size_t)a * n;
    float *xyz = smem ? reinterpret_cast<float *>(s_raw + sizeof(double) * kFpsSmemPoints) : g_xyz + (size_t)a * n * 3;
    int *row = smem ? reinterpret_cast<int *>(s_raw + (sizeof(double) + 3 * sizeof(float)) * kFpsSmemPoints) : g_row + (size_t)a * n;
    for_members<kFpsThreads>(bits, n, words, a, [&](int r, int i) {
        if (r >= m) return;
        const float4 p = reinterpret_cast<const float4 *>(points)[i];
        xyz[3 * r] = p.x; xyz[3 * r + 1] = p.y; xyz[3 * r + 2] = p.z;
        dist[r] = INFINITY;
        row[r] = i;
    });
    __syncthreads();
    int pick = 0;
    for (int s = 0; s < k; ++s) {
        if (threadIdx.x == 0 && base + s < capacity)
            reinterpret_cast<float4 *>(out)[base + s] = reinterpret_cast<const float4 *>(points)[row[pick]];
        if (s + 1 == k) break;
        const double px = xyz[3 * pick], py = xyz[3 * pick + 1], pz = xyz[3 * pick + 2];
        Best b = {-1.0, 0x7fffffff};
        for (int r = threadIdx.x; r < m; r += kFpsThreads) {
            const double dx = __dsub_rn((double)xyz[3 * r], px), dy = __dsub_rn((double)xyz[3 * r + 1], py),
                         dz = __dsub_rn((double)xyz[3 * r + 2], pz);
            const double d = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(dx, dx), __dmul_rn(dy, dy)), __dmul_rn(dz, dz)));
            const double md = fmin(dist[r], d);
            dist[r] = md;
            b = better(b, Best{md, r});
        }
#pragma unroll
        for (int o = 16; o; o >>= 1) b = better(b, Best{__shfl_xor_sync(0xffffffffu, b.d, o), __shfl_xor_sync(0xffffffffu, b.i, o)});
        if ((threadIdx.x & 31) == 0) s_best[threadIdx.x >> 5] = b;
        __syncthreads();
        if (threadIdx.x == 0) {
            Best t = s_best[0];
            for (int w = 1; w < kFpsThreads / 32; ++w) t = better(t, s_best[w]);
            s_pick = t.i;
        }
        __syncthreads();
        pick = s_pick;
    }
}

// the frame's size after sparsify: kept rows + k per valid pyramid
__global__ void fps_total_kernel(int num_ids, const int *__restrict__ counts, int min_count, int k, int *__restrict__ num) {
    int v = 0;
    for (int a = 0; a < num_ids; ++a) v += counts[a] > min_count;
    num[0] += v * k;
}

// ------------------------------------------------------------------------------------------------ swap
struct Ratio { float p1[3], v0[3], v1[3], v2[3], sc[3], n0, n1, n2; };

// get_points_ratio's constants of one pyramid [15]: surface centre ((p1 + p2) + p3) + p4) / 4, vectors and their squared norms
__device__ __forceinline__ Ratio ratio_of(const float *__restrict__ q) {
    Ratio r;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        r.p1[c] = q[3 + c];
        r.sc[c] = __fdiv_rn(__fadd_rn(__fadd_rn(__fadd_rn(q[3 + c], q[6 + c]), q[9 + c]), q[12 + c]), 4.0f);
        r.v0[c] = __fsub_rn(q[6 + c], q[3 + c]);
        r.v1[c] = __fsub_rn(q[12 + c], q[3 + c]);
        r.v2[c] = __fsub_rn(q[c], r.sc[c]);
    }
    auto sq = [](const float *v) { return __fadd_rn(__fadd_rn(__fmul_rn(v[0], v[0]), __fmul_rn(v[1], v[1])), __fmul_rn(v[2], v[2])); };
    r.n0 = sq(r.v0); r.n1 = sq(r.v1); r.n2 = sq(r.v2);
    return r;
}

__device__ __forceinline__ float dot3(float x, float y, float z, const float *o, const float *v) {
    return __fadd_rn(__fadd_rn(__fmul_rn(__fsub_rn(x, o[0]), v[0]), __fmul_rn(__fsub_rn(y, o[1]), v[1])), __fmul_rn(__fsub_rn(z, o[2]), v[2]));
}

// a point of pyramid `from` re-expressed in pyramid `to`; its intensity through the min / max ratio of the two sets
__device__ __forceinline__ float4 transfer(float4 p, const Ratio &from, const Ratio &to, float lo_from, float span_from, float lo_to,
                                           float range_to) {
    const float al = __fdiv_rn(dot3(p.x, p.y, p.z, from.p1, from.v0), from.n0);
    const float be = __fdiv_rn(dot3(p.x, p.y, p.z, from.p1, from.v1), from.n1);
    const float ga = __fdiv_rn(dot3(p.x, p.y, p.z, from.sc, from.v2), from.n2);
    float o[3];
#pragma unroll
    for (int c = 0; c < 3; ++c)
        o[c] = __fadd_rn(__fadd_rn(__fadd_rn(__fmul_rn(al, to.v0[c]), __fmul_rn(be, to.v1[c])), to.p1[c]), __fmul_rn(ga, to.v2[c]));
    const float ratio = __fdiv_rn(__fsub_rn(p.w, lo_from), span_from);
    return make_float4(o[0], o[1], o[2], __fadd_rn(__fmul_rn(ratio, range_to), lo_to));
}

// one CTA per pair p: list entries p (to_swap) and num_pairs + p (swapped)
__global__ void __launch_bounds__(kSadaThreads) swap_kernel(const float *__restrict__ points, int n, const int *__restrict__ d_n, const uint32_t *__restrict__ bits,
                                                            int words, int num_pairs, const int *__restrict__ counts,
                                                            const float *__restrict__ pyramids, int num_pyramids, const int *__restrict__ ids,
                                                            float *__restrict__ out, int capacity, const int *__restrict__ num_in,
                                                            int *__restrict__ num_out) {
    using Reduce = cub::BlockReduce<float, kSadaThreads>;
    __shared__ typename Reduce::TempStorage s_red;
    __shared__ float s_mm[4];
    const int p = blockIdx.x, q = num_pairs + p;
    n = rows_of(n, d_n);
    int base = num_in[0];
    for (int t = 0; t < p; ++t) base += counts[t] + counts[num_pairs + t];
    if (p == num_pairs - 1 && threadIdx.x == 0) *num_out = base + counts[p] + counts[q];
    const int ia = ids[p], ib = ids[q];
    if ((unsigned)ia >= (unsigned)num_pyramids || (unsigned)ib >= (unsigned)num_pyramids) return;   // such ids hold no points
    // the min / max intensity of each set (exact: order does not matter)
    float mn[2] = {INFINITY, INFINITY}, mx[2] = {-INFINITY, -INFINITY};
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
        const uint32_t *bw = bits + (size_t)i * words;
        const float w = points[4 * (size_t)i + 3];
        if ((bw[p >> 5] >> (p & 31)) & 1u) { mn[0] = fminf(mn[0], w); mx[0] = fmaxf(mx[0], w); }
        if ((bw[q >> 5] >> (q & 31)) & 1u) { mn[1] = fminf(mn[1], w); mx[1] = fmaxf(mx[1], w); }
    }
#pragma unroll
    for (int s = 0; s < 2; ++s) {
        const float a = Reduce(s_red).Reduce(mn[s], [](float x, float y) { return fminf(x, y); });
        __syncthreads();
        const float b = Reduce(s_red).Reduce(mx[s], [](float x, float y) { return fmaxf(x, y); });
        __syncthreads();
        if (threadIdx.x == 0) { s_mm[2 * s] = a; s_mm[2 * s + 1] = b; }
    }
    __syncthreads();
    const float lo_a = s_mm[0], hi_a = s_mm[1], lo_b = s_mm[2], hi_b = s_mm[3];
    const float rng_a = __fsub_rn(hi_a, lo_a), rng_b = __fsub_rn(hi_b, lo_b);
    // np.clip(max - min, 1e-6, 1) in fp32
    const float span_a = fminf(fmaxf(rng_a, 9.99999997e-07f), 1.0f), span_b = fminf(fmaxf(rng_b, 9.99999997e-07f), 1.0f);
    const Ratio ra = ratio_of(pyramids + 15 * (size_t)ia), rb = ratio_of(pyramids + 15 * (size_t)ib);
    const int cb = counts[q];
    // new_to_swap: the swapped set's points in the to_swap pyramid, then new_swapped: the to_swap set's points in the swapped pyramid
    for_members<kSadaThreads>(bits, n, words, q, [&](int r, int i) {
        if (r < cb && base + r < capacity)
            reinterpret_cast<float4 *>(out)[base + r] = transfer(reinterpret_cast<const float4 *>(points)[i], rb, ra, lo_b, span_b, lo_a, rng_a);
    });
    const int ca = counts[p];
    for_members<kSadaThreads>(bits, n, words, p, [&](int r, int i) {
        if (r < ca && base + cb + r < capacity)
            reinterpret_cast<float4 *>(out)[base + cb + r] = transfer(reinterpret_cast<const float4 *>(points)[i], ra, rb, lo_a, span_a, lo_b,
                                                                      rng_b);
    });
}

// ------------------------------------------------------------------------------------------------ shuffle
__global__ void __launch_bounds__(kSadaThreads) shuffle_kernel(const float *__restrict__ points, const int *__restrict__ frame_off,
                                                               const int *__restrict__ perm, float *__restrict__ out) {
    const int b = blockIdx.y;
    const int off = frame_off[b], np = frame_off[b + 1] - off;
    for (int k = blockIdx.x * blockDim.x + threadIdx.x; k < np; k += gridDim.x * blockDim.x) {
        const int src = perm[off + k];
        if ((unsigned)src >= (unsigned)np) continue;     // not a frame-local permutation: the row is left unwritten
        reinterpret_cast<float4 *>(out)[off + k] = reinterpret_cast<const float4 *>(points)[off + src];
    }
}

}  // namespace sessd

using namespace sessd;

static bool misaligned(const void *p) { return ((uintptr_t)p) & 15; }

extern "C" int sessd_sada_pyramids(const float *d_boxes, int num_boxes, float *d_pyramids, float *d_planes, void *stream) {
    if (num_boxes < 0 || !d_boxes || !d_pyramids || !d_planes) return SESSD_EINVAL;
    if (num_boxes > kSadaMaxIds / 6) return SESSD_ECAPACITY;
    if (num_boxes == 0) return SESSD_OK;
    SESSD_LAUNCH(pyramids_kernel, div_up(num_boxes * 6, kSadaThreads), kSadaThreads, 0, (cudaStream_t)stream, d_boxes, num_boxes, d_pyramids,
                 d_planes);
    return last_error();
}

extern "C" int sessd_sada_membership(const float *d_points, int n, const int *d_n, const float *d_planes, int num_pyramids, const int *d_ids, int num_ids,
                                     uint32_t *d_bits, int *d_counts, void *stream) {
    if (n < 0 || num_pyramids < 0 || num_ids < 0 || !d_counts) return SESSD_EINVAL;
    if ((n > 0 && !d_points) || (num_ids > 0 && !d_ids) || (num_pyramids > 0 && !d_planes)) return SESSD_EINVAL;
    if (misaligned(d_points)) return SESSD_EINVAL;
    if (num_ids > kSadaMaxIds) return SESSD_ECAPACITY;
    cudaStream_t st = (cudaStream_t)stream;
    if (num_ids == 0) return SESSD_OK;
    SESSD_CUDA_TRY(cudaMemsetAsync(d_counts, 0, sizeof(int) * num_ids, st));
    if (n == 0) return SESSD_OK;
    const int words = div_up(num_ids, 32);
    SESSD_LAUNCH(member_kernel, std::min(div_up(n, kSadaThreads), 1024), kSadaThreads, sizeof(int) * num_ids, st, d_points, n, d_n,
                 d_planes, num_pyramids, d_ids, num_ids, words, d_bits, d_counts);
    return last_error();
}

extern "C" size_t sessd_sada_compact_workspace_bytes(int n) { return n < 0 ? 0 : scan_scratch_bytes(n); }

extern "C" int sessd_sada_compact(const float *d_points, int n, const int *d_n, const uint32_t *d_bits, int num_ids, const int *d_counts, int min_count,
                                  void *d_workspace, size_t workspace_bytes, float *d_out, int capacity, int *d_num_out, void *stream) {
    if (n < 0 || num_ids < 0 || capacity < 0 || !d_num_out || !d_workspace || !d_out) return SESSD_EINVAL;
    if ((n > 0 && !d_points) || (n > 0 && num_ids > 0 && (!d_bits || !d_counts))) return SESSD_EINVAL;
    if (misaligned(d_points) || misaligned(d_out)) return SESSD_EINVAL;
    if (num_ids > kSadaMaxIds) return SESSD_ECAPACITY;
    if (workspace_bytes < scan_scratch_bytes(n)) return SESSD_EWORKSPACE;
    if (capacity < n) return SESSD_ECAPACITY;
    // the rows: *d_n (clamped to [0, n] by the scan) or n
    device_scan(NotRemoved{d_bits, div_up(num_ids, 32), num_ids, min_count, d_counts}, StoreKept{d_points, d_out, capacity}, d_n, d_n ? 1 : n,
                n, (int *)d_workspace, d_num_out, (cudaStream_t)stream);
    return last_error();
}

extern "C" size_t sessd_sada_fps_workspace_bytes(int n, int num_ids) {
    if (n < 0 || num_ids < 0) return 0;
    return (size_t)n * num_ids * (3 * sizeof(float) + sizeof(double) + sizeof(int)) + 16;
}

extern "C" int sessd_sada_fps(const float *d_points, int n, const int *d_n, const uint32_t *d_bits, int num_ids, const int *d_counts, int min_count, int k,
                              void *d_workspace, size_t workspace_bytes, float *d_out, int capacity, int *d_num, void *stream) {
    if (n < 0 || num_ids < 0 || k <= 0 || min_count < k - 1 || capacity < 0 || !d_num || !d_out) return SESSD_EINVAL;
    if (num_ids > 0 && n > 0 && (!d_points || !d_bits || !d_counts || !d_workspace)) return SESSD_EINVAL;
    if (misaligned(d_points) || misaligned(d_out) || misaligned(d_workspace)) return SESSD_EINVAL;
    if (num_ids > kSadaMaxIds) return SESSD_ECAPACITY;
    if (workspace_bytes < sessd_sada_fps_workspace_bytes(n, num_ids)) return SESSD_EWORKSPACE;
    if ((long long)capacity < (long long)n + (long long)k * num_ids) return SESSD_ECAPACITY;
    if (num_ids == 0 || n == 0) return SESSD_OK;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t smem = (sizeof(double) + 3 * sizeof(float) + sizeof(int)) * kFpsSmemPoints;
    SESSD_CUDA_TRY(cudaFuncSetAttribute(fps_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    char *w = (char *)d_workspace;
    double *g_dist = (double *)w;
    float *g_xyz = (float *)(w + sizeof(double) * (size_t)n * num_ids);
    int *g_row = (int *)(w + (sizeof(double) + 3 * sizeof(float)) * (size_t)n * num_ids);
    SESSD_LAUNCH(fps_kernel, num_ids, kFpsThreads, smem, st, d_points, n, d_n, d_bits, div_up(num_ids, 32), num_ids, d_counts, min_count, k,
                 g_xyz, g_dist, g_row, d_out, capacity, d_num);
    SESSD_LAUNCH(fps_total_kernel, 1, 1, 0, st, num_ids, d_counts, min_count, k, d_num);
    return last_error();
}

extern "C" int sessd_sada_swap(const float *d_points, int n, const int *d_n, const uint32_t *d_bits, int num_pairs, const int *d_counts,
                               const float *d_pyramids, int num_pyramids, const int *d_ids, int max_swap_points, float *d_out, int capacity,
                               const int *d_num_in, int *d_num_out, void *stream) {
    if (n < 0 || num_pairs < 0 || num_pyramids < 0 || max_swap_points < 0 || capacity < 0 || !d_num_in || !d_num_out || !d_out)
        return SESSD_EINVAL;
    if (num_pairs > 0 && (!d_bits || !d_counts || !d_pyramids || !d_ids || (n > 0 && !d_points))) return SESSD_EINVAL;
    if (misaligned(d_points) || misaligned(d_out)) return SESSD_EINVAL;
    if (2 * num_pairs > kSadaMaxIds) return SESSD_ECAPACITY;
    if ((long long)capacity < (long long)n + max_swap_points) return SESSD_ECAPACITY;
    cudaStream_t st = (cudaStream_t)stream;
    if (num_pairs == 0) {
        SESSD_CUDA_TRY(cudaMemcpyAsync(d_num_out, d_num_in, sizeof(int), cudaMemcpyDeviceToDevice, st));
        return SESSD_OK;
    }
    SESSD_LAUNCH(swap_kernel, num_pairs, kSadaThreads, 0, st, d_points, n, d_n, d_bits, div_up(2 * num_pairs, 32), num_pairs, d_counts, d_pyramids,
                 num_pyramids, d_ids, d_out, capacity, d_num_in, d_num_out);
    return last_error();
}

extern "C" int sessd_sada_shuffle(const float *d_points, const int *d_frame_off, int batch, int max_frame_points, const int *d_perm,
                                  float *d_out, void *stream) {
    if (batch <= 0 || max_frame_points < 0 || !d_frame_off || !d_perm || !d_points || !d_out) return SESSD_EINVAL;
    if (misaligned(d_points) || misaligned(d_out)) return SESSD_EINVAL;
    if (max_frame_points == 0) return SESSD_OK;
    dim3 grid(std::min(div_up(max_frame_points, kSadaThreads), 1024), batch);
    SESSD_LAUNCH(shuffle_kernel, grid, kSadaThreads, 0, (cudaStream_t)stream, d_points, d_frame_off, d_perm, d_out);
    return last_error();
}
