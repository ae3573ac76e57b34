// wgrad_mma.cuh -- the tensor-core core shared by the weight-gradient kernels (spconv_grad.cu: sparse encoder, bevgrad.cu: neck and head).
//
// Both compute per work item an [M][N] product  sum_r A[r][m] G[r][n]  over K rows r (rulebook pairs, output pixels) and write it as an
// fp32 partial; wgrad_reduce sums the partials of a result tile in ascending item order (bitwise run-to-run deterministic, no float
// atomic).  A ROUND stages up to kWgKC rows ROW-MAJOR, as the (hi, lo) planes lie in global memory: [hi | lo][row][channel], 16-byte
// cp.async per 8 channels, double-buffered so the next round's copies fly while this round multiplies.  Rows are padded by 8 halves: the
// eight 16-byte rows an ldmatrix phase reads fall in eight different bank groups.  The rows are the K dimension of both operands, so
// ldmatrix.trans turns them into the fragments of mma.sync.m16n8k16 (A = in^T: [channel][row], B = g: [row][channel]), with the forward's
// three-product fp16 split: a_hi g_hi into the main accumulator, a_hi g_lo + a_lo g_hi into the cross accumulator, summed RN once per item.
// A kernel supplies only where its rounds come from and which global rows its copies read.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace sessd {

constexpr int kWgThreads = 256;              // eight warps
constexpr int kWgKC = 64;                    // K rows staged per round

__device__ __forceinline__ void mma_f16_16816(float *d, const uint32_t *a, uint32_t b0, uint32_t b1) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b0), "r"(b1));
}
__device__ __forceinline__ void wg_cp_async16(uint32_t dst, const void *src, bool valid) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(dst), "l"(src), "r"(valid ? 16 : 0) : "memory");   // 0: zero fill
}
__device__ __forceinline__ void ldsm_x4_trans(uint32_t *r, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.trans.shared.b16 {%0,%1,%2,%3}, [%4];\n" : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3]) : "r"(addr));
}
__device__ __forceinline__ void ldsm_x2_trans(uint32_t *r, uint32_t addr) {
    asm volatile("ldmatrix.sync.aligned.m8n8.x2.trans.shared.b16 {%0,%1}, [%2];\n" : "=r"(r[0]), "=r"(r[1]) : "r"(addr));
}

// Staging layout of M input channels (A) and N gradient channels (G) in dynamic shared memory, and the warp tiling of the [M][N] result:
// eight warps in m16 slabs x kNT n8 tiles each.
template <int M, int N>
struct WgLayout {
    static constexpr int kPitchA = M + 8, kPitchG = N + 8;                  // halves
    static constexpr int kBufHalves = 2 * kWgKC * (kPitchA + kPitchG);       // one buffer: A hi, A lo, G hi, G lo
    static constexpr int kSmem = 2 * kBufHalves * 2;                         // bytes, two buffers
    static constexpr int kMSlabs = M / 16;
    static constexpr int kNT = (M / 16) * (N / 8) / 8;                       // n8 tiles per warp
    static_assert(kNT >= 1 && (M / 16) * (N / 8) % 8 == 0, "eight warps must tile the result");
    static_assert(kNT == 1 || kNT % 2 == 0, "B fragments are loaded two n8 tiles at a time");

    uint32_t s0;                                                             // shared address of the dynamic shared memory
    // buffer b: A half h at s0 + 2 (b kBufHalves + h kWgKC kPitchA), G half h after the two A halves
    __device__ __forceinline__ uint32_t a(int b, int h, int p, int c) const {
        return s0 + 2u * (uint32_t)(b * kBufHalves + (h * kWgKC + p) * kPitchA + c);
    }
    __device__ __forceinline__ uint32_t g(int b, int h, int p, int c) const {
        return s0 + 2u * (uint32_t)(b * kBufHalves + 2 * kWgKC * kPitchA + (h * kWgKC + p) * kPitchG + c);
    }
};

// Work item blockIdx.x, one CTA of kWgThreads.  The kernel describes its rounds (all block-uniform) by
//   first(r)     sets r to the item's first round
//   valid(r)     whether r is a round of the item (false once the rounds are exhausted, or at once for an empty item)
//   next(r)      advances r to the following round
//   rows(r)      K rows of round r (at most kWgKC)
//   stage(r, b)  issues the copies of round r into buffer b of L; slots from rows(r) up to the next multiple of 16 must read as zero
//                (the mma reads whole k16 steps)
// and the item writes partial[blockIdx.x][m][n] = acc_m + acc_c (RN).
template <int M, int N, class Round, class First, class Valid, class Next, class Rows, class Stage>
__device__ __forceinline__ void wgrad_mma_item(const WgLayout<M, N> &L, First first, Valid valid, Next next, Rows rows, Stage stage,
                                               float *partial) {
    using C = WgLayout<M, N>;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gq = lane >> 2, tq = lane & 3;
    const int lr = lane & 7, lm = lane >> 3;                           // ldmatrix: row within an 8x8 matrix, matrix index
    // warp w: m16 slab w % kMSlabs, n8 tiles from (w / kMSlabs) kNT on.  With eight slabs that is slab w and every tile, spelled out
    // because the compiler cannot know w < 8 (the general form costs the M = 128 kernels registers and their 64-bit partial stores)
    const int m0 = (C::kMSlabs == 8 ? warp : warp % C::kMSlabs) * 16, n0 = C::kMSlabs == 8 ? 0 : (warp / C::kMSlabs) * C::kNT * 8;
    float acc_m[C::kNT][4], acc_c[C::kNT][4];
#pragma unroll
    for (int j = 0; j < C::kNT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) { acc_m[j][q] = 0.f; acc_c[j][q] = 0.f; }

    Round cur;
    first(cur);
    if (valid(cur)) stage(cur, 0);
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    int buf = 0;
    while (valid(cur)) {                                                // block-uniform
        Round nxt = cur;
        next(nxt);
        if (valid(nxt)) stage(nxt, buf ^ 1);
        asm volatile("cp.async.commit_group;\n" ::: "memory");
        asm volatile("cp.async.wait_group 1;\n" ::: "memory");          // this round's copies (the next round's stay in flight)
        __syncthreads();
        const int steps = (int)((rows(cur) + 15) >> 4);
        for (int s = 0; s < steps; ++s) {
            const int k0 = s * 16;
            // A fragments: matrix lm covers rows k0 + 8 (lm >> 1) .., channels m0 + 8 (lm & 1) ..  ->  a0..a3 of m16n8k16
            uint32_t ah[4], al[4];
            ldsm_x4_trans(ah, L.a(buf, 0, k0 + lr + 8 * (lm >> 1), m0 + 8 * (lm & 1)));
            ldsm_x4_trans(al, L.a(buf, 1, k0 + lr + 8 * (lm >> 1), m0 + 8 * (lm & 1)));
#pragma unroll
            for (int j = 0; j < C::kNT; j += (C::kNT == 1 ? 1 : 2)) {
                // B fragments: matrix lm covers rows k0 + 8 (lm & 1) .., channels n0 + 8 (j + (lm >> 1)) ..  ->  (b0, b1) of tile j (, j + 1)
                uint32_t bh[4], bl[4];
                const int gp = k0 + lr + 8 * (lm & 1), gc = n0 + 8 * j + 8 * (lm >> 1);
                if constexpr (C::kNT == 1) {
                    ldsm_x2_trans(bh, L.g(buf, 0, gp, n0));
                    ldsm_x2_trans(bl, L.g(buf, 1, gp, n0));
                } else {
                    ldsm_x4_trans(bh, L.g(buf, 0, gp, gc));
                    ldsm_x4_trans(bl, L.g(buf, 1, gp, gc));
                }
#pragma unroll
                for (int u = 0; u < (C::kNT == 1 ? 1 : 2); ++u) {
                    mma_f16_16816(acc_m[j + u], ah, bh[2 * u], bh[2 * u + 1]);     // main  += a_hi g_hi
                    mma_f16_16816(acc_c[j + u], ah, bl[2 * u], bl[2 * u + 1]);     // cross += a_hi g_lo
                    mma_f16_16816(acc_c[j + u], al, bh[2 * u], bh[2 * u + 1]);     // cross += a_lo g_hi
                }
            }
        }
        __syncthreads();                                                // buffer `buf` is free for the round after next
        cur = nxt;
        buf ^= 1;
    }
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
    // this thread holds rows m0 + gq (+8), columns n0 + 2 tq (+1) of every n8 tile
    float *dst = partial + (size_t)(int)blockIdx.x * (M * N);
#pragma unroll
    for (int j = 0; j < C::kNT; ++j) {
        const int n = n0 + 8 * j + 2 * tq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + gq + 8 * h;
            *reinterpret_cast<float2 *>(dst + (size_t)m * N + n) =
                make_float2(acc_m[j][2 * h] + acc_c[j][2 * h], acc_m[j][2 * h + 1] + acc_c[j][2 * h + 1]);
        }
    }
}

// one CTA of kWgThreads per work item; the kernel's dynamic shared-memory limit is raised on its first launch
template <auto Kernel, int M, int N, class... Args>
static int wgrad_launch(int items, cudaStream_t st, const Args &...args) {
    constexpr int kSmem = WgLayout<M, N>::kSmem;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(Kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
        if (e != cudaSuccess) return (int)e;
        attr_done = true;
    }
    SESSD_LAUNCH(Kernel, items, kWgThreads, kSmem, st, args...);
    return last_error();
}

// gw[t][ci][co] = s (1 / S_in) (1 / S_g), s the sum over the chunks of its group, ascending, of partial[group][chunk][ci % bm][co % bn],
// group = (t mblocks + ci / bm) nblocks + co / bn; S_in = in_info[1], S_g = g_info[1], each info pointer nullable (scale 1).  The sparse
// kernels pass bm = cin, bn = cout (one group per offset).  The scales are powers of two, so both products are exact while s / S_in is a
// normal float, however small the two abs-maxes (a single factor 1 / (S_in S_g) would flush to zero beyond S_in S_g = 2^149).
// Defined in spconv_grad.cu.
int wgrad_reduce(const float *partial, int ntaps, int cin, int cout, int bm, int bn, int chunks, const float *in_info, const float *g_info,
                 float *gw, cudaStream_t st);

}  // namespace sessd
