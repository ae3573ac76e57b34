// bevconv_p2.cuh -- BEV conv / deconv (+BN+ReLU+residual) on the Hopper tensor cores (wgmma) from PRE-SPLIT fp16 planes
// (the product's default path, bevconv_p2.cu) or from an fp32 input split inside the kernel (the lab formats, bevconv_split.cu).
//
// Replaces the cuDNN conv blocks of det3d/models/necks/rpn_v1.py:135-210 and the 1x1 head convs of
// det3d/models/bbox_heads/mg_head_sessd.py:202-230 (fp32 in, fp32 out, fp32 accumulate).  Numerics: x = (x_hi + x_lo) / S with fp16
// hi / lo and an exact power-of-two scale S (22+ significand bits); three fp16 products per MAC accumulated in fp32 registers
// (a_hi*b_hi -> main, a_hi*b_lo + a_lo*b_hi -> cross, summed in RN fp32 by the epilogue).  The activations TRAVEL BETWEEN LAYERS as
// fp16 (hi, lo) planes [2][B*H*W][C] written by the producing layer's epilogue, so that
//   * the main loop is pure TMA -> shared memory -> wgmma (both operands from shared memory): no in-kernel fp32 -> fp16 conversion;
//   * the scale of an OUTPUT tensor has to be known before its first element is written: S_out comes from a rigorous bound
//     |out| <= amax_in * G + max|shift| (+ amax_residual), G = max_n sum_k |w[k][n]| |bn_scale[n]| (host, at weight-load time) and
//     amax_in = the measured abs-max of the input (device scalar, raised by the producer's epilogue).  The bound maps into
//     [2^14, 2^15): fp16 keeps 22 bits of every element down to 2^-17 of the bound, far more slack than the bound is loose;
//   * the two TMA loops (patch, weight tiles) run warp-uniform with one ELECTED issuing lane, so descriptors and addresses stay in uniform
//     registers.
// Geometry: tile = 8 (u) x 16 (v) output pixels = 128 rows, row = v*8 + u, so that one 8-row swizzle group = 8 consecutive u; each of
// the two consumer warpgroups owns 64 rows (8 v rows).  For every distinct tap shift along u (and v parity, strided convs) ONE copy of
// the input patch [v rows][8 u][32 channels] is TMA-loaded per plane: a tap then addresses a canonical K-major SWIZZLE_64B operand at
// copy + v_shift * 512 B (group stride 512 B): plain descriptors, no base-offset tricks.  u / v are mapped to (y, x) or (x, y),
// whichever tiles the map with fewer tiles.
// Warps: 0-7 consumers (two warpgroups: wgmma issue, then BN/ReLU/residual -> fp32 and / or fp16 planes + running abs-max from the
// accumulator registers), 8 patch TMA, 9 weight TMA.
#pragma once
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace sessd {

constexpr int kP2TileU = 8, kP2TileV = 16;
constexpr int kP2MaxCopies = 6, kP2MaxRowsV = 18;
constexpr int kP2BStages = 6, kP2MaxBStages = 12;
constexpr int kP2BStageBytes = 2 * 128 * 64;              // [b_hi ; b_lo] planes, up to 128 rows of 64 B each
constexpr int kP2BRing = kP2BStages * kP2BStageBytes;     // bytes of the weight-stage ring
constexpr int kP2MmaWarps = 8;
constexpr int kP2PatchWarp = 8, kP2WeightWarp = 9;
constexpr int kP2Threads = 320;                           // 10 warps
constexpr int kP2MaxSmem = 227 * 1024;
// operand source of the A side: pre-split fp16 planes (TMA straight into the operand layout), or an fp32 NHWC input that TMA stages in
// shared memory and the consumer warpgroups split there -- into fp16 (hi, lo) with the power-of-two scale of its abs-max (32-channel
// chunks), or into tf32 hi = truncate(x), lo = x - hi for three tf32 products (16-channel chunks, fp32 weights [2][taps][cout_pad][cin])
enum { kP2Planes = 0, kP2SplitF16 = 1, kP2SplitTf32 = 2 };

struct P2Params {
    int batch, cin, cout;
    int in_stride;                     // 1 or 2 (input position = output position * in_stride + tap offset)
    int out_h, out_w;                  // output tensor extent (pixels)
    int grid_u, grid_v;                // output positions computed per class along u / v
    int u_is_x;                        // 1: u = x, v = y;  0: u = y, v = x
    int out_stride, nclass;
    int cls_ntaps[4], cls_off_u[4], cls_off_v[4];
    int tap_copy[4][9], tap_row[4][9], tap_w[4][9];      // per (class, tap): patch copy, first v row inside the copy, weight tap
    int ncopies, rows_v;
    int copy_u[kP2MaxCopies], copy_v[kP2MaxCopies];       // input coordinate of the copy's first element relative to (u0, v0) * in_stride
    int copy_bytes, patch_bytes, npatch;                  // bytes of one copy plane, of one patch buffer (ncopies x 2 planes), 1 or 2 buffers
    int chunk;                         // input channels per K stage: 32 (fp16 operands) or 16 (tf32 operands); 64-byte operand rows either way
    int load_bytes, staging_bytes;     // TMA bytes per patch buffer; fp32 staging bytes per patch buffer (split modes, else 0)
    int bring_bytes;                   // bytes of the weight-stage ring
    int out_info_scale;                // 1: out_info = {abs-max, S_out} (planes chain); 0: out_info is a single running abs-max
    const float *in_amax;              // split fp16 mode: abs-max of the fp32 input (nullable: scale 1)
    int relu, n_tile, nblocks;
    int bstages, bstage_bytes;         // weight-stage ring: count and bytes per stage
    int tiles_u, tiles_v, tiles, total;                   // pixel tiles, work items = nclass * nblocks * tiles
    int cls_order[4];
    const float *in_info;              // [2] = {abs-max of the input tensor, scale S_in of its planes}
    const float *resid_info;           // nullable [2]
    float gain, shift_max;             // bound of the output: amax_in * gain + shift_max (+ amax_resid)
    float *out_info;                   // [2] = {running abs-max of the output (atomicMax), S_out}
    long long out_plane_stride;        // elements between the hi and the lo plane of the output
};

struct P2Item { int cls, n0, b, u0, v0, ntaps; };

__device__ __forceinline__ P2Item p2_decode(const P2Params &p, int g) {
    P2Item it;
    const int per_cls = p.nblocks * p.tiles;
    const int cr = g / per_cls;
    int rem = g - cr * per_cls;
    const int nb = rem / p.tiles;
    int t = rem - nb * p.tiles;
    it.cls = p.cls_order[cr];
    it.n0 = nb * p.n_tile;
    const int tu = t % p.tiles_u; t /= p.tiles_u;
    const int tv = t % p.tiles_v;
    it.b = t / p.tiles_v;
    it.u0 = tu * kP2TileU; it.v0 = tv * kP2TileV;
    it.ntaps = p.cls_ntaps[it.cls];
    return it;
}

template <int NT, int MODE>
__device__ __forceinline__ void p2_wgmma(float *d, uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (MODE == kP2SplitTf32) {
        if constexpr (NT == 32) wgmma_tf32_n32(d, da, db, accumulate);
        else wgmma_tf32_n128(d, da, db, accumulate);
    } else {
        if constexpr (NT == 32) wgmma_f16_n32(d, da, db, accumulate);
        else wgmma_f16_n128(d, da, db, accumulate);
    }
}

__device__ __forceinline__ float p2_tf32_rn(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}

// split modes: the fp32 staging copy of patch buffer pb -> the (hi, lo) operand planes in the SWIZZLE_64B layout (16-byte chunk j of a
// 64-byte row r lands at chunk j ^ ((r >> 1) & 3)); run by the 256 consumer threads, which then sync among themselves
template <int MODE>
__device__ __forceinline__ void p2_split_patch(const P2Params &p, const unsigned char *staging, unsigned char *planes, float s_in, int ctid) {
    const int rows = p.rows_v * kP2TileU;
    const int copy_in = p.staging_bytes / p.ncopies;
    const int items = p.ncopies * rows * 4;
    for (int i = ctid; i < items; i += kP2MmaWarps * 32) {
        const int j = i & 3, r = (i >> 2) % rows, c = (i >> 2) / rows;
        unsigned char *hi = planes + 2 * c * p.copy_bytes + r * 64 + ((j ^ ((r >> 1) & 3)) << 4);
        if constexpr (MODE == kP2SplitF16) {          // 32 fp32 per staging row -> 8 of them per 16-byte fp16 chunk
            const float4 *src = reinterpret_cast<const float4 *>(staging + c * copy_in + r * 128 + j * 32);
            const float4 a = src[0], b = src[1];
            const float x[8] = {a.x * s_in, a.y * s_in, a.z * s_in, a.w * s_in, b.x * s_in, b.y * s_in, b.z * s_in, b.w * s_in};
            __align__(16) __half h[8], l[8];
#pragma unroll
            for (int t = 0; t < 8; ++t) { h[t] = __float2half_rn(x[t]); l[t] = __float2half_rn(x[t] - __half2float(h[t])); }
            *reinterpret_cast<uint4 *>(hi) = *reinterpret_cast<const uint4 *>(h);
            *reinterpret_cast<uint4 *>(hi + p.copy_bytes) = *reinterpret_cast<const uint4 *>(l);
        } else {                                      // 16 fp32 per staging row -> 4 of them per 16-byte tf32 chunk
            const float4 x = *reinterpret_cast<const float4 *>(staging + c * copy_in + r * 64 + j * 16);
            const float4 h = make_float4(__uint_as_float(__float_as_uint(x.x) & ~0x1FFFu), __uint_as_float(__float_as_uint(x.y) & ~0x1FFFu),
                                         __uint_as_float(__float_as_uint(x.z) & ~0x1FFFu), __uint_as_float(__float_as_uint(x.w) & ~0x1FFFu));
            *reinterpret_cast<float4 *>(hi) = h;
            // lo rounded to the nearest tf32 here: the tensor core would truncate it (a bias that grows with K)
            *reinterpret_cast<float4 *>(hi + p.copy_bytes) = make_float4(p2_tf32_rn(x.x - h.x), p2_tf32_rn(x.y - h.y), p2_tf32_rn(x.z - h.z),
                                                                         p2_tf32_rn(x.w - h.w));
        }
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic-proxy writes -> visible to wgmma
    asm volatile("bar.sync 1, %0;\n" ::"n"(kP2MmaWarps * 32) : "memory");
}

template <int NT, int MODE>
__global__ void __launch_bounds__(kP2Threads, 1) bev_conv_p2_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                   const __grid_constant__ CUtensorMap map_b,
                                                                   const float *__restrict__ scale, const float *__restrict__ shift,
                                                                   const float *__restrict__ resid, float *__restrict__ out_f32,
                                                                   __half *__restrict__ out_planes, P2Params p) {
    extern __shared__ unsigned char smem_raw[];
    unsigned char *tiles = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    unsigned char *patches = tiles + p.bring_bytes;
    unsigned char *staging = patches + p.npatch * p.patch_bytes;
    uint64_t *bars = (uint64_t *)(staging + p.npatch * p.staging_bytes);
    uint64_t *patch_full = bars, *patch_empty = bars + 2, *b_full = bars + 4, *b_empty = bars + 4 + kP2MaxBStages;
    uint32_t *s_aoff = (uint32_t *)(b_empty + kP2MaxBStages);      // [4 classes][9 taps]

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == kP2PatchWarp * 32) prefetch_tensormap(&map_a);    // descriptor fetches overlap barrier init
    if (threadIdx.x == kP2WeightWarp * 32) prefetch_tensormap(&map_b);
    const int nchunks = p.cin / p.chunk;
    const uint32_t b_plane_bytes = (uint32_t)p.n_tile * 64u;      // bytes of the b_hi (or b_lo) rows per (tap, chunk)

    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) { mbar_init(&patch_full[s], 1); mbar_init(&patch_empty[s], kP2MmaWarps); }
        for (int s = 0; s < p.bstages; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], kP2MmaWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    // operand offset of every (class, tap) inside a patch buffer, in 16-byte units
    for (int idx = threadIdx.x; idx < p.nclass * 9; idx += blockDim.x) {
        const int c = idx / 9, t = idx - c * 9;
        s_aoff[idx] = (uint32_t)((2 * p.tap_copy[c][t] * p.copy_bytes + p.tap_row[c][t] * 512) >> 4);
    }
    __syncthreads();

    if (warp == kP2PatchWarp) {
        // ===================== activation patches: per (item, 32-channel chunk) ncopies x (hi, lo) boxes =====================
        int pb = 0;
        uint32_t pph = 0;
        const uint32_t patches_u32 = smem_u32(patches);
        for (int g = blockIdx.x; g < p.total; g += gridDim.x) {
            const P2Item it = p2_decode(p, g);
            const int bu = it.u0 * p.in_stride, bv = it.v0 * p.in_stride;
            for (int cc = 0; cc < nchunks; ++cc) {
                mbar_wait(&patch_empty[pb], pph ^ 1u);
                if (elect_one()) {
                    mbar_expect_tx(&patch_full[pb], (uint32_t)p.load_bytes);
                    if constexpr (MODE == kP2Planes) {
                        uint32_t dst = patches_u32 + (uint32_t)(pb * p.patch_bytes);
                        for (int c = 0; c < p.ncopies; ++c, dst += 2u * (uint32_t)p.copy_bytes) {
                            const int cu = bu + p.copy_u[c], cv = bv + p.copy_v[c];
                            tma_load_5d(dst, &map_a, &patch_full[pb], cc * p.chunk, cu, cv, it.b, 0);
                            tma_load_5d(dst + (uint32_t)p.copy_bytes, &map_a, &patch_full[pb], cc * p.chunk, cu, cv, it.b, 1);
                        }
                    } else {
                        const uint32_t copy_in = (uint32_t)(p.staging_bytes / p.ncopies);
                        uint32_t dst = smem_u32(staging) + (uint32_t)(pb * p.staging_bytes);
                        for (int c = 0; c < p.ncopies; ++c, dst += copy_in)
                            tma_load_5d(dst, &map_a, &patch_full[pb], cc * p.chunk, bu + p.copy_u[c], bv + p.copy_v[c], it.b, 0);
                    }
                }
                __syncwarp();
                if (++pb == p.npatch) { pb = 0; pph ^= 1u; }
            }
        }
    } else if (warp == kP2WeightWarp) {
        // ===================== weight tiles: one [b_hi ; b_lo] stage per (item, chunk, tap) =====================
        int S = 0;
        uint32_t bph = 0;
        for (int g = blockIdx.x; g < p.total; g += gridDim.x) {
            const P2Item it = p2_decode(p, g);
            for (int cc = 0; cc < nchunks; ++cc)
                for (int tap = 0; tap < it.ntaps; ++tap) {
                    mbar_wait(&b_empty[S], bph ^ 1u);
                    if (elect_one()) {
                        unsigned char *st = tiles + S * p.bstage_bytes;
                        const int wtap = p.tap_w[it.cls][tap];
                        mbar_expect_tx(&b_full[S], 2 * b_plane_bytes);
                        tma_load_4d(st, &map_b, &b_full[S], cc * p.chunk, it.n0, wtap, 0);
                        tma_load_4d(st + b_plane_bytes, &map_b, &b_full[S], cc * p.chunk, it.n0, wtap, 1);
                    }
                    __syncwarp();
                    if (++S == p.bstages) { S = 0; bph ^= 1u; }
                }
        }
    } else {
        // ===================== consumers (warps 0-7): wgmma over (chunk, tap), then BN / ReLU / residual / stores =====================
        const int wg = warp >> 2, wq = warp & 3;
        constexpr int kAcc = NT / 2;
        const uint32_t a_rows = (uint32_t)(wg * 64 * 64) >> 4;         // this warpgroup's 64 rows (8 swizzle groups of 512 B), 16-byte units
        const uint32_t tiles_lo = desc_lo(smem_u32(tiles));
        const uint32_t patch_lo = desc_lo(smem_u32(patches)) + a_rows;
        const uint32_t plane_lo = b_plane_bytes >> 4;
        const uint32_t copy_lo = (uint32_t)(p.copy_bytes >> 4), patch_sz = (uint32_t)(p.patch_bytes >> 4);
        float amax_in = 0.f, s_in = 1.f;
        if constexpr (MODE == kP2Planes) { amax_in = __ldg(p.in_info); s_in = __ldg(p.in_info + 1); }
        if constexpr (MODE == kP2SplitF16) if (p.in_amax) { amax_in = __ldg(p.in_amax); s_in = pow2_scale_for_bound(amax_in); }
        const float inv_sa = 1.f / s_in;                 // exact: power of two
        float bound = amax_in * p.gain + p.shift_max;
        if (p.resid_info) bound += __ldg(p.resid_info);
        const float s_out = pow2_scale_for_bound(bound);
        if (blockIdx.x == 0 && threadIdx.x == 0 && p.out_info && p.out_info_scale) p.out_info[1] = s_out;
        float vmax = 0.f;
        const int per_cls = p.nblocks * p.tiles;
        int S = 0, pb = 0;
        uint32_t bph = 0, pph = 0;
        for (int g = blockIdx.x; g < p.total; g += gridDim.x) {
            const int cls = p.cls_order[g / per_cls];
            const int ntaps = p.cls_ntaps[cls];
            const uint32_t *aoff = s_aoff + cls * 9;
            float acc_m[kAcc], acc_c[kAcc], tot[MODE == kP2SplitTf32 ? kAcc : 1];
#pragma unroll
            for (int i = 0; i < kAcc; ++i) { acc_m[i] = 0.f; acc_c[i] = 0.f; }
#pragma unroll
            for (int i = 0; i < (MODE == kP2SplitTf32 ? kAcc : 1); ++i) tot[i] = 0.f;
            int prevS = -1, prev_pb = -1;
            bool first = true;
            for (int cc = 0; cc < nchunks; ++cc) {
                mbar_wait(&patch_full[pb], pph);
                if constexpr (MODE != kP2Planes)
                    p2_split_patch<MODE>(p, staging + pb * p.staging_bytes, patches + pb * p.patch_bytes, s_in, threadIdx.x);
                const uint32_t pbase = patch_lo + (uint32_t)pb * patch_sz;
#pragma unroll 1
                for (int tap = 0; tap < ntaps; ++tap) {
                    mbar_wait(&b_full[S], bph);
                    if constexpr (MODE == kP2SplitTf32) {
                        // the weights' lo plane rounded to the nearest tf32 in place (the tensor core would truncate it)
                        float *wl = reinterpret_cast<float *>(tiles + S * p.bstage_bytes + b_plane_bytes);
                        for (int i = threadIdx.x; i < (int)(b_plane_bytes / 4); i += kP2MmaWarps * 32) wl[i] = p2_tf32_rn(wl[i]);
                        asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");
                        asm volatile("bar.sync 1, %0;\n" ::"n"(kP2MmaWarps * 32) : "memory");
                    }
                    const uint64_t da_hi = kDescSw64Hi | (uint64_t)(pbase + aoff[tap]);
                    const uint64_t da_lo = da_hi + (uint64_t)copy_lo;
                    const uint64_t db_hi = kDescSw64Hi | (uint64_t)(tiles_lo + (uint32_t)(S * (p.bstage_bytes >> 4)));
                    const uint64_t db_lo = db_hi + (uint64_t)plane_lo;
                    const uint32_t acc = first ? 0u : 1u;
                    // K = 16 fp16 / 8 tf32 per instruction = 32 bytes of the 64-byte row
                    wgmma_fence();
                    // tf32: the main accumulator restarts every chunk (its chunk partial is added into `tot` in RN fp32 below)
                    const uint32_t acc_main = MODE == kP2SplitTf32 ? (tap != 0 ? 1u : 0u) : acc;
                    p2_wgmma<NT, MODE>(acc_m, da_hi, db_hi, acc_main);       // main  (+)= a_hi x b_hi
                    p2_wgmma<NT, MODE>(acc_m, da_hi + 2, db_hi + 2, 1u);
                    p2_wgmma<NT, MODE>(acc_c, da_hi, db_lo, acc);            // cross (+)= a_hi x b_lo
                    p2_wgmma<NT, MODE>(acc_c, da_hi + 2, db_lo + 2, 1u);
                    p2_wgmma<NT, MODE>(acc_c, da_lo, db_hi, 1u);             // cross  += a_lo x b_hi
                    p2_wgmma<NT, MODE>(acc_c, da_lo + 2, db_hi + 2, 1u);
                    wgmma_commit();
                    first = false;
                    wgmma_wait<1>();                                         // the previous step's operands are no longer read
                    if (lane == 0) {
                        if (prevS >= 0) mbar_arrive(&b_empty[prevS]);
                        if (prev_pb >= 0) mbar_arrive(&patch_empty[prev_pb]);
                    }
                    prevS = S;
                    prev_pb = (tap == ntaps - 1) ? pb : -1;
                    if (++S == p.bstages) { S = 0; bph ^= 1u; }
                }
                if (p.npatch == 1 || MODE == kP2SplitTf32) {
                    // one patch buffer: the next chunk's patch can only land once this one is released, so release it now rather
                    // than after the next chunk's first step (that step would wait for the patch forever); tf32: drain the chunk
                    // and fold its main partial
                    wgmma_wait<0>();
                    if (lane == 0) {
                        mbar_arrive(&b_empty[prevS]);
                        mbar_arrive(&patch_empty[pb]);
                    }
                    prevS = prev_pb = -1;
                    if constexpr (MODE == kP2SplitTf32) {
                        wgmma_fence_regs<kAcc>(acc_m);
#pragma unroll
                        for (int i = 0; i < kAcc; ++i) tot[i] += acc_m[i];
                    }
                }
                if (++pb == p.npatch) { pb = 0; pph ^= 1u; }
            }
            wgmma_wait<0>();
            wgmma_fence_regs<kAcc>(acc_m);
            wgmma_fence_regs<kAcc>(acc_c);
            if (lane == 0) {
                if (prevS >= 0) mbar_arrive(&b_empty[prevS]);
                if (prev_pb >= 0) mbar_arrive(&patch_empty[prev_pb]);
            }
            // epilogue: this thread holds tile rows r0 and r0 + 8, two adjacent channels of every 8-channel group
            const P2Item it = p2_decode(p, g);
            const int r0 = wg * 64 + wq * 16 + (lane >> 2);
            const int c2 = 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r0 + 8 * h;
                const int lv = r / kP2TileU, lu = r % kP2TileU;
                const int gu = it.u0 + lu, gv = it.v0 + lv;
                if (it.b >= p.batch || gu >= p.grid_u || gv >= p.grid_v) continue;
                const int ou = gu * p.out_stride + p.cls_off_u[it.cls], ov = gv * p.out_stride + p.cls_off_v[it.cls];
                const int oy = p.u_is_x ? ov : ou, ox = p.u_is_x ? ou : ov;
                const size_t opix = ((size_t)it.b * p.out_h + (size_t)oy) * p.out_w + (size_t)ox;
#pragma unroll
                for (int gi = 0; gi < NT / 8; ++gi) {
                    const int n = it.n0 + 8 * gi + c2, i = 4 * gi + 2 * h;
                    if (n >= p.cout) continue;                          // cout % 8 == 0: both channels of the pair exist or neither
                    const float2 sc = scale ? __ldg(reinterpret_cast<const float2 *>(scale + n)) : make_float2(1.f, 1.f);
                    const float2 sh = shift ? __ldg(reinterpret_cast<const float2 *>(shift + n)) : make_float2(0.f, 0.f);
                    const float m0 = MODE == kP2SplitTf32 ? tot[i] : acc_m[i], m1 = MODE == kP2SplitTf32 ? tot[i + 1] : acc_m[i + 1];
                    float o0 = fmaf((m0 + acc_c[i]) * inv_sa, sc.x, sh.x);
                    float o1 = fmaf((m1 + acc_c[i + 1]) * inv_sa, sc.y, sh.y);
                    if (p.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                    const size_t off = opix * p.cout + n;
                    if (resid) {
                        const float2 rr = __ldg(reinterpret_cast<const float2 *>(resid + off));
                        o0 += rr.x; o1 += rr.y;
                    }
                    vmax = fmaxf(vmax, fmaxf(fabsf(o0), fabsf(o1)));
                    if (out_f32) *reinterpret_cast<float2 *>(out_f32 + off) = make_float2(o0, o1);
                    if (out_planes) {
                        const float x0 = o0 * s_out, x1 = o1 * s_out;
                        const __half2 hi = __floats2half2_rn(x0, x1);
                        const float2 f = __half22float2(hi);
                        *reinterpret_cast<__half2 *>(out_planes + off) = hi;
                        *reinterpret_cast<__half2 *>(out_planes + p.out_plane_stride + off) = __floats2half2_rn(x0 - f.x, x1 - f.y);
                    }
                }
            }
        }
        if (p.out_info) {
            const unsigned m = __reduce_max_sync(0xFFFFFFFFu, __float_as_uint(vmax));     // non-negative floats order like their bits
            if (lane == 0 && m != 0u) atomicMax(reinterpret_cast<unsigned *>(p.out_info), m);
        }
    }
}

static int encode_map_nd(CUtensorMap *m, const void *base, int rank, const cuuint64_t *dims, const cuuint64_t *strides_bytes /*rank-1*/,
                         const cuuint32_t *box, const cuuint32_t *estr, CUtensorMapSwizzle swz,
                         CUtensorMapDataType dtype = CU_TENSOR_MAP_DATA_TYPE_FLOAT16) {
    EncodeTiledFn enc = get_tensor_map_encoder();
    if (!enc) return SESSD_EINVAL;
    CUresult r = enc(m, dtype, (cuuint32_t)rank, const_cast<void *>(base), dims, strides_bytes, box, estr,
                     CU_TENSOR_MAP_INTERLEAVE_NONE, swz, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    return r == CUDA_SUCCESS ? 0 : 700 + (int)r;
}

// taps: per class (dy, dx, weight tap); fills the geometry of p and launches
struct P2Taps { int n, dy[9], dx[9], w[9]; };

// MODE kP2Planes: d_in = fp16 planes [2][B][H][W][C], d_in_info = {abs-max, S}; split modes: d_in = fp32 NHWC, d_in_info = the input's
// abs-max (split fp16; nullable) or unused (tf32), weights fp32 [2][taps][cout_pad][cin] in the tf32 mode; d_out_info is {abs-max, S_out}
// in the planes mode and a single running abs-max otherwise
template <int MODE>
static int launch_p2(const void *d_in_planes, int in_h, int in_w, const float *d_in_info, const void *d_w, int w_taps, int cout_pad,
                     const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info, float gain,
                     float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info, P2Params &p, const P2Taps *cls, int grid_h,
                     int grid_w, void *stream) {
    if (!d_in_planes || !d_w || (!d_out_f32 && !d_out_planes)) return SESSD_EINVAL;
    if (MODE == kP2Planes && (!d_in_info || !d_scale)) return SESSD_EINVAL;
    if (MODE != kP2Planes && d_out_planes) return SESSD_EINVAL;
    if (p.cin < 64 || p.cin % 64 || p.cout < 8 || p.cout % 8) return SESSD_EINVAL;      // whole 64-channel groups; 8-byte stores
    const int n_tile = p.cout <= 32 ? 32 : 128;
    if (cout_pad % n_tile || cout_pad < p.cout) return SESSD_EINVAL;
    // orientation: the in-group dimension u has the 8-pixel tile edge; pick the mapping with fewer tiles
    const int t_ux = div_up(grid_w, kP2TileU) * div_up(grid_h, kP2TileV), t_uy = div_up(grid_h, kP2TileU) * div_up(grid_w, kP2TileV);
    p.u_is_x = t_ux <= t_uy ? 1 : 0;
    p.grid_u = p.u_is_x ? grid_w : grid_h;
    p.grid_v = p.u_is_x ? grid_h : grid_w;
    // patch copies: one per distinct (tap shift along u, tap shift along v modulo the input stride)
    const int s = p.in_stride;
    p.ncopies = 0;
    int key_u[kP2MaxCopies], key_vm[kP2MaxCopies], vmin[kP2MaxCopies], vmax[kP2MaxCopies];
    for (int c = 0; c < p.nclass; ++c)
        for (int t = 0; t < cls[c].n; ++t) {
            const int tu = p.u_is_x ? cls[c].dx[t] : cls[c].dy[t], tv = p.u_is_x ? cls[c].dy[t] : cls[c].dx[t];
            const int vm = ((tv % s) + s) % s;
            int k = 0;
            for (; k < p.ncopies; ++k)
                if (key_u[k] == tu && key_vm[k] == vm) break;
            if (k == p.ncopies) {
                if (p.ncopies == kP2MaxCopies) return SESSD_EINVAL;
                key_u[k] = tu; key_vm[k] = vm; vmin[k] = tv; vmax[k] = tv;
                ++p.ncopies;
            }
            vmin[k] = min(vmin[k], tv); vmax[k] = max(vmax[k], tv);
        }
    p.rows_v = 0;
    for (int k = 0; k < p.ncopies; ++k) p.rows_v = max(p.rows_v, kP2TileV + (vmax[k] - vmin[k]) / s);
    if (p.rows_v > kP2MaxRowsV) return SESSD_EINVAL;
    for (int k = 0; k < p.ncopies; ++k) { p.copy_u[k] = key_u[k]; p.copy_v[k] = vmin[k]; }
    for (int c = 0; c < p.nclass; ++c) {
        p.cls_ntaps[c] = cls[c].n;
        for (int t = 0; t < cls[c].n; ++t) {
            const int tu = p.u_is_x ? cls[c].dx[t] : cls[c].dy[t], tv = p.u_is_x ? cls[c].dy[t] : cls[c].dx[t];
            const int vm = ((tv % s) + s) % s;
            int k = 0;
            for (; k < p.ncopies; ++k)
                if (key_u[k] == tu && key_vm[k] == vm) break;
            p.tap_copy[c][t] = k;
            p.tap_row[c][t] = (tv - vmin[k]) / s;
            p.tap_w[c][t] = cls[c].w[t];
        }
    }
    p.chunk = MODE == kP2SplitTf32 ? 16 : 32;
    p.copy_bytes = p.rows_v * kP2TileU * 64;
    p.patch_bytes = p.ncopies * 2 * p.copy_bytes;
    // fp32 staging: 32 channels = 128-byte rows (split fp16) or 16 channels = 64-byte rows (tf32)
    p.staging_bytes = MODE == kP2Planes ? 0 : p.ncopies * p.rows_v * kP2TileU * p.chunk * 4;
    p.load_bytes = MODE == kP2Planes ? p.patch_bytes : p.staging_bytes;
    const int per_buf = p.patch_bytes + p.staging_bytes, bstage = 2 * (p.cout <= 32 ? 32 : 128) * 64;
    // weight ring: kP2BRing when it fits next to two patch buffers or one, else shrunk (>= 2 stages) next to one buffer
    p.bring_bytes = kP2BRing;
    p.npatch = (kP2BRing + 1536 + 2 * per_buf <= kP2MaxSmem) ? 2 : 1;
    if (kP2BRing + 1536 + per_buf > kP2MaxSmem) p.bring_bytes = (kP2MaxSmem - 1536 - per_buf) / bstage * bstage;
    if (p.bring_bytes < 2 * bstage) return SESSD_EINVAL;
    const int smem = p.bring_bytes + 1536 + p.npatch * per_buf;
    CUtensorMap map_a, map_b;
    const cuuint64_t es = MODE == kP2SplitTf32 ? 4 : 2;               // weight element bytes
    if (MODE != kP2Planes) {   // fp32 NHWC [B][H][W][C] viewed as {C, U, V, B, 1}, staged unswizzled
        const cuuint64_t row_w = (cuuint64_t)p.cin * 4, row_h = (cuuint64_t)in_w * p.cin * 4;
        const cuuint64_t dims[5] = {(cuuint64_t)p.cin, (cuuint64_t)(p.u_is_x ? in_w : in_h), (cuuint64_t)(p.u_is_x ? in_h : in_w),
                                    (cuuint64_t)p.batch, 1};
        const cuuint64_t strides[4] = {p.u_is_x ? row_w : row_h, p.u_is_x ? row_h : row_w, (cuuint64_t)in_h * in_w * p.cin * 4,
                                       (cuuint64_t)p.batch * in_h * in_w * p.cin * 4};
        const cuuint32_t box[5] = {(cuuint32_t)p.chunk, (cuuint32_t)(kP2TileU * s), (cuuint32_t)(p.rows_v * s), 1, 1};
        const cuuint32_t estr[5] = {1, (cuuint32_t)s, (cuuint32_t)s, 1, 1};
        int rc = encode_map_nd(&map_a, d_in_planes, 5, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
        if (rc) return rc;
    } else {   // planes [2][B][H][W][C] fp16 viewed as {C, U, V, B, plane}
        const cuuint64_t row_w = (cuuint64_t)p.cin * 2, row_h = (cuuint64_t)in_w * p.cin * 2;
        const cuuint64_t dims[5] = {(cuuint64_t)p.cin, (cuuint64_t)(p.u_is_x ? in_w : in_h), (cuuint64_t)(p.u_is_x ? in_h : in_w),
                                    (cuuint64_t)p.batch, 2};
        const cuuint64_t strides[4] = {p.u_is_x ? row_w : row_h, p.u_is_x ? row_h : row_w, (cuuint64_t)in_h * in_w * p.cin * 2,
                                       (cuuint64_t)p.batch * in_h * in_w * p.cin * 2};
        const cuuint32_t box[5] = {(cuuint32_t)p.chunk, (cuuint32_t)(kP2TileU * s), (cuuint32_t)(p.rows_v * s), 1, 1};
        const cuuint32_t estr[5] = {1, (cuuint32_t)s, (cuuint32_t)s, 1, 1};
        int rc = encode_map_nd(&map_a, d_in_planes, 5, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_64B);
        if (rc) return rc;
    }
    {   // weights [2 (hi|lo)][taps][cout_pad][cin] fp16 (fp32 tf32 split in the tf32 mode): 64-byte rows of one K stage
        const cuuint64_t dims[4] = {(cuuint64_t)p.cin, (cuuint64_t)cout_pad, (cuuint64_t)w_taps, 2};
        const cuuint64_t strides[3] = {(cuuint64_t)p.cin * es, (cuuint64_t)cout_pad * p.cin * es, (cuuint64_t)w_taps * cout_pad * p.cin * es};
        const cuuint32_t box[4] = {(cuuint32_t)p.chunk, (cuuint32_t)n_tile, 1, 1};
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        int rc = encode_map_nd(&map_b, d_w, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_64B,
                               MODE == kP2SplitTf32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16);
        if (rc) return rc;
    }
    static bool attr_done = false;
    if (!attr_done) {
        SESSD_CUDA_TRY(cudaFuncSetAttribute(bev_conv_p2_kernel<32, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kP2MaxSmem));
        SESSD_CUDA_TRY(cudaFuncSetAttribute(bev_conv_p2_kernel<128, MODE>, cudaFuncAttributeMaxDynamicSharedMemorySize, kP2MaxSmem));
        attr_done = true;
    }
    p.n_tile = n_tile;
    p.bstage_bytes = 2 * n_tile * 64;
    p.bstages = p.bring_bytes / p.bstage_bytes < kP2MaxBStages ? p.bring_bytes / p.bstage_bytes : kP2MaxBStages;
    p.tiles_u = div_up(p.grid_u, kP2TileU);
    p.tiles_v = div_up(p.grid_v, kP2TileV);
    p.tiles = p.tiles_u * p.tiles_v * p.batch;
    p.nblocks = cout_pad / n_tile;
    p.total = p.nclass * p.nblocks * p.tiles;
    for (int c = 0; c < p.nclass; ++c) p.cls_order[c] = c;
    for (int i = 1; i < p.nclass; ++i)            // insertion sort by descending tap count (heavy items first)
        for (int k = i; k > 0 && p.cls_ntaps[p.cls_order[k]] > p.cls_ntaps[p.cls_order[k - 1]]; --k) {
            const int tmp = p.cls_order[k]; p.cls_order[k] = p.cls_order[k - 1]; p.cls_order[k - 1] = tmp;
        }
    p.in_info = MODE == kP2Planes ? d_in_info : nullptr;
    p.in_amax = MODE == kP2SplitF16 ? d_in_info : nullptr;
    p.resid_info = d_residual ? d_resid_info : nullptr;
    if (d_residual && d_out_planes && !d_resid_info) return SESSD_EINVAL;      // the residual's abs-max enters the output planes' bound
    p.gain = gain; p.shift_max = shift_max; p.out_info = d_out_info;
    p.out_info_scale = MODE == kP2Planes ? 1 : 0;
    if (d_out_planes && !d_out_info) return SESSD_EINVAL;
    p.out_plane_stride = (long long)p.batch * p.out_h * p.out_w * p.cout;
    static int num_sms = 0;
    if (!num_sms) {
        int dev = 0;
        SESSD_CUDA_TRY(cudaGetDevice(&dev));
        SESSD_CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    }
    const int grid = p.total < num_sms ? p.total : num_sms;                 // persistent, one CTA per SM
    if (n_tile == 32)
        SESSD_LAUNCH((bev_conv_p2_kernel<32, MODE>), grid, kP2Threads, smem, (cudaStream_t)stream, map_a, map_b, d_scale, d_shift, d_residual, d_out_f32,
                     (__half *)d_out_planes, p);
    else
        SESSD_LAUNCH((bev_conv_p2_kernel<128, MODE>), grid, kP2Threads, smem, (cudaStream_t)stream, map_a, map_b, d_scale, d_shift, d_residual, d_out_f32,
                     (__half *)d_out_planes, p);
    return last_error();
}


// one tap-list conv (sessd_conv_desc) / the four-class deconv through launch_p2<MODE>
template <int MODE>
static int p2_conv(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                   const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                   float *d_out_f32, void *d_out_planes, float *d_out_info, const sessd_conv_desc *desc, void *stream) {
    if (!desc) return SESSD_EINVAL;
    const sessd_conv_desc &d = *desc;
    if (d.batch < 1 || d.ntaps < 1 || d.ntaps > 9 || (d.in_stride != 1 && d.in_stride != 2) || d.out_stride < 1 || d.grid_h < 1 || d.grid_w < 1)
        return SESSD_EINVAL;
    if ((d.grid_h - 1) * d.out_stride + d.out_off_y >= d.out_h || (d.grid_w - 1) * d.out_stride + d.out_off_x >= d.out_w) return SESSD_EINVAL;
    P2Params p = {};
    p.batch = d.batch; p.cin = d.cin; p.cout = d.cout; p.in_stride = d.in_stride;
    p.out_h = d.out_h; p.out_w = d.out_w; p.out_stride = d.out_stride; p.relu = d.relu;
    p.nclass = 1;
    P2Taps t = {};
    t.n = d.ntaps;
    for (int i = 0; i < d.ntaps; ++i) { t.dy[i] = d.tap_dy[i]; t.dx[i] = d.tap_dx[i]; t.w[i] = i; }
    // class offsets are expressed along (u, v) inside launch_p2 once the orientation is known: pass (y, x) through the first slots
    const int off_y = d.out_off_y, off_x = d.out_off_x;
    const int t_ux = div_up(d.grid_w, kP2TileU) * div_up(d.grid_h, kP2TileV), t_uy = div_up(d.grid_h, kP2TileU) * div_up(d.grid_w, kP2TileV);
    const bool u_is_x = t_ux <= t_uy;
    p.cls_off_u[0] = u_is_x ? off_x : off_y; p.cls_off_v[0] = u_is_x ? off_y : off_x;
    return launch_p2<MODE>(d_in_planes, d.in_h, d.in_w, d_in_info, d_weight_h2, d.ntaps, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain,
                     shift_max, d_out_f32, d_out_planes, d_out_info, p, &t, d.grid_h, d.grid_w, stream);
}

template <int MODE>
static int p2_deconv(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                     const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                     float *d_out_f32, void *d_out_planes, float *d_out_info, int batch, int in_h, int in_w, int cin, int cout,
                     int relu, void *stream) {
    if (batch < 1 || in_h < 1 || in_w < 1) return SESSD_EINVAL;
    P2Params p = {};
    p.batch = batch; p.cin = cin; p.cout = cout; p.in_stride = 1;
    p.out_h = 2 * in_h; p.out_w = 2 * in_w; p.out_stride = 2; p.relu = relu;
    p.nclass = 4;
    P2Taps cls[4] = {};
    const int t_ux = div_up(in_w, kP2TileU) * div_up(in_h, kP2TileV), t_uy = div_up(in_h, kP2TileU) * div_up(in_w, kP2TileV);
    const bool u_is_x = t_ux <= t_uy;
    for (int py = 0; py < 2; ++py)
        for (int px = 0; px < 2; ++px) {
            const int c = py * 2 + px;
            p.cls_off_u[c] = u_is_x ? px : py; p.cls_off_v[c] = u_is_x ? py : px;
            // out[2y+py] receives in[y+dy] * W[ky] with 2y+py = 2(y+dy) - 1 + ky:  py=0 -> (ky=1,dy=0);  py=1 -> (ky=0,dy=1), (ky=2,dy=0)
            const int kys[2] = {py == 0 ? 1 : 0, 2}, dys[2] = {py == 0 ? 0 : 1, 0}, ny = py == 0 ? 1 : 2;
            const int kxs[2] = {px == 0 ? 1 : 0, 2}, dxs[2] = {px == 0 ? 0 : 1, 0}, nx = px == 0 ? 1 : 2;
            int t = 0;
            for (int a = 0; a < ny; ++a)
                for (int bb = 0; bb < nx; ++bb) {
                    cls[c].dy[t] = dys[a]; cls[c].dx[t] = dxs[bb]; cls[c].w[t] = kys[a] * 3 + kxs[bb];
                    ++t;
                }
            cls[c].n = t;
        }
    return launch_p2<MODE>(d_in_planes, in_h, in_w, d_in_info, d_weight_h2, 9, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain, shift_max,
                     d_out_f32, d_out_planes, d_out_info, p, cls, in_h, in_w, stream);
}

}  // namespace sessd

