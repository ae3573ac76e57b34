// bevconv_p2.cuh -- BEV conv / deconv (+BN+ReLU+residual) on the Hopper tensor cores (wgmma) from PRE-SPLIT fp16 planes
// (the product's default path, bevconv_p2.cu) or from an fp32 input split into fp16 planes inside the kernel (the lab's h2 mode,
// bevconv_split.cu: the bitwise reference of the folded wgmma, three separate products per MAC).
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
// Stride-1 launches from planes (REGA) feed A from registers instead: ONE patch [rows_v][pitch_u = 8 + the taps' u extent][32 channels]
// per plane serves every tap, because ldmatrix takes one address per row and so reads the 16 tile rows of a warp at any row shift of
// the swizzled patch, where a shared-memory descriptor needs whole 8-row swizzle groups.  A 3x3 patch is 2 x 18 x 10 rows instead of
// 3 x 2 x 18 x 8; the wgmma's, their order and the accumulators are the same (bit-identical outputs).
// Warps: 0-7 consumers (two warpgroups: wgmma issue, then BN/ReLU/residual -> fp32 and / or fp16 planes + running abs-max from the
// accumulator registers), 8 patch TMA, 9 weight TMA (REGA: and 10, 11, which only complete the producers' warpgroup).
#pragma once
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace sessd {

constexpr int kP2TileU = 8, kP2TileV = 16;
constexpr int kP2MaxCopies = 6, kP2MaxRowsV = 18;
// weight-stage ring ([b_lo ; b_hi] planes of n_tile 64-byte rows each per stage): as many stages as fit next to the patch buffers, at
// most kP2MaxBStages; two patch buffers when that leaves at least kP2BStages stages
constexpr int kP2BStages = 6, kP2MaxBStages = 12;
constexpr int kP2MmaWarps = 8;
constexpr int kP2PatchWarp = 8, kP2WeightWarp = 9;
constexpr int kP2Threads = 320;                           // 10 warps
// REGA: 12 warps, so that the producers' warpgroup (warps 8-11; 10 and 11 do nothing else) is whole and can hand registers to the two
// consumer warpgroups, which hold the A fragments next to the accumulators.  The CTA owns 384 x 168 registers (what ptxas gives a
// 384-thread kernel) and no more: the consumers' 8 x 32 x (232 - 168) must not exceed the producers' 4 x 32 x (168 - 40), or the
// raise never returns.
constexpr int kP2ThreadsRegA = 384, kP2RegsConsumer = 232, kP2RegsProducer = 40;
static_assert(2 * (kP2RegsConsumer - 168) <= 168 - kP2RegsProducer, "the consumers take what the producers release");
constexpr int kP2MaxSmem = 227 * 1024;
constexpr int kP2Chunk = 32;                              // input channels per K stage: one 64-byte fp16 operand row
// optional device item list (bevskip.cu): int32 record, word 0 = number of items to run, the item indices from word kP2ItemsHeader on
constexpr int kP2ItemsHeader = 32;
// optional device segment list (bevskip.cu, register-A launches only): word 0 = number of items to run, the groups from word
// kP2SegHeader on.  A group is kP2SegSlots = 16 segments of kP2TileU pixels along u in one v row, one int32 each: class << 24 | segment
// index ((b * grid_v + v) * tiles_u + u / 8), -1 for an empty slot (only after the group's last segment); item k runs group
// k / nblocks on n-block k % nblocks.  Slot s takes the place of tile v row s: rows 8 s .. 8 s + 7 of the item.
constexpr int kP2SegHeader = 32, kP2SegSlots = kP2TileV;
// operand source of the A side: pre-split fp16 planes (TMA straight into the operand layout), or an fp32 NHWC input that TMA stages in
// shared memory and the consumer warpgroups split there into fp16 (hi, lo) with the power-of-two scale of its abs-max
enum { kP2Planes = 0, kP2SplitF16 = 1 };
// lab instantiations: the product kernel with clock counters (P2Prof), or with counters and consumers that only wait on the full
// barriers and release them -- no wgmma, no epilogue: what the two TMA producers alone can pull from L2
enum { kP2NoProbe = 0, kP2ProbeClocks = 1, kP2ProbeLoads = 2 };

struct P2Params {
    int batch, cin, cout;
    int in_stride;                     // 1 or 2 (input position = output position * in_stride + tap offset)
    int out_h, out_w;                  // output tensor extent (pixels)
    int grid_u, grid_v;                // output positions computed per class along u / v
    int u_is_x;                        // 1: u = x, v = y;  0: u = y, v = x
    int out_stride, nclass;
    int cls_ntaps[4], cls_off_u[4], cls_off_v[4];
    // per (class, tap): patch copy, first v row inside the copy (REGA: first patch row, v * pitch_u + u), weight tap
    int tap_copy[4][9], tap_row[4][9], tap_w[4][9];
    int ncopies, rows_v, pitch_u;                         // copies, v rows and u positions per v row (8; REGA: 8 + the taps' u extent) of a copy
    int copy_u[kP2MaxCopies], copy_v[kP2MaxCopies];       // input coordinate of the copy's first element relative to (u0, v0) * in_stride
    int copy_bytes, patch_bytes, npatch;                  // bytes of one copy plane, of one patch buffer (ncopies x 2 planes), 1 or 2 buffers
    int load_bytes, staging_bytes;     // TMA bytes per patch buffer; fp32 staging bytes per patch buffer (split mode, else 0)
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
    const int *items;                  // nullable: run only the listed work items (count + indices, see kP2ItemsHeader), else all p.total
    const int *segs;                   // nullable (REGA only): run the listed segment groups (see kP2SegHeader) instead of tiles
    int slot_rows;                     // REGA: patch rows from one tile v row (segment slot) to the next: pitch_u (segments: a slot)
    long long *prof;                   // probe instantiations only: [grid][kP2ProfWords] clock counters (P2Prof)
};

// Stall profile of the probe instantiations (lab library): each CTA writes its clock64() counts to record blockIdx.x of p.prof.
// Consumer counters come from thread 0 (warpgroup 0), the producer counters from lane 0 of warps 8 and 9.
enum P2Prof {
    kProfCta,           // clocks from the end of the set-up to the end of the consumer loop
    kProfItems,         // work items run
    kProfSteps,         // tap steps (one [b_lo ; b_hi] stage each)
    kProfItemClk,       // clocks inside the item loop (main loop + epilogue)
    kProfBFull,         // clocks waiting on b_full
    kProfPatchFull,     // clocks waiting on patch_full
    kProfMmaWait,       // clocks inside wgmma_wait (in-loop and the drain before the epilogue)
    kProfEpilogue,      // clocks of the epilogue (after the drain)
    kProfPatchEmpty,    // patch producer: clocks waiting on patch_empty
    kProfPatchTotal,    // patch producer: clocks of its whole loop
    kProfBEmpty,        // weight producer: clocks waiting on b_empty
    kProfBTotal,        // weight producer: clocks of its whole loop
    kP2ProfWords = 16
};

// number of work items this launch runs and the k-th of them (every warp role walks the same sequence)
__device__ __forceinline__ int p2_item_count(const P2Params &p) { return p.segs ? __ldg(p.segs) : p.items ? __ldg(p.items) : p.total; }
__device__ __forceinline__ int p2_item(const P2Params &p, int k) { return p.items ? __ldg(p.items + kP2ItemsHeader + k) : k; }

// work item g -> (class rank in the heavy-first order, n-block, pixel tile): the item encoding of the kernel and of the skip planner
struct P2ItemIndex { int rank, nb, t; };
__host__ __device__ __forceinline__ P2ItemIndex p2_item_index(int g, int nblocks, int tiles) {
    const int rank = g / (nblocks * tiles), rem = g - rank * (nblocks * tiles), nb = rem / tiles;
    return {rank, nb, rem - nb * tiles};
}

struct P2Item { int cls, n0, b, u0, v0, ntaps; };

__device__ __forceinline__ P2Item p2_decode(const P2Params &p, int g) {
    P2Item it;
    const P2ItemIndex ix = p2_item_index(g, p.nblocks, p.tiles);
    int t = ix.t;
    it.cls = p.cls_order[ix.rank];
    it.n0 = ix.nb * p.n_tile;
    const int tu = t % p.tiles_u; t /= p.tiles_u;
    const int tv = t % p.tiles_v;
    it.b = t / p.tiles_v;
    it.u0 = tu * kP2TileU; it.v0 = tv * kP2TileV;
    it.ntaps = p.cls_ntaps[it.cls];
    return it;
}

// segment list: the 16 entries of item k's group, and one entry's frame, first pixel along u and v row
__device__ __forceinline__ const int *p2_seg_group(const P2Params &p, int k) {
    return p.segs + kP2SegHeader + (k / p.nblocks) * kP2SegSlots;
}
struct P2Seg { int b, u0, v; };
__device__ __forceinline__ P2Seg p2_seg(const P2Params &p, int e) {
    const int s = e & 0xFFFFFF, rest = s / p.tiles_u;
    return {rest / p.grid_v, (s - rest * p.tiles_u) * kP2TileU, rest % p.grid_v};
}

// N output columns: NT (one plane of the weight stage) or 2 NT (the whole [b_lo ; b_hi] stage)
template <int N>
__device__ __forceinline__ void p2_wgmma(float *d, uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (N == 32) wgmma_f16_n32(d, da, db, accumulate);
    else if constexpr (N == 64) wgmma_f16_n64(d, da, db, accumulate);
    else if constexpr (N == 128) wgmma_f16_n128(d, da, db, accumulate);
    else wgmma_f16_n256(d, da, db, accumulate);
}

// the same with the A fragment (one k16 of this warp's 16 rows, ldsm_x4) in registers
template <int N>
__device__ __forceinline__ void p2_wgmma_ra(float *d, const uint32_t *a, uint64_t db, uint32_t accumulate) {
    if constexpr (N == 32) wgmma_f16_ra_n32(d, a, db, accumulate);
    else if constexpr (N == 64) wgmma_f16_ra_n64(d, a, db, accumulate);
    else if constexpr (N == 128) wgmma_f16_ra_n128(d, a, db, accumulate);
    else wgmma_f16_ra_n256(d, a, db, accumulate);
}

// PROFILE only: clock64() at the start of a timed span, and the span's clocks added to clk (no code otherwise)
template <bool PROFILE>
__device__ __forceinline__ long long p2_tick() {
    if constexpr (PROFILE) return clock64();
    return 0;
}
template <bool PROFILE>
__device__ __forceinline__ void p2_tock(long long &clk, long long t0) {
    if constexpr (PROFILE) clk += clock64() - t0;
}

// split mode: the fp32 staging copy of patch buffer pb -> the (hi, lo) operand planes in the SWIZZLE_64B layout (16-byte chunk j of a
// 64-byte row r lands at chunk j ^ ((r >> 1) & 3)); run by the 256 consumer threads, which then sync among themselves
__device__ __forceinline__ void p2_split_patch(const P2Params &p, const unsigned char *staging, unsigned char *planes, float s_in, int ctid) {
    const int rows = p.rows_v * kP2TileU;
    const int copy_in = p.staging_bytes / p.ncopies;
    const int items = p.ncopies * rows * 4;
    for (int i = ctid; i < items; i += kP2MmaWarps * 32) {
        const int j = i & 3, r = (i >> 2) % rows, c = (i >> 2) / rows;
        unsigned char *hi = planes + 2 * c * p.copy_bytes + r * 64 + ((j ^ ((r >> 1) & 3)) << 4);
        // 32 fp32 per staging row -> 8 of them per 16-byte fp16 chunk
        const float4 *src = reinterpret_cast<const float4 *>(staging + c * copy_in + r * 128 + j * 32);
        const float4 a = src[0], b = src[1];
        const float x[8] = {a.x * s_in, a.y * s_in, a.z * s_in, a.w * s_in, b.x * s_in, b.y * s_in, b.z * s_in, b.w * s_in};
        __align__(16) __half h[8], l[8];
#pragma unroll
        for (int t = 0; t < 8; ++t) { h[t] = __float2half_rn(x[t]); l[t] = __float2half_rn(x[t] - __half2float(h[t])); }
        *reinterpret_cast<uint4 *>(hi) = *reinterpret_cast<const uint4 *>(h);
        *reinterpret_cast<uint4 *>(hi + p.copy_bytes) = *reinterpret_cast<const uint4 *>(l);
    }
    asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory");      // generic-proxy writes -> visible to wgmma
    asm volatile("bar.sync 1, %0;\n" ::"n"(kP2MmaWarps * 32) : "memory");
}

template <int NT, int MODE, bool REGA = false, int PROBE = kP2NoProbe>
__global__ void __launch_bounds__(REGA ? kP2ThreadsRegA : kP2Threads, 1) bev_conv_p2_kernel(const __grid_constant__ CUtensorMap map_a,
                                                                   const __grid_constant__ CUtensorMap map_b,
                                                                   const float *__restrict__ scale, const float *__restrict__ shift,
                                                                   const float *__restrict__ resid, float *__restrict__ out_f32,
                                                                   __half *__restrict__ out_planes, P2Params p) {
    static_assert(!REGA || MODE == kP2Planes, "register-fed A reads the TMA-written planes");
    constexpr bool PROFILE = PROBE != kP2NoProbe, LOADS_ONLY = PROBE == kP2ProbeLoads;
    extern __shared__ unsigned char smem_raw[];
    unsigned char *tiles = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    unsigned char *patches = tiles + p.bring_bytes;
    unsigned char *staging = patches + p.npatch * p.patch_bytes;
    uint64_t *bars = (uint64_t *)(staging + p.npatch * p.staging_bytes);
    uint64_t *patch_full = bars, *patch_empty = bars + 2, *b_full = bars + 4, *b_empty = bars + 4 + kP2MaxBStages;
    uint32_t *s_aoff = (uint32_t *)(b_empty + kP2MaxBStages);      // [4 classes][9 taps]
    // the epilogue's folded BN scale and shift, [p.cout] each: read from shared memory, so that no epilogue step waits on a global load
    // behind the main loops' TMA traffic
    float *s_scale = (float *)(((uintptr_t)(s_aoff + 4 * 9) + 15) & ~(uintptr_t)15), *s_shift = s_scale + p.cout;

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (threadIdx.x == kP2PatchWarp * 32) prefetch_tensormap(&map_a);    // descriptor fetches overlap barrier init
    if (threadIdx.x == kP2WeightWarp * 32) prefetch_tensormap(&map_b);
    const int nchunks = p.cin / kP2Chunk;
    const int nitems = p2_item_count(p);
    const uint32_t b_plane_bytes = (uint32_t)p.n_tile * 64u;      // bytes of the b_hi (or b_lo) rows per (tap, chunk)

    if (threadIdx.x == 0) {
        for (int s = 0; s < 2; ++s) { mbar_init(&patch_full[s], 1); mbar_init(&patch_empty[s], kP2MmaWarps); }
        for (int s = 0; s < p.bstages; ++s) { mbar_init(&b_full[s], 1); mbar_init(&b_empty[s], kP2MmaWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    // operand offset of every (class, tap) inside a patch buffer, in 16-byte units (REGA: in patch rows)
    for (int idx = threadIdx.x; idx < p.nclass * 9; idx += blockDim.x) {
        const int c = idx / 9, t = idx - c * 9;
        s_aoff[idx] = REGA ? (uint32_t)p.tap_row[c][t] : (uint32_t)((2 * p.tap_copy[c][t] * p.copy_bytes + p.tap_row[c][t] * 512) >> 4);
    }
    for (int n = threadIdx.x; n < p.cout; n += blockDim.x) {
        s_scale[n] = scale ? __ldg(scale + n) : 1.f;
        s_shift[n] = shift ? __ldg(shift + n) : 0.f;
    }
    __syncthreads();
    long long clk[kP2ProfWords] = {};          // PROFILE only (P2Prof)
    const long long t_start = p2_tick<PROFILE>();
    long long *prof_rec = PROFILE ? p.prof + (size_t)blockIdx.x * kP2ProfWords : nullptr;

    if (warp >= kP2MmaWarps) {
        if constexpr (REGA) setmaxnreg_dec<kP2RegsProducer>();
        if (warp == kP2PatchWarp) {
            // ===================== activation patches: per (item, 32-channel chunk) ncopies x (hi, lo) boxes =====================
            int pb = 0;
            uint32_t pph = 0;
            const uint32_t patches_u32 = smem_u32(patches);
            for (int k = blockIdx.x; k < nitems; k += gridDim.x) {
                if (REGA && p.segs) {
                    // one window [rows][pitch_u] per segment and plane into its slot: lane l loads plane l & 1 of slot l / 2
                    const int e = __ldg(p2_seg_group(p, k) + (lane >> 1));
                    const P2Seg sg = p2_seg(p, e);
                    const uint32_t bytes = (uint32_t)__popc(__ballot_sync(0xFFFFFFFFu, e >= 0)) * (uint32_t)p.load_bytes;
                    const uint32_t dst0 = patches_u32 + (uint32_t)((lane & 1) * p.copy_bytes + (lane >> 1) * p.slot_rows * 64);
                    for (int cc = 0; cc < nchunks; ++cc) {
                        { const long long t0 = p2_tick<PROFILE>(); mbar_wait<REGA>(&patch_empty[pb], pph ^ 1u); p2_tock<PROFILE>(clk[kProfPatchEmpty], t0); }
                        if (elect_one()) mbar_expect_tx(&patch_full[pb], bytes);
                        __syncwarp();
                        if (e >= 0)
                            tma_load_5d(dst0 + (uint32_t)(pb * p.patch_bytes), &map_a, &patch_full[pb], cc * kP2Chunk, sg.u0 + p.copy_u[0],
                                        sg.v + p.copy_v[0], sg.b, lane & 1);
                        __syncwarp();
                        if (++pb == p.npatch) { pb = 0; pph ^= 1u; }
                    }
                    continue;
                }
                const P2Item it = p2_decode(p, p2_item(p, k));
                const int bu = it.u0 * p.in_stride, bv = it.v0 * p.in_stride;
                for (int cc = 0; cc < nchunks; ++cc) {
                    { const long long t0 = p2_tick<PROFILE>(); mbar_wait<REGA>(&patch_empty[pb], pph ^ 1u); p2_tock<PROFILE>(clk[kProfPatchEmpty], t0); }
                    if (elect_one()) {
                        mbar_expect_tx(&patch_full[pb], (uint32_t)p.load_bytes);
                        if constexpr (MODE == kP2Planes) {
                            uint32_t dst = patches_u32 + (uint32_t)(pb * p.patch_bytes);
                            for (int c = 0; c < p.ncopies; ++c, dst += 2u * (uint32_t)p.copy_bytes) {
                                const int cu = bu + p.copy_u[c], cv = bv + p.copy_v[c];
                                tma_load_5d(dst, &map_a, &patch_full[pb], cc * kP2Chunk, cu, cv, it.b, 0);
                                tma_load_5d(dst + (uint32_t)p.copy_bytes, &map_a, &patch_full[pb], cc * kP2Chunk, cu, cv, it.b, 1);
                            }
                        } else {
                            const uint32_t copy_in = (uint32_t)(p.staging_bytes / p.ncopies);
                            uint32_t dst = smem_u32(staging) + (uint32_t)(pb * p.staging_bytes);
                            for (int c = 0; c < p.ncopies; ++c, dst += copy_in)
                                tma_load_5d(dst, &map_a, &patch_full[pb], cc * kP2Chunk, bu + p.copy_u[c], bv + p.copy_v[c], it.b, 0);
                        }
                    }
                    __syncwarp();
                    if (++pb == p.npatch) { pb = 0; pph ^= 1u; }
                }
            }
            if constexpr (PROFILE)
                if (lane == 0) {
                    prof_rec[kProfPatchEmpty] = clk[kProfPatchEmpty];
                    prof_rec[kProfPatchTotal] = clock64() - t_start;
                }
        } else if (warp == kP2WeightWarp) {
            // ===================== weight tiles: one [b_lo ; b_hi] stage per (item, chunk, tap) =====================
            int S = 0;
            uint32_t bph = 0;
            for (int k = blockIdx.x; k < nitems; k += gridDim.x) {
                P2Item it;
                if (REGA && p.segs) {
                    it.cls = __ldg(p2_seg_group(p, k)) >> 24;
                    it.n0 = (k % p.nblocks) * p.n_tile;
                    it.ntaps = p.cls_ntaps[it.cls];
                } else {
                    it = p2_decode(p, p2_item(p, k));
                }
                for (int cc = 0; cc < nchunks; ++cc)
                    for (int tap = 0; tap < it.ntaps; ++tap) {
                        { const long long t0 = p2_tick<PROFILE>(); mbar_wait<REGA>(&b_empty[S], bph ^ 1u); p2_tock<PROFILE>(clk[kProfBEmpty], t0); }
                        if (elect_one()) {
                            unsigned char *st = tiles + S * p.bstage_bytes;
                            const int wtap = p.tap_w[it.cls][tap];
                            mbar_expect_tx(&b_full[S], 2 * b_plane_bytes);
                            tma_load_4d(st + b_plane_bytes, &map_b, &b_full[S], cc * kP2Chunk, it.n0, wtap, 0);
                            tma_load_4d(st, &map_b, &b_full[S], cc * kP2Chunk, it.n0, wtap, 1);
                        }
                        __syncwarp();
                        if (++S == p.bstages) { S = 0; bph ^= 1u; }
                    }
            }
            if constexpr (PROFILE)
                if (lane == 0) {
                    prof_rec[kProfBEmpty] = clk[kProfBEmpty];
                    prof_rec[kProfBTotal] = clock64() - t_start;
                }
        }
    } else {
        if constexpr (REGA) setmaxnreg_inc<kP2RegsConsumer>();
        // ===================== consumers (warps 0-7): wgmma over (chunk, tap), then BN / ReLU / residual / stores =====================
        const int wg = warp >> 2, wq = warp & 3;
        constexpr int kAcc = NT / 2;
        const uint32_t a_rows = (uint32_t)(wg * 64 * 64) >> 4;         // this warpgroup's 64 rows (8 swizzle groups of 512 B), 16-byte units
        const uint32_t tiles_lo = desc_lo(smem_u32(tiles));
        const uint32_t patch_lo = desc_lo(smem_u32(patches)) + a_rows;
        const uint32_t plane_lo = b_plane_bytes >> 4;
        const uint32_t copy_lo = (uint32_t)(p.copy_bytes >> 4), patch_sz = (uint32_t)(p.patch_bytes >> 4);
        // REGA: lane l gives ldmatrix the address of row l % 8 of matrix l / 8 -- matrices 0, 1 = tile rows 0-7, 8-15 of this warp's
        // 16 (one v row of 8 u each), matrices 2, 3 the same rows 16 bytes on.  Its patch row before the tap's shift, and 16-byte chunk:
        // (segments: the first row of slot v instead of tile v row v)
        const uint32_t a_row = (uint32_t)((wg * 8 + wq * 2 + ((lane >> 3) & 1)) * p.slot_rows + (lane & 7)), a_chunk = (uint32_t)(lane >> 4);
        const uint32_t patches_u32 = smem_u32(patches);
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
        for (int k = blockIdx.x; k < nitems; k += gridDim.x) {
            const long long t_item = p2_tick<PROFILE>();
            const int g = p2_item(p, k);
            const int *grp = REGA && p.segs ? p2_seg_group(p, k) : nullptr;
            const int cls = grp ? __ldg(grp) >> 24 : p.cls_order[g / per_cls];
            const int ntaps = p.cls_ntaps[cls];
            const uint32_t *aoff = s_aoff + cls * 9;
            // acc[0, kAcc): cross a_hi x b_lo + a_lo x b_hi, acc[kAcc, NT): main a_hi x b_hi -- the fragment of an m64n(2 NT) over the
            // whole [b_lo ; b_hi] weight stage.  The cross half comes first: ptxas serializes every wgmma of the kernel when one of them
            // accumulates into a part of another's fragment that does not start at its first register.
            float acc[NT];
#pragma unroll
            for (int i = 0; i < NT; ++i) acc[i] = 0.f;
            int prevS = -1, prev_pb = -1;
            bool first = true;
            if constexpr (REGA) {
                // the A fragments of a tap step, {a_hi k 0-15, a_hi k 16-31, a_lo k 0-15, a_lo k 16-31}.  Two sets, taken in turn: the
                // tensor core reads a step's set until the wgmma_wait<1> of the NEXT step has retired the step.
                uint32_t frag[2][16];
                int tap = 0;
                uint32_t pbase = 0;
                // the A fragments of the step at (pb, tap) -> fa
                auto load_frags = [&](uint32_t *fa) {
                    if (tap == 0) {
                        { const long long t0 = p2_tick<PROFILE>(); mbar_wait<REGA>(&patch_full[pb], pph); p2_tock<PROFILE>(clk[kProfPatchFull], t0); }
                        pbase = patches_u32 + (uint32_t)(pb * p.patch_bytes);
                    }
                    if constexpr (!LOADS_ONLY) {
                        // patch row r is 64 bytes at r * 64, its 16-byte chunk j at j ^ ((r >> 1) & 3) (SWIZZLE_64B); k 16-31 = chunk + 2
                        const uint32_t r = a_row + aoff[tap];
                        const uint32_t a_hi = pbase + r * 64u + ((a_chunk ^ ((r >> 1) & 3u)) << 4), a_lo = a_hi + (uint32_t)p.copy_bytes;
                        ldsm_x4(fa, a_hi);
                        ldsm_x4(fa + 4, a_hi ^ 32u);
                        ldsm_x4(fa + 8, a_lo);
                        ldsm_x4(fa + 12, a_lo ^ 32u);
                    }
                };
                // one tap step from the fragments fa: the planes sequence of the descriptor path below, its a_hi and its a_lo instructions
                // as two groups; between them, once the previous step has retired, the next step's fragments load into that step's set fn,
                // so that their latency runs under the a_lo group's issue
                auto step_ra = [&](const uint32_t *fa, uint32_t *fn, bool more) {
                    { const long long t0 = p2_tick<PROFILE>(); mbar_wait<REGA>(&b_full[S], bph); p2_tock<PROFILE>(clk[kProfBFull], t0); }
                    const uint64_t db_lo = kDescSw64Hi | (uint64_t)(tiles_lo + (uint32_t)(S * (p.bstage_bytes >> 4)));
                    const uint64_t db_hi = db_lo + (uint64_t)plane_lo;
                    if constexpr (!LOADS_ONLY) {
                        wgmma_fence();
                        p2_wgmma_ra<2 * NT>(acc, fa, db_lo, first ? 0u : 1u);
                        p2_wgmma_ra<2 * NT>(acc, fa + 4, db_lo + 2, 1u);
                        wgmma_commit();
                    }
                    first = false;
                    if constexpr (PROFILE) ++clk[kProfSteps];
                    // all but this step's a_hi group has retired: the previous step's stage and fragment set are free
                    { const long long t0 = p2_tick<PROFILE>(); wgmma_wait<1>(); p2_tock<PROFILE>(clk[kProfMmaWait], t0); }
                    if (lane == 0 && prevS >= 0) mbar_arrive(&b_empty[prevS]);
                    prevS = S;
                    if (++S == p.bstages) { S = 0; bph ^= 1u; }
                    if (++tap == ntaps) {      // the chunk's last fragments are in registers: its patch is free
                        tap = 0;
                        if (lane == 0) mbar_arrive(&patch_empty[pb]);
                        if (++pb == p.npatch) { pb = 0; pph ^= 1u; }
                    }
                    if (more) load_frags(fn);
                    if constexpr (!LOADS_ONLY) {
                        wgmma_fence();
                        p2_wgmma_ra<NT>(acc, fa + 8, db_hi, 1u);                          // cross  += a_lo x b_hi
                        p2_wgmma_ra<NT>(acc, fa + 12, db_hi + 2, 1u);
                        wgmma_commit();
                    }
                };
                const int nsteps = nchunks * ntaps;
                load_frags(frag[0]);
#pragma unroll 1
                for (int st = 0; st + 1 < nsteps; st += 2) { step_ra(frag[0], frag[1], true); step_ra(frag[1], frag[0], st + 2 < nsteps); }
                if (nsteps & 1) step_ra(frag[0], frag[1], false);
            } else {
                for (int cc = 0; cc < nchunks; ++cc) {
                    { const long long t0 = p2_tick<PROFILE>(); mbar_wait(&patch_full[pb], pph); p2_tock<PROFILE>(clk[kProfPatchFull], t0); }
                    if constexpr (MODE == kP2SplitF16)
                        p2_split_patch(p, staging + pb * p.staging_bytes, patches + pb * p.patch_bytes, s_in, threadIdx.x);
                    const uint32_t pbase = patch_lo + (uint32_t)pb * patch_sz;
#pragma unroll 1
                    for (int tap = 0; tap < ntaps; ++tap) {
                        { const long long t0 = p2_tick<PROFILE>(); mbar_wait(&b_full[S], bph); p2_tock<PROFILE>(clk[kProfBFull], t0); }
                        if constexpr (!LOADS_ONLY) {
                            const uint64_t da_hi = kDescSw64Hi | (uint64_t)(pbase + aoff[tap]);
                            const uint64_t da_lo = da_hi + (uint64_t)copy_lo;
                            const uint64_t db_lo = kDescSw64Hi | (uint64_t)(tiles_lo + (uint32_t)(S * (p.bstage_bytes >> 4)));
                            const uint64_t db_hi = db_lo + (uint64_t)plane_lo;
                            const uint32_t accum = first ? 0u : 1u;
                            // K = 16 fp16 per instruction = 32 bytes of the 64-byte row
                            wgmma_fence();
                            if constexpr (MODE == kP2Planes) {
                                // one m64n(2 NT) per k16 over the stacked stage: cross (+)= a_hi x b_lo and main (+)= a_hi x b_hi read
                                // a_hi once.  Each accumulator sums in the order of the three-product sequence below (the h2 mode's
                                // bitwise reference).
                                p2_wgmma<2 * NT>(acc, da_hi, db_lo, accum);
                                p2_wgmma<2 * NT>(acc, da_hi + 2, db_lo + 2, 1u);
                            } else {
                                p2_wgmma<NT>(acc + kAcc, da_hi, db_hi, accum);       // main  (+)= a_hi x b_hi
                                p2_wgmma<NT>(acc + kAcc, da_hi + 2, db_hi + 2, 1u);
                                p2_wgmma<NT>(acc, da_hi, db_lo, accum);              // cross (+)= a_hi x b_lo
                                p2_wgmma<NT>(acc, da_hi + 2, db_lo + 2, 1u);
                            }
                            p2_wgmma<NT>(acc, da_lo, db_hi, 1u);                     // cross  += a_lo x b_hi
                            p2_wgmma<NT>(acc, da_lo + 2, db_hi + 2, 1u);
                            wgmma_commit();
                        }
                        first = false;
                        if constexpr (PROFILE) ++clk[kProfSteps];
                        // the previous step's operands are no longer read
                        { const long long t0 = p2_tick<PROFILE>(); wgmma_wait<1>(); p2_tock<PROFILE>(clk[kProfMmaWait], t0); }
                        if (lane == 0) {
                            if (prevS >= 0) mbar_arrive(&b_empty[prevS]);
                            if (prev_pb >= 0) mbar_arrive(&patch_empty[prev_pb]);
                        }
                        prevS = S;
                        prev_pb = (tap == ntaps - 1) ? pb : -1;
                        if (++S == p.bstages) { S = 0; bph ^= 1u; }
                    }
                    if (p.npatch == 1) {
                        // one patch buffer: the next chunk's patch can only land once this one is released, so release it now rather
                        // than after the next chunk's first step (that step would wait for the patch forever)
                        { const long long t0 = p2_tick<PROFILE>(); wgmma_wait<0>(); p2_tock<PROFILE>(clk[kProfMmaWait], t0); }
                        if (lane == 0) {
                            mbar_arrive(&b_empty[prevS]);
                            mbar_arrive(&patch_empty[pb]);
                        }
                        prevS = prev_pb = -1;
                    }
                    if (++pb == p.npatch) { pb = 0; pph ^= 1u; }
                }
            }
            // segments: the entries of this thread's two slots (rows r0 and r0 + 8 below), loaded while the last wgmmas drain
            int seg_e[2] = {-1, -1};
            if (grp) { seg_e[0] = __ldg(grp + wg * 8 + wq * 2); seg_e[1] = __ldg(grp + wg * 8 + wq * 2 + 1); }
            { const long long t0 = p2_tick<PROFILE>(); wgmma_wait<0>(); p2_tock<PROFILE>(clk[kProfMmaWait], t0); }
            const long long t_epi = p2_tick<PROFILE>();
            wgmma_fence_regs<NT>(acc);
            if (lane == 0) {
                if (prevS >= 0) mbar_arrive(&b_empty[prevS]);
                if (prev_pb >= 0) mbar_arrive(&patch_empty[prev_pb]);
            }
            // epilogue: this thread holds tile rows r0 and r0 + 8, two adjacent channels of every 8-channel group; a transpose inside
            // each quad of lanes (one row) gives every lane 8 whole channels, stored 16 bytes at a time
#pragma unroll
            for (int i = 0; i < kAcc; ++i) acc[i] = acc[kAcc + i] + acc[i];      // main + cross
            P2Item it = grp ? P2Item{cls, (k % p.nblocks) * p.n_tile, 0, 0, 0, ntaps} : p2_decode(p, g);
            const int q = lane & 3;
            const int r0 = wg * 64 + wq * 16 + (lane >> 2);
            bool rows_ok[2];
            size_t opixs[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r0 + 8 * h;
                const int lv = r / kP2TileU, lu = r % kP2TileU;
                if (grp) {      // slot lv holds segment seg_e[h]: its pixels along u are this item's rows 8 lv .. 8 lv + 7
                    const P2Seg sg = p2_seg(p, seg_e[h]);
                    it.b = seg_e[h] >= 0 ? sg.b : p.batch; it.u0 = sg.u0; it.v0 = sg.v - lv;
                }
                const int gu = it.u0 + lu, gv = it.v0 + lv;
                rows_ok[h] = it.b < p.batch && gu < p.grid_u && gv < p.grid_v;      // the same in the four lanes of a quad
                const int ou = gu * p.out_stride + p.cls_off_u[it.cls], ov = gv * p.out_stride + p.cls_off_v[it.cls];
                const int oy = p.u_is_x ? ov : ou, ox = p.u_is_x ? ou : ov;
                opixs[h] = ((size_t)it.b * p.out_h + (size_t)oy) * p.out_w + (size_t)ox;
            }
#pragma unroll
            for (int j = 0; j < (LOADS_ONLY ? 0 : NT / 32); ++j)      // the loads probe has nothing to store
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const bool row_ok = rows_ok[h];
                    const size_t opix = opixs[h];
                    float v[8], o[8] = {};
                    quad_transpose8(acc + 16 * j + 2 * h, q, v);
                    const int n = it.n0 + 32 * j + 8 * q;      // this lane's 8 channels; cout % 8 == 0: all exist or none
                    const size_t off = opix * p.cout + n;
                    if (row_ok && n < p.cout) {
                        float sc[8], sh[8];
#pragma unroll
                        for (int t = 0; t < 8; t += 4) {
                            const float4 a = *reinterpret_cast<const float4 *>(s_scale + n + t);
                            const float4 b = *reinterpret_cast<const float4 *>(s_shift + n + t);
                            sc[t] = a.x; sc[t + 1] = a.y; sc[t + 2] = a.z; sc[t + 3] = a.w;
                            sh[t] = b.x; sh[t + 1] = b.y; sh[t + 2] = b.z; sh[t + 3] = b.w;
                        }
#pragma unroll
                        for (int t = 0; t < 8; ++t) {
                            o[t] = fmaf(v[t] * inv_sa, sc[t], sh[t]);
                            if (p.relu) o[t] = fmaxf(o[t], 0.f);
                        }
                        if (resid) {
#pragma unroll
                            for (int t = 0; t < 8; t += 4) {
                                const float4 rr = __ldg(reinterpret_cast<const float4 *>(resid + off + t));
                                o[t] += rr.x; o[t + 1] += rr.y; o[t + 2] += rr.z; o[t + 3] += rr.w;
                            }
                        }
#pragma unroll
                        for (int t = 0; t < 8; ++t) vmax = fmaxf(vmax, fabsf(o[t]));
                        if (out_planes) {
                            __align__(16) __half2 hi[4], lo[4];
#pragma unroll
                            for (int t = 0; t < 4; ++t) {
                                const float x0 = o[2 * t] * s_out, x1 = o[2 * t + 1] * s_out;
                                hi[t] = __floats2half2_rn(x0, x1);
                                const float2 f = __half22float2(hi[t]);
                                lo[t] = __floats2half2_rn(x0 - f.x, x1 - f.y);
                            }
                            *reinterpret_cast<uint4 *>(out_planes + off) = *reinterpret_cast<const uint4 *>(hi);
                            *reinterpret_cast<uint4 *>(out_planes + p.out_plane_stride + off) = *reinterpret_cast<const uint4 *>(lo);
                        }
                    }
                    if (out_f32) {
                        // lanes q and q ^ 2 trade half groups, so that each of the two stores of a quad covers 16 whole channels
                        // (groups 0-1, then 2-3 of the block): lane q keeps half (q >> 1) of group q, gets the same half of group q ^ 2
                        const bool up = q & 2;
                        float keep[4], recv[4];
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            keep[t] = up ? o[4 + t] : o[t];
                            recv[t] = __shfl_xor_sync(0xFFFFFFFFu, up ? o[t] : o[4 + t], 2);
                        }
                        const int n_lo = it.n0 + 32 * j + 8 * (q & 1), c_lo = n_lo + 4 * (q >> 1);
                        const float4 w_lo = up ? make_float4(recv[0], recv[1], recv[2], recv[3]) : make_float4(keep[0], keep[1], keep[2], keep[3]);
                        const float4 w_hi = up ? make_float4(keep[0], keep[1], keep[2], keep[3]) : make_float4(recv[0], recv[1], recv[2], recv[3]);
                        if (row_ok && n_lo < p.cout) *reinterpret_cast<float4 *>(out_f32 + opix * p.cout + c_lo) = w_lo;
                        if (row_ok && n_lo + 16 < p.cout) *reinterpret_cast<float4 *>(out_f32 + opix * p.cout + c_lo + 16) = w_hi;
                    }
                }
            if constexpr (PROFILE) {
                const long long t_end = clock64();
                clk[kProfEpilogue] += t_end - t_epi;
                clk[kProfItemClk] += t_end - t_item;
                ++clk[kProfItems];
            }
        }
        if constexpr (PROFILE)
            if (threadIdx.x == 0) {
                clk[kProfCta] = clock64() - t_start;
                for (int w = kProfCta; w <= kProfEpilogue; ++w) prof_rec[w] = clk[w];
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

// per class: the taps (dy, dx, weight tap) and the (y, x) offset of its output positions (output = grid position * out_stride + offset)
struct P2Taps { int n, dy[9], dx[9], w[9], off_y, off_x; };

// ConvTranspose2d(k3, s2, p1, op1) as four output-parity classes c = 2 py + px over the input grid, output offset (py, px):
// out[2y+py] receives in[y+dy] * W[ky] with 2y+py = 2(y+dy) - 1 + ky, i.e. ky = py + 1 - 2 dy for dy = py .. 0 (the same along x)
static void p2_deconv_classes(P2Taps cls[4]) {
    for (int c = 0; c < 4; ++c) {
        P2Taps &k = cls[c];
        k = {};
        k.off_y = c >> 1; k.off_x = c & 1;
        for (int dy = k.off_y; dy >= 0; --dy)
            for (int dx = k.off_x; dx >= 0; --dx, ++k.n) {
                k.dy[k.n] = dy; k.dx[k.n] = dx; k.w[k.n] = (k.off_y + 1 - 2 * dy) * 3 + (k.off_x + 1 - 2 * dx);
            }
    }
}

constexpr int p2_n_tile(int cout) { return cout <= 32 ? 32 : 128; }      // output channels per work item

// The work items of one launch (the launcher's and the skip planner's): the class grid cut into 8 (u) x 16 (v) pixel tiles, u / v
// mapped to (y, x) or (x, y), whichever gives fewer tiles; n-blocks of n_tile channels over the packed weight width cout_pad; classes
// heavy first (descending tap count).  Item g = (rank * nblocks + n-block) * tiles + tile, tile = (b * tiles_v + tv) * tiles_u + tu.
struct P2Geometry {
    int u_is_x, grid_u, grid_v, tiles_u, tiles_v, tiles;
    int n_tile, nblocks, nclass, total;
    int ntaps[4], off_u[4], off_v[4], order[4];
};

static int p2_geometry(P2Geometry &g, int batch, int grid_h, int grid_w, int cout, int cout_pad, const P2Taps *cls, int nclass) {
    g = {};
    if (batch < 1 || grid_h < 1 || grid_w < 1 || cout < 8 || cout % 8) return SESSD_EINVAL;      // 8-channel stores
    g.n_tile = p2_n_tile(cout);
    if (cout_pad % g.n_tile || cout_pad < cout) return SESSD_EINVAL;
    // orientation: the in-group dimension u has the 8-pixel tile edge; pick the mapping with fewer tiles
    g.u_is_x = div_up(grid_w, kP2TileU) * div_up(grid_h, kP2TileV) <= div_up(grid_h, kP2TileU) * div_up(grid_w, kP2TileV);
    g.grid_u = g.u_is_x ? grid_w : grid_h; g.grid_v = g.u_is_x ? grid_h : grid_w;
    g.tiles_u = div_up(g.grid_u, kP2TileU); g.tiles_v = div_up(g.grid_v, kP2TileV);
    g.tiles = g.tiles_u * g.tiles_v * batch;
    g.nblocks = cout_pad / g.n_tile;
    g.nclass = nclass; g.total = nclass * g.nblocks * g.tiles;
    for (int c = 0; c < nclass; ++c) {
        g.ntaps[c] = cls[c].n;
        g.off_u[c] = g.u_is_x ? cls[c].off_x : cls[c].off_y;
        g.off_v[c] = g.u_is_x ? cls[c].off_y : cls[c].off_x;
        g.order[c] = c;
    }
    for (int i = 1; i < nclass; ++i)            // insertion sort by descending tap count
        for (int k = i; k > 0 && g.ntaps[g.order[k]] > g.ntaps[g.order[k - 1]]; --k) {
            const int tmp = g.order[k]; g.order[k] = g.order[k - 1]; g.order[k - 1] = tmp;
        }
    return 0;
}

// The launch plan: work-item geometry (p2_geometry), the patch copies and every (class, tap)'s copy, row and weight tap, and the
// shared-memory split between the patch buffers and the weight-stage ring.  Reads p.batch, p.cin, p.cout and p.in_stride, fills the
// plan fields of p and *smem (dynamic shared memory bytes), or returns SESSD_EINVAL for a launch the kernel cannot run.  Host only.
// segs (register A only): the items are segment groups (kP2SegHeader): each of the 16 slots gets its own window of the taps' v extent
// x pitch_u rows, padded to whole 512-byte swizzle periods, and the launch always keeps two patch buffers.
static int p2_plan(P2Params &p, const P2Taps *cls, int nclass, int grid_h, int grid_w, int cout_pad, int mode, bool reg_a, int *smem,
                   bool segs = false) {
    if (reg_a && (mode != kP2Planes || p.in_stride != 1)) return SESSD_EINVAL;
    if (segs && !reg_a) return SESSD_EINVAL;
    if (p.cin < 64 || p.cin % 64) return SESSD_EINVAL;      // whole 64-channel groups
    P2Geometry g;
    if (p2_geometry(g, p.batch, grid_h, grid_w, p.cout, cout_pad, cls, nclass)) return SESSD_EINVAL;
    p.u_is_x = g.u_is_x; p.grid_u = g.grid_u; p.grid_v = g.grid_v;
    p.tiles_u = g.tiles_u; p.tiles_v = g.tiles_v; p.tiles = g.tiles;
    p.n_tile = g.n_tile; p.nblocks = g.nblocks; p.nclass = g.nclass; p.total = g.total;
    for (int c = 0; c < 4; ++c) {
        p.cls_ntaps[c] = g.ntaps[c]; p.cls_off_u[c] = g.off_u[c]; p.cls_off_v[c] = g.off_v[c]; p.cls_order[c] = g.order[c];
    }
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
    p.pitch_u = kP2TileU;
    for (int k = 0; k < p.ncopies; ++k) p.rows_v = max(p.rows_v, kP2TileV + (vmax[k] - vmin[k]) / s);
    if (p.rows_v > kP2MaxRowsV) return SESSD_EINVAL;
    for (int k = 0; k < p.ncopies; ++k) { p.copy_u[k] = key_u[k]; p.copy_v[k] = vmin[k]; }
    if (reg_a) {      // the same taps from one copy: from their least shift, wide and tall enough for their greatest (one TMA box)
        int umin = key_u[0], umax = key_u[0];
        for (int k = 1; k < p.ncopies; ++k) {
            umin = min(umin, key_u[k]); umax = max(umax, key_u[k]);
            vmin[0] = min(vmin[0], vmin[k]); vmax[0] = max(vmax[0], vmax[k]);
        }
        p.ncopies = 1;
        p.copy_u[0] = umin; p.copy_v[0] = vmin[0];
        p.pitch_u = kP2TileU + umax - umin; p.rows_v = kP2TileV + vmax[0] - vmin[0];
        if (p.pitch_u > 256 || p.rows_v > 256) return SESSD_EINVAL;
    }
    for (int c = 0; c < p.nclass; ++c) {
        for (int t = 0; t < cls[c].n; ++t) {
            const int tu = p.u_is_x ? cls[c].dx[t] : cls[c].dy[t], tv = p.u_is_x ? cls[c].dy[t] : cls[c].dx[t];
            const int vm = ((tv % s) + s) % s;
            int k = 0;
            for (; k < p.ncopies; ++k)
                if (key_u[k] == tu && key_vm[k] == vm) break;
            p.tap_copy[c][t] = reg_a ? 0 : k;
            p.tap_row[c][t] = reg_a ? (tv - p.copy_v[0]) * p.pitch_u + (tu - p.copy_u[0]) : (tv - vmin[k]) / s;
            p.tap_w[c][t] = cls[c].w[t];
        }
    }
    p.copy_bytes = (p.rows_v * p.pitch_u * 64 + 511) & ~511;      // whole 512-byte swizzle periods: every copy starts one
    p.slot_rows = p.pitch_u;
    if (segs) {
        const int win = (p.rows_v - kP2TileV + 1) * p.pitch_u;       // rows of one segment's window
        p.slot_rows = (win + 7) & ~7;
        p.copy_bytes = kP2SegSlots * p.slot_rows * 64;
    }
    p.patch_bytes = p.ncopies * 2 * p.copy_bytes;
    // fp32 staging (split mode): 32 channels = 128-byte rows
    p.staging_bytes = mode == kP2Planes ? 0 : p.ncopies * p.rows_v * kP2TileU * kP2Chunk * 4;
    p.load_bytes = mode == kP2Planes ? p.ncopies * 2 * p.rows_v * p.pitch_u * 64 : p.staging_bytes;
    if (segs) p.load_bytes = (p.rows_v - kP2TileV + 1) * p.pitch_u * 64;      // one window of one plane
    const int per_buf = p.patch_bytes + p.staging_bytes, bstage = 2 * p.n_tile * 64;
    // after the ring and the patch buffers: barriers and tap offsets (1536 B with the 1 KB alignment slack), then scale / shift
    const int tail = 1536 + 16 + 2 * 4 * p.cout;
    // two patch buffers when kP2BStages weight stages fit next to them, else one; then every stage that fits (>= 2), up to kP2MaxBStages
    p.npatch = (segs || kP2BStages * bstage + tail + 2 * per_buf <= kP2MaxSmem) ? 2 : 1;
    p.bstage_bytes = bstage;
    p.bstages = min((kP2MaxSmem - tail - p.npatch * per_buf) / bstage, kP2MaxBStages);
    if (p.bstages < 2) return SESSD_EINVAL;
    p.bring_bytes = p.bstages * bstage;
    *smem = p.bring_bytes + tail + p.npatch * per_buf;
    return 0;
}

// MODE kP2Planes: d_in = fp16 planes [2][B][H][W][C], d_in_info = {abs-max, S}; kP2SplitF16: d_in = fp32 NHWC, d_in_info = the input's
// abs-max (nullable); d_out_info is {abs-max, S_out} in the planes mode and a single running abs-max otherwise
template <int MODE, int PROBE = kP2NoProbe>
static int launch_p2(const void *d_in_planes, int in_h, int in_w, const float *d_in_info, const void *d_w, int w_taps, int cout_pad,
                     const float *d_scale, const float *d_shift, const float *d_residual, const float *d_resid_info, float gain,
                     float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info, P2Params &p, const P2Taps *cls, int nclass,
                     int grid_h, int grid_w, bool reg_a, void *stream) {
    if (!d_in_planes || !d_w || (!d_out_f32 && !d_out_planes)) return SESSD_EINVAL;
    if (MODE == kP2Planes && (!d_in_info || !d_scale)) return SESSD_EINVAL;
    if (MODE != kP2Planes && d_out_planes) return SESSD_EINVAL;
    // the epilogue reads and writes 16 bytes at a time
    if (((uintptr_t)d_scale | (uintptr_t)d_shift | (uintptr_t)d_residual | (uintptr_t)d_out_f32 | (uintptr_t)d_out_planes) & 15)
        return SESSD_EINVAL;
    int smem = 0;
    if (p.items && p.segs) return SESSD_EINVAL;
    if (p2_plan(p, cls, nclass, grid_h, grid_w, cout_pad, MODE, reg_a, &smem, p.segs != nullptr)) return SESSD_EINVAL;
    // a skip-plan record numbers the items of the width the runner packs: any other width decodes them to other classes / n-blocks
    if ((p.items || p.segs) && cout_pad != div_up(p.cout, p.n_tile) * p.n_tile) return SESSD_EINVAL;
    // segment entries hold the segment index in 24 bits
    if (p.segs && (long long)p.batch * p.grid_v * p.tiles_u >= (1 << 24)) return SESSD_EINVAL;
    const int s = p.in_stride;
    CUtensorMap map_a, map_b;
    if (MODE != kP2Planes) {   // fp32 NHWC [B][H][W][C] viewed as {C, U, V, B, 1}, staged unswizzled
        const cuuint64_t row_w = (cuuint64_t)p.cin * 4, row_h = (cuuint64_t)in_w * p.cin * 4;
        const cuuint64_t dims[5] = {(cuuint64_t)p.cin, (cuuint64_t)(p.u_is_x ? in_w : in_h), (cuuint64_t)(p.u_is_x ? in_h : in_w),
                                    (cuuint64_t)p.batch, 1};
        const cuuint64_t strides[4] = {p.u_is_x ? row_w : row_h, p.u_is_x ? row_h : row_w, (cuuint64_t)in_h * in_w * p.cin * 4,
                                       (cuuint64_t)p.batch * in_h * in_w * p.cin * 4};
        const cuuint32_t box[5] = {(cuuint32_t)kP2Chunk, (cuuint32_t)(kP2TileU * s), (cuuint32_t)(p.rows_v * s), 1, 1};
        const cuuint32_t estr[5] = {1, (cuuint32_t)s, (cuuint32_t)s, 1, 1};
        int rc = encode_map_nd(&map_a, d_in_planes, 5, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_DATA_TYPE_FLOAT32);
        if (rc) return rc;
    } else {   // planes [2][B][H][W][C] fp16 viewed as {C, U, V, B, plane}
        const cuuint64_t row_w = (cuuint64_t)p.cin * 2, row_h = (cuuint64_t)in_w * p.cin * 2;
        const cuuint64_t dims[5] = {(cuuint64_t)p.cin, (cuuint64_t)(p.u_is_x ? in_w : in_h), (cuuint64_t)(p.u_is_x ? in_h : in_w),
                                    (cuuint64_t)p.batch, 2};
        const cuuint64_t strides[4] = {p.u_is_x ? row_w : row_h, p.u_is_x ? row_h : row_w, (cuuint64_t)in_h * in_w * p.cin * 2,
                                       (cuuint64_t)p.batch * in_h * in_w * p.cin * 2};
        // segments: one window of the taps' v extent per box
        const int box_v = p.segs ? p.rows_v - kP2TileV + 1 : p.rows_v;
        const cuuint32_t box[5] = {(cuuint32_t)kP2Chunk, (cuuint32_t)(p.pitch_u * s), (cuuint32_t)(box_v * s), 1, 1};
        const cuuint32_t estr[5] = {1, (cuuint32_t)s, (cuuint32_t)s, 1, 1};
        int rc = encode_map_nd(&map_a, d_in_planes, 5, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_64B);
        if (rc) return rc;
    }
    {   // weights [2 (hi|lo)][taps][cout_pad][cin] fp16: 64-byte rows of one K stage
        const cuuint64_t dims[4] = {(cuuint64_t)p.cin, (cuuint64_t)cout_pad, (cuuint64_t)w_taps, 2};
        const cuuint64_t strides[3] = {(cuuint64_t)p.cin * 2, (cuuint64_t)cout_pad * p.cin * 2, (cuuint64_t)w_taps * cout_pad * p.cin * 2};
        const cuuint32_t box[4] = {(cuuint32_t)kP2Chunk, (cuuint32_t)p.n_tile, 1, 1};
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        int rc = encode_map_nd(&map_b, d_w, 4, dims, strides, box, estr, CU_TENSOR_MAP_SWIZZLE_64B);
        if (rc) return rc;
    }
    // A from registers only in the planes mode: the split mode writes its operand planes from the consumer threads
    constexpr bool kRegA = MODE == kP2Planes;
    auto kernel = bev_conv_p2_kernel<128, MODE, false, PROBE>;
    if (p.n_tile == 32) kernel = reg_a ? bev_conv_p2_kernel<32, MODE, kRegA, PROBE> : bev_conv_p2_kernel<32, MODE, false, PROBE>;
    else if (reg_a) kernel = bev_conv_p2_kernel<128, MODE, kRegA, PROBE>;
    static bool attr_done[2][2] = {};
    if (!attr_done[p.n_tile == 32][reg_a]) {
        SESSD_CUDA_TRY(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, kP2MaxSmem));
        attr_done[p.n_tile == 32][reg_a] = true;
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
    SESSD_LAUNCH(kernel, grid, reg_a ? kP2ThreadsRegA : kP2Threads, smem, (cudaStream_t)stream, map_a, map_b, d_scale, d_shift, d_residual, d_out_f32,
                 (__half *)d_out_planes, p);
    return last_error();
}


// the fields of P2Params that describe a tap-list conv (sessd_conv_desc) / the four-class deconv, and its tap classes
static int p2_conv_params(const sessd_conv_desc &d, P2Params &p, P2Taps &t) {
    if (d.ntaps < 1 || d.ntaps > 9 || (d.in_stride != 1 && d.in_stride != 2) || d.out_stride < 1) return SESSD_EINVAL;
    if ((d.grid_h - 1) * d.out_stride + d.out_off_y >= d.out_h || (d.grid_w - 1) * d.out_stride + d.out_off_x >= d.out_w) return SESSD_EINVAL;
    p = {};
    p.batch = d.batch; p.cin = d.cin; p.cout = d.cout; p.in_stride = d.in_stride;
    p.out_h = d.out_h; p.out_w = d.out_w; p.out_stride = d.out_stride; p.relu = d.relu;
    t = {};
    t.n = d.ntaps; t.off_y = d.out_off_y; t.off_x = d.out_off_x;
    for (int i = 0; i < d.ntaps; ++i) { t.dy[i] = d.tap_dy[i]; t.dx[i] = d.tap_dx[i]; t.w[i] = i; }
    return 0;
}

static void p2_deconv_params(int batch, int in_h, int in_w, int cin, int cout, int relu, P2Params &p, P2Taps cls[4]) {
    p = {};
    p.batch = batch; p.cin = cin; p.cout = cout; p.in_stride = 1;
    p.out_h = 2 * in_h; p.out_w = 2 * in_w; p.out_stride = 2; p.relu = relu;
    p2_deconv_classes(cls);
}

// one tap-list conv (sessd_conv_desc) / the four-class deconv through launch_p2<MODE, PROBE>; d_prof: [grid][kP2ProfWords] (probes).
// Stride-1 launches from planes take A from registers (one patch copy); smem_a (the loads probe) plans them for the shared-memory
// descriptors instead, for comparison.
template <int MODE, int PROBE = kP2NoProbe>
static int p2_conv(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                   const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                   float *d_out_f32, void *d_out_planes, float *d_out_info, const sessd_conv_desc *desc, void *stream,
                   const int *d_items = nullptr, long long *d_prof = nullptr, bool smem_a = false, const int *d_segs = nullptr) {
    if (!desc || (PROBE != kP2NoProbe && !d_prof)) return SESSD_EINVAL;
    const sessd_conv_desc &d = *desc;
    P2Params p;
    P2Taps t;
    if (p2_conv_params(d, p, t)) return SESSD_EINVAL;
    p.items = d_items;
    p.segs = d_segs;
    p.prof = d_prof;
    return launch_p2<MODE, PROBE>(d_in_planes, d.in_h, d.in_w, d_in_info, d_weight_h2, d.ntaps, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain,
                     shift_max, d_out_f32, d_out_planes, d_out_info, p, &t, 1, d.grid_h, d.grid_w, MODE == kP2Planes && d.in_stride == 1 && !smem_a,
                     stream);
}

template <int MODE, int PROBE = kP2NoProbe>
static int p2_deconv(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                     const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                     float *d_out_f32, void *d_out_planes, float *d_out_info, int batch, int in_h, int in_w, int cin, int cout,
                     int relu, void *stream, const int *d_items = nullptr, long long *d_prof = nullptr, const int *d_segs = nullptr) {
    if (PROBE != kP2NoProbe && !d_prof) return SESSD_EINVAL;
    P2Params p;
    P2Taps cls[4];
    p2_deconv_params(batch, in_h, in_w, cin, cout, relu, p, cls);
    p.items = d_items;
    p.segs = d_segs;
    p.prof = d_prof;
    return launch_p2<MODE, PROBE>(d_in_planes, in_h, in_w, d_in_info, d_weight_h2, 9, cout_pad, d_scale, d_shift, d_residual, d_resid_info, gain, shift_max,
                     d_out_f32, d_out_planes, d_out_info, p, cls, 4, in_h, in_w, MODE == kP2Planes, stream);
}

}  // namespace sessd

