// spconv_cg.cu -- sparse 3-D convolution (SubM / strided, + folded BN + ReLU) on the Hopper tensor cores (wgmma) whose operand traffic
// is proportional to the number of rulebook PAIRS: only the neighbour rows that exist are fetched.
//
// Replaces spconv 1.x's per-offset gather -> sgemm -> scatter-add used by det3d/models/backbones/scn.py:106-149 (SpMiddleFHD).
// Numerics: fp16 (hi, lo) planes with an exact power-of-two scale, three fp16 products per MAC (a_hi b_hi into the main accumulator,
// a_hi b_lo + a_lo b_hi into the cross accumulator, both fp32), summed in RN fp32 by the epilogue.
//   * the rulebook is regrouped ONCE per build (sessd_rulebook_tile_lists; a SubM rulebook serves 2-3 layers) into per-tile, per-offset
//     lists of (input row, tile row) pairs + row masks; a tile's record (~3-8 KB) is copied to shared memory;
//   * eight producer warps copy the listed rows with 16-byte cp.async (global/L2 -> shared, no registers) straight into the K-major
//     SWIZZLE_128B layout the wgmma descriptors address; rows without a neighbour are never touched;
//   * a stage's missing rows must read as zeros: each producer warp remembers (registers) which of its rows of its stage hold data and
//     clears (st.shared) only the rows that were valid for the stage's previous offset and are not for the new one -- the stages are
//     zeroed once per CTA;
//   * the 32-channel layers stage the weights as [b_hi rows ; b_lo rows] of 64 bytes (SWIZZLE_64B), the 64-channel layers as
//     [b_hi ; b_lo] tiles of 128-byte rows (SWIZZLE_128B);
//   * two consumer warpgroups (64 tile rows each) issue the wgmmas of every offset, keep one offset's group in flight while they wait
//     for the next stage, and run the epilogue from the accumulator registers;
//   * CTAs are persistent (one per SM), so barrier / zero-fill setup is paid once, not per 128 rows;
//   * the epilogue writes the NEXT layer's operand format directly -- fp16 (hi, lo) planes scaled by a power of two derived from a
//     rigorous bound |out| <= amax_in * G + max|shift| (G from the weights, host; amax_in measured by the producing layer's epilogue) --
//     and raises the output's abs-max: no separate split kernel.
// Each stage has its own producer group (8 / kStages warps): the group copies, waits for ITS copies (cp.async.wait_all), makes them and
// the clears visible to the async proxy (fence.proxy.async by the writing threads) and arrives on the stage's mbarrier, while the other
// groups' fills are in flight.
// Warps: 0-7 producers, 8-15 consumers (warpgroups 2 and 3), 16 weight-tile TMA.
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace sessd {

constexpr int kCgBM = 128;
constexpr int kCgMaxK = 27;
constexpr int kCgProdWarps = 8;
constexpr int kCgMmaWarps = 8;
constexpr int kCgWeightWarp = kCgProdWarps + kCgMmaWarps;
constexpr int kCgThreads = (kCgWeightWarp + 1) * 32;

// DEEP = 1: twice the stages -- for launches whose tiles do not fill the machine (a single frame: ~100 tiles on 132 SMs), where the
// layer's time is the serial chain of a tile's fills (latency-bound): more fills in flight shorten it
template <int CP, int COUT, int DEEP = 0>
struct CgCfg {
    static constexpr bool kWide = (CP == 64);
    static constexpr int kATile = (kWide ? 2 : 1) * kCgBM * 128;              // bytes: [hi tile ; lo tile] (wide) or one [hi | lo] tile
    static constexpr int kBTile = (kWide ? 2 : 1) * COUT * 128;               // wide: [b_hi ; b_lo] of 128-byte rows; narrow: 64-byte rows
    static constexpr int kStage = kATile + (kBTile + 1023) / 1024 * 1024;
    static constexpr int kStages = (kWide ? 2 : 4) * (DEEP ? 2 : 1);           // must divide the 8 producer warps (one group per stage)
    static constexpr int kMeta = kCgBM * kCgMaxK * 4 /*lists*/ + kCgMaxK * 16 /*valid*/ + 32 * 4 /*cnt*/ + 33 * 4 /*klist, nact*/ + 32 * 4 /*off*/ +
                                 3 * kStages * 8 /*barriers*/ + 24;
    static constexpr int kSmem = kStages * kStage + kMeta + 1024;
    static constexpr int kCPO = COUT > 32 ? 64 : 32;                          // channels per plane row of the OUTPUT
};

struct CgArgs {
    const __half *planes;              // input [rows][2][CP] fp16, x = (hi + lo) / in_info[1]
    const float *in_info;              // {abs-max of the input tensor, its plane scale}
    const unsigned int *tiles;         // per-tile pair lists (sessd_rulebook_tile_lists), tile_stride words per tile
    int tile_stride;
    const int *d_n_out;
    int kvol, max_out, relu;
    const float *scale, *shift;        // folded BN (scale already times the per-channel weight exponent 2^-e)
    float gain, shift_max;             // |out| <= amax_in * gain + shift_max
    float *out_f32;                    // nullable [max_out][COUT]
    __half *out_planes;                // nullable [max_out (+1)][2][kCPO]
    float *out_info;                   // nullable {abs-max of the output (atomicMax), plane scale}
};

// 16-byte global -> shared copy that bypasses L1 (the gathered rows are not re-read from L1)
__device__ __forceinline__ void cg_cp_async16(uint32_t smem_dst, const void *gsrc) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(smem_dst), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void cg_fence_proxy_async() { asm volatile("fence.proxy.async.shared::cta;\n" ::: "memory"); }
__device__ __forceinline__ void cg_sts_zero16(uint32_t saddr) {
    asm volatile("st.shared.v4.b32 [%0], {%1, %1, %1, %1};\n" ::"r"(saddr), "r"(0) : "memory");
}

template <int COUT>
__device__ __forceinline__ void cg_wgmma(float *d, uint64_t da, uint64_t db, uint32_t accumulate) {
    if constexpr (COUT == 32) wgmma_f16_n32(d, da, db, accumulate);
    else wgmma_f16_n64(d, da, db, accumulate);
}

template <int CP, int COUT, int DEEP>
__global__ void __launch_bounds__(kCgThreads, 1) spconv_cg_kernel(const __grid_constant__ CUtensorMap map_w, const CgArgs a) {
    using C = CgCfg<CP, COUT, DEEP>;
    const int n_out = min(*a.d_n_out, a.max_out);
    const int ntiles = (n_out + kCgBM - 1) / kCgBM;
    if ((int)blockIdx.x >= ntiles) return;                       // whole CTA leaves together (before any barrier use)
    const int kvol = a.kvol;
    if (threadIdx.x == kCgWeightWarp * 32) prefetch_tensormap(&map_w);      // the weight-TMA warp's first load finds the descriptor cached

    extern __shared__ unsigned char smem_raw[];
    unsigned char *tiles = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint32_t *s_list = (uint32_t *)(tiles + C::kStages * C::kStage);      // [kvol][128]: (input row << 7) | tile row
    uint32_t *s_valid = s_list + kCgBM * kCgMaxK;                        // [kvol][4]: 128-bit row mask per offset
    int *s_cnt = (int *)(s_valid + kCgMaxK * 4);                         // [32]
    int *s_klist = s_cnt + 32;                                           // [32] + nact
    int *s_nact = s_klist + 32;
    int *s_off = s_nact + 1;                                             // [32] first list entry of every offset
    uint64_t *bars = (uint64_t *)(((uintptr_t)(s_off + 32) + 7) & ~(uintptr_t)7);
    uint64_t *full_a = bars, *full_b = bars + C::kStages, *empty = bars + 2 * C::kStages;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t tiles_u32 = smem_u32(tiles);

    if (tid == 0) {
        for (int s = 0; s < C::kStages; ++s) { mbar_init(&full_a[s], kCgProdWarps / C::kStages); mbar_init(&full_b[s], 1); mbar_init(&empty[s], kCgMmaWarps); }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    // every A tile starts as zeros (the B halves of the stages are always fully overwritten by the TMA)
    for (int s = 0; s < C::kStages; ++s)
        for (int o = tid * 16; o < C::kATile; o += kCgThreads * 16) cg_sts_zero16(tiles_u32 + (uint32_t)(s * C::kStage + o));
    cg_fence_proxy_async();
    __syncthreads();

    const float amax_in = __ldg(a.in_info), s_in = __ldg(a.in_info + 1);
    const float inv_act = 1.f / s_in;                            // exact: power of two
    const float s_out = pow2_scale_for_bound(amax_in * a.gain + a.shift_max);
    if (blockIdx.x == 0 && tid == 0 && a.out_info) a.out_info[1] = s_out;
    float vmax = 0.f;
    uint32_t dirty[4] = {0u, 0u, 0u, 0u};                        // rows of this warp's share of its stage that hold data (producer warps)
    int st0 = 0;                                                 // stage of this tile's first fill (all roles advance it alike)
    uint32_t ph0 = 0;                                            // phase bit of stage st0

    for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
        const int row0 = tile * kCgBM;
        const int rows = min(kCgBM, n_out - row0);
        // ---------------------------------------------------------------- the tile's per-offset pair lists (built once per rulebook by
        // sessd_rulebook_tile_lists: counts, row masks, (input row << 7 | tile row) entries grouped by offset) -> shared memory
        {
            const unsigned int *rec = a.tiles + (size_t)tile * (size_t)a.tile_stride;
            const int c = (int)__ldg(rec + lane);                        // every warp ranks the 32 counts itself: no extra block-wide sync
            // the first list entries are requested together with the counts (one L2 round trip instead of two for most tiles; the record
            // is 160 + 128 kvol words long, so the speculative reads stay inside it)
            unsigned int spec[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) spec[u] = (tid + u * kCgThreads < 128 * kvol) ? __ldg(rec + 160 + tid + u * kCgThreads) : 0u;
            const int incl = warp_incl_scan(c, lane);
            const int total = __shfl_sync(0xffffffffu, incl, 31);
            if (warp == 0) {
                s_cnt[lane] = c;
                s_off[lane] = incl - c;
                const unsigned int m = __ballot_sync(0xffffffffu, c > 0);
                if (c > 0) s_klist[__popc(m & ((1u << lane) - 1u))] = lane;
                if (lane == 0) *s_nact = __popc(m);
            }
            if (tid < kvol * 4) s_valid[tid] = __ldg(rec + 32 + tid);
#pragma unroll
            for (int u = 0; u < 4; ++u)
                if (tid + u * kCgThreads < total) s_list[tid + u * kCgThreads] = spec[u];
            for (int e = tid + 4 * kCgThreads; e < total; e += kCgThreads) s_list[e] = __ldg(rec + 160 + e);
        }
        __syncthreads();
        const int nact = *s_nact;

        if (warp == kCgWeightWarp) {
            // ===================== weight tiles (TMA, one elected lane): [b_hi ; b_lo] =====================
            int s = st0;
            uint32_t ph = ph0;
            for (int j = 0; j < nact; ++j) {
                const int k = s_klist[j];
                mbar_wait(&empty[s], ph ^ 1u);
                if (elect_one()) {
                    mbar_expect_tx(&full_b[s], C::kBTile);
                    unsigned char *b_tile = tiles + s * C::kStage + C::kATile;
                    tma_load_4d(b_tile, &map_w, &full_b[s], 0, 0, 0, k);
                    tma_load_4d(b_tile + C::kBTile / 2, &map_w, &full_b[s], 0, 0, 1, k);
                }
                __syncwarp();
                if (++s == C::kStages) { s = 0; ph ^= 1u; }
            }
        } else if (warp >= kCgProdWarps) {
            // ===================== consumers: wgmma per offset, then the epilogue from the accumulator registers =====================
            const int cw = warp - kCgProdWarps, wg = cw >> 2, wq = cw & 3;
            constexpr int kAcc = COUT / 2;
            float acc_m[kAcc], acc_c[kAcc];
#pragma unroll
            for (int i = 0; i < kAcc; ++i) { acc_m[i] = 0.f; acc_c[i] = 0.f; }
            const uint32_t a_rows = (uint32_t)(wg * 64 * 128);   // this warpgroup's 64 rows of the 128-byte-row A tile
            int s = st0, prev = -1;
            uint32_t ph = ph0;
            for (int j = 0; j < nact; ++j) {
                mbar_wait(&full_b[s], ph);
                mbar_wait(&full_a[s], ph);
                const uint32_t st = tiles_u32 + (uint32_t)(s * C::kStage);
                const uint64_t dA = kDescSw128Hi | desc_lo(st + a_rows);
                const uint32_t first = j != 0 ? 1u : 0u;
                wgmma_fence();
                if constexpr (C::kWide) {
                    const uint64_t dAl = dA + ((kCgBM * 128) >> 4);
                    const uint64_t dBh = kDescSw128Hi | desc_lo(st + C::kATile);
                    const uint64_t dBl = dBh + ((COUT * 128) >> 4);
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) cg_wgmma<COUT>(acc_m, dA + 2 * kk, dBh + 2 * kk, first | (kk != 0));      // main  += a_hi x b_hi
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) cg_wgmma<COUT>(acc_c, dA + 2 * kk, dBl + 2 * kk, first | (kk != 0));      // cross += a_hi x b_lo
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) cg_wgmma<COUT>(acc_c, dAl + 2 * kk, dBh + 2 * kk, 1u);                    // cross += a_lo x b_hi
                } else {
                    // A line = [hi 32 | lo 32] (SWIZZLE_128B); B stage = [b_hi rows ; b_lo rows] of 64 bytes each (SWIZZLE_64B)
                    const uint64_t dBh = kDescSw64Hi | desc_lo(st + C::kATile);
                    const uint64_t dBl = dBh + ((COUT * 64) >> 4);
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) cg_wgmma<COUT>(acc_m, dA + 2 * kk, dBh + 2 * kk, first | (kk != 0));
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) cg_wgmma<COUT>(acc_c, dA + 2 * kk, dBl + 2 * kk, first | (kk != 0));
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) cg_wgmma<COUT>(acc_c, dA + 4 + 2 * kk, dBh + 2 * kk, 1u);
                }
                wgmma_commit();
                wgmma_wait<1>();                                 // the previous offset's products are done: its stage may be refilled
                if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
                prev = s;
                if (++s == C::kStages) { s = 0; ph ^= 1u; }
            }
            wgmma_wait<0>();
            wgmma_fence_regs<kAcc>(acc_m);
            wgmma_fence_regs<kAcc>(acc_c);
            if (prev >= 0 && lane == 0) mbar_arrive(&empty[prev]);
            // BN / ReLU -> planes and / or fp32 rows; this thread holds rows r0 and r0 + 8, two adjacent channels per 8-channel group
            const int r0 = wg * 64 + wq * 16 + (lane >> 2);
            const int c2 = 2 * (lane & 3);
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int r = r0 + 8 * h;
                if (r >= rows) continue;
                const size_t orow = (size_t)(row0 + r);
#pragma unroll
                for (int g = 0; g < COUT / 8; ++g) {
                    const int n = 8 * g + c2, i = 4 * g + 2 * h;
                    const float2 sc = __ldg(reinterpret_cast<const float2 *>(a.scale + n));
                    const float2 sh = a.shift ? __ldg(reinterpret_cast<const float2 *>(a.shift + n)) : make_float2(0.f, 0.f);
                    float o0 = fmaf((acc_m[i] + acc_c[i]) * inv_act, sc.x, sh.x);
                    float o1 = fmaf((acc_m[i + 1] + acc_c[i + 1]) * inv_act, sc.y, sh.y);
                    if (a.relu) { o0 = fmaxf(o0, 0.f); o1 = fmaxf(o1, 0.f); }
                    vmax = fmaxf(vmax, fmaxf(fabsf(o0), fabsf(o1)));
                    if (a.out_f32) *reinterpret_cast<float2 *>(a.out_f32 + orow * COUT + n) = make_float2(o0, o1);
                    if (a.out_planes) {
                        const float x0 = o0 * s_out, x1 = o1 * s_out;
                        const __half2 hi = __floats2half2_rn(x0, x1);
                        const float2 f = __half22float2(hi);
                        const __half2 lo = __floats2half2_rn(x0 - f.x, x1 - f.y);
                        __half2 *dst = reinterpret_cast<__half2 *>(a.out_planes + orow * (2 * C::kCPO) + n);
                        dst[0] = hi;
                        dst[C::kCPO / 2] = lo;
                    }
                }
            }
        } else {
            // ===================== producers: copy the rows that exist, clear the rows that stopped existing =====================
            // One producer GROUP per stage (kStages groups of 8 / kStages warps): a group fills only "its" stage, waits for its own copies
            // (cp.async.wait_all), fences them into the async proxy and arrives; the other groups' fills are in flight meanwhile.
            constexpr int kGroupWarps = kCgProdWarps / C::kStages;       // 1, 2 or 4
            constexpr int kGroupThreads = kGroupWarps * 32;
            constexpr int kOwnRows = kCgBM / kGroupWarps;                // rows of the stage whose zero state this warp maintains: 128, 64 or 32
            constexpr int kOwnWords = kOwnRows / 32;
            constexpr int kLanesPerRow = C::kWide ? 16 : 8;
            constexpr int kRowsPerPass = kGroupThreads / kLanesPerRow;
            const int grp = warp / kGroupWarps, gw = warp % kGroupWarps;
            const int gtid = tid - grp * kGroupThreads;
            const int slot = gtid / kLanesPerRow;
            const int c = gtid % kLanesPerRow;
            const int half = c >> 3, cc = c & 7;                         // wide: chunk c of the 256-byte row = (hi | lo tile, 16-byte chunk)
            const uint32_t a_base = tiles_u32 + (uint32_t)(grp * C::kStage);
            // this tile's fills that land in stage `grp`: j = j0, j0 + kStages, ...; the phase bit of fill j follows the ring position
            for (int j = (grp - st0 + C::kStages) % C::kStages; j < nact; j += C::kStages) {
                const uint32_t ph = ph0 ^ ((uint32_t)((st0 + j) / C::kStages) & 1u);
                const int k = s_klist[j];
                if (lane == 0) mbar_wait(&empty[grp], ph ^ 1u);
                __syncwarp();
#pragma unroll
                for (int w = 0; w < kOwnWords; ++w) {
                    const uint32_t vs = s_valid[k * 4 + gw * kOwnWords + w];
                    const uint32_t z = dirty[w] & ~vs;                     // rows that hold data of the stage's previous offset and get none now
                    dirty[w] = vs;
                    if (z) {
#pragma unroll
                        for (int q4 = 0; q4 < 8; ++q4) {
                            const int r32 = q4 * 4 + (lane >> 3);
                            if ((z >> r32) & 1u) {
                                const uint32_t dst = a_base + (uint32_t)((gw * kOwnRows + w * 32 + r32) * 128 + (lane & 7) * 16);
                                cg_sts_zero16(dst);
                                if constexpr (C::kWide) cg_sts_zero16(dst + kCgBM * 128);
                            }
                        }
                    }
                }
                const int n = s_cnt[k];
                const uint32_t *lst = s_list + s_off[k];
                auto copy_row = [&](uint32_t e) {
                    const uint32_t r = e & 127u;
                    const size_t src = (size_t)(e >> 7);
                    if constexpr (C::kWide)
                        cg_cp_async16(a_base + (uint32_t)half * (kCgBM * 128) + r * 128u + (((uint32_t)cc ^ (r & 7u)) << 4),
                                      a.planes + src * 128 + half * 64 + cc * 8);
                    else
                        cg_cp_async16(a_base + r * 128u + (((uint32_t)cc ^ (r & 7u)) << 4), a.planes + src * 64 + cc * 8);
                };
                // four list entries per round: the shared-memory reads of a round are in flight together
                int i = slot;
                for (; i + 3 * kRowsPerPass < n; i += 4 * kRowsPerPass) {
                    const uint32_t e0 = lst[i], e1 = lst[i + kRowsPerPass], e2 = lst[i + 2 * kRowsPerPass], e3 = lst[i + 3 * kRowsPerPass];
                    copy_row(e0); copy_row(e1); copy_row(e2); copy_row(e3);
                }
                for (; i < n; i += kRowsPerPass) copy_row(lst[i]);
                asm volatile("cp.async.wait_all;\n" ::: "memory");
                cg_fence_proxy_async();                                  // copies and clears (generic proxy) -> visible to the tensor core
                __syncwarp();
                if (lane == 0) mbar_arrive(&full_a[grp]);
            }
        }
        {   // advance the ring position by this tile's fills
            const int adv = st0 + nact;
            ph0 ^= (uint32_t)(adv / C::kStages) & 1u;
            st0 = adv % C::kStages;
        }
        __syncthreads();                                         // lists are rebuilt next; every role is done reading them
    }
    if (warp >= kCgProdWarps && warp < kCgWeightWarp && a.out_info) {
        const unsigned m = __reduce_max_sync(0xFFFFFFFFu, __float_as_uint(vmax));     // non-negative floats order like their bits
        if (lane == 0 && m != 0u) atomicMax(reinterpret_cast<unsigned *>(a.out_info), m);
    }
}

static int g_cg_deep = 0;          // 1: deep pipeline (sessd_set_sp_cg_deep)

template <int CP, int COUT, int DEEP>
static int launch_spconv_cg(const CgArgs &a, const void *w_h2, cudaStream_t st) {
    using C = CgCfg<CP, COUT, DEEP>;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(spconv_cg_kernel<CP, COUT, DEEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem);
        if (e != cudaSuccess) return (int)e;
        attr_done = true;
    }
    CUtensorMap map_w;
    int rc;
    if (C::kWide) {       // [kvol][2 (hi|lo)][Cout][64]
        const cuuint64_t dims[4] = {64, (cuuint64_t)COUT, 2, (cuuint64_t)a.kvol};
        const cuuint32_t box[4] = {64, (cuuint32_t)COUT, 1, 1};
        rc = encode_map_4d(&map_w, w_h2, dims, box, nullptr, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 2);
    } else {              // [kvol][2 (hi|lo)][Cout][32]: 64-byte rows, SWIZZLE_64B
        EncodeTiledFn enc = get_tensor_map_encoder();
        if (!enc) return SESSD_EINVAL;
        const cuuint64_t dims[4] = {32, (cuuint64_t)COUT, 2, (cuuint64_t)a.kvol};
        const cuuint64_t strides[3] = {64, (cuuint64_t)COUT * 64, (cuuint64_t)COUT * 128};
        const cuuint32_t box[4] = {32, (cuuint32_t)COUT, 1, 1};
        const cuuint32_t estr[4] = {1, 1, 1, 1};
        CUresult r = enc(&map_w, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, 4, const_cast<void *>(w_h2), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                         CU_TENSOR_MAP_SWIZZLE_64B, CU_TENSOR_MAP_L2_PROMOTION_L2_128B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
        rc = r == CUDA_SUCCESS ? 0 : 700 + (int)r;
    }
    if (rc) return rc;
    static int num_sms = 0;
    if (!num_sms) {
        int dev = 0;
        SESSD_CUDA_TRY(cudaGetDevice(&dev));
        SESSD_CUDA_TRY(cudaDeviceGetAttribute(&num_sms, cudaDevAttrMultiProcessorCount, dev));
    }
    const int tiles = div_up(a.max_out, kCgBM);
    const int grid = tiles < num_sms ? tiles : num_sms;                          // persistent, one CTA per SM
    SESSD_LAUNCH((spconv_cg_kernel<CP, COUT, DEEP>), grid, kCgThreads, C::kSmem, st, map_w, a);
    return last_error();
}

}  // namespace sessd

using namespace sessd;

// 1: twice the stages (launches with fewer tiles than SMs, e.g. single frames: the serial fill chain of a tile is latency-bound);
// 0 (default): the shorter ring (many tiles: throughput)
extern "C" void sessd_set_sp_cg_deep(int on) { sessd::g_cg_deep = on ? 1 : 0; }

// S4 (scn.py:106-149), pair-proportional tensor-core path.  d_in_planes [plane_rows][2][cp] fp16 with d_in_info = {abs-max, scale};
// weights / d_scale from ops.pack_weight_sp_h2 (cp = 64: [kvol][2][Cout][64], cp = 32: [kvol][2][Cout][32]; d_scale = BN scale *
// 2^-e[c]); gain / shift_max bound the output (see the header).  Outputs (each nullable, at least one): fp32 rows [max_out][cout],
// planes [>= max_out][2][cout <= 32 ? 32 : 64] + d_out_info = {abs-max (zero it once per frame), scale}.
// Supported (cp, cout): (32,32), (32,64), (64,64).
extern "C" int sessd_spconv_forward_cg(const void *d_in_planes, int cp, int plane_rows, const float *d_in_info, const void *d_tiles, int kvol,
                                       const int *d_n_out, int max_out, const void *d_weight_h2, int cout, const float *d_scale,
                                       const float *d_shift, int relu, float gain, float shift_max, float *d_out_f32, void *d_out_planes,
                                       float *d_out_info, void *stream) {
    if (!d_in_planes || !d_in_info || !d_tiles || !d_n_out || !d_weight_h2 || !d_scale || (!d_out_f32 && !d_out_planes) || max_out < 1 ||
        kvol < 1 || kvol > kCgMaxK || plane_rows < 1 || plane_rows > (1 << 25))
        return SESSD_EINVAL;
    if (d_out_planes && !d_out_info) return SESSD_EINVAL;
    CgArgs a;
    a.planes = (const __half *)d_in_planes; a.in_info = d_in_info; a.tiles = (const unsigned int *)d_tiles; a.tile_stride = 160 + 128 * kvol; a.d_n_out = d_n_out; a.kvol = kvol; a.max_out = max_out;
    a.relu = relu; a.scale = d_scale; a.shift = d_shift; a.gain = gain; a.shift_max = shift_max; a.out_f32 = d_out_f32;
    a.out_planes = (__half *)d_out_planes; a.out_info = d_out_info;
    cudaStream_t st = (cudaStream_t)stream;
#define SESSD_CG_CASE(CPV, CO) \
    if (cp == CPV && cout == CO) return g_cg_deep ? launch_spconv_cg<CPV, CO, 1>(a, d_weight_h2, st) : launch_spconv_cg<CPV, CO, 0>(a, d_weight_h2, st);
    SESSD_CG_CASE(32, 32)
    SESSD_CG_CASE(32, 64)
    SESSD_CG_CASE(64, 64)
#undef SESSD_CG_CASE
    return SESSD_EINVAL;
}
