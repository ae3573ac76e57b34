// spconv_cg.cu -- sparse 3-D convolution (SubM / strided, + folded BN + ReLU) on the Hopper tensor cores (wgmma) whose operand traffic
// is proportional to the number of rulebook PAIRS: only the neighbour rows that exist are fetched.
//
// Replaces spconv 1.x's per-offset gather -> sgemm -> scatter-add used by det3d/models/backbones/scn.py:106-149 (SpMiddleFHD).
// Numerics: fp16 (hi, lo) planes with an exact power-of-two scale, three fp16 products per MAC (a_hi b_hi into the main accumulator,
// a_hi b_lo + a_lo b_hi into the cross accumulator, both fp32), summed in RN fp32 by the epilogue.
//   * the rulebook is regrouped ONCE per build (sessd_rulebook_tile_lists; a SubM rulebook serves 2-3 layers) into per-tile, per-offset
//     lists of (input row, tile row) pairs + row masks; a tile's record (~3-8 KB) is copied to shared memory;
//   * four producer warps copy the listed rows with 16-byte cp.async (global/L2 -> shared, no registers) straight into the K-major
//     SWIZZLE_128B layout the wgmma descriptors address; rows without a neighbour are never touched;
//   * a stage's missing rows must read as zeros: each producer warp remembers (registers) which of its rows of its stages hold data and
//     clears (st.shared) only the rows that were valid for the stage's previous offset and are not for the new one -- the stages are
//     zeroed once per CTA;
//   * the 32-channel layers stage the weights as [b_lo rows ; b_hi rows] of 64 bytes (SWIZZLE_64B), the 64-channel layers as
//     [b_lo ; b_hi] tiles of 128-byte rows (SWIZZLE_128B); per k16, three m64nCOUT compute a_hi b_lo and a_lo b_hi into the cross
//     accumulator and a_hi b_hi into the main one;
//   * two consumer warpgroups (64 tile rows each) issue the wgmmas of every offset, wait for them and release the stage at once, so its
//     next fill starts while the following offset's fill is still in flight (a single frame's layers are bound by this chain of fills,
//     see DEEP; measurements in DESIGN section 4), and run the epilogue from the accumulator registers: a 4 x 4 transpose inside each
//     quad of lanes gives every lane 8 whole channels of one row, stored 16 bytes at a time (each warp store covers whole 32-byte
//     sectors), with the folded BN scale / shift read from shared memory (copied there once per CTA);
//   * CTAs are persistent, so barrier / zero-fill setup is paid once, not per 128 rows; two fit on an SM (384 threads, <= 113 KB of
//     shared memory), so one tile's chain of fills runs while the other CTA's wgmmas or epilogue do;
//   * the epilogue writes the NEXT layer's operand format directly -- fp16 (hi, lo) planes scaled by a power of two derived from a
//     rigorous bound |out| <= amax_in * G + max|shift| (G from the weights, host; amax_in measured by the producing layer's epilogue) --
//     and raises the output's abs-max: no separate split kernel.
// Stages are owned by producer groups (2 stages: two groups of 2 warps; 4 stages: one warp each; 8 stages: two per warp): after the
// stage's empty wait the group loads its weight tile with TMA from one lane, copies the A rows, waits for ITS copies (cp.async.wait_all),
// makes them and the clears visible to the async proxy (fence.proxy.async by the writing threads) and arrives on the stage's mbarrier,
// while the other groups' fills are in flight.
// Warps: 0-3 producers (warpgroup 0, 48 registers), 4-11 consumers (warpgroups 1 and 2, 96 registers).
#include <cuda_fp16.h>

#include "tc_common.cuh"
#include "tile_lists.cuh"

namespace sessd {

constexpr int kCgBM = 128;
constexpr int kCgMaxK = 27;
constexpr int kCgProdWarps = 4;
constexpr int kCgMmaWarps = 8;
constexpr int kCgThreads = (kCgProdWarps + kCgMmaWarps) * 32;
// 80 registers per thread at launch fit two CTAs on an SM; setmaxnreg then moves them from the producers to the consumers'
// accumulators: 128 x 48 + 256 x 96 = 384 x 80
constexpr int kCgRegsProducer = 48, kCgRegsConsumer = 96;

// DEEP = 1: twice the stages -- for launches whose tiles do not fill the machine (a single frame: ~100 tiles on 132 SMs), where the
// layer's time is the serial chain of a tile's fills (latency-bound): more fills in flight shorten it
template <int CP, int COUT, int DEEP = 0>
struct CgCfg {
    static constexpr bool kWide = (CP == 64);
    static constexpr int kATile = (kWide ? 2 : 1) * kCgBM * 128;              // bytes: [hi tile ; lo tile] (wide) or one [hi | lo] tile
    static constexpr int kBTile = (kWide ? 2 : 1) * COUT * 128;               // wide: [b_lo ; b_hi] of 128-byte rows; narrow: 64-byte rows
    static constexpr int kStage = kATile + (kBTile + 1023) / 1024 * 1024;
    static constexpr int kStages = (kWide ? 2 : 4) * (DEEP ? 2 : 1);
    // producer groups: group g owns stages g, g + kGroups, ... and fills them in ring order
    static constexpr int kGroups = kStages < kCgProdWarps ? kStages : kCgProdWarps;
    static constexpr int kGroupWarps = kCgProdWarps / kGroups;                // 2 or 1
    static constexpr int kGroupStages = kStages / kGroups;                    // 1 or 2
    static constexpr int kMeta = kCgBM * kCgMaxK * 4 /*lists*/ + kCgMaxK * 16 /*valid*/ + 2 * COUT * 4 /*scale, shift*/ + 32 * 4 /*cnt*/ +
                                 33 * 4 /*klist, nact*/ + 32 * 4 /*off*/ + 3 * kStages * 8 /*barriers*/ + 24;
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

// N = COUT output columns: one plane of the weight stage
template <int N>
__device__ __forceinline__ void cg_wgmma(float *d, uint64_t da, uint64_t db, uint32_t accumulate) {
    static_assert(N == 32 || N == 64, "COUT is 32 or 64");
    if constexpr (N == 32) wgmma_f16_n32(d, da, db, accumulate);
    else wgmma_f16_n64(d, da, db, accumulate);
}

template <int CP, int COUT, int DEEP>
__global__ void __launch_bounds__(kCgThreads, 2) spconv_cg_kernel(const __grid_constant__ CUtensorMap map_w, const CgArgs a) {
    using C = CgCfg<CP, COUT, DEEP>;
    static_assert(DEEP || C::kSmem <= 113 * 1024, "two CTAs per SM: 228 KB of shared memory less 1 KB reserved per CTA");
    static_assert(kCgProdWarps * 32 * kCgRegsProducer + kCgMmaWarps * 32 * kCgRegsConsumer <= kCgThreads * 80, "setmaxnreg budget");
    const int n_out = min(*a.d_n_out, a.max_out);
    const int ntiles = (n_out + kCgBM - 1) / kCgBM;
    if ((int)blockIdx.x >= ntiles) return;                       // whole CTA leaves together (before any barrier use)
    const int kvol = a.kvol;
    if (threadIdx.x == 0) prefetch_tensormap(&map_w);            // the producers' first weight load finds the descriptor cached

    extern __shared__ unsigned char smem_raw[];
    unsigned char *tiles = (unsigned char *)(((uintptr_t)smem_raw + 1023) & ~(uintptr_t)1023);
    uint32_t *s_list = (uint32_t *)(tiles + C::kStages * C::kStage);      // [kvol][128]: (input row << 7) | tile row
    uint32_t *s_valid = s_list + kCgBM * kCgMaxK;                        // [kvol][4]: 128-bit row mask per offset
    float *s_scale = (float *)(s_valid + kCgMaxK * 4);                   // [COUT] folded BN scale, 16-byte aligned
    float *s_shift = s_scale + COUT;                                     // [COUT] folded BN shift (zeros without one)
    int *s_cnt = (int *)(s_shift + COUT);                                // [32]
    int *s_klist = s_cnt + 32;                                           // [32] + nact
    int *s_nact = s_klist + 32;
    int *s_off = s_nact + 1;                                             // [32] first list entry of every offset
    uint64_t *bars = (uint64_t *)(((uintptr_t)(s_off + 32) + 7) & ~(uintptr_t)7);
    uint64_t *full_a = bars, *full_b = bars + C::kStages, *empty = bars + 2 * C::kStages;

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const uint32_t tiles_u32 = smem_u32(tiles);

    if (tid == 0) {
        for (int s = 0; s < C::kStages; ++s) {
            mbar_init(&full_a[s], C::kGroupWarps);
            mbar_init(&full_b[s], 1);
            mbar_init(&empty[s], kCgMmaWarps);
        }
        asm volatile("fence.mbarrier_init.release.cluster;\n" ::: "memory");
    }
    if (tid < COUT) {
        s_scale[tid] = __ldg(a.scale + tid);
        s_shift[tid] = a.shift ? __ldg(a.shift + tid) : 0.f;
    }
    // every A tile starts as zeros (the B halves of the stages are always fully overwritten by the TMA)
    for (int s = 0; s < C::kStages; ++s)
        for (int o = tid * 16; o < C::kATile; o += kCgThreads * 16) cg_sts_zero16(tiles_u32 + (uint32_t)(s * C::kStage + o));
    cg_fence_proxy_async();
    __syncthreads();

    // The tile's per-offset pair lists (built once per rulebook by sessd_rulebook_tile_lists: counts, row masks, (input row << 7 | tile
    // row) entries grouped by offset) -> shared memory.  Every thread of both roles runs it at the head of a tile, then a __syncthreads.
    auto load_lists = [&](int tile) {
        const unsigned int *rec = a.tiles + (size_t)tile * (size_t)a.tile_stride;
        const int c = (int)__ldg(rec + lane);                    // every warp ranks the 32 counts itself: no extra block-wide sync
        // the first list entries are requested together with the counts (one L2 round trip instead of two for most tiles; the record
        // is tile_list_stride(kvol) words long, so the speculative reads stay inside it)
        unsigned int spec[4];
#pragma unroll
        for (int u = 0; u < 4; ++u) spec[u] = (tid + u * kCgThreads < kTlRows * kvol) ? __ldg(rec + kTlHeader + tid + u * kCgThreads) : 0u;
        const int incl = warp_incl_scan(c, lane);
        const int total = __shfl_sync(0xffffffffu, incl, 31);
        if (warp == 0) {
            s_cnt[lane] = c;
            s_off[lane] = incl - c;
            const unsigned int m = __ballot_sync(0xffffffffu, c > 0);
            if (c > 0) s_klist[__popc(m & ((1u << lane) - 1u))] = lane;
            if (lane == 0) *s_nact = __popc(m);
        }
        if (tid < kvol * 4) s_valid[tid] = __ldg(rec + kTlMask + tid);
#pragma unroll
        for (int u = 0; u < 4; ++u)
            if (tid + u * kCgThreads < total) s_list[tid + u * kCgThreads] = spec[u];
        for (int e = tid + 4 * kCgThreads; e < total; e += kCgThreads) s_list[e] = __ldg(rec + kTlHeader + e);
    };
    // Ring position of a tile's first fill: stage st0, phase bit ph0.  Both roles advance it alike by each tile's nact fills.
    int st0 = 0;
    uint32_t ph0 = 0;
    auto advance_ring = [&](int nact) {
        const int adv = st0 + nact;
        ph0 ^= (uint32_t)(adv / C::kStages) & 1u;
        st0 = adv % C::kStages;
    };

    if (warp < kCgProdWarps) {
        setmaxnreg_dec<kCgRegsProducer>();
        // ===================== producers: weight tile (TMA), copy the rows that exist, clear the rows that stopped existing ============
        // Group grp fills the ring positions p = grp (mod kGroups), i.e. its stages grp, grp + kGroups, ... in turn; it waits for its
        // own copies (cp.async.wait_all), fences them into the async proxy and arrives, while the other groups' fills are in flight.
        constexpr int kGroups = C::kGroups, kGroupWarps = C::kGroupWarps, kGroupStages = C::kGroupStages;
        constexpr int kGroupThreads = kGroupWarps * 32;
        constexpr int kOwnRows = kCgBM / kGroupWarps;                // rows of a stage whose zero state this warp maintains: 128 or 64
        constexpr int kOwnWords = kOwnRows / 32;
        constexpr int kLanesPerRow = C::kWide ? 16 : 8;
        constexpr int kRowsPerPass = kGroupThreads / kLanesPerRow;
        const int grp = warp / kGroupWarps, gw = warp % kGroupWarps;
        const int gtid = tid - grp * kGroupThreads;
        const int slot = gtid / kLanesPerRow;
        const int c = gtid % kLanesPerRow;
        const int half = c >> 3, cc = c & 7;                         // wide: chunk c of the 256-byte row = (hi | lo tile, 16-byte chunk)
        // rows of this warp's share of each of its stages that hold data; dirty[0] is the stage of the group's next fill
        uint32_t dirty[kGroupStages][kOwnWords];
#pragma unroll
        for (int g = 0; g < kGroupStages; ++g)
#pragma unroll
            for (int w = 0; w < kOwnWords; ++w) dirty[g][w] = 0u;
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            load_lists(tile);
            __syncthreads();
            const int nact = *s_nact;
            for (int j = (grp - st0 % kGroups + kGroups) % kGroups; j < nact; j += kGroups) {
                const int pos = st0 + j;                             // the phase bit of fill j follows the ring position
                const int s = pos % C::kStages;
                const uint32_t ph = ph0 ^ ((uint32_t)(pos / C::kStages) & 1u);
                const int k = s_klist[j];
                const uint32_t a_base = tiles_u32 + (uint32_t)(s * C::kStage);
                if (lane == 0) {
                    mbar_wait<true>(&empty[s], ph ^ 1u);
                    if (gw == 0) {                                   // weight tile [b_lo ; b_hi]
                        mbar_expect_tx(&full_b[s], C::kBTile);
                        unsigned char *b_tile = tiles + s * C::kStage + C::kATile;
                        tma_load_4d(b_tile + C::kBTile / 2, &map_w, &full_b[s], 0, 0, 0, k);      // plane 0 = b_hi
                        tma_load_4d(b_tile, &map_w, &full_b[s], 0, 0, 1, k);                      // plane 1 = b_lo
                    }
                }
                __syncwarp();
#pragma unroll
                for (int w = 0; w < kOwnWords; ++w) {
                    const uint32_t vs = s_valid[k * 4 + gw * kOwnWords + w];
                    const uint32_t z = dirty[0][w] & ~vs;    // rows that hold data of the stage's previous offset and get none now
                    dirty[0][w] = vs;
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
                    const uint32_t r = tl_tile_row(e);
                    const size_t src = (size_t)tl_in_row(e);
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
                cg_fence_proxy_async();                              // copies and clears (generic proxy) -> visible to the tensor core
                __syncwarp();
                if (lane == 0) mbar_arrive(&full_a[s]);
                if constexpr (kGroupStages > 1) {                    // the group's next fill lands in its next stage
#pragma unroll
                    for (int w = 0; w < kOwnWords; ++w) {
                        const uint32_t d = dirty[0][w];
#pragma unroll
                        for (int g = 0; g + 1 < kGroupStages; ++g) dirty[g][w] = dirty[g + 1][w];
                        dirty[kGroupStages - 1][w] = d;
                    }
                }
            }
            advance_ring(nact);
            __syncthreads();                                         // lists are rebuilt next; every role is done reading them
        }
    } else {
        setmaxnreg_inc<kCgRegsConsumer>();
        // ===================== consumers: wgmma per offset, then the epilogue from the accumulator registers =====================
        const int cw = warp - kCgProdWarps, wg = cw >> 2, wq = cw & 3;
        constexpr int kAcc = COUT / 2;
        const float amax_in = __ldg(a.in_info), s_in = __ldg(a.in_info + 1);
        const float inv_act = 1.f / s_in;                        // exact: power of two
        const float s_out = pow2_scale_for_bound(amax_in * a.gain + a.shift_max);
        if (blockIdx.x == 0 && cw == 0 && lane == 0 && a.out_info) a.out_info[1] = s_out;
        float vmax = 0.f;
        const uint32_t a_rows = (uint32_t)(wg * 64 * 128);       // this warpgroup's 64 rows of the 128-byte-row A tile
        for (int tile = blockIdx.x; tile < ntiles; tile += gridDim.x) {
            load_lists(tile);
            __syncthreads();
            const int nact = *s_nact;
            const int row0 = tile * kCgBM;
            const int rows = min(kCgBM, n_out - row0);
            // m64nCOUT fragments: cross a_hi x b_lo + a_lo x b_hi, main a_hi x b_hi
            float acc[kAcc], acc_main[kAcc];
#pragma unroll
            for (int i = 0; i < kAcc; ++i) acc[i] = acc_main[i] = 0.f;
            int s = st0;
            uint32_t ph = ph0;
            for (int j = 0; j < nact; ++j) {
                mbar_wait<true>(&full_b[s], ph);
                mbar_wait<true>(&full_a[s], ph);
                const uint32_t st = tiles_u32 + (uint32_t)(s * C::kStage);
                const uint64_t dA = kDescSw128Hi | desc_lo(st + a_rows);
                const uint32_t first = j != 0 ? 1u : 0u;
                // per k16: cross (+)= a_hi x b_lo and main (+)= a_hi x b_hi, then cross += a_lo x b_hi.  Each accumulator sums the same
                // products in the same order as one m64n(2 COUT) over the stacked stage followed by an m64nCOUT would; that wider form
                // needs more registers than a consumer has with two CTAs on an SM (ptxas then ignores setmaxnreg or fails at 80).
                wgmma_fence();
                if constexpr (C::kWide) {
                    const uint64_t dAl = dA + ((kCgBM * 128) >> 4);
                    const uint64_t dBl = kDescSw128Hi | desc_lo(st + C::kATile);
                    const uint64_t dBh = dBl + ((COUT * 128) >> 4);
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) {
                        cg_wgmma<COUT>(acc, dA + 2 * kk, dBl + 2 * kk, first | (kk != 0));
                        cg_wgmma<COUT>(acc_main, dA + 2 * kk, dBh + 2 * kk, first | (kk != 0));
                    }
#pragma unroll
                    for (int kk = 0; kk < 4; ++kk) cg_wgmma<COUT>(acc, dAl + 2 * kk, dBh + 2 * kk, 1u);
                } else {
                    // A line = [hi 32 | lo 32] (SWIZZLE_128B); B stage = [b_lo rows ; b_hi rows] of 64 bytes each (SWIZZLE_64B)
                    const uint64_t dBl = kDescSw64Hi | desc_lo(st + C::kATile);
                    const uint64_t dBh = dBl + ((COUT * 64) >> 4);
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) {
                        cg_wgmma<COUT>(acc, dA + 2 * kk, dBl + 2 * kk, first | (kk != 0));
                        cg_wgmma<COUT>(acc_main, dA + 2 * kk, dBh + 2 * kk, first | (kk != 0));
                    }
#pragma unroll
                    for (int kk = 0; kk < 2; ++kk) cg_wgmma<COUT>(acc, dA + 4 + 2 * kk, dBh + 2 * kk, 1u);
                }
                wgmma_commit();
                // release the stage as soon as its own products are done, not one offset later: the producers start its next fill
                // while this offset's successor is still being filled, so with two stages two fills overlap instead of one.  A
                // single frame's tiles are bound by this chain of fills; the wait costs little since the next offset's stage is
                // rarely full by then anyway
                wgmma_wait<0>();
                if (lane == 0) mbar_arrive(&empty[s]);
                if (++s == C::kStages) { s = 0; ph ^= 1u; }
            }
            wgmma_fence_regs<kAcc>(acc);
            wgmma_fence_regs<kAcc>(acc_main);
            // BN / ReLU -> planes and / or fp32 rows.  This thread holds rows r0 and r0 + 8, two adjacent channels of every 8-channel
            // group; a transpose inside each quad of lanes (one row) gives every lane 8 whole channels, stored 16 bytes at a time
#pragma unroll
            for (int i = 0; i < kAcc; ++i) acc[i] = acc_main[i] + acc[i];        // main + cross
            const int q = lane & 3;
            const int r0 = wg * 64 + wq * 16 + (lane >> 2);
#pragma unroll
            for (int jb = 0; jb < COUT / 32; ++jb)
#pragma unroll
                for (int h = 0; h < 2; ++h) {
                    const int r = r0 + 8 * h;
                    const bool row_ok = r < rows;                // the same in the four lanes of a quad
                    const size_t orow = (size_t)(row0 + r);
                    float v[8], o[8];
                    quad_transpose8(acc + 16 * jb + 2 * h, q, v);
                    const int n = 32 * jb + 8 * q;               // this lane's 8 channels
#pragma unroll
                    for (int t = 0; t < 8; t += 4) {
                        const float4 sc = *reinterpret_cast<const float4 *>(s_scale + n + t);
                        const float4 sh = *reinterpret_cast<const float4 *>(s_shift + n + t);
                        o[t] = fmaf(v[t] * inv_act, sc.x, sh.x);
                        o[t + 1] = fmaf(v[t + 1] * inv_act, sc.y, sh.y);
                        o[t + 2] = fmaf(v[t + 2] * inv_act, sc.z, sh.z);
                        o[t + 3] = fmaf(v[t + 3] * inv_act, sc.w, sh.w);
                    }
                    if (a.relu) {
#pragma unroll
                        for (int t = 0; t < 8; ++t) o[t] = fmaxf(o[t], 0.f);
                    }
                    if (row_ok) {
#pragma unroll
                        for (int t = 0; t < 8; ++t) vmax = fmaxf(vmax, fabsf(o[t]));
                    }
                    if (a.out_planes && row_ok) {
                        __align__(16) __half2 hi[4], lo[4];
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            const float x0 = o[2 * t] * s_out, x1 = o[2 * t + 1] * s_out;
                            hi[t] = __floats2half2_rn(x0, x1);
                            const float2 f = __half22float2(hi[t]);
                            lo[t] = __floats2half2_rn(x0 - f.x, x1 - f.y);
                        }
                        __half *dst = a.out_planes + orow * (2 * C::kCPO) + n;
                        *reinterpret_cast<uint4 *>(dst) = *reinterpret_cast<const uint4 *>(hi);
                        *reinterpret_cast<uint4 *>(dst + C::kCPO) = *reinterpret_cast<const uint4 *>(lo);
                    }
                    if (a.out_f32) {
                        // lanes q and q ^ 2 trade half groups, so that each of the two stores of a quad covers 16 whole channels (two whole
                        // 32-byte sectors): lane q keeps half (q >> 1) of group q and gets the same half of group q ^ 2
                        const bool up = q & 2;
                        float keep[4], recv[4];
#pragma unroll
                        for (int t = 0; t < 4; ++t) {
                            keep[t] = up ? o[4 + t] : o[t];
                            recv[t] = __shfl_xor_sync(0xFFFFFFFFu, up ? o[t] : o[4 + t], 2);
                        }
                        const float4 w_lo = up ? make_float4(recv[0], recv[1], recv[2], recv[3]) : make_float4(keep[0], keep[1], keep[2], keep[3]);
                        const float4 w_hi = up ? make_float4(keep[0], keep[1], keep[2], keep[3]) : make_float4(recv[0], recv[1], recv[2], recv[3]);
                        float *dst = a.out_f32 + orow * COUT + 32 * jb + 8 * (q & 1) + 4 * (q >> 1);
                        if (row_ok) {
                            *reinterpret_cast<float4 *>(dst) = w_lo;
                            *reinterpret_cast<float4 *>(dst + 16) = w_hi;
                        }
                    }
                }
            advance_ring(nact);
            __syncthreads();                                         // lists are rebuilt next; every role is done reading them
        }
        if (a.out_info) {
            const unsigned m = __reduce_max_sync(0xFFFFFFFFu, __float_as_uint(vmax));     // non-negative floats order like their bits
            if (lane == 0 && m != 0u) atomicMax(reinterpret_cast<unsigned *>(a.out_info), m);
        }
    }
}

static int g_cg_deep = 0;          // 1: deep pipeline (sessd_set_sp_cg_deep)

// CTAs of spconv_cg_kernel<CP, COUT, DEEP> that are resident on one SM at once (registers, shared memory, threads).  The first call also
// raises the kernel's dynamic shared-memory limit.
template <int CP, int COUT, int DEEP>
static cudaError_t cg_blocks_per_sm(int *blocks) {
    using C = CgCfg<CP, COUT, DEEP>;
    static int cached = 0;
    if (!cached) {
        cudaError_t e = cudaFuncSetAttribute(spconv_cg_kernel<CP, COUT, DEEP>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem);
        if (e == cudaSuccess)
            e = cudaOccupancyMaxActiveBlocksPerMultiprocessor(&cached, spconv_cg_kernel<CP, COUT, DEEP>, kCgThreads, C::kSmem);
        if (e != cudaSuccess) { cached = 0; return e; }
        if (!cached) return cudaErrorInvalidConfiguration;
    }
    *blocks = cached;
    return cudaSuccess;
}

template <int CP, int COUT, int DEEP>
static int launch_spconv_cg(const CgArgs &a, const void *w_h2, cudaStream_t st) {
    using C = CgCfg<CP, COUT, DEEP>;
    int blocks_per_sm = 0;
    SESSD_CUDA_TRY((cg_blocks_per_sm<CP, COUT, DEEP>(&blocks_per_sm)));
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
    const int grid = tiles < blocks_per_sm * num_sms ? tiles : blocks_per_sm * num_sms;     // persistent, every CTA resident at once
    SESSD_LAUNCH((spconv_cg_kernel<CP, COUT, DEEP>), grid, kCgThreads, C::kSmem, st, map_w, a);
    return last_error();
}

}  // namespace sessd

using namespace sessd;

// 1: twice the stages (launches with fewer tiles than SMs, e.g. single frames: the serial fill chain of a tile is latency-bound);
// 0 (default): the shorter ring (many tiles: throughput)
extern "C" void sessd_set_sp_cg_deep(int on) { sessd::g_cg_deep = on ? 1 : 0; }

template <int CP, int COUT>
static int cg_blocks_per_sm_or_error(int deep) {
    int blocks = 0;
    const cudaError_t e = deep ? cg_blocks_per_sm<CP, COUT, 1>(&blocks) : cg_blocks_per_sm<CP, COUT, 0>(&blocks);
    return e == cudaSuccess ? blocks : -(int)e;
}

// CTAs of the (cp, cout, deep) instantiation resident on one SM of the current device (the grid is that many per SM at most);
// SESSD_EINVAL for an unsupported (cp, cout), -cudaError on a CUDA error
extern "C" int sessd_spconv_cg_blocks_per_sm(int cp, int cout, int deep) {
    if (cp == 32 && cout == 32) return cg_blocks_per_sm_or_error<32, 32>(deep);
    if (cp == 32 && cout == 64) return cg_blocks_per_sm_or_error<32, 64>(deep);
    if (cp == 64 && cout == 32) return cg_blocks_per_sm_or_error<64, 32>(deep);
    if (cp == 64 && cout == 64) return cg_blocks_per_sm_or_error<64, 64>(deep);
    return SESSD_EINVAL;
}

// S4 (scn.py:106-149), pair-proportional tensor-core path.  d_in_planes [plane_rows][2][cp] fp16 with d_in_info = {abs-max, scale};
// weights / d_scale from ops.pack_weight_sp_h2 (cp = 64: [kvol][2][Cout][64], cp = 32: [kvol][2][Cout][32]; d_scale = BN scale *
// 2^-e[c]); gain / shift_max bound the output (see the header).  Outputs (each nullable, at least one): fp32 rows [max_out][cout],
// planes [>= max_out][2][cout <= 32 ? 32 : 64] + d_out_info = {abs-max (zero it once per frame), scale}.
// Supported (cp, cout): (32,32), (32,64), (64,32), (64,64).
extern "C" int sessd_spconv_forward_cg(const void *d_in_planes, int cp, int plane_rows, const float *d_in_info, const void *d_tiles, int kvol,
                                       const int *d_n_out, int max_out, const void *d_weight_h2, int cout, const float *d_scale,
                                       const float *d_shift, int relu, float gain, float shift_max, float *d_out_f32, void *d_out_planes,
                                       float *d_out_info, void *stream) {
    if (!d_in_planes || !d_in_info || !d_tiles || !d_n_out || !d_weight_h2 || !d_scale || (!d_out_f32 && !d_out_planes) || max_out < 1 ||
        kvol < 1 || kvol > kCgMaxK || plane_rows < 1 || plane_rows > (1 << 25))
        return SESSD_EINVAL;
    if (d_out_planes && !d_out_info) return SESSD_EINVAL;
    if (((uintptr_t)d_out_f32 | (uintptr_t)d_out_planes) & 15) return SESSD_EINVAL;     // the epilogue writes 16 bytes at a time
    CgArgs a;
    a.planes = (const __half *)d_in_planes; a.in_info = d_in_info; a.tiles = (const unsigned int *)d_tiles; a.tile_stride = tile_list_stride(kvol); a.d_n_out = d_n_out; a.kvol = kvol; a.max_out = max_out;
    a.relu = relu; a.scale = d_scale; a.shift = d_shift; a.gain = gain; a.shift_max = shift_max; a.out_f32 = d_out_f32;
    a.out_planes = (__half *)d_out_planes; a.out_info = d_out_info;
    cudaStream_t st = (cudaStream_t)stream;
#define SESSD_CG_CASE(CPV, CO) \
    if (cp == CPV && cout == CO) return g_cg_deep ? launch_spconv_cg<CPV, CO, 1>(a, d_weight_h2, st) : launch_spconv_cg<CPV, CO, 0>(a, d_weight_h2, st);
    SESSD_CG_CASE(32, 32)
    SESSD_CG_CASE(32, 64)
    SESSD_CG_CASE(64, 32)     // data gradient of the 32 -> 64 strided layer
    SESSD_CG_CASE(64, 64)
#undef SESSD_CG_CASE
    return SESSD_EINVAL;
}
