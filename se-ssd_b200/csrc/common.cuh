// common.cuh -- shared device/host helpers for the sessd_b200 kernels (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>

#include "../../include/sessd_b200.h"

namespace sessd {

constexpr int kNumSMs = 132;   // H100 SXM; grids are sized in multiples of this

extern long long g_launches;   // counted per kernel launch (sessd_launch_count)

#define SESSD_LAUNCH(kernel, grid, block, smem, stream, ...)                                         \
    do {                                                                                             \
        kernel<<<(grid), (block), (smem), (cudaStream_t)(stream)>>>(__VA_ARGS__);                    \
        ++::sessd::g_launches;                                                                       \
    } while (0)

#define SESSD_CUDA_TRY(expr)                                                                         \
    do {                                                                                             \
        cudaError_t _e = (expr);                                                                     \
        if (_e != cudaSuccess) return (int)_e;                                                       \
    } while (0)

// exact power-of-two scale that maps `bound` (> 0, finite) into [2^14, 2^15): the scale of fp16 (hi, lo) activation planes whose
// elements are bounded by `bound` (1 when the bound is 0 / not finite).  x * S < 2^15 < 65504 for every |x| <= bound.
__host__ __device__ __forceinline__ float pow2_scale_for_bound(float bound) {
    union { float f; uint32_t u; } v;
    v.f = bound;
    const uint32_t e = (v.u >> 23) & 0xFFu;
    if (e == 0 || e == 255) return 1.f;
    int bits = 268 - (int)e;                                  // biased exponent of 2^(14 - (e - 127))
    bits = bits < 2 ? 2 : (bits > 252 ? 252 : bits);
    v.u = (uint32_t)bits << 23;
    return v.f;
}

static inline int last_error() { return (int)cudaGetLastError(); }

static inline int div_up(long long a, long long b) { return (int)((a + b - 1) / b); }

// persistent-style grid: enough CTAs to fill the machine `waves` times, never more than the work needs
static inline int persistent_grid(long long work_items, int block, int ctas_per_sm = 8) {
    long long need = (work_items + block - 1) / block;
    long long cap = (long long)kNumSMs * ctas_per_sm;
    if (need < 1) need = 1;
    return (int)(need < cap ? need : cap);
}

// the frame that owns row i of a batch with non-decreasing offsets off [batch + 1]: the largest b < batch with off[b] <= i (0 when none),
// so an empty frame never owns a row
__device__ __forceinline__ int find_frame(const int *__restrict__ off, int batch, int i) {
    int lo = 0, hi = batch;   // off[lo] <= i < off[hi]
    while (hi - lo > 1) {
        int mid = (lo + hi) >> 1;
        if (i >= off[mid]) lo = mid; else hi = mid;
    }
    return lo;
}

// ---------------------------------------------------------------------------------------------
// 64-bit open-addressing hash: slot = key << 24 | value (value < 2^24), empty = all ones.
// Used by the voxeliser (value = first point index, atomicMin) and the level-0 coordinate index
// (value = row).
// ---------------------------------------------------------------------------------------------
constexpr unsigned long long kHashEmpty = 0xFFFFFFFFFFFFFFFFull;
constexpr int kHashValBits = 24;
constexpr unsigned long long kHashValMask = (1ull << kHashValBits) - 1;

__device__ __forceinline__ unsigned int hash_mix(unsigned long long k) {
    k ^= k >> 33;
    k *= 0xff51afd7ed558ccdull;
    k ^= k >> 33;
    k *= 0xc4ceb9fe1a85ec53ull;
    k ^= k >> 33;
    return (unsigned int)k;
}

// insert (key, val); on duplicate keys the smallest value wins.  returns the slot.
__device__ __forceinline__ int hash_insert_min(unsigned long long *tbl, int cap_mask, unsigned long long key,
                                               unsigned int val) {
    const unsigned long long entry = (key << kHashValBits) | val;
    unsigned int h = hash_mix(key) & cap_mask;
    while (true) {
        unsigned long long cur = tbl[h];
        if (cur == kHashEmpty) {
            cur = atomicCAS(&tbl[h], kHashEmpty, entry);
            if (cur == kHashEmpty) return (int)h;
        }
        if ((cur >> kHashValBits) == key) {
            if (entry < cur) atomicMin(&tbl[h], entry);
            return (int)h;
        }
        h = (h + 1) & cap_mask;
    }
}

__device__ __forceinline__ int hash_lookup(const unsigned long long *__restrict__ tbl, int cap_mask,
                                           unsigned long long key) {
    unsigned int h = hash_mix(key) & cap_mask;
    while (true) {
        unsigned long long cur = __ldg(&tbl[h]);
        if (cur == kHashEmpty) return -1;
        if ((cur >> kHashValBits) == key) return (int)(cur & kHashValMask);
        h = (h + 1) & cap_mask;
    }
}

// ---------------------------------------------------------------------------------------------
// Device-wide exclusive scan of 32-bit counts (three launches, no spin-waits => nothing can hang).
//   pass 1: per-tile reduce, pass 2: one CTA scans the tile sums, pass 3: per-tile scan + offset.
// The item count lives in device memory (d_n; nullptr => the host constant n_mul); launches are sized from the capacity, and every
// kernel clamps the count to [0, capacity], so a device count past the buffer never reads or writes past it.
// `Load` is a functor int(long long i).  out[i] = sum_{j<i} load(j); out[n] = total.
// ---------------------------------------------------------------------------------------------
constexpr int kScanThreads = 256;
constexpr int kScanItems = 8;
constexpr int kScanTile = kScanThreads * kScanItems;

__device__ __forceinline__ int warp_incl_scan(int v, int lane) {
#pragma unroll
    for (int d = 1; d < 32; d <<= 1) {
        int t = __shfl_up_sync(0xffffffffu, v, d);
        if (lane >= d) v += t;
    }
    return v;
}

// block-wide exclusive scan of one value per thread (256 threads); returns exclusive prefix, total in *total
__device__ __forceinline__ int block_excl_scan(int v, int *smem /*>= 9 ints*/, int *total) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    int incl = warp_incl_scan(v, lane);
    if (lane == 31) smem[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        int w = (lane < (int)(blockDim.x >> 5)) ? smem[lane] : 0;
        int wi = warp_incl_scan(w, lane);
        if (lane < (int)(blockDim.x >> 5)) smem[lane] = wi - w;
        if (lane == 31) smem[32] = wi;
    }
    __syncthreads();
    int res = incl - v + smem[warp];
    *total = smem[32];
    __syncthreads();
    return res;
}

__device__ __forceinline__ long long scan_count(const int *d_n, long long n_mul, long long cap) {
    const long long n = d_n ? (long long)(*d_n) * n_mul : n_mul;
    return n < 0 ? 0 : (n < cap ? n : cap);
}

template <class Load>
__global__ void __launch_bounds__(kScanThreads) scan_reduce_kernel(Load load, const int *__restrict__ d_n,
                                                                   long long n_mul, long long cap, int *__restrict__ tile_sums) {
    __shared__ int sm[40];
    const long long n = scan_count(d_n, n_mul, cap);
    const long long base = (long long)blockIdx.x * kScanTile;
    if (base >= n) return;
    int s = 0;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        long long i = base + (long long)j * kScanThreads + threadIdx.x;
        if (i < n) s += load(i);
    }
    int tot;
    block_excl_scan(s, sm, &tot);
    if (threadIdx.x == 0) tile_sums[blockIdx.x] = tot;
}

static __global__ void __launch_bounds__(1024) scan_tiles_kernel(const int *__restrict__ d_n, long long n_mul, long long cap,
                                                          int *__restrict__ tile_sums, int *__restrict__ d_total) {
    __shared__ int sm[40];
    __shared__ int carry;
    const long long n = scan_count(d_n, n_mul, cap);
    const int tiles = (int)((n + kScanTile - 1) / kScanTile);
    if (threadIdx.x == 0) carry = 0;
    __syncthreads();
    for (int b = 0; b < tiles; b += blockDim.x) {
        int i = b + threadIdx.x;
        int v = (i < tiles) ? tile_sums[i] : 0;
        int tot;
        int ex = block_excl_scan(v, sm, &tot);
        if (i < tiles) tile_sums[i] = ex + carry;
        __syncthreads();
        if (threadIdx.x == 0) carry += tot;
        __syncthreads();
    }
    if (threadIdx.x == 0 && d_total) *d_total = carry;
}

// SELF_PREFIX: tile_sums holds the raw per-tile sums of scan_reduce_kernel and every CTA adds up the sums of the tiles before it itself (a few
// hundred ints) -- saves the one-CTA scan_tiles launch for mid-sized inputs (two launches instead of three); the last tile writes the total.
template <class Load, class Store, bool SELF_PREFIX>
__global__ void __launch_bounds__(kScanThreads) scan_apply_kernel(Load load, Store store, const int *__restrict__ d_n,
                                                                  long long n_mul, long long cap, const int *__restrict__ tile_sums,
                                                                  int *__restrict__ d_total) {
    __shared__ int sm[40];
    const long long n = scan_count(d_n, n_mul, cap);
    const long long base = (long long)blockIdx.x * kScanTile;
    if (SELF_PREFIX && n <= 0 && blockIdx.x == 0 && threadIdx.x == 0 && d_total) *d_total = 0;
    if (base >= n) return;
    int tile_off = 0;
    if (SELF_PREFIX) {
        int part = 0;
        for (int t = threadIdx.x; t < (int)blockIdx.x; t += kScanThreads) part += tile_sums[t];
        int tot;
        block_excl_scan(part, sm, &tot);
        tile_off = tot;
    } else {
        tile_off = tile_sums[blockIdx.x];
    }
    // thread owns kScanItems consecutive items (blocked arrangement keeps the scan order trivial)
    int v[kScanItems];
    int s = 0;
    const long long first = base + (long long)threadIdx.x * kScanItems;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        long long i = first + j;
        v[j] = (i < n) ? load(i) : 0;
        s += v[j];
    }
    int tot;
    int ex = block_excl_scan(s, sm, &tot) + tile_off;
#pragma unroll
    for (int j = 0; j < kScanItems; ++j) {
        long long i = first + j;
        if (i < n) store(i, ex, v[j]);
        ex += v[j];
    }
    if (SELF_PREFIX && d_total && threadIdx.x == 0 && base + kScanTile >= n) *d_total = tile_off + tot;     // the last tile
}

// Small inputs (a frame's point list, the bitmaps of the coarse levels): ONE launch of one 1024-thread CTA that walks the items in chunks with a
// running carry -- the three-launch scan costs ~12 us of launch latency per use at batch 1, more than the work itself.
constexpr int kScanSmallThreads = 1024;
constexpr int kScanSelfPrefixTiles = 1024;               // up to this many tiles every apply CTA sums the preceding tile sums itself
constexpr long long kScanSmallMax = 16 * 1024;          // capacity (items) up to which the one-CTA scan is used (measured: 5.5 k / 2.2 k bitmap words -6 us, 48 k words +30 us)

template <class Load, class Store>
__global__ void __launch_bounds__(kScanSmallThreads) scan_small_kernel(Load load, Store store, const int *__restrict__ d_n, long long n_mul,
                                                                       long long cap, int *__restrict__ d_total) {
    __shared__ int sm[40];
    const long long n = scan_count(d_n, n_mul, cap);
    int carry = 0;
    for (long long base = 0; base < n; base += (long long)kScanSmallThreads * kScanItems) {
        int v[kScanItems];
        int s = 0;
        const long long first = base + (long long)threadIdx.x * kScanItems;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            const long long i = first + j;
            v[j] = (i < n) ? load(i) : 0;
            s += v[j];
        }
        int tot;
        int ex = block_excl_scan(s, sm, &tot) + carry;
#pragma unroll
        for (int j = 0; j < kScanItems; ++j) {
            const long long i = first + j;
            if (i < n) store(i, ex, v[j]);
            ex += v[j];
        }
        carry += tot;
    }
    if (threadIdx.x == 0 && d_total) *d_total = carry;
}

// host driver.  scratch: ints[ceil(cap/kScanTile) + 1].  d_n * n_mul items; cap = capacity in items.
template <class Load, class Store>
static inline void device_scan(Load load, Store store, const int *d_n, long long n_mul, long long cap_items,
                               int *scratch, int *d_total, cudaStream_t st) {
    if (cap_items <= kScanSmallMax) {
        SESSD_LAUNCH((scan_small_kernel<Load, Store>), 1, kScanSmallThreads, 0, st, load, store, d_n, n_mul, cap_items, d_total);
        return;
    }
    int tiles = (int)((cap_items + kScanTile - 1) / kScanTile);
    if (tiles < 1) tiles = 1;
    SESSD_LAUNCH((scan_reduce_kernel<Load>), tiles, kScanThreads, 0, st, load, d_n, n_mul, cap_items, scratch);
    if (tiles <= kScanSelfPrefixTiles) {
        SESSD_LAUNCH((scan_apply_kernel<Load, Store, true>), tiles, kScanThreads, 0, st, load, store, d_n, n_mul, cap_items, scratch,
                     d_total);
        return;
    }
    SESSD_LAUNCH(scan_tiles_kernel, 1, 1024, 0, st, d_n, n_mul, cap_items, scratch, d_total);
    SESSD_LAUNCH((scan_apply_kernel<Load, Store, false>), tiles, kScanThreads, 0, st, load, store, d_n, n_mul, cap_items, scratch,
                     d_total);
}

static inline size_t scan_scratch_bytes(long long cap_items) {
    return sizeof(int) * (size_t)((cap_items + kScanTile - 1) / kScanTile + 2);
}

}  // namespace sessd
