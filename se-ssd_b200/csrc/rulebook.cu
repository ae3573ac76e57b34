// rulebook.cu -- sparse-convolution rulebook ("indice pairs") construction on the GPU.
//
// Replaces the indice-pair builders of spconv 1.x that det3d/models/backbones/scn.py:106-149,182-183 triggers
// (one per SubM indice_key + one per strided SparseConv3d = 8 builds per forward).  spconv builds per-offset pair
// lists with global atomic counters (nondeterministic order).  Here the rulebook is OUTPUT-MAJOR and deterministic:
//     nbr[o, k] = row of the input voxel at  pos_o * stride - pad + k   (or -1),
// which is exactly what the output-stationary gather-GEMM in spconv.cu consumes (no scatter-add, no atomics on
// features), and which the tensor-core conv (spconv_cg.cu) reads regrouped into per-tile pair lists
// (sessd_rulebook_tile_lists, at the end of this file).
//
// Two coordinate indices:
//   * hash   : 64-bit open addressing over linear cell index -> row, for coordinates given in arbitrary order
//              (level 0: the voxeliser's first-appearance order);
//   * bitmap : one bit per cell + exclusive popcount prefix per 32-cell word (uint2).  A strided conv marks its
//              reachable outputs in the bitmap; ranking the bits yields the output rows in ascending linear index
//              -- the canonical order -- without any sort, and the same structure answers lookups with ONE 8-byte
//              read (bit test + popc).  Level-1..4 bitmaps are 3 MB ... 18 KB per frame: L2 resident.
// HBM traffic per build: reads 16 B/input row, writes 4*kvol B/output row (nbr) + 16 B/output row (coords); the
// bitmap/hash probes hit L2.  All counts are device-resident (d_n), grids are persistent.
#include <cuda_fp16.h>

#include "common.cuh"
#include "tile_lists.cuh"

namespace sessd {

struct GridDims { int B, D, H, W; };

__device__ __forceinline__ unsigned long long lin_index(GridDims g, int b, int z, int y, int x) {
    return (((unsigned long long)b * g.D + z) * g.H + y) * g.W + x;
}

struct HashIndex {
    const unsigned long long *tbl;
    int mask;
    __device__ __forceinline__ int find(unsigned long long lin) const { return hash_lookup(tbl, mask, lin); }
    // rows of the cells (row_base + x0 + c), c = 0..n-1, of one x-line; -1 outside [0, W) or where no voxel lives
    __device__ __forceinline__ void find_line(unsigned long long row_base, int x0, int n, int W, int *dst) const {
        for (int c = 0; c < n; ++c) {
            const int x = x0 + c;
            dst[c] = (x >= 0 && x < W) ? find(row_base + x) : -1;
        }
    }
};

struct BitmapIndex {
    const uint2 *words;
    __device__ __forceinline__ int find(unsigned long long lin) const {
        const uint2 e = __ldg(&words[lin >> 5]);
        const unsigned int bit = (unsigned int)lin & 31u;
        if (!((e.x >> bit) & 1u)) return -1;
        return (int)e.y + __popc(e.x & ((1u << bit) - 1u));
    }
    __device__ __forceinline__ void find_line(unsigned long long row_base, int x0, int n, int W, int *dst) const {
        unsigned long long cached = ~0ull;
        uint2 e = make_uint2(0u, 0u);
        for (int c = 0; c < n; ++c) {
            const int x = x0 + c;
            int res = -1;
            if (x >= 0 && x < W) {
                const unsigned long long lin = row_base + x;
                if ((lin >> 5) != cached) { cached = lin >> 5; e = __ldg(&words[cached]); }
                const unsigned int bit = (unsigned int)lin & 31u;
                if ((e.x >> bit) & 1u) res = (int)e.y + __popc(e.x & ((1u << bit) - 1u));
            }
            dst[c] = res;
        }
    }
};

__global__ void __launch_bounds__(256) hash_build_kernel(const int4 *__restrict__ coors, const int *__restrict__ d_n, int max_rows,
                                                         GridDims g, unsigned long long *tbl, int mask) {
    const int n = min(*d_n, max_rows);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int4 c = coors[i];
        hash_insert_min(tbl, mask, lin_index(g, c.x, c.y, c.z, c.w), (unsigned int)i);
    }
}

// nbr table: one thread per (output row, kernel z, kernel y) = one x-line of the kernel window.  The kw cells of the line are
// consecutive in the input grid, so a bitmap-indexed level answers them from one (rarely two) 8-byte words; index arithmetic and the
// coordinate load are shared by the line, and the thread writes kw consecutive ints (warp: one contiguous segment of the table).
// KD..SW > 0: kernel shape / stride known at compile time (the SpMiddleFHD shapes) -- the per-thread divisions and modulos become
// multiplies and shifts (ncu: the runtime-divisor version was ALU-bound, sm 67 %, at 16 % of the DRAM write peak); KD = 0: runtime values.
// IdxT = unsigned int when the work-item count fits 31 bits (host check), long long otherwise.
template <class Index, class IdxT, int KD, int KH, int KW, int SD, int SH, int SW>
__global__ void __launch_bounds__(256) nbr_kernel(const int4 *__restrict__ out_coors, const int *__restrict__ d_n_out, int max_out,
                                                  GridDims gin, Index index, int kd_, int kh_, int kw_, int sd_, int sh_, int sw_,
                                                  int pd, int ph, int pw, int *__restrict__ nbr) {
    const int kd = KD ? KD : kd_, kh = KD ? KH : kh_, kw = KD ? KW : kw_;
    const int sd = KD ? SD : sd_, sh = KD ? SH : sh_, sw = KD ? SW : sw_;
    const int lines = kd * kh;
    const IdxT total = (IdxT)min(*d_n_out, max_out) * (IdxT)lines;
    for (IdxT t = (IdxT)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (IdxT)gridDim.x * blockDim.x) {
        const int o = (int)(t / (IdxT)lines);
        const int l = (int)(t - (IdxT)o * (IdxT)lines);
        const int a = l / kh, bb = l - a * kh;
        const int4 oc = __ldg(&out_coors[o]);
        const int z = oc.y * sd - pd + a, y = oc.z * sh - ph + bb, x0 = oc.w * sw - pw;
        int *dst = nbr + (size_t)t * kw;           // == nbr[o * kvol + (a * kh + bb) * kw]
        if (z < 0 || z >= gin.D || y < 0 || y >= gin.H) {
            for (int c = 0; c < kw; ++c) dst[c] = -1;
            continue;
        }
        index.find_line(lin_index(gin, oc.x, z, y, 0), x0, kw, gin.W, dst);
    }
}

// strided conv, step 1: mark every reachable output cell.  One thread per (input voxel, kernel z, kernel y): along each axis only the
// taps with (i + pad - k) divisible by the stride reach an output (1 or 2 of 3 for k3 s2); the thread walks the kw taps of its x-line.
template <class IdxT, int KD, int KH, int KW, int SD, int SH, int SW>
__global__ void __launch_bounds__(256) mark_outputs_kernel(const int4 *__restrict__ in_coors, const int *__restrict__ d_n_in, int max_in,
                                                           GridDims gout, int kd_, int kh_, int kw_, int sd_, int sh_, int sw_,
                                                           int pd, int ph, int pw, uint2 *bitmap) {
    const int kd = KD ? KD : kd_, kh = KD ? KH : kh_, kw = KD ? KW : kw_;
    const int sd = KD ? SD : sd_, sh = KD ? SH : sh_, sw = KD ? SW : sw_;
    const int lines = kd * kh;
    const IdxT total = (IdxT)min(*d_n_in, max_in) * (IdxT)lines;
    for (IdxT t = (IdxT)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (IdxT)gridDim.x * blockDim.x) {
        const int i = (int)(t / (IdxT)lines);
        const int l = (int)(t - (IdxT)i * (IdxT)lines);
        const int a = l / kh, bb = l - a * kh;
        const int4 ic = __ldg(&in_coors[i]);
        const int nz = ic.y + pd - a, ny = ic.z + ph - bb;
        if (nz < 0 || ny < 0 || nz % sd || ny % sh) continue;
        const int z = nz / sd, y = ny / sh;
        if (z >= gout.D || y >= gout.H) continue;
        const unsigned long long row = lin_index(gout, ic.x, z, y, 0);
        for (int c = 0; c < kw; ++c) {
            const int nx = ic.w + pw - c;
            if (nx < 0 || nx % sw) continue;
            const int x = nx / sw;
            if (x >= gout.W) continue;
            const unsigned long long lin = row + x;
            unsigned int *w = &bitmap[lin >> 5].x;
            const unsigned int bit = 1u << ((unsigned int)lin & 31u);
            if (!(*(volatile unsigned int *)w & bit)) atomicOr(w, bit);
        }
    }
}

// host dispatch over the compile-time shapes of SpMiddleFHD (scn.py:106-149): 3x3x3 s1 (SubM), 3x3x3 s2, (3,1,1) s(2,1,1); else generic
template <class Index>
static void launch_nbr(int grid_sz, cudaStream_t st, const int4 *coors, const int *d_n, int max_out, GridDims g, Index idx, const int k[3],
                       const int s[3], const int p[3], int *nbr) {
    const bool small = (long long)max_out * k[0] * k[1] < (1ll << 31);
#define SESSD_NBR(IT, KD, KH, KW, SD, SH, SW)                                                                                             \
    SESSD_LAUNCH((nbr_kernel<Index, IT, KD, KH, KW, SD, SH, SW>), grid_sz, 256, 0, st, coors, d_n, max_out, g, idx, k[0], k[1], k[2], s[0], \
                 s[1], s[2], p[0], p[1], p[2], nbr)
    if (!small) SESSD_NBR(long long, 0, 0, 0, 0, 0, 0);
    else if (k[0] == 3 && k[1] == 3 && k[2] == 3 && s[0] == 1 && s[1] == 1 && s[2] == 1) SESSD_NBR(unsigned int, 3, 3, 3, 1, 1, 1);
    else if (k[0] == 3 && k[1] == 3 && k[2] == 3 && s[0] == 2 && s[1] == 2 && s[2] == 2) SESSD_NBR(unsigned int, 3, 3, 3, 2, 2, 2);
    else if (k[0] == 3 && k[1] == 1 && k[2] == 1 && s[0] == 2 && s[1] == 1 && s[2] == 1) SESSD_NBR(unsigned int, 3, 1, 1, 2, 1, 1);
    else SESSD_NBR(unsigned int, 0, 0, 0, 0, 0, 0);
#undef SESSD_NBR
}

static void launch_mark(cudaStream_t st, const int4 *coors, const int *d_n, int max_in, GridDims g, const int k[3], const int s[3],
                        const int p[3], uint2 *bm) {
    const int grid_sz = persistent_grid((long long)max_in * k[0] * k[1], 256);
    const bool small = (long long)max_in * k[0] * k[1] < (1ll << 31);
#define SESSD_MARK(IT, KD, KH, KW, SD, SH, SW)                                                                                           \
    SESSD_LAUNCH((mark_outputs_kernel<IT, KD, KH, KW, SD, SH, SW>), grid_sz, 256, 0, st, coors, d_n, max_in, g, k[0], k[1], k[2], s[0], s[1], \
                 s[2], p[0], p[1], p[2], bm)
    if (!small) SESSD_MARK(long long, 0, 0, 0, 0, 0, 0);
    else if (k[0] == 3 && k[1] == 3 && k[2] == 3 && s[0] == 2 && s[1] == 2 && s[2] == 2) SESSD_MARK(unsigned int, 3, 3, 3, 2, 2, 2);
    else if (k[0] == 3 && k[1] == 1 && k[2] == 1 && s[0] == 2 && s[1] == 1 && s[2] == 1) SESSD_MARK(unsigned int, 3, 1, 1, 2, 1, 1);
    else SESSD_MARK(unsigned int, 0, 0, 0, 0, 0, 0);
#undef SESSD_MARK
}

struct PopcLoad {
    const uint2 *words;
    __device__ __forceinline__ int operator()(long long i) const { return __popc(words[i].x); }
};
struct PrefixStore {
    uint2 *words;
    __device__ __forceinline__ void operator()(long long i, int ex, int) const { words[i].y = (unsigned int)ex; }
};

// strided conv, step 3: emit output coordinates in ascending linear index, clamp the count.  On overflow (more sites than max_out) the
// level keeps its first max_out sites in canonical order: the thread that owns a word also clears the bits ranked >= max_out, so every
// later lookup through the bitmap index (SubM rulebook, next strided rulebook, dense gather, skip plan) sees exactly the kept sites and
// never returns a row >= max_out.  The ranks of the kept bits are unchanged.
__global__ void __launch_bounds__(256) enumerate_kernel(uint2 *__restrict__ bitmap, long long nwords, GridDims gout,
                                                        const int *__restrict__ d_total, int max_out, int4 *__restrict__ out_coors,
                                                        int *__restrict__ d_n_out, int *__restrict__ d_status) {
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        const int tot = *d_total;
        *d_n_out = tot < max_out ? tot : max_out;
        if (tot > max_out && d_status) atomicOr(d_status, 1);
    }
    const bool small = nwords < (1ll << 27);
    for (long long w = (long long)blockIdx.x * blockDim.x + threadIdx.x; w < nwords; w += (long long)gridDim.x * blockDim.x) {
        const uint2 e = bitmap[w];
        unsigned int bits = e.x;
        int pos = (int)e.y;
        if ((long long)pos + __popc(bits) > max_out) {    // overflow: keep the lowest (max_out - pos) bits, if any
            unsigned int keep = 0u;
            for (int r = pos; r < max_out && bits; ++r) { keep |= bits & (0u - bits); bits &= bits - 1; }
            bits = keep;
            bitmap[w].x = keep;
        }
        while (bits) {
            const int b = __ffs(bits) - 1;
            bits &= bits - 1;
            if (small) {                                   // < 2^32 cells (every level below the input grid): 32-bit divisions
                unsigned int lin = (unsigned int)w * 32u + (unsigned int)b;
                const unsigned int q1 = lin / (unsigned int)gout.W, x = lin - q1 * (unsigned int)gout.W;
                const unsigned int q2 = q1 / (unsigned int)gout.H, y = q1 - q2 * (unsigned int)gout.H;
                const unsigned int q3 = q2 / (unsigned int)gout.D, z = q2 - q3 * (unsigned int)gout.D;
                out_coors[pos] = make_int4((int)q3, (int)z, (int)y, (int)x);
            } else {
                unsigned long long lin = (unsigned long long)w * 32 + b;
                const int x = (int)(lin % gout.W); lin /= gout.W;
                const int y = (int)(lin % gout.H); lin /= gout.H;
                const int z = (int)(lin % gout.D); lin /= gout.D;
                out_coors[pos] = make_int4((int)lin, z, y, x);
            }
            ++pos;
        }
    }
}

static GridDims to_dims(sessd_grid g) { GridDims d; d.B = g.batch; d.D = g.shape[0]; d.H = g.shape[1]; d.W = g.shape[2]; return d; }


// ---------------------------------------------------------------------------------------------------------------------------------
// Tile lists: the neighbour table regrouped for the pair-proportional tensor-core conv (spconv_cg.cu), record format in tile_lists.cuh.
// Built once per rulebook (a SubM rulebook serves 2-3 layers); deterministic (warp ballots + popcount ranks, no atomics).
template <int KV>
__global__ void __launch_bounds__(kTlRows) tile_lists_kernel(const int *__restrict__ nbr, int kvol_, const int *__restrict__ d_n_out, int max_out,
                                                             unsigned int *__restrict__ tiles) {
    const int kvol = KV ? KV : kvol_;
    const int n_out = min(*d_n_out, max_out);
    const int row0 = blockIdx.x * kTlRows;
    if (row0 >= n_out) return;
    __shared__ unsigned int s_mask[32][4];
    __shared__ int s_off[33];
    const int r = threadIdx.x, warp = r >> 5, lane = r & 31;
    const bool live = row0 + r < n_out;
    int v[KV ? KV : 27];
    const int *src = nbr + (size_t)(row0 + r) * kvol;
#pragma unroll
    for (int k = 0; k < (KV ? KV : 27); ++k) {
        v[k] = (k < kvol && live) ? __ldg(src + k) : -1;
        const unsigned int m = __ballot_sync(0xffffffffu, v[k] >= 0);
        if (lane == 0 && k < kvol) s_mask[k][warp] = m;
    }
    __syncthreads();
    if (r < 32) {                                        // exclusive prefix of the per-offset counts (kvol <= 27 < 32)
        int c = 0;
        if (r < kvol) c = __popc(s_mask[r][0]) + __popc(s_mask[r][1]) + __popc(s_mask[r][2]) + __popc(s_mask[r][3]);
        const int incl = warp_incl_scan(c, lane);
        s_off[r + 1] = incl;
        if (r == 0) s_off[0] = 0;
    }
    __syncthreads();
    unsigned int *rec = tiles + (size_t)blockIdx.x * tile_list_stride(kvol);
    if (r < 32) rec[r] = (unsigned int)(s_off[r + 1] - s_off[r]);
    for (int e = r; e < kvol * 4; e += kTlRows) rec[kTlMask + e] = s_mask[e >> 2][e & 3];
    const unsigned int lt = (1u << lane) - 1u;
#pragma unroll
    for (int k = 0; k < (KV ? KV : 27); ++k) {
        if (k < kvol && v[k] >= 0) {
            int pos = s_off[k] + __popc(s_mask[k][warp] & lt);
            for (int w = 0; w < warp; ++w) pos += __popc(s_mask[k][w]);
            rec[kTlHeader + pos] = tl_entry(v[k], r);
        }
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" size_t sessd_hash_bytes(int max_rows, int *capacity_out) {
    int cap = 1024;
    while (cap < 2 * max_rows) cap <<= 1;
    if (capacity_out) *capacity_out = cap;
    return sizeof(unsigned long long) * (size_t)cap;
}

extern "C" int sessd_hash_build(const int *d_coors, const int *d_n, int max_rows, sessd_grid grid, uint64_t *d_table, int capacity,
                                void *stream) {
    if (!d_coors || !d_n || !d_table || max_rows < 1 || capacity < 2 * max_rows || (capacity & (capacity - 1))) return SESSD_EINVAL;
    if ((long long)max_rows >= (1ll << kHashValBits)) return SESSD_ECAPACITY;
    const unsigned long long cells = (unsigned long long)grid.batch * grid.shape[0] * grid.shape[1] * grid.shape[2];
    if (cells >= (1ull << (64 - kHashValBits))) return SESSD_ECAPACITY;
    cudaStream_t st = (cudaStream_t)stream;
    SESSD_CUDA_TRY(cudaMemsetAsync(d_table, 0xff, sizeof(unsigned long long) * (size_t)capacity, st));
    SESSD_LAUNCH(hash_build_kernel, persistent_grid(max_rows, 256), 256, 0, st, (const int4 *)d_coors, d_n, max_rows, to_dims(grid),
                 (unsigned long long *)d_table, capacity - 1);
    return last_error();
}

extern "C" size_t sessd_bitmap_words(sessd_grid grid) {
    const unsigned long long cells = (unsigned long long)grid.batch * grid.shape[0] * grid.shape[1] * grid.shape[2];
    return (size_t)((cells + 31) / 32);
}

extern "C" size_t sessd_scan_scratch_bytes(size_t n_items) { return scan_scratch_bytes((long long)n_items) + 256; }

extern "C" int sessd_subm_rulebook(const int *d_coors, const int *d_n, int max_rows, sessd_grid grid, const int ksize[3],
                                   int index_kind, const void *d_index, int hash_capacity, int *d_nbr, void *stream) {
    if (!d_coors || !d_n || !d_index || !d_nbr || max_rows < 1 || !ksize) return SESSD_EINVAL;
    const int kd = ksize[0], kh = ksize[1], kw = ksize[2];
    if (kd < 1 || kh < 1 || kw < 1 || !(kd & 1) || !(kh & 1) || !(kw & 1)) return SESSD_EINVAL;
    const GridDims g = to_dims(grid);
    const int grid_sz = persistent_grid((long long)max_rows * kd * kh, 256);
    const int one[3] = {1, 1, 1}, pad[3] = {kd / 2, kh / 2, kw / 2};
    if (index_kind == 0) {
        HashIndex idx{(const unsigned long long *)d_index, hash_capacity - 1};
        launch_nbr(grid_sz, (cudaStream_t)stream, (const int4 *)d_coors, d_n, max_rows, g, idx, ksize, one, pad, d_nbr);
    } else if (index_kind == 1) {
        BitmapIndex idx{(const uint2 *)d_index};
        launch_nbr(grid_sz, (cudaStream_t)stream, (const int4 *)d_coors, d_n, max_rows, g, idx, ksize, one, pad, d_nbr);
    } else {
        return SESSD_EINVAL;
    }
    return last_error();
}

extern "C" int sessd_strided_rulebook(const int *d_in_coors, const int *d_n_in, int max_in, sessd_grid in_grid, int in_index_kind,
                                      const void *d_in_index, int in_hash_capacity, const int ksize[3], const int stride[3],
                                      const int padding[3], sessd_grid out_grid, void *d_out_bitmap, void *d_scan_scratch,
                                      int *d_out_coors, int *d_n_out, int max_out, int *d_nbr, int *d_status, void *stream) {
    if (!d_in_coors || !d_n_in || !d_in_index || !d_out_bitmap || !d_scan_scratch || !d_out_coors || !d_n_out || !d_nbr || !ksize ||
        !stride || !padding || max_in < 1 || max_out < 1)
        return SESSD_EINVAL;
    for (int j = 0; j < 3; ++j) {
        if (ksize[j] < 1 || stride[j] < 1 || padding[j] < 0) return SESSD_EINVAL;
        if (out_grid.shape[j] != (in_grid.shape[j] + 2 * padding[j] - ksize[j]) / stride[j] + 1) return SESSD_EINVAL;
    }
    if (out_grid.batch != in_grid.batch) return SESSD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const GridDims gi = to_dims(in_grid), go = to_dims(out_grid);
    const size_t words = sessd_bitmap_words(out_grid);
    if (words >= (1ull << 31)) return SESSD_ECAPACITY;
    uint2 *bm = (uint2 *)d_out_bitmap;
    SESSD_CUDA_TRY(cudaMemsetAsync(bm, 0, sizeof(uint2) * words, st));
    launch_mark(st, (const int4 *)d_in_coors, d_n_in, max_in, go, ksize, stride, padding, bm);
    int *scratch = (int *)d_scan_scratch;
    int *d_total = scratch;                    // first int: total; tile sums follow (256-byte offset)
    PopcLoad ld{bm};
    PrefixStore stf{bm};
    device_scan(ld, stf, nullptr, (long long)words, (long long)words, scratch + 64, d_total, st);
    SESSD_LAUNCH(enumerate_kernel, persistent_grid((long long)words, 256), 256, 0, st, bm, (long long)words, go, d_total, max_out,
                 (int4 *)d_out_coors, d_n_out, d_status);
    const int grid_sz = persistent_grid((long long)max_out * ksize[0] * ksize[1], 256);
    if (in_index_kind == 0) {
        HashIndex idx{(const unsigned long long *)d_in_index, in_hash_capacity - 1};
        launch_nbr(grid_sz, st, (const int4 *)d_out_coors, d_n_out, max_out, gi, idx, ksize, stride, padding, d_nbr);
    } else if (in_index_kind == 1) {
        BitmapIndex idx{(const uint2 *)d_in_index};
        launch_nbr(grid_sz, st, (const int4 *)d_out_coors, d_n_out, max_out, gi, idx, ksize, stride, padding, d_nbr);
    } else {
        return SESSD_EINVAL;
    }
    return last_error();
}

// dense() as ONE gather pass over the output (no memset + scatter): thread = 4 consecutive output channels of one BEV cell; the rows of
// the D z-slices of the cell come from the level's bitmap index (bit test + popcount rank).  NHWC [B, H, W, C*D], channel = c*D + d
// (== NCDHW .view(N, C*D, H, W) of det3d/models/backbones/scn.py:184-187, channels-last).  Writes every output byte exactly once with
// 16-byte stores; reads each feature row once.
template <bool PLANES>
__global__ void __launch_bounds__(256) dense_gather_kernel(const float *__restrict__ feat, BitmapIndex index, GridDims g, int C,
                                                           int max_rows, float4 *__restrict__ out, const float *__restrict__ amax,
                                                           float *__restrict__ info, __half *__restrict__ planes, long long plane_stride) {
    const unsigned int cd4 = (unsigned int)(C * g.D) >> 2;
    const unsigned int total = (unsigned int)g.B * g.H * g.W * cd4;          // < 2^31 (checked by the host)
    float s = 1.f;
    if (PLANES) {
        const float am = __ldg(amax);
        s = pow2_scale_for_bound(am);
        if (blockIdx.x == 0 && threadIdx.x == 0) { info[0] = am; info[1] = s; }
    }
    for (unsigned int t = blockIdx.x * blockDim.x + threadIdx.x; t < total; t += gridDim.x * blockDim.x) {
        const unsigned int cell = t / cd4;
        const int j = (int)(t - cell * cd4) * 4;
        const unsigned int r = cell / (unsigned int)g.W;
        const int x = (int)(cell - r * g.W);
        const int b = (int)(r / (unsigned int)g.H), y = (int)(r - (r / (unsigned int)g.H) * g.H);
        float v[4];
        int last_d = -1, row = -1;
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int ch = j + e;
            const int c = ch / g.D, d = ch - c * g.D;
            if (d != last_d) { row = index.find(lin_index(g, b, d, y, x)); last_d = d; }
            v[e] = (row >= 0 && row < max_rows) ? __ldg(&feat[(size_t)row * C + c]) : 0.f;    // rows past the capacity were dropped (status flag)
        }
        if (PLANES) {
            __align__(8) __half hi[4], lo[4];
#pragma unroll
            for (int e = 0; e < 4; ++e) {
                const float a = v[e] * s;
                hi[e] = __float2half_rn(a);
                lo[e] = __float2half_rn(a - __half2float(hi[e]));
            }
            *reinterpret_cast<uint2 *>(planes + 4 * (size_t)t) = *reinterpret_cast<const uint2 *>(hi);
            *reinterpret_cast<uint2 *>(planes + plane_stride + 4 * (size_t)t) = *reinterpret_cast<const uint2 *>(lo);
        } else {
            out[t] = make_float4(v[0], v[1], v[2], v[3]);
        }
    }
}

extern "C" int sessd_sparse_to_dense_indexed(const float *d_feat, int max_rows, const void *d_bitmap_index, int channels, sessd_grid grid,
                                             float *d_out, void *stream) {
    if (!d_feat || !d_bitmap_index || !d_out || channels < 1 || max_rows < 1 || ((channels * grid.shape[0]) & 3)) return SESSD_EINVAL;
    const GridDims g = to_dims(grid);
    BitmapIndex idx{(const uint2 *)d_bitmap_index};
    const long long total = (long long)g.B * g.H * g.W * ((channels * g.D) >> 2);
    if (total >= (1ll << 31)) return SESSD_ECAPACITY;
    SESSD_LAUNCH(dense_gather_kernel<false>, persistent_grid(total, 256), 256, 0, stream, d_feat, idx, g, channels, max_rows, (float4 *)d_out,
                 nullptr, nullptr, nullptr, 0ll);
    return last_error();
}

// dense() straight into the fp16 (hi, lo) planes [2][B][H][W][C*D] the BEV neck reads (sessd_bev_conv_p2): d_amax = abs-max of the feature
// rows (raised by the producing sparse conv), d_info[2] receives {abs-max, scale}
extern "C" int sessd_sparse_to_dense_planes(const float *d_feat, int max_rows, const void *d_bitmap_index, int channels, sessd_grid grid,
                                            const float *d_amax, float *d_info, void *d_planes, void *stream) {
    if (!d_feat || !d_bitmap_index || !d_amax || !d_info || !d_planes || channels < 1 || max_rows < 1 || ((channels * grid.shape[0]) & 3))
        return SESSD_EINVAL;
    const GridDims g = to_dims(grid);
    BitmapIndex idx{(const uint2 *)d_bitmap_index};
    const long long total = (long long)g.B * g.H * g.W * ((channels * g.D) >> 2);
    if (total >= (1ll << 31)) return SESSD_ECAPACITY;
    SESSD_LAUNCH(dense_gather_kernel<true>, persistent_grid(total, 256), 256, 0, stream, d_feat, idx, g, channels, max_rows, nullptr, d_amax,
                 d_info, (__half *)d_planes, total * 4);
    return last_error();
}

// words per tile record of sessd_rulebook_tile_lists (128 output rows per tile)
extern "C" int sessd_tile_list_stride(int kvol) { return tile_list_stride(kvol); }

// nbr table -> per-tile pair lists for sessd_spconv_forward_cg (see tile_lists_kernel).  d_tiles: uint32 [ceil(max_out / 128)][stride].
extern "C" int sessd_rulebook_tile_lists(const int *d_nbr, int kvol, const int *d_n_out, int max_out, void *d_tiles, void *stream) {
    if (!d_nbr || !d_n_out || !d_tiles || kvol < 1 || kvol > 27 || max_out < 1) return SESSD_EINVAL;
    const int nblk = div_up(max_out, kTlRows);
    if (kvol == 27)
        SESSD_LAUNCH((tile_lists_kernel<27>), nblk, kTlRows, 0, stream, d_nbr, kvol, d_n_out, max_out, (unsigned int *)d_tiles);
    else if (kvol == 3)
        SESSD_LAUNCH((tile_lists_kernel<3>), nblk, kTlRows, 0, stream, d_nbr, kvol, d_n_out, max_out, (unsigned int *)d_tiles);
    else
        SESSD_LAUNCH((tile_lists_kernel<0>), nblk, kTlRows, 0, stream, d_nbr, kvol, d_n_out, max_out, (unsigned int *)d_tiles);
    return last_error();
}
