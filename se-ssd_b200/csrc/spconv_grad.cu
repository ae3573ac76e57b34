// spconv_grad.cu -- backward of the sparse 3-D convolutions of SpMiddleFHD (det3d/models/backbones/scn.py:106-149): the pieces the data
// gradient needs around the forward kernels, and the weight gradient.
//
// Rulebook form (oracle/spconv_grad_ref.py): out[o] = sum_k in[nbr[o, k]] @ W[k]
//   dgrad  gin[i] = sum_k gout[nbr_t[i, k]] @ W[k]^T   -- the FORWARD kernels (spconv_rows.cu / spconv_cg.cu) run over the transposed table
//          (strided layers: sessd_rulebook_transpose; SubM layers: the same table with W'[k] = W[K-1-k]^T), no kernel of its own;
//   wgrad  gW[k]   = sum_{o : nbr[o, k] >= 0} in[nbr[o, k]]^T gout[o]  -- here.
// Weight gradient: the pairs are the reduction (K) dimension.  The forward's per-tile pair lists (sessd_rulebook_tile_lists) already group
// every (input row, output row) pair by offset, so a work ITEM is (offset k, a fixed range of tiles): it walks the pairs of offset k in
// those tiles, in list order, and writes its own fp32 partial [Cin][Cout] to the workspace.  The item decomposition depends on max_out and
// kvol only (wgrad_chunks), so a reduce kernel that sums the partials of an offset in ascending item order makes the result bitwise
// run-to-run deterministic without a float atomic.
//   * rows (Cin <= 16, layers 0-2): fp32 SIMT fmaf chains over the item's pairs, in list order;
//   * cg   (Cin >= 32): the input planes saved by the forward and the gradient planes (sessd_sparse_split_planes) -- fp16 (hi, lo) at an
//     exact power-of-two scale -- on the tensor cores (wgrad_mma.cuh), the pairs being the K rows; the reduce divides by S_in S_g (exact).
#include <cuda_fp16.h>

#include "tile_lists.cuh"
#include "wgrad_mma.cuh"

namespace sessd {

constexpr int kGrMaxK = 27;
constexpr int kGrThreads = 256;
constexpr int kGrKC = 64;                    // pairs staged per round (fp32 SIMT kernel)
constexpr int kGrItemsTarget = 4 * kNumSMs;  // items per launch the decomposition aims at (several per SM)

// chunks (tile ranges) per offset; a function of (max_out, kvol) only: the summation order of the result never depends on the data
static inline void wgrad_chunks(int max_out, int kvol, int *chunks, int *tiles_per_item) {
    const int nt = div_up(max_out, kTlRows);
    int c = div_up(kGrItemsTarget, kvol);
    if (c > nt) c = nt;
    const int t = div_up(nt, c);
    *tiles_per_item = t;
    *chunks = div_up(nt, t);
}

// ---------------------------------------------------------------------------------------------------------------- fp32 SIMT wgrad
template <int CIN, int COUT>
__global__ void __launch_bounds__(kGrThreads) wgrad_rows_kernel(const float *__restrict__ in_feat, const float *__restrict__ gout,
                                                                const unsigned int *__restrict__ tiles, int kvol, const int *__restrict__ d_n_out,
                                                                int max_out, int chunks, int tpi, float *__restrict__ partial) {
    constexpr int kOut = CIN * COUT;
    constexpr int kPer = (kOut + kGrThreads - 1) / kGrThreads;
    __shared__ float s_in[kGrKC][CIN];
    __shared__ float s_g[kGrKC][COUT];
    const int item = blockIdx.x, k = item / chunks, ch = item - k * chunks;
    const int n_out = min(*d_n_out, max_out);
    const int ntiles = (n_out + kTlRows - 1) / kTlRows;
    const int t0 = ch * tpi, t1 = min(ntiles, t0 + tpi);
    const int tid = threadIdx.x;
    float acc[kPer];
#pragma unroll
    for (int j = 0; j < kPer; ++j) acc[j] = 0.f;
    for (int t = t0; t < t1; ++t) {
        const unsigned int *rec = tiles + (size_t)t * tile_list_stride(kvol);
        const int cnt = (int)__ldg(rec + k);
        if (cnt == 0) continue;                                             // block-uniform
        const unsigned int *lst = rec + kTlHeader + tl_offset_start(rec, k);
        for (int p0 = 0; p0 < cnt; p0 += kGrKC) {
            const int np = min(kGrKC, cnt - p0);
            for (int e = tid; e < np * CIN; e += kGrThreads) {
                const int p = e / CIN, c = e - p * CIN;
                s_in[p][c] = __ldg(in_feat + (size_t)tl_in_row(__ldg(lst + p0 + p)) * CIN + c);
            }
            for (int e = tid; e < np * COUT; e += kGrThreads) {
                const int p = e / COUT, n = e - p * COUT;
                const unsigned int en = __ldg(lst + p0 + p);
                s_g[p][n] = __ldg(gout + ((size_t)t * kTlRows + tl_tile_row(en)) * COUT + n);
            }
            __syncthreads();
#pragma unroll
            for (int j = 0; j < kPer; ++j) {
                const int e = tid + j * kGrThreads;
                if (e < kOut) {
                    const int c = e / COUT, n = e - c * COUT;
                    for (int p = 0; p < np; ++p) acc[j] = fmaf(s_in[p][c], s_g[p][n], acc[j]);
                }
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int j = 0; j < kPer; ++j) {
        const int e = tid + j * kGrThreads;
        if (e < kOut) partial[(size_t)item * kOut + e] = acc[j];
    }
}

// ---------------------------------------------------------------------------------------------------------------- tensor-core wgrad
// one round of an item: up to kWgKC pairs of offset k in tile t, from entry p0 on (block-uniform)
struct WgRound {
    int t, p0, cnt;
    const unsigned int *lst;
    bool live;                               // false: past the item's last round
};

// the first tile in [t, t1) with pairs of offset k
__device__ __forceinline__ bool wg_seek(const unsigned int *tiles, int kvol, int k, int t, int t1, WgRound &r) {
    for (; t < t1; ++t) {
        const unsigned int *rec = tiles + (size_t)t * tile_list_stride(kvol);
        const int cnt = (int)__ldg(rec + k);
        if (cnt > 0) {
            r.t = t; r.p0 = 0; r.cnt = cnt;
            r.lst = rec + kTlHeader + tl_offset_start(rec, k);
            return true;
        }
    }
    return false;
}

__device__ __forceinline__ bool wg_next(const unsigned int *tiles, int kvol, int k, int t1, WgRound &r) {
    if (r.p0 + kWgKC < r.cnt) { r.p0 += kWgKC; return true; }
    return wg_seek(tiles, kvol, k, r.t + 1, t1, r);
}

// CP input channels (plane width), COUT output channels (= the gradient plane width); a round's K rows are pairs, the A row of a pair is
// its input row's plane row, the G row its output row's
template <int CP, int COUT>
__global__ void __launch_bounds__(kWgThreads) wgrad_cg_kernel(const __half *__restrict__ in_planes, const __half *__restrict__ g_planes,
                                                              const unsigned int *__restrict__ tiles, int kvol, const int *__restrict__ d_n_out,
                                                              int max_out, int chunks, int tpi, float *__restrict__ partial) {
    extern __shared__ __align__(16) unsigned char wg_smem[];
    const WgLayout<CP, COUT> L{(uint32_t)__cvta_generic_to_shared(wg_smem)};
    const int item = blockIdx.x, k = item / chunks, ch = item - k * chunks;
    const int n_out = min(*d_n_out, max_out);
    const int ntiles = (n_out + kTlRows - 1) / kTlRows;
    const int t0 = ch * tpi, t1 = min(ntiles, t0 + tpi);
    const int tid = threadIdx.x;

    // copy a round's rows into buffer b: pair slots [np, 16 ceil(np / 16)) are zero-filled (the mma reads whole k16 steps)
    auto stage = [&](const WgRound &r, int b) {
        const int np = min(kWgKC, r.cnt - r.p0);
        const int kp = (np + 15) & ~15;
        constexpr int kAChunks = 2 * CP / 8, kGChunks = 2 * COUT / 8;
        for (int e = tid; e < kp * (kAChunks + kGChunks); e += kWgThreads) {
            const int p = e / (kAChunks + kGChunks), q = e - p * (kAChunks + kGChunks);
            const bool valid = p < np;
            const unsigned int en = valid ? __ldg(r.lst + r.p0 + p) : 0u;
            if (q < kAChunks) {
                const int h = q / (CP / 8), c0 = (q % (CP / 8)) * 8;
                wg_cp_async16(L.a(b, h, p, c0), in_planes + (size_t)tl_in_row(en) * (2 * CP) + h * CP + c0, valid);
            } else {
                const int qq = q - kAChunks, h = qq / (COUT / 8), c0 = (qq % (COUT / 8)) * 8;
                const size_t o = (size_t)r.t * kTlRows + tl_tile_row(en);
                wg_cp_async16(L.g(b, h, p, c0), g_planes + o * (2 * COUT) + h * COUT + c0, valid);
            }
        }
    };
    wgrad_mma_item<CP, COUT, WgRound>(
        L, [&](WgRound &r) { r.live = wg_seek(tiles, kvol, k, t0, t1, r); }, [](const WgRound &r) { return r.live; },
        [&](WgRound &r) { r.live = wg_next(tiles, kvol, k, t1, r); },
        [](const WgRound &r) { return min(kWgKC, r.cnt - r.p0); }, stage, partial);
}

// ---------------------------------------------------------------------------------------------------------------- reduce
// gw[t][ci][co]: see wgrad_mma.cuh.  Block row blockIdx.y = t.
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float *__restrict__ partial, int cin, int cout, int bm, int bn, int chunks,
                                                           const float *__restrict__ in_info, const float *__restrict__ g_info,
                                                           float *__restrict__ gw) {
    const float inv_a = in_info ? 1.f / __ldg(in_info + 1) : 1.f;         // exact: powers of two
    const float inv_g = g_info ? 1.f / __ldg(g_info + 1) : 1.f;
    const int t = blockIdx.y, per_tile = bm * bn, mblocks = cin / bm, nblocks = cout / bn;
    for (int r = blockIdx.x * blockDim.x + threadIdx.x; r < cin * cout; r += gridDim.x * blockDim.x) {
        const int ci = r / cout, co = r - ci * cout;
        const int mb = ci / bm, nb = co / bn;
        const float *p = partial + (size_t)((t * mblocks + mb) * nblocks + nb) * chunks * per_tile + (ci - mb * bm) * bn + (co - nb * bn);
        float s = 0.f;
        for (int c = 0; c < chunks; ++c) s += __ldg(p + (size_t)c * per_tile);
        gw[(size_t)t * cin * cout + r] = s * inv_a * inv_g;
    }
}

int wgrad_reduce(const float *partial, int ntaps, int cin, int cout, int bm, int bn, int chunks, const float *in_info, const float *g_info,
                 float *gw, cudaStream_t st) {
    const dim3 grid(div_up(persistent_grid((long long)ntaps * cin * cout, 256), ntaps), ntaps);
    SESSD_LAUNCH(wgrad_reduce_kernel, grid, 256, 0, st, partial, cin, cout, bm, bn, chunks, in_info, g_info, gw);
    return last_error();
}

// ---------------------------------------------------------------------------------------------------------------- helpers
// nbr_t[i, k] = o with nbr[o, k] = i, else -1.  Each (i, k) has at most one o, so the scatter is deterministic.
__global__ void __launch_bounds__(256) rulebook_transpose_kernel(const int *__restrict__ nbr, int kvol, const int *__restrict__ d_n_out,
                                                                 int max_out, int max_in, int *__restrict__ nbr_t) {
    const long long total = (long long)min(*d_n_out, max_out) * kvol;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int i = __ldg(nbr + t);
        if (i >= 0 && i < max_in) {
            const int o = (int)(t / kvol), k = (int)(t - (long long)o * kvol);
            nbr_t[(size_t)i * kvol + k] = o;
        }
    }
}

// fp32 rows -> (hi, lo) planes at S = pow2_scale_for_bound(info[0]) (the epilogues' rule); channels [C, cp) of a row are zero
__global__ void __launch_bounds__(256) sparse_split_planes_kernel(const float *__restrict__ x, const int *__restrict__ d_n, int max_rows, int channels,
                                                                  int cp, float *__restrict__ info, __half *__restrict__ planes) {
    const float s = pow2_scale_for_bound(__ldg(info));
    if (blockIdx.x == 0 && threadIdx.x == 0) info[1] = s;
    const long long total = (long long)min(*d_n, max_rows) * cp;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int r = (int)(t / cp), c = (int)(t - (long long)r * cp);
        const float v = c < channels ? __ldg(x + (size_t)r * channels + c) * s : 0.f;
        const __half hi = __float2half_rn(v);
        planes[(size_t)r * 2 * cp + c] = hi;
        planes[(size_t)r * 2 * cp + cp + c] = __float2half_rn(v - __half2float(hi));
    }
}

// adjoint of dense(): rows[r][c] = grad[b, y, x, c D + z] for (b, z, y, x) = coors[r]
__global__ void __launch_bounds__(256) dense_grad_gather_kernel(const float *__restrict__ grad, const int4 *__restrict__ coors,
                                                                const int *__restrict__ d_n, int max_rows, int C, int D, int H, int W,
                                                                float *__restrict__ out) {
    const long long total = (long long)min(*d_n, max_rows) * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int row = (int)(t / C), c = (int)(t - (long long)row * C);
        const int4 q = __ldg(&coors[row]);
        out[t] = __ldg(grad + (((size_t)q.x * H + q.z) * W + q.w) * (size_t)(C * D) + (size_t)c * D + q.y);
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" int sessd_rulebook_transpose(const int *d_nbr, int kvol, const int *d_n_out, int max_out, int max_in, int *d_nbr_t, void *stream) {
    if (!d_nbr || !d_n_out || !d_nbr_t || kvol < 1 || kvol > kGrMaxK || max_out < 1 || max_in < 1) return SESSD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    SESSD_CUDA_TRY(cudaMemsetAsync(d_nbr_t, 0xFF, sizeof(int) * (size_t)max_in * kvol, st));
    SESSD_LAUNCH(rulebook_transpose_kernel, persistent_grid((long long)max_out * kvol, 256), 256, 0, st, d_nbr, kvol, d_n_out, max_out, max_in,
                 d_nbr_t);
    return last_error();
}

extern "C" int sessd_sparse_split_planes(const float *d_x, const int *d_n, int max_rows, int channels, float *d_info, void *d_planes, int cp,
                                         void *stream) {
    if (!d_x || !d_n || !d_info || !d_planes || max_rows < 1 || channels < 1 || cp < channels || (cp != 32 && cp != 64)) return SESSD_EINVAL;
    SESSD_LAUNCH(sparse_split_planes_kernel, persistent_grid((long long)max_rows * cp, 256), 256, 0, stream, d_x, d_n, max_rows, channels, cp,
                 d_info, (__half *)d_planes);
    return last_error();
}

extern "C" int sessd_dense_grad_gather(const float *d_grad, const int *d_coors, const int *d_n, int max_rows, int channels, sessd_grid grid,
                                       float *d_out, void *stream) {
    if (!d_grad || !d_coors || !d_n || !d_out || max_rows < 1 || channels < 1) return SESSD_EINVAL;
    SESSD_LAUNCH(dense_grad_gather_kernel, persistent_grid((long long)max_rows * channels, 256), 256, 0, stream, d_grad, (const int4 *)d_coors,
                 d_n, max_rows, channels, grid.shape[0], grid.shape[1], grid.shape[2], d_out);
    return last_error();
}

extern "C" int sessd_spconv_wgrad_items(int max_out, int kvol) {
    if (max_out < 1 || kvol < 1 || kvol > kGrMaxK) return SESSD_EINVAL;
    int chunks, tpi;
    wgrad_chunks(max_out, kvol, &chunks, &tpi);
    return kvol * chunks;
}

extern "C" size_t sessd_spconv_wgrad_workspace_bytes(int max_out, int kvol, int cin, int cout) {
    const int items = sessd_spconv_wgrad_items(max_out, kvol);
    if (items < 1 || cin < 1 || cout < 1) return 0;
    return sizeof(float) * (size_t)items * (size_t)cin * (size_t)cout;
}

extern "C" int sessd_spconv_wgrad_rows(const float *d_in_feat, int cin, const float *d_gout, int cout, const void *d_tiles, int kvol,
                                       const int *d_n_out, int max_out, float *d_gw, void *d_ws, size_t ws_bytes, void *stream) {
    if (!d_in_feat || !d_gout || !d_tiles || !d_n_out || !d_gw || !d_ws || max_out < 1 || kvol < 1 || kvol > kGrMaxK) return SESSD_EINVAL;
    if (ws_bytes < sessd_spconv_wgrad_workspace_bytes(max_out, kvol, cin, cout)) return SESSD_EWORKSPACE;
    int chunks, tpi;
    wgrad_chunks(max_out, kvol, &chunks, &tpi);
    cudaStream_t st = (cudaStream_t)stream;
    float *part = (float *)d_ws;
    const unsigned int *tl = (const unsigned int *)d_tiles;
#define GR_CASE(CI, CO)                                                                                                          \
    if (cin == CI && cout == CO) {                                                                                               \
        SESSD_LAUNCH((wgrad_rows_kernel<CI, CO>), kvol * chunks, kGrThreads, 0, st, d_in_feat, d_gout, tl, kvol, d_n_out, max_out, \
                     chunks, tpi, part);                                                                                         \
        return wgrad_reduce(part, kvol, CI, CO, CI, CO, chunks, nullptr, nullptr, d_gw, st);                                    \
    }
    GR_CASE(4, 16)
    GR_CASE(16, 16)
    GR_CASE(16, 32)
#undef GR_CASE
    return SESSD_EINVAL;
}

extern "C" int sessd_spconv_wgrad_cg(const void *d_in_planes, int cp, const float *d_in_info, const void *d_g_planes, int cout,
                                     const float *d_g_info, const void *d_tiles, int kvol, const int *d_n_out, int max_out, float *d_gw,
                                     void *d_ws, size_t ws_bytes, void *stream) {
    if (!d_in_planes || !d_in_info || !d_g_planes || !d_g_info || !d_tiles || !d_n_out || !d_gw || !d_ws || max_out < 1 || kvol < 1 ||
        kvol > kGrMaxK)
        return SESSD_EINVAL;
    if (ws_bytes < sessd_spconv_wgrad_workspace_bytes(max_out, kvol, cp, cout)) return SESSD_EWORKSPACE;
    int chunks, tpi;
    wgrad_chunks(max_out, kvol, &chunks, &tpi);
    cudaStream_t st = (cudaStream_t)stream;
    float *part = (float *)d_ws;
    const unsigned int *tl = (const unsigned int *)d_tiles;
#define WG_CASE(CPV, CO)                                                                                                              \
    if (cp == CPV && cout == CO) {                                                                                                    \
        const int rc = wgrad_launch<wgrad_cg_kernel<CPV, CO>, CPV, CO>(kvol * chunks, st, (const __half *)d_in_planes,                  \
                                                                       (const __half *)d_g_planes, tl, kvol, d_n_out, max_out, chunks, \
                                                                       tpi, part);                                                     \
        return rc ? rc : wgrad_reduce(part, kvol, CPV, CO, CPV, CO, chunks, d_in_info, d_g_info, d_gw, st);                           \
    }
    WG_CASE(32, 32)
    WG_CASE(32, 64)
    WG_CASE(64, 64)
#undef WG_CASE
    return SESSD_EINVAL;
}
