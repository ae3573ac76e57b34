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
//     exact power-of-two scale -- are copied pair-major by double-buffered 16-byte cp.async and fed to mma.sync.m16n8k16 through
//     ldmatrix.trans (the pairs are K, so both operands are transposed on the way to the fragments); three products per MAC as in the forward (a_hi g_hi into the main accumulator,
//     a_hi g_lo + a_lo g_hi into the cross accumulator, fp32), summed RN once per item; the reduce divides by S_in S_g (exact).
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace sessd {

constexpr int kGrTile = 128;                 // output rows per tile-list record
constexpr int kGrHeader = 160;               // words before the pair entries of a record (rulebook.cu)
constexpr int kGrMaxK = 27;
constexpr int kGrThreads = 256;
constexpr int kGrKC = 64;                    // pairs staged per round
constexpr int kGrItemsTarget = 4 * kNumSMs;  // items per launch the decomposition aims at (several per SM)

__host__ __device__ inline int gr_stride(int kvol) { return kGrHeader + kGrTile * kvol; }

// chunks (tile ranges) per offset; a function of (max_out, kvol) only: the summation order of the result never depends on the data
static inline void wgrad_chunks(int max_out, int kvol, int *chunks, int *tiles_per_item) {
    const int nt = div_up(max_out, kGrTile);
    int c = div_up(kGrItemsTarget, kvol);
    if (c > nt) c = nt;
    const int t = div_up(nt, c);
    *tiles_per_item = t;
    *chunks = div_up(nt, t);
}

// the item's offset and tile range; the entries of offset k in a record start after the counts of offsets < k
__device__ __forceinline__ int gr_offset_start(const unsigned int *rec, int k) {
    int s = 0;
    for (int j = 0; j < k; ++j) s += (int)__ldg(rec + j);
    return s;
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
    const int ntiles = (n_out + kGrTile - 1) / kGrTile;
    const int t0 = ch * tpi, t1 = min(ntiles, t0 + tpi);
    const int tid = threadIdx.x;
    float acc[kPer];
#pragma unroll
    for (int j = 0; j < kPer; ++j) acc[j] = 0.f;
    for (int t = t0; t < t1; ++t) {
        const unsigned int *rec = tiles + (size_t)t * gr_stride(kvol);
        const int cnt = (int)__ldg(rec + k);
        if (cnt == 0) continue;                                             // block-uniform
        const unsigned int *lst = rec + kGrHeader + gr_offset_start(rec, k);
        for (int p0 = 0; p0 < cnt; p0 += kGrKC) {
            const int np = min(kGrKC, cnt - p0);
            for (int e = tid; e < np * CIN; e += kGrThreads) {
                const int p = e / CIN, c = e - p * CIN;
                s_in[p][c] = __ldg(in_feat + (size_t)(__ldg(lst + p0 + p) >> 7) * CIN + c);
            }
            for (int e = tid; e < np * COUT; e += kGrThreads) {
                const int p = e / COUT, n = e - p * COUT;
                const unsigned int en = __ldg(lst + p0 + p);
                s_g[p][n] = __ldg(gout + ((size_t)t * kGrTile + (en & 127u)) * COUT + n);
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
// CP input channels (plane width), COUT output channels (= the gradient plane width).  Eight warps tile the [CP][COUT] result in m16 slabs
// x NT n8 tiles each.  A round stages up to kGrKC pairs PAIR-MAJOR, exactly as the planes lie in global memory: [hi | lo][pair][channel],
// 16-byte cp.async per 8 channels (slots past the round's pairs are zero-filled by the copy itself), double-buffered so the next round's
// copies fly while this round multiplies.  Rows are padded to CP + 8 halves: the eight 16-byte rows an ldmatrix phase reads fall in eight
// different bank groups.  The mma fragments (A = in^T: [channel][pair], B = gout: [pair][channel]) come out of ldmatrix.trans.
template <int CP, int COUT>
struct WgCfg {
    static constexpr int kPitchA = CP + 8, kPitchG = COUT + 8;             // halves
    static constexpr int kBufHalves = 2 * kGrKC * (kPitchA + kPitchG);       // one buffer: A hi, A lo, G hi, G lo
    static constexpr int kSmem = 2 * kBufHalves * 2;                         // bytes, two buffers
    static constexpr int kMSlabs = CP / 16;
    static constexpr int kNT = (CP / 16) * (COUT / 8) / 8;     // n8 tiles per warp
    static_assert(kNT >= 1 && (CP / 16) * (COUT / 8) % 8 == 0, "eight warps must tile the result");
    static_assert(kNT == 1 || kNT % 2 == 0, "B fragments are loaded two n8 tiles at a time");
};

// one round of an item: up to kGrKC pairs of offset k in tile t, from entry p0 on (block-uniform)
struct WgRound {
    int t, p0, cnt;
    const unsigned int *lst;
};

// the first tile in [t, t1) with pairs of offset k
__device__ __forceinline__ bool wg_seek(const unsigned int *tiles, int kvol, int k, int t, int t1, WgRound &r) {
    for (; t < t1; ++t) {
        const unsigned int *rec = tiles + (size_t)t * gr_stride(kvol);
        const int cnt = (int)__ldg(rec + k);
        if (cnt > 0) {
            r.t = t; r.p0 = 0; r.cnt = cnt;
            r.lst = rec + kGrHeader + gr_offset_start(rec, k);
            return true;
        }
    }
    return false;
}

__device__ __forceinline__ bool wg_next(const unsigned int *tiles, int kvol, int k, int t1, WgRound &r) {
    if (r.p0 + kGrKC < r.cnt) { r.p0 += kGrKC; return true; }
    return wg_seek(tiles, kvol, k, r.t + 1, t1, r);
}

template <int CP, int COUT>
__global__ void __launch_bounds__(kGrThreads) wgrad_cg_kernel(const __half *__restrict__ in_planes, const __half *__restrict__ g_planes,
                                                              const unsigned int *__restrict__ tiles, int kvol, const int *__restrict__ d_n_out,
                                                              int max_out, int chunks, int tpi, float *__restrict__ partial) {
    using C = WgCfg<CP, COUT>;
    extern __shared__ __align__(16) unsigned char wg_smem[];
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(wg_smem);
    // buffer b: A half h at s0 + 2 (b kBufHalves + h kGrKC kPitchA), G half h after the two A halves
    auto a_addr = [&](int b, int h, int p, int c) { return s0 + 2u * (uint32_t)(b * C::kBufHalves + (h * kGrKC + p) * C::kPitchA + c); };
    auto g_addr = [&](int b, int h, int p, int c) {
        return s0 + 2u * (uint32_t)(b * C::kBufHalves + 2 * kGrKC * C::kPitchA + (h * kGrKC + p) * C::kPitchG + c);
    };
    const int item = blockIdx.x, k = item / chunks, ch = item - k * chunks;
    const int n_out = min(*d_n_out, max_out);
    const int ntiles = (n_out + kGrTile - 1) / kGrTile;
    const int t0 = ch * tpi, t1 = min(ntiles, t0 + tpi);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gq = lane >> 2, tq = lane & 3;
    const int lr = lane & 7, lm = lane >> 3;                           // ldmatrix: row within an 8x8 matrix, matrix index
    const int m0 = (warp % C::kMSlabs) * 16, n0 = (warp / C::kMSlabs) * C::kNT * 8;
    float acc_m[C::kNT][4], acc_c[C::kNT][4];
#pragma unroll
    for (int j = 0; j < C::kNT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) { acc_m[j][q] = 0.f; acc_c[j][q] = 0.f; }

    // copy a round's rows into buffer b: pair slots [np, 16 ceil(np / 16)) are zero-filled (the mma reads whole k16 steps)
    auto stage = [&](const WgRound &r, int b) {
        const int np = min(kGrKC, r.cnt - r.p0);
        const int kp = (np + 15) & ~15;
        constexpr int kAChunks = 2 * CP / 8, kGChunks = 2 * COUT / 8;
        for (int e = tid; e < kp * (kAChunks + kGChunks); e += kGrThreads) {
            const int p = e / (kAChunks + kGChunks), q = e - p * (kAChunks + kGChunks);
            const bool valid = p < np;
            const unsigned int en = valid ? __ldg(r.lst + r.p0 + p) : 0u;
            if (q < kAChunks) {
                const int h = q / (CP / 8), c0 = (q % (CP / 8)) * 8;
                wg_cp_async16(a_addr(b, h, p, c0), in_planes + (size_t)(en >> 7) * (2 * CP) + h * CP + c0, valid);
            } else {
                const int qq = q - kAChunks, h = qq / (COUT / 8), c0 = (qq % (COUT / 8)) * 8;
                const size_t o = (size_t)r.t * kGrTile + (en & 127u);
                wg_cp_async16(g_addr(b, h, p, c0), g_planes + o * (2 * COUT) + h * COUT + c0, valid);
            }
        }
    };

    WgRound cur;
    bool have = wg_seek(tiles, kvol, k, t0, t1, cur);
    if (have) stage(cur, 0);
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    int buf = 0;
    while (have) {                                                      // block-uniform
        WgRound nxt = cur;
        const bool more = wg_next(tiles, kvol, k, t1, nxt);
        if (more) stage(nxt, buf ^ 1);
        asm volatile("cp.async.commit_group;\n" ::: "memory");
        asm volatile("cp.async.wait_group 1;\n" ::: "memory");          // this round's copies (the next round's stay in flight)
        __syncthreads();
        const int steps = (min(kGrKC, cur.cnt - cur.p0) + 15) >> 4;
        for (int s = 0; s < steps; ++s) {
            const int k0 = s * 16;
            // A fragments: matrix lm covers pairs k0 + 8 (lm >> 1) .., channels m0 + 8 (lm & 1) ..  ->  a0..a3 of m16n8k16
            uint32_t ah[4], al[4];
            ldsm_x4_trans(ah, a_addr(buf, 0, k0 + lr + 8 * (lm >> 1), m0 + 8 * (lm & 1)));
            ldsm_x4_trans(al, a_addr(buf, 1, k0 + lr + 8 * (lm >> 1), m0 + 8 * (lm & 1)));
#pragma unroll
            for (int j = 0; j < C::kNT; j += (C::kNT == 1 ? 1 : 2)) {
                // B fragments: matrix lm covers pairs k0 + 8 (lm & 1) .., channels n0 + 8 (j + (lm >> 1)) ..  ->  (b0, b1) of tile j (, j + 1)
                uint32_t bh[4], bl[4];
                const int gp = k0 + lr + 8 * (lm & 1), gc = n0 + 8 * j + 8 * (lm >> 1);
                if constexpr (C::kNT == 1) {
                    ldsm_x2_trans(bh, g_addr(buf, 0, gp, n0));
                    ldsm_x2_trans(bl, g_addr(buf, 1, gp, n0));
                } else {
                    ldsm_x4_trans(bh, g_addr(buf, 0, gp, gc));
                    ldsm_x4_trans(bl, g_addr(buf, 1, gp, gc));
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
        have = more;
        buf ^= 1;
    }
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
    // partial[item][c][n] = acc_m + acc_c (RN); this thread holds rows m0 + gq (+8), columns 2 tq (+1) of every n8 tile
    float *dst = partial + (size_t)item * (CP * COUT);
#pragma unroll
    for (int j = 0; j < C::kNT; ++j) {
        const int n = n0 + 8 * j + 2 * tq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + gq + 8 * h;
            *reinterpret_cast<float2 *>(dst + (size_t)m * COUT + n) =
                make_float2(acc_m[j][2 * h] + acc_c[j][2 * h], acc_m[j][2 * h + 1] + acc_c[j][2 * h + 1]);
        }
    }
}

template <int CP, int COUT>
static int launch_wgrad_cg(const __half *in_planes, const __half *g_planes, const unsigned int *tl, int kvol, const int *d_n_out, int max_out,
                           int chunks, int tpi, float *part, cudaStream_t st) {
    constexpr int kSmem = WgCfg<CP, COUT>::kSmem;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(wgrad_cg_kernel<CP, COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
        if (e != cudaSuccess) return (int)e;
        attr_done = true;
    }
    SESSD_LAUNCH((wgrad_cg_kernel<CP, COUT>), kvol * chunks, kGrThreads, kSmem, st, in_planes, g_planes, tl, kvol, d_n_out,
                 max_out, chunks, tpi, part);
    return last_error();
}

// gW[k][e] = (sum over the chunks of offset k, ascending, of partial[k chunks + c][e]) / S_in / S_g  (info pointers nullable: scale 1)
__global__ void __launch_bounds__(256) wgrad_reduce_kernel(const float *__restrict__ partial, int kvol, int chunks, int per_item,
                                                           const float *__restrict__ in_info, const float *__restrict__ g_info,
                                                           float *__restrict__ gw) {
    const float inv_a = in_info ? 1.f / __ldg(in_info + 1) : 1.f;         // exact: powers of two
    const float inv_g = g_info ? 1.f / __ldg(g_info + 1) : 1.f;
    const long long total = (long long)kvol * per_item;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int k = (int)(t / per_item), e = (int)(t - (long long)k * per_item);
        const float *p = partial + (size_t)k * chunks * per_item + e;
        float s = 0.f;
        for (int c = 0; c < chunks; ++c) s += __ldg(p + (size_t)c * per_item);
        gw[t] = s * inv_a * inv_g;
    }
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

static int wgrad_reduce(const float *partial, int kvol, int chunks, int per_item, const float *in_info, const float *g_info, float *gw,
                        cudaStream_t st) {
    SESSD_LAUNCH(wgrad_reduce_kernel, persistent_grid((long long)kvol * per_item, 256), 256, 0, st, partial, kvol, chunks, per_item, in_info,
                 g_info, gw);
    return last_error();
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
        return wgrad_reduce(part, kvol, chunks, CI * CO, nullptr, nullptr, d_gw, st);                                           \
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
        const int rc = launch_wgrad_cg<CPV, CO>((const __half *)d_in_planes, (const __half *)d_g_planes, tl, kvol, d_n_out, max_out,   \
                                                chunks, tpi, part, st);                                                               \
        return rc ? rc : wgrad_reduce(part, kvol, chunks, CPV * CO, d_in_info, d_g_info, d_gw, st);                                   \
    }
    WG_CASE(32, 32)
    WG_CASE(32, 64)
    WG_CASE(64, 64)
#undef WG_CASE
    return SESSD_EINVAL;
}
