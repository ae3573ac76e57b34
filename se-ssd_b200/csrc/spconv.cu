// spconv.cu -- sparse 3-D convolution forward (output-stationary gather -> GEMM -> fused BN+ReLU) and dense().
//
// Replaces spconv 1.x SubMConv3d / SparseConv3d forward (per offset: gather rows -> sgemm -> scatter-add; up to
// 27 small GEMMs + 54 gather/scatter launches per layer) followed by the unfused BatchNorm1d + ReLU of
// det3d/models/backbones/scn.py:106-149, and SparseConvTensor.dense() + view (scn.py:184-187).
//
// One launch per layer.  A CTA owns a tile of TM=128 output voxels and walks the kernel offsets that have at least
// one neighbour inside the tile (offsets with none are skipped): for offset k it gathers the TM input rows
// nbr[o,k] (zero rows where missing) and W[k] into shared memory with cp.async (double buffered against the math of
// the previous offset) and accumulates  acc[o,:] += A_k[o,:] @ W[k]  in registers.  The epilogue applies the folded
// BatchNorm scale/shift and ReLU and writes each output row exactly once -- no scatter-add, no atomics, no
// intermediate buffers (spconv writes/reads 2 x sum(P_k) x C floats of gather/scatter buffers per layer).
// Algorithmic HBM bytes per layer: 4 (N_in Cin + N_out Cout) + 4 kvol N_out (nbr) + 4 kvol Cin Cout (weights);
// FLOPs: 2 sum(P_k) Cin Cout.  This SIMT fp32 version is the numerics baseline for the tensor-core path.
#include "common.cuh"

namespace sessd {

__device__ __forceinline__ void cp_async16(void *smem, const void *gmem, bool valid) {
    const unsigned int s = (unsigned int)__cvta_generic_to_shared(smem);
    const int sz = valid ? 16 : 0;   // src-size 0 => 16 bytes of zeros are written
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

constexpr int kSpTM = 128;
constexpr int kSpThreads = 256;
constexpr int kSpMaxK = 32;

template <int CIN, int COUT>
struct SpCfg {
    static constexpr int kAStride = CIN + 4;                  // floats; +4 keeps 16-byte alignment and spreads banks
    static constexpr int kTn = COUT / 4;                      // threads along cout (float4 each)
    static constexpr int kTm = kSpThreads / kTn;              // threads along rows
    static constexpr int kRm = kSpTM / kTm;                   // rows per thread
    static constexpr int kABytes = kSpTM * kAStride * 4;
    static constexpr int kWBytes = CIN * COUT * 4;
    static constexpr int kStageBytes = kABytes + kWBytes;
    static constexpr int kSmem = 2 * kStageBytes + kSpTM * kSpMaxK * 4 + 256;
};

template <int CIN, int COUT>
__global__ void __launch_bounds__(kSpThreads) spconv_gemm_kernel(const float *__restrict__ in_feat, const int *__restrict__ nbr,
                                                                 int kvol, const int *__restrict__ d_n_out, int max_out,
                                                                 const float *__restrict__ weight, const float *__restrict__ scale,
                                                                 const float *__restrict__ shift, int relu,
                                                                 float *__restrict__ out_feat) {
    using C = SpCfg<CIN, COUT>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *stage[2] = {reinterpret_cast<float *>(smem_raw), reinterpret_cast<float *>(smem_raw + C::kStageBytes)};
    int *s_nbr = reinterpret_cast<int *>(smem_raw + 2 * C::kStageBytes);
    int *s_klist = s_nbr + kSpTM * kSpMaxK;      // [kSpMaxK] active offsets
    int *s_nact = s_klist + kSpMaxK;
    unsigned int *s_kmask = reinterpret_cast<unsigned int *>(s_nact + 1);

    const int n_out = min(*d_n_out, max_out);
    const int tiles = (n_out + kSpTM - 1) / kSpTM;
    const int tid = threadIdx.x;
    const int tn = tid % C::kTn, tm = tid / C::kTn;

    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
        const int row0 = tile * kSpTM;
        const int rows = min(kSpTM, n_out - row0);
        if (tid == 0) *s_kmask = 0u;
        __syncthreads();
        // neighbour tile (contiguous in global memory) + per-offset occupancy
        unsigned int mymask = 0;
        for (int e = tid; e < kSpTM * kvol; e += kSpThreads) {
            const int r = e / kvol, k = e - r * kvol;
            int v = -1;
            if (r < rows) v = nbr[(size_t)row0 * kvol + e];
            s_nbr[r * kSpMaxK + k] = v;
            if (v >= 0) mymask |= 1u << k;
        }
        mymask = __reduce_or_sync(0xffffffffu, mymask);
        if ((tid & 31) == 0 && mymask) atomicOr(s_kmask, mymask);
        __syncthreads();
        if (tid == 0) {
            unsigned int m = *s_kmask;
            int c = 0;
            while (m) { const int k = __ffs(m) - 1; m &= m - 1; s_klist[c++] = k; }
            *s_nact = c;
        }
        __syncthreads();
        const int nact = *s_nact;

        float acc[C::kRm][4];
#pragma unroll
        for (int i = 0; i < C::kRm; ++i) { acc[i][0] = acc[i][1] = acc[i][2] = acc[i][3] = 0.f; }

        auto prefetch = [&](int st, int k) {
            float *sA = stage[st];
            float *sW = sA + kSpTM * C::kAStride;
            constexpr int kChunksPerRow = CIN / 4;
            for (int e = tid; e < kSpTM * kChunksPerRow; e += kSpThreads) {
                const int r = e / kChunksPerRow, c4 = e - r * kChunksPerRow;
                const int src = s_nbr[r * kSpMaxK + k];
                const float *g = in_feat + (size_t)(src >= 0 ? src : 0) * CIN + c4 * 4;
                cp_async16(sA + r * C::kAStride + c4 * 4, g, src >= 0);
            }
            const float *gw = weight + (size_t)k * CIN * COUT;
            for (int e = tid; e < CIN * COUT / 4; e += kSpThreads) cp_async16(sW + e * 4, gw + e * 4, true);
            cp_async_commit();
        };

        if (nact > 0) prefetch(0, s_klist[0]);
        for (int j = 0; j < nact; ++j) {
            if (j + 1 < nact) { prefetch((j + 1) & 1, s_klist[j + 1]); cp_async_wait<1>(); }
            else cp_async_wait<0>();
            __syncthreads();
            const float *sA = stage[j & 1];
            const float *sW = sA + kSpTM * C::kAStride;
#pragma unroll 2
            for (int c = 0; c < CIN; c += 4) {
                float4 w0 = *reinterpret_cast<const float4 *>(sW + (c + 0) * COUT + tn * 4);
                float4 w1 = *reinterpret_cast<const float4 *>(sW + (c + 1) * COUT + tn * 4);
                float4 w2 = *reinterpret_cast<const float4 *>(sW + (c + 2) * COUT + tn * 4);
                float4 w3 = *reinterpret_cast<const float4 *>(sW + (c + 3) * COUT + tn * 4);
#pragma unroll
                for (int i = 0; i < C::kRm; ++i) {
                    const float4 a = *reinterpret_cast<const float4 *>(sA + (tm * C::kRm + i) * C::kAStride + c);
                    acc[i][0] = fmaf(a.x, w0.x, acc[i][0]); acc[i][1] = fmaf(a.x, w0.y, acc[i][1]);
                    acc[i][2] = fmaf(a.x, w0.z, acc[i][2]); acc[i][3] = fmaf(a.x, w0.w, acc[i][3]);
                    acc[i][0] = fmaf(a.y, w1.x, acc[i][0]); acc[i][1] = fmaf(a.y, w1.y, acc[i][1]);
                    acc[i][2] = fmaf(a.y, w1.z, acc[i][2]); acc[i][3] = fmaf(a.y, w1.w, acc[i][3]);
                    acc[i][0] = fmaf(a.z, w2.x, acc[i][0]); acc[i][1] = fmaf(a.z, w2.y, acc[i][1]);
                    acc[i][2] = fmaf(a.z, w2.z, acc[i][2]); acc[i][3] = fmaf(a.z, w2.w, acc[i][3]);
                    acc[i][0] = fmaf(a.w, w3.x, acc[i][0]); acc[i][1] = fmaf(a.w, w3.y, acc[i][1]);
                    acc[i][2] = fmaf(a.w, w3.z, acc[i][2]); acc[i][3] = fmaf(a.w, w3.w, acc[i][3]);
                }
            }
            __syncthreads();
        }
        // epilogue: folded BatchNorm1d (eval) + ReLU, one float4 store per row
        float4 sc = make_float4(1.f, 1.f, 1.f, 1.f), sh = make_float4(0.f, 0.f, 0.f, 0.f);
        if (scale) sc = *reinterpret_cast<const float4 *>(scale + tn * 4);
        if (shift) sh = *reinterpret_cast<const float4 *>(shift + tn * 4);
#pragma unroll
        for (int i = 0; i < C::kRm; ++i) {
            const int r = tm * C::kRm + i;
            if (r < rows) {
                float4 o;
                o.x = fmaf(acc[i][0], sc.x, sh.x); o.y = fmaf(acc[i][1], sc.y, sh.y);
                o.z = fmaf(acc[i][2], sc.z, sh.z); o.w = fmaf(acc[i][3], sc.w, sh.w);
                if (relu) { o.x = fmaxf(o.x, 0.f); o.y = fmaxf(o.y, 0.f); o.z = fmaxf(o.z, 0.f); o.w = fmaxf(o.w, 0.f); }
                *reinterpret_cast<float4 *>(out_feat + (size_t)(row0 + r) * COUT + tn * 4) = o;
            }
        }
        __syncthreads();
    }
}

// dense(): NHWC [B, H, W, C*D], channel = c*D + d   (== NCDHW .view(N, C*D, H, W) of scn.py:186-187, channels-last)
__global__ void __launch_bounds__(256) dense_scatter_kernel(const float *__restrict__ feat, const int4 *__restrict__ coors,
                                                            const int *__restrict__ d_n, int max_rows, int C, int D, int H, int W,
                                                            float *__restrict__ out) {
    const long long total = (long long)min(*d_n, max_rows) * C;
    for (long long t = (long long)blockIdx.x * blockDim.x + threadIdx.x; t < total; t += (long long)gridDim.x * blockDim.x) {
        const int row = (int)(t / C), c = (int)(t - (long long)row * C);
        const int4 q = __ldg(&coors[row]);   // b, z, y, x
        out[(((size_t)q.x * H + q.z) * W + q.w) * (size_t)(C * D) + (size_t)c * D + q.y] = feat[t];
    }
}

template <int CIN, int COUT>
static int launch_spconv(const float *in, const int *nbr, int kvol, const int *d_n, int max_out, const float *w, const float *sc,
                         const float *sh, int relu, float *out, cudaStream_t st) {
    using C = SpCfg<CIN, COUT>;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(spconv_gemm_kernel<CIN, COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, C::kSmem);
        if (e != cudaSuccess) return (int)e;
        attr_done = true;
    }
    const int tiles = div_up(max_out, kSpTM);
    const int grid = tiles < 2 * kNumSMs ? tiles : 2 * kNumSMs;
    SESSD_LAUNCH((spconv_gemm_kernel<CIN, COUT>), grid, kSpThreads, C::kSmem, st, in, nbr, kvol, d_n, max_out, w, sc, sh, relu, out);
    return last_error();
}

// abs-max over the first *d_n rows of a [max_rows, channels] fp32 tensor (rows beyond the device-side count hold stale data)
__global__ void __launch_bounds__(256) absmax_rows_kernel(const float *__restrict__ feat, const int *__restrict__ d_n, int max_rows, int channels,
                                                          float *__restrict__ amax) {
    const int n = min(*d_n, max_rows);
    const long long total4 = ((long long)n * channels) >> 2;
    float m = 0.f;
    for (long long i = blockIdx.x * (long long)blockDim.x + threadIdx.x; i < total4; i += (long long)gridDim.x * blockDim.x) {
        const float4 v = __ldg(reinterpret_cast<const float4 *>(feat) + i);
        m = fmaxf(m, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
    }
    const unsigned w = __reduce_max_sync(0xFFFFFFFFu, __float_as_uint(m));
    if ((threadIdx.x & 31) == 0 && w != 0u) atomicMax(reinterpret_cast<unsigned *>(amax), w);
}

}  // namespace sessd

using namespace sessd;

extern "C" int sessd_absmax_rows(const float *d_feat, const int *d_n, int max_rows, int channels, float *d_amax, void *stream) {
    if (!d_feat || !d_n || !d_amax || max_rows < 1 || channels < 4 || (channels & 3)) return SESSD_EINVAL;
    SESSD_LAUNCH(absmax_rows_kernel, persistent_grid(((long long)max_rows * channels) >> 2, 256), 256, 0, stream, d_feat, d_n, max_rows, channels,
                 d_amax);
    return last_error();
}


extern "C" int sessd_spconv_forward(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out, int max_out,
                                    const float *d_weight, int cout, const float *d_scale, const float *d_shift, int relu,
                                    float *d_out_feat, void *stream) {
    if (!d_in_feat || !d_nbr || !d_n_out || !d_weight || !d_out_feat || max_out < 1 || kvol < 1 || kvol > kSpMaxK) return SESSD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
#define SP_CASE(CI, CO) \
    if (cin == CI && cout == CO) return launch_spconv<CI, CO>(d_in_feat, d_nbr, kvol, d_n_out, max_out, d_weight, d_scale, d_shift, relu, d_out_feat, st)
    SP_CASE(4, 16);
    SP_CASE(16, 16);
    SP_CASE(16, 32);
    SP_CASE(32, 32);
    SP_CASE(32, 64);
    SP_CASE(64, 64);
#undef SP_CASE
    return SESSD_EINVAL;
}

extern "C" int sessd_sparse_to_dense(const float *d_feat, const int *d_coors, const int *d_n, int max_rows, int channels,
                                     sessd_grid grid, float *d_out, void *stream) {
    if (!d_feat || !d_coors || !d_n || !d_out || max_rows < 1 || channels < 1) return SESSD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t bytes = sizeof(float) * (size_t)grid.batch * grid.shape[0] * grid.shape[1] * grid.shape[2] * channels;
    SESSD_CUDA_TRY(cudaMemsetAsync(d_out, 0, bytes, st));
    SESSD_LAUNCH(dense_scatter_kernel, persistent_grid((long long)max_rows * channels, 256), 256, 0, st, d_feat, (const int4 *)d_coors,
                 d_n, max_rows, channels, grid.shape[0], grid.shape[1], grid.shape[2], d_out);
    return last_error();
}
