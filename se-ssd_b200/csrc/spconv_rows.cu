// spconv_rows.cu -- sparse 3-D convolution for the NARROW layers (Cin <= 32) of SpMiddleFHD with work proportional to the number of
// rulebook PAIRS (fp32 SIMT), + folded BN + ReLU.
//
// Why a second formulation: the output-stationary tensor-core kernels (spconv_tc.cu, spconv_h2.cu) move and multiply a full 128-row
// operand tile for every kernel offset, i.e. N_out x 27 row slots per layer whatever the neighbour fill.  On the first two levels of
// det3d/models/backbones/scn.py:106-131 the fill is low (SubM level 0: ~1 of 27 slots, the stride-2 SparseConv3d layers: 1-3 of 27,
// SubM level 1: ~6 of 27 on KITTI-like and on the dense synthetic clouds alike) and the channels are few (4..32), so > 75 % of that work
// is zeros and the layers are bound by operand movement, not by math.  Here a warp owns 4 output rows and touches ONLY their valid
// (row, offset) pairs:
//   * persistent CTAs of 32 warps; ALL kvol weight slices of the layer (7 .. 110 KB fp32) are loaded into shared memory once per CTA
//     and stay there: no per-offset staging, no block-wide synchronisation in the main loop;
//   * per tile of 128 output rows the neighbour table is staged in shared memory; lane k of a warp holds nbr[row][k], a ballot gives
//     the row's valid offsets, and the warp walks them in ascending k: the input row is one coalesced 16-128 byte segment (lane c
//     holds channel c; the first pair of each of the warp's 4 rows is requested up front, further pairs 4 at a time), acc[cout] += in[c] * W[k][c][cout] with the input value broadcast
//     by warp shuffle and the weights read as consecutive lanes = consecutive output channels (conflict-free);
//   * epilogue per row: folded BatchNorm1d scale / shift + ReLU, coalesced row store, running abs-max of the output (feeds the fp16
//     split of the next tensor-core layer).
// Same contract and results as sessd_spconv_forward (fp32 FMA accumulation; only the summation order over offsets is the same too:
// ascending k).  Algorithmic work: 2 P Cin Cout flops, 4 (P Cin + N_out Cout) + 4 kvol N_out bytes.
#include <cuda_fp16.h>

#include "common.cuh"

namespace sessd {

constexpr int kRwRows = 128;
constexpr int kRwWarps = 32;
constexpr int kRwThreads = kRwWarps * 32;
constexpr int kRwRpw = kRwRows / kRwWarps;          // rows per warp
constexpr int kRwMaxK = 27;
constexpr int kRwBatch = 4;                         // input rows in flight per warp beyond the prefetched first pair of each row

template <int CIN, int COUT>
struct RwCfg {
    static constexpr int kJ = (COUT + 31) / 32;                  // output channels per lane
    static constexpr int kWFloats = CIN * COUT;                  // per kernel offset
    static constexpr size_t smem(int kvol) { return (size_t)kvol * kWFloats * 4 + 2 * (size_t)kRwRows * kRwMaxK * 4 + 64; }   // weights + two neighbour tables
};

template <int CIN, int COUT>
__global__ void __launch_bounds__(kRwThreads, 1) spconv_rows_kernel(const float *__restrict__ in_feat, const int *__restrict__ nbr, int kvol,
                                                                    const int *__restrict__ d_n_out, int max_out,
                                                                    const float *__restrict__ weight, const float *__restrict__ scale,
                                                                    const float *__restrict__ shift, int relu, float *__restrict__ out_feat,
                                                                    float *__restrict__ amax_out, const float *__restrict__ amax_in, float gain,
                                                                    float shift_max, __half *__restrict__ out_planes, int cpo) {
    using C = RwCfg<CIN, COUT>;
    extern __shared__ __align__(16) unsigned char smem_raw[];
    float *s_w = reinterpret_cast<float *>(smem_raw);                              // [kvol][CIN][COUT], resident for the CTA's lifetime
    int *s_nbr = reinterpret_cast<int *>(s_w + (size_t)kvol * C::kWFloats);        // [2][128][kvol]

    const int n_out = min(*d_n_out, max_out);
    const int tiles = (n_out + kRwRows - 1) / kRwRows;
    if ((int)blockIdx.x >= tiles) return;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    // all weight slices of the layer (7 .. 110 KB): loaded once, every (row, offset) pair of every tile of this CTA reads them from here
    {
        const float4 *gw = reinterpret_cast<const float4 *>(weight);
        float4 *sw4 = reinterpret_cast<float4 *>(s_w);
        const int n4 = kvol * C::kWFloats / 4;
        for (int e = tid; e < n4; e += kRwThreads) sw4[e] = __ldg(gw + e);
    }
    float sc[C::kJ], sh[C::kJ];
#pragma unroll
    for (int j = 0; j < C::kJ; ++j) {
        const int co = lane + 32 * j;
        sc[j] = (scale && co < COUT) ? scale[co] : 1.f;
        sh[j] = (shift && co < COUT) ? shift[co] : 0.f;
    }
    float wmax = 0.f;
    // optional second output: the fp16 (hi, lo) planes [row][2][cpo] the tensor-core layers read, scaled by the power of two that maps
    // the bound |out| <= amax_in * gain + shift_max into [2^14, 2^15) (same rule as spconv_cg.cu / bevconv_p2.cu); amax_out[1] <- scale
    float s_out = 1.f;
    if (out_planes) {
        s_out = pow2_scale_for_bound(__ldg(amax_in) * gain + shift_max);
        if (blockIdx.x == 0 && tid == 0) amax_out[1] = s_out;
    }

    // the tile's neighbour table is contiguous in global memory; the NEXT tile's table is copied (cp.async) while this one is processed
    auto stage_nbr = [&](int t, int b) {
        const int r0 = t * kRwRows;
        const int nent = min(kRwRows, n_out - r0) * kvol;
        const uint32_t dst = (uint32_t)__cvta_generic_to_shared(s_nbr + b * (kRwRows * kRwMaxK));
        const int *src = nbr + (size_t)r0 * kvol;
        for (int e = tid; e < nent; e += kRwThreads)
            asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"(dst + 4u * (uint32_t)e), "l"(src + e) : "memory");
    };
    int buf = 0;
    stage_nbr(blockIdx.x, 0);
    for (int tile = blockIdx.x; tile < tiles; tile += gridDim.x, buf ^= 1) {
        const int row0 = tile * kRwRows;
        const int rows = min(kRwRows, n_out - row0);
        asm volatile("cp.async.wait_all;\n" ::: "memory");
        __syncthreads();                      // this tile's table landed; every warp is done with the other buffer (and s_w is written, first iteration)
        if (tile + (int)gridDim.x < tiles) stage_nbr(tile + (int)gridDim.x, buf ^ 1);
        const int *s_nbr_t = s_nbr + buf * (kRwRows * kRwMaxK);
        // each warp walks the valid (row, offset) pairs of its rows; no block-wide synchronisation inside.  The input row of the FIRST pair
        // of each of the warp's rows is requested up front (on these layers most rows have one to three pairs: with one row at a time the
        // warp sat through one L2 / HBM round trip per row)
        int mine[kRwRpw];                                                        // lane k holds nbr[row][k]
        unsigned int m[kRwRpw];
        float v0[kRwRpw];
#pragma unroll
        for (int r = 0; r < kRwRpw; ++r) {
            const int row = warp * kRwRpw + r;
            mine[r] = (row < rows && lane < kvol) ? s_nbr_t[row * kvol + lane] : -1;
            m[r] = __ballot_sync(0xffffffffu, mine[r] >= 0);
            v0[r] = 0.f;
            if (m[r]) {                                                          // warp-uniform
                const int src = __shfl_sync(0xffffffffu, mine[r], __ffs(m[r]) - 1);
                if (lane < CIN) v0[r] = __ldg(&in_feat[(size_t)src * CIN + lane]);
            }
        }
#pragma unroll
        for (int r = 0; r < kRwRpw; ++r) {
            const int row = warp * kRwRpw + r;
            if (row >= rows) break;                                              // warp-uniform
            float acc[C::kJ];
#pragma unroll
            for (int j = 0; j < C::kJ; ++j) acc[j] = 0.f;
            auto mac = [&](int k, float v) {                                     // acc[cout] += in[c] * W[k][c][cout], c ascending
                const float *sw = s_w + (size_t)k * C::kWFloats;
#pragma unroll
                for (int c = 0; c < CIN; ++c) {
                    const float a = __shfl_sync(0xffffffffu, v, c);
#pragma unroll
                    for (int j = 0; j < C::kJ; ++j) {
                        const int co = lane + 32 * j;
                        const float wv = sw[c * COUT + (COUT >= 32 ? co : (co & (COUT - 1)))];
                        acc[j] = fmaf(a, wv, acc[j]);
                    }
                }
            };
            unsigned int mr = m[r];
            if (mr) {
                mac(__ffs(mr) - 1, v0[r]);
                mr &= mr - 1;
            }
            // the row's remaining pairs, up to kRwBatch at a time: their input rows are requested back to back, then multiplied (ascending k)
            while (mr) {
                int ks[kRwBatch];
                float vs[kRwBatch];
#pragma unroll
                for (int i = 0; i < kRwBatch; ++i) {
                    ks[i] = -1;
                    vs[i] = 0.f;
                    if (mr) {                                                    // warp-uniform
                        const int k = __ffs(mr) - 1;
                        mr &= mr - 1;
                        ks[i] = k;
                        const int src = __shfl_sync(0xffffffffu, mine[r], k);
                        if (lane < CIN) vs[i] = __ldg(&in_feat[(size_t)src * CIN + lane]);
                    }
                }
#pragma unroll
                for (int i = 0; i < kRwBatch; ++i) {
                    if (ks[i] < 0) break;
                    mac(ks[i], vs[i]);
                }
            }
            // epilogue: folded BatchNorm1d (eval) + ReLU, one coalesced segment per row
#pragma unroll
            for (int j = 0; j < C::kJ; ++j) {
                const int co = lane + 32 * j;
                if (co < COUT) {
                    float o = fmaf(acc[j], sc[j], sh[j]);
                    if (relu) o = fmaxf(o, 0.f);
                    wmax = fmaxf(wmax, fabsf(o));
                    if (out_feat) out_feat[(size_t)(row0 + row) * COUT + co] = o;
                    if (out_planes) {
                        const float x = o * s_out;
                        const __half hi = __float2half_rn(x);
                        __half *dst = out_planes + (size_t)(row0 + row) * (2 * cpo) + co;
                        dst[0] = hi;
                        dst[cpo] = __float2half_rn(x - __half2float(hi));
                    }
                }
            }
        }
    }
    if (amax_out) {
        const unsigned mm = __reduce_max_sync(0xFFFFFFFFu, __float_as_uint(wmax));
        if (lane == 0 && mm != 0u) atomicMax(reinterpret_cast<unsigned *>(amax_out), mm);
    }
}

template <int CIN, int COUT>
static int launch_rows(const float *in, const int *nbr, int kvol, const int *d_n, int max_out, const float *w, const float *sc, const float *sh,
                       int relu, float *out, float *amax_out, const float *amax_in, float gain, float shift_max, void *out_planes, int cpo,
                       cudaStream_t st) {
    using C = RwCfg<CIN, COUT>;
    const size_t smem = C::smem(kvol);
    if (smem > 227 * 1024) return SESSD_ECAPACITY;
    static size_t attr_smem = 0;
    if (smem > attr_smem) {
        cudaError_t e = cudaFuncSetAttribute(spconv_rows_kernel<CIN, COUT>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) return (int)e;
        attr_smem = smem;
    }
    const int tiles = div_up(max_out, kRwRows);
    const int per_sm = smem <= 100 * 1024 ? 2 : 1;                         // 1024 threads per CTA: at most two resident CTAs
    const int grid = tiles < per_sm * kNumSMs ? tiles : per_sm * kNumSMs;  // persistent
    SESSD_LAUNCH((spconv_rows_kernel<CIN, COUT>), grid, kRwThreads, smem, st, in, nbr, kvol, d_n, max_out, w, sc, sh, relu, out, amax_out, amax_in,
                 gain, shift_max, (__half *)out_planes, cpo);
    return last_error();
}

}  // namespace sessd

using namespace sessd;

static int rows_dispatch(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out, int max_out, const float *d_weight,
                         int cout, const float *d_scale, const float *d_shift, int relu, float *d_out_feat, float *d_amax_out,
                         const float *d_amax_in, float gain, float shift_max, void *d_out_planes, int cpo, void *stream) {
    if (!d_in_feat || !d_nbr || !d_n_out || !d_weight || (!d_out_feat && !d_out_planes) || max_out < 1 || kvol < 1 || kvol > kRwMaxK)
        return SESSD_EINVAL;
    if (d_out_planes && (!d_amax_in || !d_amax_out || cpo < cout || (cpo != 32 && cpo != 64))) return SESSD_EINVAL;
    cudaStream_t st = (cudaStream_t)stream;
#define RW_CASE(CI, CO) \
    if (cin == CI && cout == CO) return launch_rows<CI, CO>(d_in_feat, d_nbr, kvol, d_n_out, max_out, d_weight, d_scale, d_shift, relu, d_out_feat, d_amax_out, d_amax_in, gain, shift_max, d_out_planes, cpo, st)
    RW_CASE(4, 16);
    RW_CASE(16, 16);
    RW_CASE(16, 32);
    RW_CASE(32, 16);     // data gradient of the 16 -> 32 strided layer
    RW_CASE(32, 32);
#undef RW_CASE
    return SESSD_EINVAL;
}

// Same arguments as sessd_spconv_forward plus d_amax_out (nullable): running abs-max of the output.  Supported (Cin, Cout): (4,16),
// (16,16), (16,32), (32,16), (32,32) -- the whole weight tensor must fit in shared memory.
extern "C" int sessd_spconv_forward_rows(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out, int max_out,
                                         const float *d_weight, int cout, const float *d_scale, const float *d_shift, int relu,
                                         float *d_out_feat, float *d_amax_out, void *stream) {
    if (!d_out_feat) return SESSD_EINVAL;
    return rows_dispatch(d_in_feat, cin, d_nbr, kvol, d_n_out, max_out, d_weight, cout, d_scale, d_shift, relu, d_out_feat, d_amax_out, nullptr,
                         0.f, 0.f, nullptr, 0, stream);
}

// ... and the output also (d_out_feat nullable: only) as fp16 (hi, lo) planes [row][2][cpo] for the tensor-core layers: d_out_info =
// {abs-max of the output (atomicMax; zero it once per frame), plane scale}; the scale comes from the bound *d_amax_in * gain + shift_max
// (d_amax_in = abs-max of the INPUT features, gain = max_n sum_{k,c} |w[k][c][n] bn_scale[n]|, shift_max = max_n |shift[n]|).
extern "C" int sessd_spconv_forward_rows_planes(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out, int max_out,
                                                const float *d_weight, int cout, const float *d_scale, const float *d_shift, int relu,
                                                const float *d_amax_in, float gain, float shift_max, float *d_out_feat, void *d_out_planes,
                                                int cpo, float *d_out_info, void *stream) {
    if (!d_out_planes) return SESSD_EINVAL;
    return rows_dispatch(d_in_feat, cin, d_nbr, kvol, d_n_out, max_out, d_weight, cout, d_scale, d_shift, relu, d_out_feat, d_out_info, d_amax_in,
                         gain, shift_max, d_out_planes, cpo, stream);
}
