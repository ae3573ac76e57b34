// bevgrad.cu -- weight gradient of the BEV neck and head convs (training of SSFA, det3d/models/necks/rpn_v1.py:135-210, and of the
// head's 1x1 convs, det3d/models/bbox_heads/mg_head_sessd.py:202-215).
//
// Tap-list form of the forward (sessd_bev_conv): out[b, y, x] = sum_t in[b, y s + dy_t, x s + dx_t] @ W[t]   (zero outside the input)
//   wgrad  gW[t][ci][co] = sum_{b, y, x} in[b, y s + dy_t, x s + dx_t, ci] g[b, y, x, co]   -- here;
//   dgrad  is the forward kernels (bevconv_p2.cu) with re-packed weights, no kernel of its own (sessd_b200/bev_grad.py).
// The deconv (k3, s2, p1, op1) has no mode of its own: its weight gradient is the stride-2 conv's with the roles swapped (input = the
// deconv's output gradient, gradient = the deconv's input), transposed on the host.
//
// A per-tap GEMM [Cin x P] [P x Cout] whose K dimension is the P = batch * out_h * out_w output pixels.  A work ITEM is (tap, 128-channel
// block of Cin, NC-channel block of Cout, fixed range of pixel rounds); the decomposition depends on the descriptor only (bg_chunks), every
// item writes its fp32 partial [128][NC] to the workspace, and a reduce sums the partials of a tile in ascending item order: bitwise
// run-to-run deterministic without a float atomic, the contract of sessd_spconv_wgrad_*.
// A round stages kBgKC consecutive output pixels PIXEL-MAJOR, as the planes lie in global memory: [hi | lo][pixel][channel], 16-byte
// cp.async per 8 channels, double-buffered.  The shifted input pixel of a tap that falls outside the map, and the slots past the item's
// last pixel, are zero-filled by the copy itself (the padding taps).  ldmatrix.trans feeds mma.sync.m16n8k16 (both operands are
// K-major, K = pixels) with the forward's three-product fp16 split: a_hi g_hi into the main accumulator, a_hi g_lo + a_lo g_hi into the
// cross accumulator, summed RN once per item; the reduce divides by S_in S_g (exact: powers of two).
#include <cuda_fp16.h>

#include "tc_common.cuh"

namespace sessd {

constexpr int kBgThreads = 256;
constexpr int kBgKC = 64;                    // pixels staged per round
constexpr int kBgM = 128;                    // Cin channels per item (eight warps x one m16 slab)
constexpr int kBgItemsTarget = 4 * kNumSMs;  // most items per launch: four waves at one CTA per SM

// item geometry of one launch; a function of the descriptor only: the summation order of the result never depends on the data
struct BgGeom {
    int nc;                  // Cout channels per item: 128, or 64 for a 64-channel gradient (the head's, zero-padded)
    int mblocks, nblocks;    // 128-channel blocks of Cin, nc-channel blocks of Cout
    int groups;              // ntaps * mblocks * nblocks result tiles
    int chunks, rpc;         // items per tile, pixel rounds per item
    long long pixels;        // batch * out_h * out_w
};

static int bg_geometry(const sessd_conv_desc &d, BgGeom &g) {
    if (d.batch < 1 || d.in_h < 1 || d.in_w < 1 || d.out_h < 1 || d.out_w < 1) return SESSD_EINVAL;
    if (d.ntaps < 1 || d.ntaps > 9 || (d.in_stride != 1 && d.in_stride != 2)) return SESSD_EINVAL;
    if (d.out_stride != 1 || d.out_off_y != 0 || d.out_off_x != 0 || d.grid_h != d.out_h || d.grid_w != d.out_w) return SESSD_EINVAL;
    if (d.cin < kBgM || d.cin % kBgM) return SESSD_EINVAL;
    if (d.cout % 128 == 0 && d.cout >= 128) g.nc = 128;
    else if (d.cout == 64) g.nc = 64;
    else return SESSD_EINVAL;
    g.mblocks = d.cin / kBgM;
    g.nblocks = d.cout / g.nc;
    g.groups = d.ntaps * g.mblocks * g.nblocks;
    g.pixels = (long long)d.batch * d.out_h * d.out_w;
    const long long rounds = (g.pixels + kBgKC - 1) / kBgKC;
    // at most kBgItemsTarget items (four waves of one CTA per SM): a fifth, nearly empty wave would cost a fifth of the launch
    long long c = kBgItemsTarget / g.groups;
    if (c < 1) c = 1;
    if (c > rounds) c = rounds;
    g.rpc = div_up(rounds, c);
    g.chunks = div_up(rounds, g.rpc);
    return 0;
}

template <int NC>
struct BgCfg {
    static constexpr int kPitchA = kBgM + 8, kPitchG = NC + 8;             // halves: the eight rows of an ldmatrix phase hit eight bank groups
    static constexpr int kBufHalves = 2 * kBgKC * (kPitchA + kPitchG);      // one buffer: A hi, A lo, G hi, G lo
    static constexpr int kSmem = 2 * kBufHalves * 2;                        // bytes, two buffers
    static constexpr int kNT = NC / 8;                                      // n8 tiles per warp (a warp owns one m16 slab x all NC)
    static_assert(kNT % 2 == 0, "B fragments are loaded two n8 tiles at a time");
};

struct BgArgs {
    const __half *x;         // input planes [2][batch][in_h][in_w][cin]
    const __half *g;         // gradient planes [2][batch][out_h][out_w][cout]
    long long x_plane, g_plane;                      // halves per plane
    int in_h, in_w, cin, out_h, out_w, cout, stride;
    int tap_dy[9], tap_dx[9];
    int mblocks, nblocks, chunks, rpc;
    long long pixels;
    float *partial;
};

template <int NC>
__global__ void __launch_bounds__(kBgThreads, 1) bev_wgrad_kernel(const __grid_constant__ BgArgs a) {
    using C = BgCfg<NC>;
    extern __shared__ __align__(16) unsigned char bg_smem[];
    const uint32_t s0 = (uint32_t)__cvta_generic_to_shared(bg_smem);
    auto a_addr = [&](int b, int h, int p, int c) { return s0 + 2u * (uint32_t)(b * C::kBufHalves + (h * kBgKC + p) * C::kPitchA + c); };
    auto g_addr = [&](int b, int h, int p, int c) {
        return s0 + 2u * (uint32_t)(b * C::kBufHalves + 2 * kBgKC * C::kPitchA + (h * kBgKC + p) * C::kPitchG + c);
    };
    const int item = blockIdx.x, grp = item / a.chunks, ch = item - grp * a.chunks;
    const int nb = grp % a.nblocks, mb = (grp / a.nblocks) % a.mblocks, tap = grp / (a.nblocks * a.mblocks);
    const int dy = a.tap_dy[tap], dx = a.tap_dx[tap];
    const long long q_begin = (long long)ch * a.rpc * kBgKC;
    const long long q_end = min(a.pixels, q_begin + (long long)a.rpc * kBgKC);
    const int hw = a.out_h * a.out_w;
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int gq = lane >> 2, tq = lane & 3;
    const int lr = lane & 7, lm = lane >> 3;                           // ldmatrix: row within an 8x8 matrix, matrix index
    const int m0 = warp * 16;
    float acc_m[C::kNT][4], acc_c[C::kNT][4];
#pragma unroll
    for (int j = 0; j < C::kNT; ++j)
#pragma unroll
        for (int q = 0; q < 4; ++q) { acc_m[j][q] = 0.f; acc_c[j][q] = 0.f; }

    // copy the round of pixels [q0, q0 + kBgKC) into buffer b; pixels >= q_end and shifted input pixels outside the map read as zero
    auto stage = [&](long long q0, int b) {
        constexpr int kAChunks = 2 * kBgM / 8, kGChunks = 2 * NC / 8;
        for (int e = tid; e < kBgKC * (kAChunks + kGChunks); e += kBgThreads) {
            const int p = e / (kAChunks + kGChunks), r = e - p * (kAChunks + kGChunks);
            const long long q = q0 + p;
            bool valid = q < q_end;
            const int bi = valid ? (int)(q / hw) : 0, rem = valid ? (int)(q - (long long)bi * hw) : 0;
            const int y = rem / a.out_w, x = rem - y * a.out_w;
            if (r < kAChunks) {
                const int h = r / (kBgM / 8), c0 = mb * kBgM + (r % (kBgM / 8)) * 8;
                const int iy = y * a.stride + dy, ix = x * a.stride + dx;
                valid = valid && iy >= 0 && iy < a.in_h && ix >= 0 && ix < a.in_w;
                const size_t off = valid ? (((size_t)bi * a.in_h + iy) * a.in_w + ix) * a.cin + c0 : 0;
                wg_cp_async16(a_addr(b, h, p, c0 - mb * kBgM), a.x + h * a.x_plane + off, valid);
            } else {
                const int rr = r - kAChunks, h = rr / (NC / 8), c0 = (rr % (NC / 8)) * 8;
                const size_t off = valid ? (size_t)q * a.cout + nb * NC + c0 : 0;
                wg_cp_async16(g_addr(b, h, p, c0), a.g + h * a.g_plane + off, valid);
            }
        }
    };

    long long q0 = q_begin;
    if (q0 < q_end) stage(q0, 0);
    asm volatile("cp.async.commit_group;\n" ::: "memory");
    int buf = 0;
    while (q0 < q_end) {                                               // block-uniform
        const long long qn = q0 + kBgKC;
        if (qn < q_end) stage(qn, buf ^ 1);
        asm volatile("cp.async.commit_group;\n" ::: "memory");
        asm volatile("cp.async.wait_group 1;\n" ::: "memory");          // this round's copies (the next round's stay in flight)
        __syncthreads();
        const int steps = (int)((min((long long)kBgKC, q_end - q0) + 15) >> 4);
        for (int s = 0; s < steps; ++s) {
            const int k0 = s * 16;
            // A fragments: matrix lm covers pixels k0 + 8 (lm >> 1) .., channels m0 + 8 (lm & 1) ..  ->  a0..a3 of m16n8k16
            uint32_t ah[4], al[4];
            ldsm_x4_trans(ah, a_addr(buf, 0, k0 + lr + 8 * (lm >> 1), m0 + 8 * (lm & 1)));
            ldsm_x4_trans(al, a_addr(buf, 1, k0 + lr + 8 * (lm >> 1), m0 + 8 * (lm & 1)));
#pragma unroll
            for (int j = 0; j < C::kNT; j += 2) {
                // B fragments: matrix lm covers pixels k0 + 8 (lm & 1) .., channels 8 (j + (lm >> 1)) ..  ->  (b0, b1) of tiles j, j + 1
                uint32_t bh[4], bl[4];
                const int gp = k0 + lr + 8 * (lm & 1), gc = 8 * j + 8 * (lm >> 1);
                ldsm_x4_trans(bh, g_addr(buf, 0, gp, gc));
                ldsm_x4_trans(bl, g_addr(buf, 1, gp, gc));
#pragma unroll
                for (int u = 0; u < 2; ++u) {
                    mma_f16_16816(acc_m[j + u], ah, bh[2 * u], bh[2 * u + 1]);     // main  += a_hi g_hi
                    mma_f16_16816(acc_c[j + u], ah, bl[2 * u], bl[2 * u + 1]);     // cross += a_hi g_lo
                    mma_f16_16816(acc_c[j + u], al, bh[2 * u], bh[2 * u + 1]);     // cross += a_lo g_hi
                }
            }
        }
        __syncthreads();                                                // buffer `buf` is free for the round after next
        q0 = qn;
        buf ^= 1;
    }
    asm volatile("cp.async.wait_group 0;\n" ::: "memory");
    // partial[item][c][n] = acc_m + acc_c (RN); this thread holds rows m0 + gq (+8), columns 2 tq (+1) of every n8 tile
    float *dst = a.partial + (size_t)item * (kBgM * NC);
#pragma unroll
    for (int j = 0; j < C::kNT; ++j) {
        const int n = 8 * j + 2 * tq;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int m = m0 + gq + 8 * h;
            *reinterpret_cast<float2 *>(dst + (size_t)m * NC + n) =
                make_float2(acc_m[j][2 * h] + acc_c[j][2 * h], acc_m[j][2 * h + 1] + acc_c[j][2 * h + 1]);
        }
    }
}

// gW[t][ci][co] = (sum over the chunks of its tile, ascending, of partial[tile chunks + c][ci % 128][co % nc]) / S_in / S_g
__global__ void __launch_bounds__(256) bev_wgrad_reduce_kernel(const float *__restrict__ partial, int ntaps, int cin, int cout, int nc,
                                                               int chunks, const float *__restrict__ in_info, const float *__restrict__ g_info,
                                                               float *__restrict__ gw) {
    const float inv = 1.f / __ldg(in_info + 1) / __ldg(g_info + 1);    // exact: powers of two
    const int per_tile = kBgM * nc, mblocks = cin / kBgM, nblocks = cout / nc;
    const long long total = (long long)ntaps * cin * cout;
    for (long long e = (long long)blockIdx.x * blockDim.x + threadIdx.x; e < total; e += (long long)gridDim.x * blockDim.x) {
        const int t = (int)(e / ((long long)cin * cout)), r = (int)(e - (long long)t * cin * cout);
        const int ci = r / cout, co = r - ci * cout;
        const int grp = (t * mblocks + ci / kBgM) * nblocks + co / nc;
        const float *p = partial + (size_t)grp * chunks * per_tile + (ci % kBgM) * nc + co % nc;
        float s = 0.f;
        for (int c = 0; c < chunks; ++c) s += __ldg(p + (size_t)c * per_tile);
        gw[e] = s * inv;
    }
}

template <int NC>
static int launch_bev_wgrad(const BgArgs &a, int items, cudaStream_t st) {
    constexpr int kSmem = BgCfg<NC>::kSmem;
    static bool attr_done = false;
    if (!attr_done) {
        cudaError_t e = cudaFuncSetAttribute(bev_wgrad_kernel<NC>, cudaFuncAttributeMaxDynamicSharedMemorySize, kSmem);
        if (e != cudaSuccess) return (int)e;
        attr_done = true;
    }
    SESSD_LAUNCH(bev_wgrad_kernel<NC>, items, kBgThreads, kSmem, st, a);
    return last_error();
}

}  // namespace sessd

using namespace sessd;

extern "C" int sessd_bev_wgrad_items(const sessd_conv_desc *desc) {
    BgGeom g;
    if (!desc || bg_geometry(*desc, g)) return SESSD_EINVAL;
    return g.groups * g.chunks;
}

extern "C" size_t sessd_bev_wgrad_workspace_bytes(const sessd_conv_desc *desc) {
    BgGeom g;
    if (!desc || bg_geometry(*desc, g)) return 0;
    return sizeof(float) * (size_t)g.groups * g.chunks * kBgM * g.nc;
}

extern "C" int sessd_bev_wgrad(const void *d_in_planes, const float *d_in_info, const void *d_g_planes, const float *d_g_info,
                               const sessd_conv_desc *desc, float *d_gw, void *d_ws, size_t ws_bytes, void *stream) {
    if (!d_in_planes || !d_in_info || !d_g_planes || !d_g_info || !desc || !d_gw || !d_ws) return SESSD_EINVAL;
    if (((uintptr_t)d_in_planes | (uintptr_t)d_g_planes) & 15) return SESSD_EINVAL;     // 16-byte copies
    const sessd_conv_desc &d = *desc;
    BgGeom g;
    if (bg_geometry(d, g)) return SESSD_EINVAL;
    if (ws_bytes < sessd_bev_wgrad_workspace_bytes(desc)) return SESSD_EWORKSPACE;
    BgArgs a;
    a.x = (const __half *)d_in_planes;
    a.g = (const __half *)d_g_planes;
    a.x_plane = (long long)d.batch * d.in_h * d.in_w * d.cin;
    a.g_plane = g.pixels * d.cout;
    a.in_h = d.in_h; a.in_w = d.in_w; a.cin = d.cin; a.out_h = d.out_h; a.out_w = d.out_w; a.cout = d.cout; a.stride = d.in_stride;
    for (int t = 0; t < 9; ++t) {
        a.tap_dy[t] = t < d.ntaps ? d.tap_dy[t] : 0;
        a.tap_dx[t] = t < d.ntaps ? d.tap_dx[t] : 0;
    }
    a.mblocks = g.mblocks; a.nblocks = g.nblocks; a.chunks = g.chunks; a.rpc = g.rpc; a.pixels = g.pixels;
    a.partial = (float *)d_ws;
    cudaStream_t st = (cudaStream_t)stream;
    const int items = g.groups * g.chunks;
    const int rc = g.nc == 128 ? launch_bev_wgrad<128>(a, items, st) : launch_bev_wgrad<64>(a, items, st);
    if (rc) return rc;
    SESSD_LAUNCH(bev_wgrad_reduce_kernel, persistent_grid((long long)d.ntaps * d.cin * d.cout, 256), 256, 0, st, (const float *)d_ws, d.ntaps,
                 d.cin, d.cout, g.nc, g.chunks, d_in_info, d_g_info, d_gw);
    return last_error();
}
