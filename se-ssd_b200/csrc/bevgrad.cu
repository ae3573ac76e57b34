// bevgrad.cu -- weight gradient of the BEV neck and head convs (training of SSFA, det3d/models/necks/rpn_v1.py:135-210, and of the
// head's 1x1 convs, det3d/models/bbox_heads/mg_head_sessd.py:202-215).
//
// Tap-list form of the forward (sessd_conv_desc): out[b, y, x] = sum_t in[b, y s + dy_t, x s + dx_t] @ W[t]   (zero outside the input)
//   wgrad  gW[t][ci][co] = sum_{b, y, x} in[b, y s + dy_t, x s + dx_t, ci] g[b, y, x, co]   -- here;
//   dgrad  is the forward kernels (bevconv_p2.cu) with re-packed weights, no kernel of its own (sessd_b200/bev_grad.py).
// The deconv (k3, s2, p1, op1) has no mode of its own: its weight gradient is the stride-2 conv's with the roles swapped (input = the
// deconv's output gradient, gradient = the deconv's input), transposed on the host.
//
// A per-tap GEMM [Cin x P] [P x Cout] whose K dimension is the P = batch * out_h * out_w output pixels.  A work ITEM is (tap, 128-channel
// block of Cin, NC-channel block of Cout, fixed range of pixel rounds); the decomposition depends on the descriptor only (bg_chunks), every
// item writes its fp32 partial [128][NC] to the workspace, and a reduce sums the partials of a tile in ascending item order: bitwise
// run-to-run deterministic without a float atomic, the contract of sessd_spconv_wgrad_*.
// The item runs on the tensor cores (wgrad_mma.cuh) with the output pixels as the K rows: a round is kWgKC consecutive pixels.  The
// shifted input pixel of a tap that falls outside the map, and the slots past the item's last pixel, are zero-filled by the copy itself
// (the padding taps).  The reduce divides by S_in S_g (exact: powers of two).
#include <cuda_fp16.h>

#include "wgrad_mma.cuh"

namespace sessd {

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
    const long long rounds = (g.pixels + kWgKC - 1) / kWgKC;
    // at most kBgItemsTarget items (four waves of one CTA per SM): a fifth, nearly empty wave would cost a fifth of the launch
    long long c = kBgItemsTarget / g.groups;
    if (c < 1) c = 1;
    if (c > rounds) c = rounds;
    g.rpc = div_up(rounds, c);
    g.chunks = div_up(rounds, g.rpc);
    return 0;
}

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
__global__ void __launch_bounds__(kWgThreads, 1) bev_wgrad_kernel(const __grid_constant__ BgArgs a) {
    extern __shared__ __align__(16) unsigned char bg_smem[];
    const WgLayout<kBgM, NC> L{(uint32_t)__cvta_generic_to_shared(bg_smem)};
    const int item = blockIdx.x, grp = item / a.chunks, ch = item - grp * a.chunks;
    const int nb = grp % a.nblocks, mb = (grp / a.nblocks) % a.mblocks, tap = grp / (a.nblocks * a.mblocks);
    const int dy = a.tap_dy[tap], dx = a.tap_dx[tap];
    const long long q_begin = (long long)ch * a.rpc * kWgKC;
    const long long q_end = min(a.pixels, q_begin + (long long)a.rpc * kWgKC);
    const int hw = a.out_h * a.out_w;
    const int tid = threadIdx.x;

    // copy the round of pixels [q0, q0 + kWgKC) into buffer b; pixels >= q_end and shifted input pixels outside the map read as zero
    auto stage = [&](long long q0, int b) {
        constexpr int kAChunks = 2 * kBgM / 8, kGChunks = 2 * NC / 8;
        for (int e = tid; e < kWgKC * (kAChunks + kGChunks); e += kWgThreads) {
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
                wg_cp_async16(L.a(b, h, p, c0 - mb * kBgM), a.x + h * a.x_plane + off, valid);
            } else {
                const int rr = r - kAChunks, h = rr / (NC / 8), c0 = (rr % (NC / 8)) * 8;
                const size_t off = valid ? (size_t)q * a.cout + nb * NC + c0 : 0;
                wg_cp_async16(L.g(b, h, p, c0), a.g + h * a.g_plane + off, valid);
            }
        }
    };
    wgrad_mma_item<kBgM, NC, long long>(
        L, [&](long long &q0) { q0 = q_begin; }, [&](long long q0) { return q0 < q_end; }, [&](long long &q0) { q0 += kWgKC; },
        [&](long long q0) { return min((long long)kWgKC, q_end - q0); }, stage, a.partial);
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
    if ((long long)d.cin * d.cout > (1 << 30)) return SESSD_EINVAL;                     // the reduce indexes a tap's [cin][cout] in int
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
    const int rc = g.nc == 128 ? wgrad_launch<bev_wgrad_kernel<128>, kBgM, 128>(items, st, a)
                               : wgrad_launch<bev_wgrad_kernel<64>, kBgM, 64>(items, st, a);
    return rc ? rc : wgrad_reduce((const float *)d_ws, d.ntaps, d.cin, d.cout, kBgM, g.nc, g.chunks, d_in_info, d_g_info, d_gw, st);
}
