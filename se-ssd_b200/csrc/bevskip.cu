// bevskip.cu -- constant-region skipping for the SSFA neck + head (runners.SSFAPlanesRunner) on the bevconv_p2 kernel.
//
// dense() writes exact zeros wherever the last sparse level has no site.  Over a receptive field that lies entirely in that empty space
// and inside the map (zero padding makes the border differ), a conv sees the same operands, in the same order, at every output pixel of
// one parity class, so the kernel's result there is one value per class, bit for bit; the layers after it inherit this.  The neck's maps
// have period 1 (conv chains from the empty input) or 2 (the deconv's output-parity classes and what follows them).
//
// sessd_bev_skip_plan (one launch of one CTA per batch) marks, per frame, every pixel of every neck output that may differ from its class
// constant ("non-constant": an active BEV site, an out-of-map tap, a non-constant tap or residual) as bit maps in shared memory.  Then,
// per neck launch:
//   * every work-item tile that holds a non-constant pixel or leaves the map (partial tiles always run) is flagged;
//   * the first all-constant tile of each class is its representative: it runs like any other item, so its abs-max enters out_info;
//   * the work items to run are compacted in the launcher's own item order (class by descending tap count, n-block, tile);
//   * the skipped (class, tile) pairs are listed.
// sessd_bev_skip_fill copies, after the launch, the representative's pixel at the same tile position into every skipped pixel.  Tile
// origins are multiples of 8 (u) and 16 (v) along the class grid, so that pixel has the same parity.
//
// Most pixels of the tiles that run are constant too, so the stride-1 launches (the register-A path of bev_conv_p2, which addresses
// A per 8-row matrix) run segments instead: 8 pixels along u in one v row.  The plan kernel copies every frame's bit maps into the
// segment buffer (a separate record per launch, next to the tile record, which stays as it is); bev_skip_seg_kernel then, one CTA per
// launch so that the work runs in parallel rather than on the plan kernel's single CTA:
//   * flags every segment that holds a non-constant pixel or leaves the map;
//   * picks two representatives per class, the first all-constant segment of each v parity (a segment starts at a multiple of 8 along u,
//     but at any v, and the maps after the deconvs have period 2);
//   * packs the live segments and the representatives 16 to a group, per class in the launcher's heavy-first order, by ascending segment
//     index (a class's last group is padded with -1);
//   * lists the skipped (class, segment) pairs, which sessd_bev_skip_fill_segs fills from the representative of their v parity.
#include "bevconv_p2.cuh"

namespace sessd {

// record header (int32 words; the item list starts at kP2ItemsHeader, where bev_conv_p2_kernel reads it)
enum {
    kRecCount = 0, kRecSkipped = 1, kRecNclass = 2, kRecTiles = 3, kRecTilesU = 4, kRecTilesV = 5, kRecUisX = 6, kRecOutStride = 7,
    kRecOutH = 8, kRecOutW = 9, kRecBatch = 10, kRecOffY = 11, kRecOffX = 15, kRecRep = 19, kRecSkipOff = 23, kRecFlagOff = 24
};
// segment record header (int32 words; the groups start at kP2SegHeader, where bev_conv_p2_kernel reads them, then the skipped
// (class * segments + segment) entries and the per-(class, segment) flags); representatives at kSegRep + 2 class + v parity
enum {
    kSegCount = 0, kSegSkipped = 1, kSegGroups = 2, kSegNclass = 3, kSegPerClass = 4, kSegTilesU = 5, kSegGridV = 6, kSegUisX = 7,
    kSegOutStride = 8, kSegOutH = 9, kSegOutW = 10, kSegBatch = 11, kSegOffY = 12, kSegOffX = 16, kSegRep = 20, kSegSkipOff = 28,
    kSegFlagOff = 29
};

// bit maps of the plan kernel: the neck input, every layer output (t0 = x0 and t1 = x1 pixel for pixel: 1x1 convs) and two scratch maps
enum { kMX, kMB0a, kMB0b, kMX0, kMM0, kMM1, kMO0, kMO1, kMOut, kMTmp, kMB1a, kMB1b, kMX1, kMTmpH, kNumMaps };
constexpr int kNumFullMaps = kMTmp + 1;
constexpr int kSkipLaunches = 13;
constexpr int kSkipThreads = 1024;

struct SkipLaunch : P2Geometry {             // the launcher's work items (p2_geometry)
    int map;                                   // bit map of the launch's output
    int out_stride, out_h, out_w;
    int rec;                                   // word offset of the launch record
    int seg;                                   // word offset of the segment record, -1: tiles only (the stride-2 conv)
    int nseg, max_groups;                      // segments per class (batch * grid_v * tiles_u), groups of a record at most
};

struct SkipPlan {
    int batch, depth, h, w, h2, w2, nwf, nwh;  // nwf / nwh: 32-bit words per row of a full / half resolution map
    long long seg_words;                       // int32 words of the segment records and, from map_off, of every frame's bit maps
    long long map_off;
    int frame_words;                           // words of one frame's bit maps (the plan kernel's shared memory, same layout)
    SkipLaunch l[kSkipLaunches];
};

// one launch of the plan, with the launcher's geometry at the weight width the runner packs (round_up(cout, n_tile))
static int skip_launch(SkipLaunch &L, int map, int batch, int grid_h, int grid_w, int out_h, int out_w, int cout, bool deconv) {
    P2Taps cls[4] = {};
    if (deconv) p2_deconv_classes(cls);
    else cls[0].n = 1;                         // a conv is one class: its taps do not enter the item order
    L.map = map;
    L.out_stride = deconv ? 2 : 1;
    L.out_h = out_h; L.out_w = out_w;
    return p2_geometry(L, batch, grid_h, grid_w, cout, div_up(cout, p2_n_tile(cout)) * p2_n_tile(cout), cls, deconv ? 4 : 1);
}

// the SSFAPlanesRunner launch sequence (runners.SSFAPlanesRunner.SKIP_LAUNCHES); returns the plan's int32 words, or 0
static long long skip_plan(SkipPlan &P, int batch, int h, int w) {
    if (batch < 1 || h < 4 || w < 4 || (h & 1) || (w & 1)) return 0;
    P.batch = batch; P.h = h; P.w = w; P.h2 = h / 2; P.w2 = w / 2;
    P.nwf = div_up(w, 32); P.nwh = div_up(P.w2, 32);
    const int h2 = P.h2, w2 = P.w2;
    SkipLaunch *L = P.l;
    const int rc = skip_launch(L[0], kMB0a, batch, h, w, h, w, 128, false)     // bottom_up_block_0.1
                 | skip_launch(L[1], kMB0b, batch, h, w, h, w, 128, false)     // bottom_up_block_0.4
                 | skip_launch(L[2], kMX0, batch, h, w, h, w, 128, false)      // bottom_up_block_0.7
                 | skip_launch(L[3], kMB1a, batch, h2, w2, h2, w2, 256, false) // bottom_up_block_1.0 (stride 2)
                 | skip_launch(L[4], kMB1b, batch, h2, w2, h2, w2, 256, false) // bottom_up_block_1.3
                 | skip_launch(L[5], kMX1, batch, h2, w2, h2, w2, 256, false)  // bottom_up_block_1.6
                 | skip_launch(L[6], kMX0, batch, h, w, h, w, 128, false)      // trans_0.0 (1x1)
                 | skip_launch(L[7], kMX1, batch, h2, w2, h2, w2, 256, false)  // trans_1.0 (1x1)
                 | skip_launch(L[8], kMM0, batch, h2, w2, h, w, 128, true)     // deconv_block_0.0 (+ t0)
                 | skip_launch(L[9], kMM1, batch, h2, w2, h, w, 128, true)     // deconv_block_1.0
                 | skip_launch(L[10], kMO0, batch, h, w, h, w, 128, false)     // conv_0.0
                 | skip_launch(L[11], kMO1, batch, h, w, h, w, 128, false)     // conv_1.0
                 | skip_launch(L[12], kMOut, batch, h, w, h, w, 24, false);    // head (1x1 on the fused map)
    long long words = 0;
    P.seg_words = 0;
    for (int i = 0; i < kSkipLaunches; ++i) {
        L[i].rec = (int)words;
        words += kP2ItemsHeader + L[i].total + 2LL * L[i].nclass * L[i].tiles;
        L[i].nseg = batch * L[i].grid_v * L[i].tiles_u;
        L[i].max_groups = L[i].nclass * div_up(L[i].nseg, kP2SegSlots);
        L[i].seg = i == 3 ? -1 : (int)P.seg_words;
        if (L[i].seg >= 0) P.seg_words += kP2SegHeader + (long long)kP2SegSlots * L[i].max_groups + 2LL * L[i].nclass * L[i].nseg;
    }
    P.frame_words = kNumFullMaps * h * P.nwf + (kNumMaps - kNumFullMaps) * P.h2 * P.nwh;
    P.map_off = P.seg_words;
    P.seg_words += (long long)batch * P.frame_words;
    if (P.seg_words >= (1LL << 31) || L[0].nseg >= (1 << 24)) return 0;
    return rc ? 0 : words;
}

struct BitMap {
    uint32_t *w;
    int h, wd, nw;
    __device__ __forceinline__ bool get(int y, int x) const { return (w[y * nw + (x >> 5)] >> (x & 31)) & 1u; }
    __device__ __forceinline__ uint32_t valid(int i) const {
        const int rem = wd - 32 * i;
        return rem >= 32 ? ~0u : ((1u << rem) - 1u);
    }
};

// out = the non-constant pixels of a 3x3 / pad 1 conv of `in` (out-of-map taps count as non-constant); out may alias in
__device__ void skip_dilate3(const BitMap &in, const BitMap &tmp, const BitMap &out) {
    const int n = in.h * in.nw, last = (in.wd - 1) >> 5;
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int y = idx / in.nw, i = idx - y * in.nw;
        const uint32_t *r = in.w + y * in.nw;
        const uint32_t c = r[i], l = i > 0 ? r[i - 1] : 0u, rr = i + 1 < in.nw ? r[i + 1] : 0u;
        uint32_t hv = c | (c << 1) | (l >> 31) | (c >> 1) | (rr << 31);
        if (i == 0) hv |= 1u;
        if (i == last) hv |= 1u << ((in.wd - 1) & 31);
        tmp.w[idx] = hv & in.valid(i);
    }
    __syncthreads();
    for (int idx = threadIdx.x; idx < n; idx += blockDim.x) {
        const int y = idx / in.nw, i = idx - y * in.nw;
        out.w[idx] = (y == 0 || y == in.h - 1) ? in.valid(i) : (tmp.w[idx - in.nw] | tmp.w[idx] | tmp.w[idx + in.nw]);
    }
    __syncthreads();
}

// out(y, x) = f(y, x), one warp per 32-pixel word
template <class F>
__device__ void skip_map_from(const BitMap &out, F f) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    for (int idx = warp; idx < out.h * out.nw; idx += nwarps) {
        const int y = idx / out.nw, x = (idx - y * out.nw) * 32 + lane;
        const unsigned bits = __ballot_sync(0xFFFFFFFFu, x < out.wd && f(y, x));
        if (lane == 0) out.w[idx] = bits;
    }
    __syncthreads();
}

// n predicates -> the indices i with pred(i) at out[0..count), in ascending order; returns count (every thread)
template <class Pred>
__device__ int skip_compact(int n, Pred pred, int *out, int *s_scan) {
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nwarps = blockDim.x >> 5;
    int base = 0;
    for (int start = 0; start < n; start += blockDim.x) {
        const int i = start + threadIdx.x;
        const bool v = i < n && pred(i);
        const unsigned bal = __ballot_sync(0xFFFFFFFFu, v);
        if (lane == 0) s_scan[warp] = __popc(bal);
        __syncthreads();
        if (warp == 0) {
            const int own = lane < nwarps ? s_scan[lane] : 0;
            int x = own;
#pragma unroll
            for (int o = 1; o < 32; o <<= 1) {
                const int y = __shfl_up_sync(0xFFFFFFFFu, x, o);
                if (lane >= o) x += y;
            }
            if (lane < nwarps) s_scan[lane] = x - own;
            if (lane == 31) s_scan[32] = x;
        }
        __syncthreads();
        if (v) out[base + s_scan[warp] + __popc(bal & ((1u << lane) - 1u))] = i;
        base += s_scan[32];
        __syncthreads();
    }
    return base;
}

__global__ void __launch_bounds__(kSkipThreads) bev_skip_plan_kernel(const uint2 *__restrict__ bitmap, int *__restrict__ plan,
                                                                    int *__restrict__ segs, SkipPlan P) {
    extern __shared__ uint32_t s_bits[];
    __shared__ int s_scan[33], s_rep[4];
    BitMap m[kNumMaps];
    {
        uint32_t *p = s_bits;
        for (int i = 0; i < kNumMaps; ++i) {
            const bool full = i < kNumFullMaps;
            m[i].w = p; m[i].h = full ? P.h : P.h2; m[i].wd = full ? P.w : P.w2; m[i].nw = full ? P.nwf : P.nwh;
            p += m[i].h * m[i].nw;
        }
    }
    for (int b = 0; b < P.batch; ++b) {
        // the neck input: a BEV cell is non-constant when any of its z slices holds a site of the last sparse level
        // (one thread per 32-pixel word: the bits of a row segment are one funnel shift of two bitmap words per slice, all loads independent)
        const BitMap X = m[kMX];
        for (int idx = threadIdx.x; idx < X.h * X.nw; idx += blockDim.x) {
            const int y = idx / X.nw, i = idx - y * X.nw;
            const int nbits = min(32, X.wd - 32 * i);
            uint32_t acc = 0u;
            for (int z = 0; z < P.depth; ++z) {
                const unsigned long long lin = (((unsigned long long)b * P.depth + z) * P.h + y) * P.w + 32 * i;
                const unsigned sh = (unsigned)(lin & 31);
                const uint32_t lo = __ldg(&bitmap[lin >> 5]).x, hi = sh + nbits > 32 ? __ldg(&bitmap[(lin >> 5) + 1]).x : 0u;
                acc |= __funnelshift_r(lo, hi, sh);
            }
            X.w[idx] = acc & X.valid(i);
        }
        __syncthreads();
        skip_dilate3(m[kMX], m[kMTmp], m[kMB0a]);
        skip_dilate3(m[kMB0a], m[kMTmp], m[kMB0b]);
        skip_dilate3(m[kMB0b], m[kMTmp], m[kMX0]);
        skip_dilate3(m[kMX0], m[kMTmp], m[kMX]);                       // stride 2: the 3x3 neighbourhood of (2y, 2x)
        {
            const BitMap D = m[kMX];
            skip_map_from(m[kMB1a], [&](int y, int x) { return D.get(2 * y, 2 * x); });
        }
        skip_dilate3(m[kMB1a], m[kMTmpH], m[kMB1b]);
        skip_dilate3(m[kMB1b], m[kMTmpH], m[kMX1]);
        {   // deconv: out[2g + p] reads in[g] and, for p = 1, in[g + 1] (per axis); m0 adds the residual t0 (= x0's pixels)
            const BitMap T = m[kMX1], R = m[kMX0];
            auto tget = [&](int gy, int gx) { return gy >= T.h || gx >= T.wd || T.get(gy, gx); };
            auto dc = [&](int oy, int ox) {
                const int py = oy & 1, px = ox & 1, gy = oy >> 1, gx = ox >> 1;
                return tget(gy, gx) || (py && tget(gy + 1, gx)) || (px && tget(gy, gx + 1)) || (py && px && tget(gy + 1, gx + 1));
            };
            skip_map_from(m[kMM0], [&](int y, int x) { return dc(y, x) || R.get(y, x); });
            skip_map_from(m[kMM1], dc);
        }
        skip_dilate3(m[kMM0], m[kMTmp], m[kMO0]);
        skip_dilate3(m[kMM1], m[kMTmp], m[kMO1]);
        for (int i = threadIdx.x; i < P.h * P.nwf; i += blockDim.x) m[kMOut].w[i] = m[kMO0].w[i] | m[kMO1].w[i];
        __syncthreads();
        // per launch and class: flag the tiles of this frame that must run
        for (int li = 0; li < kSkipLaunches; ++li) {
            const SkipLaunch &L = P.l[li];
            const BitMap &o = m[L.map];
            int *flags = plan + L.rec + kP2ItemsHeader + L.total + L.nclass * L.tiles;
            const int per_frame = L.tiles_u * L.tiles_v;
            for (int idx = threadIdx.x; idx < L.nclass * per_frame; idx += blockDim.x) {
                const int c = idx / per_frame, tf = idx - c * per_frame;
                const int tu = tf % L.tiles_u, tv = tf / L.tiles_u;
                const int u0 = tu * kP2TileU, v0 = tv * kP2TileV;
                bool run = u0 + kP2TileU > L.grid_u || v0 + kP2TileV > L.grid_v;      // partial tile
                if (!run && L.out_stride == 1) {     // the tile is one aligned 8- or 16-bit field of 16 or 8 rows
                    const int y0 = L.u_is_x ? v0 : u0, x0 = L.u_is_x ? u0 : v0;
                    const int ny = L.u_is_x ? kP2TileV : kP2TileU, nx = L.u_is_x ? kP2TileU : kP2TileV;
                    const uint32_t field = (1u << nx) - 1u;
                    for (int y = y0; y < y0 + ny && !run; ++y) run = (o.w[y * o.nw + (x0 >> 5)] >> (x0 & 31)) & field;
                } else if (!run) {
                    for (int r = 0; r < kP2TileU * kP2TileV && !run; ++r) {
                        const int ou = (u0 + (r & 7)) * L.out_stride + L.off_u[c], ov = (v0 + (r >> 3)) * L.out_stride + L.off_v[c];
                        run = L.u_is_x ? o.get(ov, ou) : o.get(ou, ov);
                    }
                }
                flags[c * L.tiles + b * per_frame + tf] = run ? 1 : 0;
            }
        }
        // the frame's maps, for bev_skip_seg_kernel to flag the segments from (in parallel, off this CTA)
        for (int i = threadIdx.x; i < P.frame_words; i += blockDim.x) segs[P.map_off + (long long)b * P.frame_words + i] = (int)s_bits[i];
        __syncthreads();
    }
    // per launch: representatives, the item list, the skipped list, the header
    for (int li = 0; li < kSkipLaunches; ++li) {
        const SkipLaunch &L = P.l[li];
        int *rec = plan + L.rec;
        int *items = rec + kP2ItemsHeader, *skipped = items + L.total;
        const int *flags = skipped + L.nclass * L.tiles;
        if (threadIdx.x < 4) s_rep[threadIdx.x] = 0x7FFFFFFF;
        __syncthreads();
        for (int e = threadIdx.x; e < L.nclass * L.tiles; e += blockDim.x)
            if (!flags[e]) atomicMin(&s_rep[e / L.tiles], e % L.tiles);
        __syncthreads();
        const int count = skip_compact(L.total, [&](int g) {
            const P2ItemIndex ix = p2_item_index(g, L.nblocks, L.tiles);
            return flags[L.order[ix.rank] * L.tiles + ix.t] != 0 || ix.t == s_rep[L.order[ix.rank]];
        }, items, s_scan);
        const int nskip = skip_compact(L.nclass * L.tiles, [&](int e) {
            return flags[e] == 0 && e % L.tiles != s_rep[e / L.tiles];
        }, skipped, s_scan);
        if (threadIdx.x == 0) {
            rec[kRecCount] = count; rec[kRecSkipped] = nskip;
            rec[kRecNclass] = L.nclass; rec[kRecTiles] = L.tiles; rec[kRecTilesU] = L.tiles_u; rec[kRecTilesV] = L.tiles_v;
            rec[kRecUisX] = L.u_is_x; rec[kRecOutStride] = L.out_stride; rec[kRecOutH] = L.out_h; rec[kRecOutW] = L.out_w;
            rec[kRecBatch] = P.batch;
            for (int c = 0; c < 4; ++c) {
                rec[kRecOffY + c] = L.u_is_x ? L.off_v[c] : L.off_u[c]; rec[kRecOffX + c] = L.u_is_x ? L.off_u[c] : L.off_v[c];
                rec[kRecRep + c] = c < L.nclass && s_rep[c] != 0x7FFFFFFF ? s_rep[c] : -1;
            }
            rec[kRecSkipOff] = kP2ItemsHeader + L.total;
            rec[kRecFlagOff] = kP2ItemsHeader + L.total + L.nclass * L.tiles;
        }
        __syncthreads();
    }
}

// one CTA per launch with a segment record: the flags from the plan kernel's maps, representatives, the groups, the skipped list, the
// header
__global__ void __launch_bounds__(kSkipThreads) bev_skip_seg_kernel(int *__restrict__ segs, SkipPlan P) {
    __shared__ int s_scan[33], s_rep[8];
    const SkipLaunch &L = P.l[blockIdx.x];
    if (L.seg < 0) return;
    int *rec = segs + L.seg;
    int *groups = rec + kP2SegHeader, *skipped = groups + kP2SegSlots * L.max_groups;
    int *flags = skipped + L.nclass * L.nseg;
    const int nseg = L.nseg;
    // flags: a segment runs when it holds a non-constant pixel or leaves the map
    const bool full = L.map < kNumFullMaps;
    const int map_word = full ? L.map * P.h * P.nwf : kNumFullMaps * P.h * P.nwf + (L.map - kNumFullMaps) * P.h2 * P.nwh;
    const int seg_frame = L.grid_v * L.tiles_u;
    for (int b = 0; b < P.batch; ++b) {
        const BitMap o{reinterpret_cast<uint32_t *>(segs + P.map_off + (long long)b * P.frame_words + map_word), full ? P.h : P.h2,
                       full ? P.w : P.w2, full ? P.nwf : P.nwh};
        for (int idx = threadIdx.x; idx < L.nclass * seg_frame; idx += blockDim.x) {
            const int c = idx / seg_frame, sf = idx - c * seg_frame;
            const int v = sf / L.tiles_u, u0 = (sf - v * L.tiles_u) * kP2TileU;
            bool live = u0 + kP2TileU > L.grid_u;                        // partial segment
            if (!live && L.out_stride == 1 && L.u_is_x) {                // one aligned 8-bit field
                live = (o.w[v * o.nw + (u0 >> 5)] >> (u0 & 31)) & 0xFFu;
            } else {
                for (int i = 0; i < kP2TileU && !live; ++i) {
                    const int ou = (u0 + i) * L.out_stride + L.off_u[c], ov = v * L.out_stride + L.off_v[c];
                    live = L.u_is_x ? o.get(ov, ou) : o.get(ou, ov);
                }
            }
            flags[c * nseg + b * seg_frame + sf] = live ? 1 : 0;
        }
    }
    __syncthreads();
    auto parity = [&](int s) { return (s / L.tiles_u) % L.grid_v & 1; };
    if (threadIdx.x < 8) s_rep[threadIdx.x] = 0x7FFFFFFF;
    __syncthreads();
    for (int e = threadIdx.x; e < L.nclass * nseg; e += blockDim.x)
        if (!flags[e]) {
            const int c = e / nseg, s = e - c * nseg;
            atomicMin(&s_rep[2 * c + parity(s)], s);
        }
    __syncthreads();
    int ngroups = 0;
    for (int rank = 0; rank < L.nclass; ++rank) {
        const int c = L.order[rank];
        int *g = groups + kP2SegSlots * ngroups;
        const int n = skip_compact(nseg, [&](int s) {
            return flags[c * nseg + s] != 0 || s == s_rep[2 * c] || s == s_rep[2 * c + 1];
        }, g, s_scan);
        const int ng = (n + kP2SegSlots - 1) / kP2SegSlots;
        for (int j = threadIdx.x; j < ng * kP2SegSlots; j += blockDim.x) g[j] = j < n ? (c << 24) | g[j] : -1;
        ngroups += ng;
        __syncthreads();
    }
    const int nskip = skip_compact(L.nclass * nseg, [&](int e) {
        const int c = e / nseg, s = e - c * nseg;
        return flags[e] == 0 && s != s_rep[2 * c + parity(s)];
    }, skipped, s_scan);
    if (threadIdx.x == 0) {
        rec[kSegCount] = ngroups * L.nblocks; rec[kSegSkipped] = nskip; rec[kSegGroups] = ngroups;
        rec[kSegNclass] = L.nclass; rec[kSegPerClass] = nseg; rec[kSegTilesU] = L.tiles_u; rec[kSegGridV] = L.grid_v;
        rec[kSegUisX] = L.u_is_x; rec[kSegOutStride] = L.out_stride; rec[kSegOutH] = L.out_h; rec[kSegOutW] = L.out_w;
        rec[kSegBatch] = P.batch;
        for (int c = 0; c < 4; ++c) {
            rec[kSegOffY + c] = L.u_is_x ? L.off_v[c] : L.off_u[c]; rec[kSegOffX + c] = L.u_is_x ? L.off_u[c] : L.off_v[c];
            for (int par = 0; par < 2; ++par)
                rec[kSegRep + 2 * c + par] = c < L.nclass && s_rep[2 * c + par] != 0x7FFFFFFF ? s_rep[2 * c + par] : -1;
        }
        rec[kSegSkipOff] = kP2SegHeader + kP2SegSlots * L.max_groups;
        rec[kSegFlagOff] = kP2SegHeader + kP2SegSlots * L.max_groups + L.nclass * nseg;
    }
}

// every pixel of a skipped segment <- the pixel at the same position of the representative of its class and v parity
__global__ void __launch_bounds__(256) bev_skip_fill_segs_kernel(const int *__restrict__ rec, float *__restrict__ out_f32,
                                                                 __half *__restrict__ out_planes, int cout) {
    const int nskip = __ldg(rec + kSegSkipped);
    const int nseg = __ldg(rec + kSegPerClass), tiles_u = __ldg(rec + kSegTilesU), grid_v = __ldg(rec + kSegGridV);
    const int u_is_x = __ldg(rec + kSegUisX), os = __ldg(rec + kSegOutStride), out_h = __ldg(rec + kSegOutH), out_w = __ldg(rec + kSegOutW);
    const long long plane_stride = (long long)__ldg(rec + kSegBatch) * out_h * out_w * cout;
    const int *skipped = rec + __ldg(rec + kSegSkipOff);
    // (destination, source) pixel of position lu of skipped entry e
    auto pixels = [&](int e, int lu, size_t &dst, size_t &src) {
        const int ent = __ldg(skipped + e), c = ent / nseg, s = ent - c * nseg;
        const int oy0 = __ldg(rec + kSegOffY + c), ox0 = __ldg(rec + kSegOffX + c);
        auto pixel = [&](int ss) -> size_t {
            const int rest = ss / tiles_u, v = rest % grid_v, b = rest / grid_v, gu = (ss - rest * tiles_u) * kP2TileU + lu;
            const int gy = u_is_x ? v : gu, gx = u_is_x ? gu : v;
            return ((size_t)b * out_h + (size_t)(gy * os + oy0)) * out_w + (size_t)(gx * os + ox0);
        };
        dst = pixel(s);
        src = pixel(__ldg(rec + kSegRep + 2 * c + ((s / tiles_u) % grid_v & 1)));
    };
    const int stride = gridDim.x * blockDim.x, tid = blockIdx.x * blockDim.x + threadIdx.x;
    if (out_f32) {
        const int q = cout / 4, n = nskip * kP2TileU * q;
        for (int i = tid; i < n; i += stride) {
            const int px = i / q, j = i - px * q;
            size_t dst, src;
            pixels(px / kP2TileU, px % kP2TileU, dst, src);
            reinterpret_cast<float4 *>(out_f32 + dst * cout)[j] = reinterpret_cast<const float4 *>(out_f32 + src * cout)[j];
        }
    }
    if (out_planes) {
        const int q = cout / 8, n = nskip * kP2TileU * q;
        for (int i = tid; i < 2 * n; i += stride) {
            const int pl = i / n, k = i - pl * n, px = k / q, j = k - px * q;
            size_t dst, src;
            pixels(px / kP2TileU, px % kP2TileU, dst, src);
            reinterpret_cast<uint4 *>(out_planes + pl * plane_stride + dst * cout)[j] =
                reinterpret_cast<const uint4 *>(out_planes + pl * plane_stride + src * cout)[j];
        }
    }
}

// every pixel of a skipped tile <- the pixel at the same tile position of its class's representative (fp32 and / or both planes)
__global__ void __launch_bounds__(256) bev_skip_fill_kernel(const int *__restrict__ rec, float *__restrict__ out_f32,
                                                            __half *__restrict__ out_planes, int cout) {
    const int nskip = __ldg(rec + kRecSkipped);
    if ((int)blockIdx.x >= nskip) return;
    const int tiles = __ldg(rec + kRecTiles), tiles_u = __ldg(rec + kRecTilesU), tiles_v = __ldg(rec + kRecTilesV);
    const int u_is_x = __ldg(rec + kRecUisX), os = __ldg(rec + kRecOutStride), out_h = __ldg(rec + kRecOutH), out_w = __ldg(rec + kRecOutW);
    const long long plane_stride = (long long)__ldg(rec + kRecBatch) * out_h * out_w * cout;
    const int *skipped = rec + __ldg(rec + kRecSkipOff);
    for (int e = blockIdx.x; e < nskip; e += gridDim.x) {
        const int ent = __ldg(skipped + e);
        const int c = ent / tiles, t = ent - c * tiles, r = __ldg(rec + kRecRep + c);
        const int oy0 = __ldg(rec + kRecOffY + c), ox0 = __ldg(rec + kRecOffX + c);
        auto pixel = [&](int tt, int lu, int lv) -> size_t {
            const int tu = tt % tiles_u, rest = tt / tiles_u, tv = rest % tiles_v, b = rest / tiles_v;
            const int gu = tu * kP2TileU + lu, gv = tv * kP2TileV + lv;
            const int gy = u_is_x ? gv : gu, gx = u_is_x ? gu : gv;
            return ((size_t)b * out_h + (size_t)(gy * os + oy0)) * out_w + (size_t)(gx * os + ox0);
        };
        if (out_f32) {
            const int q = cout / 4;
            for (int i = threadIdx.x; i < kP2TileU * kP2TileV * q; i += blockDim.x) {
                const int px = i / q, j = i - px * q;
                const float4 v = reinterpret_cast<const float4 *>(out_f32 + pixel(r, px & 7, px >> 3) * cout)[j];
                reinterpret_cast<float4 *>(out_f32 + pixel(t, px & 7, px >> 3) * cout)[j] = v;
            }
        }
        if (out_planes) {
            const int q = cout / 8, n = kP2TileU * kP2TileV * q;
            for (int i = threadIdx.x; i < 2 * n; i += blockDim.x) {
                const int pl = i / n, k = i - pl * n, px = k / q, j = k - px * q;
                const __half *src = out_planes + pl * plane_stride + pixel(r, px & 7, px >> 3) * cout;
                __half *dst = out_planes + pl * plane_stride + pixel(t, px & 7, px >> 3) * cout;
                reinterpret_cast<uint4 *>(dst)[j] = reinterpret_cast<const uint4 *>(src)[j];
            }
        }
    }
}

}  // namespace sessd

using namespace sessd;

extern "C" long long sessd_bev_skip_plan_words(int batch, int h, int w, int *offsets) {
    SkipPlan P;
    const long long words = skip_plan(P, batch, h, w);
    if (words && offsets)
        for (int i = 0; i < kSkipLaunches; ++i) offsets[i] = P.l[i].rec;
    return words;
}

extern "C" long long sessd_bev_skip_seg_words(int batch, int h, int w, int *offsets) {
    SkipPlan P;
    if (!skip_plan(P, batch, h, w)) return 0;
    if (offsets)
        for (int i = 0; i < kSkipLaunches; ++i) offsets[i] = P.l[i].seg;
    return P.seg_words;
}

// d_bitmap_index: the last sparse level's bitmap index (grid = that level: shape = {D, h, w}); d_plan: sessd_bev_skip_plan_words(B, h, w),
// d_segs: sessd_bev_skip_seg_words(B, h, w)
extern "C" int sessd_bev_skip_plan(const void *d_bitmap_index, sessd_grid grid, int *d_plan, int *d_segs, void *stream) {
    if (!d_bitmap_index || !d_plan || !d_segs || grid.shape[0] < 1) return SESSD_EINVAL;
    SkipPlan P;
    if (!skip_plan(P, grid.batch, grid.shape[1], grid.shape[2])) return SESSD_EINVAL;
    P.depth = grid.shape[0];
    const int smem = 4 * P.frame_words;
    if (smem > 200 * 1024) return SESSD_EINVAL;
    static int attr_smem = 48 * 1024;     // opt in to what the maps need (the static shared memory counts against the same limit)
    if (smem > attr_smem) {
        SESSD_CUDA_TRY(cudaFuncSetAttribute(bev_skip_plan_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr_smem = smem;
    }
    SESSD_LAUNCH(bev_skip_plan_kernel, 1, kSkipThreads, smem, (cudaStream_t)stream, (const uint2 *)d_bitmap_index, d_plan, d_segs, P);
    SESSD_LAUNCH(bev_skip_seg_kernel, kSkipLaunches, kSkipThreads, 0, (cudaStream_t)stream, d_segs, P);
    return last_error();
}

// after the launch that ran d_record's items: fill its skipped tiles in d_out_f32 [B][H][W][cout] and / or d_out_planes [2][B][H][W][cout]
extern "C" int sessd_bev_skip_fill(const int *d_record, float *d_out_f32, void *d_out_planes, int cout, void *stream) {
    if (!d_record || (!d_out_f32 && !d_out_planes) || cout < 8 || cout % 8) return SESSD_EINVAL;
    SESSD_LAUNCH(bev_skip_fill_kernel, 2 * kNumSMs, 256, 0, (cudaStream_t)stream, d_record, d_out_f32, (__half *)d_out_planes, cout);
    return last_error();
}

// after the launch that ran d_seg_record's segments: fill its skipped segments in d_out_f32 [B][H][W][cout] and / or d_out_planes
extern "C" int sessd_bev_skip_fill_segs(const int *d_seg_record, float *d_out_f32, void *d_out_planes, int cout, void *stream) {
    if (!d_seg_record || (!d_out_f32 && !d_out_planes) || cout < 8 || cout % 8) return SESSD_EINVAL;
    SESSD_LAUNCH(bev_skip_fill_segs_kernel, 2 * kNumSMs, 256, 0, (cudaStream_t)stream, d_seg_record, d_out_f32, (__half *)d_out_planes, cout);
    return last_error();
}
