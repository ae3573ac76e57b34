/*
 * sessd_b200.h -- C ABI of the GPU-native (sm_90a) SE-SSD per-frame LiDAR hot path
 *                 (voxelise -> sparse 3-D conv encoder -> BEV neck/head -> rotated IoU / NMS).
 *
 * Conventions (all entry points):
 *   - plain C types only; device pointers are owned by the caller (torch's allocator in the Python host);
 *   - every call takes an explicit `stream` (a cudaStream_t passed as void*), launches asynchronously on it
 *     and performs NO hidden synchronisation or allocation, so a whole frame can be captured in a CUDA graph;
 *   - data-dependent sizes (voxel / active-site / candidate counts) live in DEVICE memory: kernels take
 *     `const int* d_count` plus a host-side capacity and are launched as persistent grids sized from the SM count;
 *   - return value 0 on success, negative SESSD_E* on argument / capacity errors, positive cudaError_t otherwise
 *     (no exit(), unlike the reference's CHECK_ERROR macro, det3d/core/iou3d/src/iou3d.cpp:13-21).
 *
 * Each function cites the reference interface (file:line under Vegeta2020/SE-SSD) it replaces.
 */
#ifndef SESSD_B200_H
#define SESSD_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define SESSD_OK 0
#define SESSD_EINVAL (-1)
#define SESSD_ECAPACITY (-2)
#define SESSD_EWORKSPACE (-3)

/* library / build information: returns e.g. "sessd_b200 0.1 (sm_90a)" */
const char *sessd_version(void);
/* number of kernel launches issued through this library since load (bench.py's gpu_launches claim) */
long long sessd_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * V1/V2/V4 + R1: voxeliser.
 * Replaces det3d/core/input/voxel_generator.py:10-32 (VoxelGenerator.generate) ->
 * det3d/ops/point_cloud/point_cloud_ops_v2.py:120-194 (points_to_voxel) and :9-62 (numba kernel),
 * batched over frames in the wire format of det3d/torchie/parallel/collate.py:154-218 (concatenated
 * voxels, coordinates with a leading batch column), with the per-voxel mean of
 * det3d/models/readers/voxel_encoder.py:205-210 (VoxelFeatureExtractorV3) fused into the same pass.
 * Results are bit-identical to the sequential reference loop (voxel id = rank of the voxel's first point in
 * input order; first max_points points kept in input order; everything after the first point that would open
 * voxel #max_voxels is dropped).
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    float voxel_size[3];      /* x, y, z */
    float range_min[3];       /* x, y, z */
    float range_max[3];
    int grid[3];              /* x, y, z cells = round((max-min)/voxel_size) in fp32 (voxel_generator.py:15-16) */
    int max_points;           /* per voxel (config: 5) */
    int max_voxels;           /* per frame (config: 20000) */
    int num_feat;             /* floats per point (4) */
} sessd_voxel_cfg;

size_t sessd_voxelize_workspace_bytes(int max_total_points, int batch, const sessd_voxel_cfg *cfg);

/* d_points [max_total_points, num_feat] f32; d_frame_off [batch+1] i32 (device; frame f owns points
 * [off[f], off[f+1])); outputs: d_voxels [batch*max_voxels, max_points, num_feat] (zero padded),
 * d_coors [batch*max_voxels, 4] i32 (b, z, y, x), d_num_points [batch*max_voxels] i32,
 * d_mean [batch*max_voxels, num_feat] f32 (nullable), d_num_voxels [batch+1] i32 (per frame; last = total). */
int sessd_voxelize(const float *d_points, const int *d_frame_off, int batch, int max_total_points,
                   const sessd_voxel_cfg *cfg, float *d_voxels, int *d_coors, int *d_num_points, float *d_mean,
                   int *d_num_voxels, void *workspace, size_t workspace_bytes, void *stream);

/* Host-buffer convenience for the numpy-level API (VoxelGenerator.generate): one frame, host in / host out,
 * allocation + H2D + D2H inside, synchronous.  Returns the voxel count (>=0) or a negative error. */
int sessd_voxelize_host(const float *h_points, int num_points, const sessd_voxel_cfg *cfg, float *h_voxels,
                        int *h_coors_zyx /*[max_voxels,3]*/, int *h_num_points);

/* ------------------------------------------------------------------------------------------------
 * S3: rulebook ("indice pairs") construction.  Replaces spconv 1.x's indice-pair builders that
 * det3d/models/backbones/scn.py:106-149,182-183 trigger (4 SubM keys + 4 strided convs per forward).
 * The rulebook is kept output-major: nbr[o, k] = input row feeding output o through kernel offset k, or -1.
 *
 * An "index" is either a hash table over given coordinates (any row order: the voxeliser's first-appearance
 * order at level 0) or a rank bitmap (rows in ascending linear index: what strided convs emit).
 * ------------------------------------------------------------------------------------------------ */
typedef struct {
    int batch;
    int shape[3];     /* D, H, W  (z, y, x) */
} sessd_grid;

/* hash index: table of `capacity` (power of two >= 2*max_rows) 64-bit slots */
size_t sessd_hash_bytes(int max_rows, int *capacity_out);
int sessd_hash_build(const int *d_coors /*[n,4] b,z,y,x*/, const int *d_n, int max_rows, sessd_grid grid,
                     uint64_t *d_table, int capacity, void *stream);

/* rank bitmap index: uint2 {bits, exclusive prefix popcount} per 32 cells; + scan scratch */
size_t sessd_bitmap_words(sessd_grid grid);
size_t sessd_scan_scratch_bytes(size_t n_items);

/* SubM rulebook over an index: nbr [max_rows, kvol] */
int sessd_subm_rulebook(const int *d_coors, const int *d_n, int max_rows, sessd_grid grid, const int ksize[3],
                        int index_kind /*0 hash, 1 bitmap*/, const void *d_index, int hash_capacity,
                        int *d_nbr, void *stream);

/* Strided sparse conv rulebook: marks reachable outputs in d_out_bitmap (zeroed by the call), ranks them
 * (ascending linear index == canonical order), emits out coords + count and the [max_out, kvol] nbr table. */
int sessd_strided_rulebook(const int *d_in_coors, const int *d_n_in, int max_in, sessd_grid in_grid,
                           int in_index_kind, const void *d_in_index, int in_hash_capacity,
                           const int ksize[3], const int stride[3], const int padding[3],
                           sessd_grid out_grid, void *d_out_bitmap /*uint2[words]*/, void *d_scan_scratch,
                           int *d_out_coors, int *d_n_out, int max_out, int *d_nbr, int *d_status, void *stream);

/* nbr table -> per-tile pair lists for sessd_spconv_forward_cg: one record of sessd_tile_list_stride(kvol) uint32 per 128 output rows:
 * [0,32) pair count per kernel offset, [32, 32 + 4 kvol) 128-bit row mask per offset, [160, ...) the pairs grouped by offset, each
 * (input row << 7) | tile row, ascending tile row (deterministic).  d_tiles: uint32 [ceil(max_out / 128)][stride].  kvol <= 27. */
int sessd_tile_list_stride(int kvol);
int sessd_rulebook_tile_lists(const int *d_nbr, int kvol, const int *d_n_out, int max_out, void *d_tiles, void *stream);

/* ------------------------------------------------------------------------------------------------
 * S4/S5: sparse convolution (gather -> GEMM -> fused BN(eval)+ReLU epilogue, output-stationary) and dense().
 * Replaces spconv.SubMConv3d / SparseConv3d forward + BatchNorm1d + ReLU (scn.py:106-149) and
 * SparseConvTensor.dense() + view (scn.py:184-187).
 * weight layout [kvol, Cin, Cout] (== spconv 1.x [kz,ky,kx,Cin,Cout] flattened); scale/shift = folded BN
 * (scale = gamma/sqrt(var+eps), shift = beta - mean*scale), nullable => identity; relu flag.
 * ------------------------------------------------------------------------------------------------ */
int sessd_spconv_forward(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out,
                         int max_out, const float *d_weight, int cout, const float *d_scale, const float *d_shift,
                         int relu, float *d_out_feat, void *stream);

/* dense(): out NHWC [batch, H, W, C*D] with channel index c*D + d (zero-filled by the call) */
int sessd_sparse_to_dense(const float *d_feat, const int *d_coors, const int *d_n, int max_rows, int channels,
                          sessd_grid grid, float *d_out, void *stream);
/* same result in one gather pass (no memset + scatter): the rows of every BEV cell are looked up in the level's bitmap index
 * (the `d_out_bitmap` that sessd_strided_rulebook filled for this level); writes each output byte exactly once. */
int sessd_sparse_to_dense_indexed(const float *d_feat, int max_rows, const void *d_bitmap_index, int channels, sessd_grid grid,
                                  float *d_out, void *stream);

/* S4, narrow layers (Cin <= 32; csrc/spconv_rows.cu): same contract and arguments as sessd_spconv_forward, fp32 SIMT, but the work is
 * proportional to the number of rulebook PAIRS instead of N_out x kvol row slots (a warp owns 8 output rows and visits only their valid
 * neighbours).  d_amax_out (nullable) receives the running abs-max of the output.  (Cin, Cout): (4,16) (16,16) (16,32) (32,16) (32,32). */
int sessd_spconv_forward_rows(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out, int max_out,
                              const float *d_weight, int cout, const float *d_scale, const float *d_shift, int relu,
                              float *d_out_feat, float *d_amax_out, void *stream);
/* ... and the output also (d_out_feat nullable: only) as fp16 (hi, lo) planes [row][2][cpo] for the tensor-core layers: d_out_info =
 * {abs-max of the output (atomicMax; zero it once per frame), plane scale S_out}; S_out = the power of two that maps the bound
 * *d_amax_in * gain + shift_max into [2^14, 2^15) (d_amax_in = abs-max of the INPUT features, gain = max_n sum_{k,c} |w[k][c][n] bn_scale[n]|,
 * shift_max = max_n |shift[n]|). */
int sessd_spconv_forward_rows_planes(const float *d_in_feat, int cin, const int *d_nbr, int kvol, const int *d_n_out, int max_out,
                                     const float *d_weight, int cout, const float *d_scale, const float *d_shift, int relu,
                                     const float *d_amax_in, float gain, float shift_max, float *d_out_feat, void *d_out_planes, int cpo,
                                     float *d_out_info, void *stream);
/* S4, the default tensor-core path of the Cin >= 32 layers (csrc/spconv_cg.cu): pair-proportional operand traffic -- the rows of the
 * neighbours that exist are copied by cp.async into the wgmma operand tiles (no row slot is spent on a missing neighbour), persistent CTAs,
 * fp16 wgmma with a two-term fp16 split of activations and weights (weight tiles: ops.pack_weight_sp_h2).  Same contract as
 * sessd_spconv_forward (spconv 1.x gather -> GEMM -> scatter-add at det3d/models/backbones/scn.py:106-149, + folded BN + ReLU).
 * The rulebook is passed as d_tiles = the per-tile pair lists sessd_rulebook_tile_lists() makes from the nbr table (once per rulebook).
 * d_in_planes [plane_rows][2][cp] fp16, x = (hi + lo) / d_in_info[1], d_in_info[0] = abs-max of the input tensor; outputs (each nullable, at
 * least one): fp32 rows [max_out][cout]; planes [>= max_out][2][cout <= 32 ? 32 : 64] with d_out_info = {abs-max of the output (atomicMax; zero
 * it once per frame), S_out}, S_out from the bound d_in_info[0] * gain + shift_max as above; both outputs are written 16 bytes at a time and
 * must be 16-byte aligned (SESSD_EINVAL otherwise).  Supported (cp, cout): (32,32) (32,64) (64,32) (64,64). */
int sessd_spconv_forward_cg(const void *d_in_planes, int cp, int plane_rows, const float *d_in_info, const void *d_tiles, int kvol,
                            const int *d_n_out, int max_out, const void *d_weight_h2, int cout, const float *d_scale, const float *d_shift,
                            int relu, float gain, float shift_max, float *d_out_f32, void *d_out_planes, float *d_out_info, void *stream);
/* 1: deep pipeline (twice the stages) for launches with fewer tiles than SMs (single frames); 0 (default): the shorter ring */
void sessd_set_sp_cg_deep(int on);
/* CTAs of sessd_spconv_forward_cg's (cp, cout, deep) kernel resident on one SM of the current device; its persistent grid is at most that
 * many per SM.  SESSD_EINVAL for an unsupported (cp, cout), -cudaError on a CUDA error. */
int sessd_spconv_cg_blocks_per_sm(int cp, int cout, int deep);
/* *d_amax = max(*d_amax, max |d_feat[i]|) over the first *d_n rows of a [max_rows, channels] fp32 tensor */
int sessd_absmax_rows(const float *d_feat, const int *d_n, int max_rows, int channels, float *d_amax, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Backward of the sparse convs (csrc/spconv_grad.cu; training of SpMiddleFHD).  The data gradient is the forward kernels run with
 * re-packed weights over the same table (SubM: W'[k] = W[K-1-k]^T) or over the transposed table (strided: W[k]^T); the weight gradient
 * gW[k] = sum over the pairs of offset k of in[i]^T gout[o] reads the forward rulebook's tile lists.
 * ------------------------------------------------------------------------------------------------ */
/* nbr [max_out, kvol] -> nbr_t [max_in, kvol]: nbr_t[i, k] = o where nbr[o, k] = i (o < *d_n_out), else -1 (every row of nbr_t is written) */
int sessd_rulebook_transpose(const int *d_nbr, int kvol, const int *d_n_out, int max_out, int max_in, int *d_nbr_t, void *stream);
/* fp32 rows [max_rows, channels] -> fp16 (hi, lo) planes [rows][2][cp] at S = the power of two that maps d_info[0] (the abs-max of the
 * tensor, sessd_absmax_rows) into [2^14, 2^15); d_info[1] <- S.  Rows >= *d_n are untouched; channels [channels, cp) are written as zero. */
int sessd_sparse_split_planes(const float *d_x, const int *d_n, int max_rows, int channels, float *d_info, void *d_planes, int cp, void *stream);
/* adjoint of sessd_sparse_to_dense: d_out[r][c] = d_grad[b, y, x, c*D + z] for (b, z, y, x) = d_coors[r], r < *d_n */
int sessd_dense_grad_gather(const float *d_grad, const int *d_coors, const int *d_n, int max_rows, int channels, sessd_grid grid,
                            float *d_out, void *stream);
/* weight gradient: work items (offset, fixed range of tiles) -- sessd_spconv_wgrad_items(max_out, kvol) of them, a function of the
 * arguments only -- each write an fp32 partial [Cin][Cout] to the workspace; a reduce sums the partials of every offset in ascending item
 * order: bitwise run-to-run deterministic, no float atomics.  d_gw [kvol][Cin][Cout] fp32.  _items: SESSD_EINVAL on invalid arguments. */
int sessd_spconv_wgrad_items(int max_out, int kvol);
size_t sessd_spconv_wgrad_workspace_bytes(int max_out, int kvol, int cin, int cout);
/* Cin <= 16 (fp32 SIMT): d_in_feat [*, cin] fp32, d_gout [max_out, cout] fp32.  (Cin, Cout): (4,16) (16,16) (16,32). */
int sessd_spconv_wgrad_rows(const float *d_in_feat, int cin, const float *d_gout, int cout, const void *d_tiles, int kvol,
                            const int *d_n_out, int max_out, float *d_gw, void *d_ws, size_t ws_bytes, void *stream);
/* Cin >= 32 (tensor cores, fp16 mma with the three-product split): d_in_planes [*][2][cp] with d_in_info = {abs-max, S_in}, d_g_planes
 * [max_out][2][cout] with d_g_info = {abs-max, S_g} (sessd_sparse_split_planes); gW = sum / S_in / S_g.  (cp, cout): (32,32) (32,64) (64,64). */
int sessd_spconv_wgrad_cg(const void *d_in_planes, int cp, const float *d_in_info, const void *d_g_planes, int cout, const float *d_g_info,
                          const void *d_tiles, int kvol, const int *d_n_out, int max_out, float *d_gw, void *d_ws, size_t ws_bytes,
                          void *stream);

/* ------------------------------------------------------------------------------------------------
 * N1/H1: BEV neck (SSFA) + head.  Replaces the cuDNN conv/deconv + BatchNorm2d + ReLU blocks of
 * det3d/models/necks/rpn_v1.py:135-235 and the four 1x1 convs of
 * det3d/models/bbox_heads/mg_head_sessd.py:202-230.  Tensors are NHWC.
 * ------------------------------------------------------------------------------------------------ */
/* One tap-list convolution:  out[b, oy*os+py, ox*os+px, :] =
 *    epilogue( sum_t in[b, oy*is + dy[t], ox*is + dx[t], :] @ W[t] )   (zero outside the input)
 * with epilogue y = acc*scale + shift (nullable), optional ReLU, optional residual add AFTER the ReLU
 * (rpn_v1.py:225: deconv_block_0(x_trans_1) + x_trans_0). */
typedef struct {
    int batch, in_h, in_w, cin;       /* input tensor  [batch, in_h, in_w, cin]  */
    int out_h, out_w, cout;           /* output tensor [batch, out_h, out_w, cout] */
    int grid_h, grid_w;               /* output positions computed by this call (per batch) */
    int in_stride;                    /* is */
    int out_stride, out_off_y, out_off_x;   /* os, py, px */
    int ntaps;
    int tap_dy[16], tap_dx[16];
    int relu;
} sessd_conv_desc;

/* ------------------------------------------------------------------------------------------------
 * BEV convs from PRE-SPLIT fp16 planes (csrc/bevconv_p2.cu): the neck's default path.  Activations travel between layers as
 * __half [2 (hi|lo)][batch][H][W][C] planes with x = (hi + lo) / S, S an exact power of two; every plane tensor has a device-side
 * info pair float[2] = {abs-max of the tensor (atomically raised by its producer; zero it once per frame), S}.  sessd_bev_conv_p2
 * runs the tap-list conv of sessd_conv_desc (rpn_v1.py:135-210, mg_head_sessd.py:202-230): in_stride 1 or 2, <= 9 taps, cin % 64 == 0,
 * cout % 8 == 0.  d_weight_h2: __half [2 (hi|lo)][ntaps][cout_pad][cin] of 2^e[n] w
 * (ops.pack_weight_h2); d_scale = folded BN scale * 2^-e[n].  gain / shift_max: |out| <= amax_in * gain + shift_max
 * (+ amax of the residual) with gain = max_n sum_{tap,c} |w[tap][c][n] * bn_scale[n]|: the producer derives the OUTPUT scale from
 * this bound before it writes the first element.  Outputs: fp32 NHWC (d_out_f32) and / or planes (d_out_planes + d_out_info). */
int sessd_bev_conv_p2(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                      const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                      float *d_out_f32, void *d_out_planes, float *d_out_info, const sessd_conv_desc *desc, const int *d_items,
                      const int *d_segs, void *stream);
int sessd_bev_deconv_p2(const void *d_in_planes, const float *d_in_info, const void *d_weight_h2, int cout_pad, const float *d_scale,
                        const float *d_shift, const float *d_residual, const float *d_resid_info, float gain, float shift_max,
                        float *d_out_f32, void *d_out_planes, float *d_out_info, int batch, int in_h, int in_w, int cin, int cout,
                        int relu, const int *d_items, const int *d_segs, void *stream);
/* Constant-region skipping of the SSFA neck + head (csrc/bevskip.cu).  Where the last sparse level has no site, dense() writes exact
 * zeros; every neck pixel whose receptive field lies in that empty space (and inside the map) then holds, bit for bit, the same value
 * as every other such pixel of its output-parity class.  sessd_bev_skip_plan derives from the level's bitmap index, per neck launch
 * (SKIP_LAUNCHES order of runners.SSFAPlanesRunner), the work items that must run plus one representative of the skipped ones, all on
 * the device.  The conv / deconv run the list (d_items = the launch's record); sessd_bev_skip_fill then copies the representative's
 * output into the skipped tiles.  sessd_bev_skip_plan_words: int32 words of the plan of a [batch, h, w] neck; offsets[13] <- the
 * word offset of every launch record.  The same plan also lists, in d_segs, the live segments (8 pixels along the launch's u in one
 * v row) of every stride-1 launch, packed 16 to a work item: the conv / deconv run them (d_segs = the launch's segment record) and
 * sessd_bev_skip_fill_segs fills the other segments.  sessd_bev_skip_seg_words: int32 words of d_segs; offsets[13] <- the word offset
 * of every segment record, -1 for the stride-2 launch (tiles only).  These three plan the one-task head (24 channels); the _head
 * variants plan a head launch of head_cout channels (24 per task of a multi-task head, a multiple of 8). */
long long sessd_bev_skip_plan_words(int batch, int h, int w, int *offsets);
long long sessd_bev_skip_seg_words(int batch, int h, int w, int *offsets);
int sessd_bev_skip_plan(const void *d_bitmap_index, sessd_grid grid, int *d_plan, int *d_segs, void *stream);
long long sessd_bev_skip_plan_words_head(int batch, int h, int w, int head_cout, int *offsets);
long long sessd_bev_skip_seg_words_head(int batch, int h, int w, int head_cout, int *offsets);
int sessd_bev_skip_plan_head(const void *d_bitmap_index, sessd_grid grid, int head_cout, int *d_plan, int *d_segs, void *stream);
int sessd_bev_skip_fill(const int *d_record, float *d_out_f32, void *d_out_planes, int cout, void *stream);
int sessd_bev_skip_fill_segs(const int *d_seg_record, float *d_out_f32, void *d_out_planes, int cout, void *stream);
/* Weight gradient of a BEV conv (csrc/bevgrad.cu; training of the neck and head, rpn_v1.py:135-210, mg_head_sessd.py:202-215):
 *    d_gw[t][ci][co] = sum_{b, y, x} in[b, y*is + dy[t], x*is + dx[t], ci] * g[b, y, x, co]     (zero outside the input)
 * for the tap list, stride and extents of the forward's descriptor (out_stride 1, no offset, grid = the output extent; relu ignored).
 * d_in_planes __half [2][batch][in_h][in_w][cin] with d_in_info = {abs-max, S_in} (the planes the forward read); d_g_planes __half
 * [2][batch][out_h][out_w][cout] with d_g_info = {abs-max, S_g} (sessd_absmax + sessd_bev_split_planes of the output gradient).
 * cin % 128 == 0; cout % 128 == 0 or cout == 64 (the head's 24-channel gradient zero-padded, as its data gradient needs).  Tensor cores,
 * fp16 mma with the three-product split, divided by S_in S_g.  A deconv (k3, s2, p1, op1) is the stride-2 conv with the roles swapped:
 * in = its output gradient, g = its input; its gradient is d_gw transposed.  Work items (tap, channel blocks, fixed pixel range) --
 * sessd_bev_wgrad_items(desc) of them, a function of the descriptor only -- each write an fp32 partial to the workspace, and a reduce
 * sums them in ascending item order: bitwise run-to-run deterministic, no float atomics.  _items: SESSD_EINVAL on an invalid descriptor;
 * _workspace_bytes: 0 then. */
int sessd_bev_wgrad_items(const sessd_conv_desc *desc);
size_t sessd_bev_wgrad_workspace_bytes(const sessd_conv_desc *desc);
int sessd_bev_wgrad(const void *d_in_planes, const float *d_in_info, const void *d_g_planes, const float *d_g_info,
                    const sessd_conv_desc *desc, float *d_gw, void *d_ws, size_t ws_bytes, void *stream);
/* fp32 [n] -> planes [2][n] scaled from d_info[0] (the tensor's abs-max, e.g. from sessd_absmax); writes the scale to d_info[1] */
int sessd_bev_split_planes(const float *d_x, long long n, float *d_info, void *d_planes, void *stream);
/* dense() (scn.py:184-187) straight into the planes the neck reads: d_amax = abs-max of the feature rows, d_info[2] <- {abs-max, S} */
int sessd_sparse_to_dense_planes(const float *d_feat, int max_rows, const void *d_bitmap_index, int channels, sessd_grid grid,
                                 const float *d_amax, float *d_info, void *d_planes, void *stream);
/* SSFA tail (rpn_v1.py:229-233): w_k = BN(conv1x1_{128->1}(x_k)) with d_w0 / d_w1 [C] and (s_k, t_k) the folded BN; softmax over the
 * pair; weighted sum of x0 and x1.  Writes the fused map as planes (d_planes + d_out_info) and, when d_out is set, as fp32;
 * d_info0 / d_info1 [2]: abs-max of x0 / x1 */
int sessd_ssfa_fuse_planes(const float *d_x0, const float *d_x1, const float *d_w0, const float *d_w1, float s0, float t0, float s1,
                           float t1, int num_pixels, int channels, float *d_out, const float *d_info0, const float *d_info1,
                           float *d_out_info, void *d_planes, void *stream);

/* *d_amax = max(*d_amax, max_i |d_x[i]|)  (for tensors produced by kernels without an abs-max epilogue) */
int sessd_absmax(const float *d_x, long long n, float *d_amax, void *stream);

/* ------------------------------------------------------------------------------------------------
 * P1/P2/P3: decode -> sigmoid -> threshold -> IoU-rectified score -> top-k -> rotated NMS -> direction fix ->
 * range mask, all on device, no host round trip.  Replaces MultiGroupHead.predict / get_task_detections
 * (mg_head_sessd.py:893-1057), box_torch_ops.second_box_decode (:81-147), box_torch_ops.rotate_nms (:527-548),
 * nms_cpu.py:37-48 and nms_cpu.h:72-168.
 * head layout per pixel: [box 2x7 | cls 2 | dir 2x2 | iou 2] = 22 floats, row stride head_stride (22, or 24 when the
 * fused 128->22 head GEMM pads its output to a multiple of 4 channels).
 * ------------------------------------------------------------------------------------------------ */

/* DI-NMS (IoU-weighted rotated NMS, nms_cpu.h:173-384 with box_torch_ops.rotate_weighted_nms's centerness) constants; the SE-SSD /
 * CIA-SSD head's values (mg_head_sessd.py:1001-1018) in brackets. */
typedef struct {
    float cnt_thresh;          /* 2.6: a pick is emitted when sum over same-label j with IoU > 0 of IoU * q_j exceeds this */
    float dist_edge[4];        /* 0, 20, 40, 60: band b = [dist_edge[b], dist_edge[b+1]) of the pick's distance to the origin */
    float sigma2[3];           /* 0.0009, 0.009, 0.1: weight exp(-(1 - IoU)^2 / sigma2[b]); no band (>= dist_edge[3]): weight 0 */
    float suppressed_thresh;   /* 0.3: members have IoU > thr; IoU >= thr suppresses */
    float centerness_pow;      /* 2 */
    int centerness;            /* 1: score *= (1 - softmax_k(|centre - anchor centre|))^centerness_pow before the loop */
} sessd_dinms_cfg;

#define SESSD_DINMS_MAX_PRE 4096   /* DI-NMS keeps a dense [pre_max, pre_max] fp32 IoU matrix per frame: 64 MB at the cap */

typedef struct {
    int batch;
    int num_anchors;           /* per frame (70400) */
    int anchors_per_loc;       /* 2 */
    int head_stride;           /* floats per pixel row of d_head (>= 22) */
    float score_thresh;        /* 0.3 */
    int nms_pre_max;           /* 1000 */
    int nms_post_max;          /* 100 */
    float nms_iou_thresh;      /* 0.01 */
    int nms_ge;                /* 1: suppress when iou >= thr (nms_cpu.h:155); 0: iou > thr (iou3d nms_kernel) */
    float post_range[6];       /* 0,-40,-5,70.4,40,5 */
    float direction_offset;    /* 0 */
    int use_frustum;           /* apply the calib frustum filter (mg_head_sessd.py:1024-1030) */
    int nms_mode;              /* 0: rotate_nms (greedy, nms_iou_thresh, nms_ge); 1: DI-NMS (rotate_weighted_nms, constants below) */
    sessd_dinms_cfg dinms;     /* read in nms_mode 1 only: a zero-initialised config keeps rotate_nms */
    int num_tasks;             /* T: one-class tasks of a MultiGroupHead (Car, Pedestrian, Cyclist); 0 or 1 = one task */
    int task_stride;           /* T > 1: floats between two tasks' 22-float blocks in a pixel row (24) */
} sessd_post_cfg;

#define SESSD_POST_MAX_TASKS 64

size_t sessd_postprocess_workspace_bytes(const sessd_post_cfg *cfg);

/* d_head [batch, num_anchors/apl, head_stride]; d_anchors [num_anchors, 7] (shared by all frames);
 * d_frustum [batch, 6, 4] plane (a,b,c,d) per surface (nullable unless use_frustum);
 * outputs: d_boxes [batch, post_max, 7], d_scores [batch, post_max], d_labels [batch, post_max] i32,
 * d_count [batch] i32, d_aux [batch, 4] i32 (candidates, pre-NMS count, NMS-selected count, reserved),
 * d_sel_anchor [batch, post_max] i32 (anchor index of each NMS-selected box, before frustum/range masks).
 * nms_mode 1 (DI-NMS): nms_pre_max <= SESSD_DINMS_MAX_PRE, and every "post_max" above is nms_pre_max (DI-NMS applies no post_max);
 * the boxes are the clusters' weighted averages, d_sel_anchor holds each emitted cluster's pick, d_aux[2] the emitted clusters and
 * d_aux[3] the loop's picks.
 * Several tasks (num_tasks = T > 1; one class and anchors_per_loc anchors per location each): task t's head floats start at
 * t * task_stride of the pixel row (head_stride >= (T - 1) * task_stride + 22), its anchors at d_anchors + t * num_anchors * 7
 * (d_anchors [T, num_anchors, 7]).  Every frame and task is one slot (b * T + t) of the same launches; each slot takes its own top
 * nms_pre_max and runs NMS within its task only (no suppression across classes) and keeps nms_post_max; score threshold, frustum,
 * direction fix and range mask are shared.  Layouts with P the per-task capacity above: d_boxes [batch, T * P, 7], d_scores and
 * d_labels [batch, T * P]: the tasks' detections concatenated in task order, label t; d_count [batch] = the frame total;
 * d_aux [batch * T, 4] per slot; d_sel_anchor [batch, T * P], task t's block at t * P, holding indices t * num_anchors + a into the
 * concatenated anchors.  The workspace carries one staging copy of each slot's detections. */
int sessd_postprocess(const float *d_head, const float *d_anchors, const float *d_frustum,
                      const sessd_post_cfg *cfg, float *d_boxes, float *d_scores, int *d_labels, int *d_count,
                      int *d_aux, int *d_sel_anchor, void *workspace, size_t workspace_bytes, void *stream);

/* Same as sessd_postprocess, plus a packed copy of the results for ONE device->host transfer per batch (the reference moves boxes,
 * scores and labels to the host separately and syncs twice per frame: box_torch_ops.py:536, mg_head_sessd.py:1026):
 * d_packed [batch, post_max, 8] = box 7 | score; d_meta [batch, 8 + post_max] i32 = count, candidates, pre-NMS count,
 * NMS-selected count, d_num_voxels[b] (0 if null), *d_status (0 if null), 0, 0, then the anchor index of every returned
 * detection (-1 beyond count).  Several tasks: d_packed [batch, T * P, 8] and d_meta [batch, 8 + T * P] follow the concatenated
 * order; the counts of the header are summed over the tasks, and the anchor index t * num_anchors + a gives the label t. */
int sessd_postprocess_packed(const float *d_head, const float *d_anchors, const float *d_frustum,
                             const sessd_post_cfg *cfg, float *d_boxes, float *d_scores, int *d_labels, int *d_count,
                             int *d_aux, int *d_sel_anchor, float *d_packed, int *d_meta, const int *d_num_voxels,
                             const int *d_status, void *workspace, size_t workspace_bytes, void *stream);

/* stand-alone rotated NMS on [n,5] (x,y,w,l,r) + scores: box_torch_ops.rotate_nms semantics
 * (top-k pre_max by score, greedy, keep <= post_max); d_keep [post_max] i32 indices into the input.
 * Scores may have either sign and are ordered as floats, -0 == +0; equal scores keep the lower index first.
 * NaN / Inf scores are out of scope. */
size_t sessd_rotate_nms_workspace_bytes(int max_boxes, int pre_max);
int sessd_rotate_nms(const float *d_boxes5, const float *d_scores, const int *d_n, int max_boxes, int pre_max,
                     int post_max, float iou_thresh, int ge, int *d_keep, int *d_num_keep, void *workspace,
                     size_t workspace_bytes, void *stream);

/* stand-alone DI-NMS: box_torch_ops.rotate_weighted_nms (box_torch_ops.py:552-621) with the C core nms_cpu.h:173-384.
 * Inputs, n = min(*d_n, max_boxes) rows: d_boxes7 [n,7] (averaged and distance-tested), d_boxes5 [n,5] (x,y,w,l,r: the IoU
 * geometry), d_scores [n] (>= 0), d_iou_preds [n] (the rectified q = (iou + 1) / 2), d_labels [n] i32, d_dirs [n] i32, d_anchors
 * [n,7] (read when cfg->centerness; nullable otherwise).  Top-k = min(n, pre_max) by score (equal scores: lower index first), then
 * the loop.  Outputs, one row per emitted cluster in pick order: d_out_boxes [pre_max,7], d_out_scores, d_out_labels,
 * d_out_dirs, d_keep (the pick's top-k position), d_selected (the pick's input index); d_count [2] = emitted clusters, picks.
 * Rows beyond the count are left unwritten.  pre_max <= SESSD_DINMS_MAX_PRE. */
size_t sessd_rotate_weighted_nms_workspace_bytes(int max_boxes, int pre_max);
int sessd_rotate_weighted_nms(const float *d_boxes7, const float *d_boxes5, const float *d_scores, const float *d_iou_preds,
                              const int *d_labels, const int *d_dirs, const float *d_anchors, const int *d_n, int max_boxes,
                              int pre_max, const sessd_dinms_cfg *cfg, float *d_out_boxes, float *d_out_scores, int *d_out_labels,
                              int *d_out_dirs, int *d_keep, int *d_selected, int *d_count, void *workspace, size_t workspace_bytes,
                              void *stream);

/* ------------------------------------------------------------------------------------------------
 * I1/I2: the iou3d_cuda extension.  Replaces det3d/core/iou3d/src/iou3d.cpp:34-281 (+ iou3d_kernel.cu
 * :270-365): same box layouts ([x1,y1,x2,y2,ry] / [x1,y1,z1,x2,y2,z2,ry]), caller-allocated outputs.
 * NMS variants take boxes already sorted by descending score (iou3d_utils.py:254-306) and do the greedy
 * reduction ON DEVICE (the reference copies the N x N/64 mask to the host, iou3d.cpp:131-158).
 * ------------------------------------------------------------------------------------------------ */
int sessd_boxes_overlap_bev(const float *d_a, int n, const float *d_b, int m, float *d_out, void *stream);
int sessd_boxes_aligned_overlap_bev(const float *d_a, const float *d_b, int n, float *d_out, void *stream);
int sessd_boxes_iou_bev(const float *d_a, int n, const float *d_b, int m, float *d_out, void *stream);
int sessd_boxes_iou3d(const float *d_a, int n, const float *d_b, int m, float *d_out, void *stream);
size_t sessd_nms_workspace_bytes(int n);
/* mode 0: rotated BEV (nms_gpu), 1: 3-D (nms_3d_gpu), 2: axis-aligned (nms_normal_gpu);
 * d_keep [n] int64 (device), d_num_keep [1] i32 (device) */
int sessd_nms_sorted(const float *d_boxes, int n, float thresh, int mode, long long *d_keep, int *d_num_keep,
                     void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * T1 (SURVEY.md 8(f) row 3): IoU target assignment of the SSD head, batched over frames on the device.
 * Replaces the DataLoader-worker path det3d/core/anchor/target_assigner.py:68-136 (TargetAssigner.assign_v2 with
 * enable_similar_type=True: every GT is class 1) -> det3d/core/anchor/target_ops_v2.py:11-126 (create_target_np) with
 * NearestIouSimilarity (det3d/core/bbox/region_similarity.py:85-98; box_np_ops.py:354-366, :1007-1046 iou_jit eps=0)
 * and second_box_encode (det3d/core/bbox/box_np_ops.py:52-113), called from AssignTarget
 * (det3d/datasets/pipelines/preprocess.py:286-358).
 *   d_anchors [A,7] (x,y,z,w,l,h,r), shared by all frames; d_gt_boxes [batch,max_gt,7] padded, d_num_gt [batch].
 *   d_labels [batch,A] (1 positive / 0 negative / -1 ignore), d_bbox_targets [batch,A,7] (zeros off the positives),
 *   d_bbox_outside_weights [batch,A] (1 on positives), d_pos_anchor / d_pos_gt_id [batch,A]: the first d_num_pos[b]
 *   entries of row b are the positive anchors in ascending order and their GT index (`positive_gt_id`).
 * labels / positive sets are bit-exact against the reference (its mixed fp32/fp64 IoU rounding is reproduced).
 * max_gt <= 1024.  Workspace: sessd_assign_workspace_bytes().  num_anchors < 1, batch < 1 or max_gt outside [0, 1024]: SESSD_EINVAL.
 * A frame uses the first min(d_num_gt[b], max_gt) GT rows: num_gt above max_gt assigns from gt[:max_gt]; num_gt <= 0 (or max_gt 0,
 * when d_gt_boxes may be null) makes every anchor of the frame background.
 * ------------------------------------------------------------------------------------------------ */
size_t sessd_assign_workspace_bytes(int num_anchors, int batch, int max_gt);
int sessd_assign_targets(const float *d_anchors, int num_anchors, const float *d_gt_boxes, const int *d_num_gt, int batch,
                         int max_gt, float matched_thr, float unmatched_thr, int *d_labels, float *d_bbox_targets,
                         float *d_bbox_outside_weights, int *d_pos_anchor, int *d_pos_gt_id, int *d_num_pos,
                         void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Training augmentation: per-object noise, global flip / rotation / scaling, shuffle (csrc/augment.cu).  Replaces the numba loops of det3d/core/sampler/preprocess.py that
 * noise_per_object_v4_ (:614-658, called from det3d/datasets/pipelines/preprocess.py:110-121) runs on every training frame.  The random
 * draws are made on the host (sessd_b200/augment.py, a numpy RandomState in the reference's order); these calls are pure functions
 * of the boxes and the draws, evaluated in fp64 like the reference (see the file header for the rounding).
 * sessd_box_collision -- box_collision_test (:944-1027, clockwise): d_out[i, j] = 1 when BEV corner set i of d_boxes [n, 4, 2] and j of
 *     d_qboxes [k, 4, 2] (fp64, box2d_to_corner_jit order) collide: standup pre-test, segment crossing, containment either way.
 * sessd_noise_per_box -- noise_per_box (:579-611) over a padded batch: d_gt_boxes [batch, max_gt, 7] f32 (x y z w l h r), d_num_gt
 *     [batch] (device), d_valid [batch, max_gt] u8 (gt_boxes_mask: the box's class is a target class), d_loc_noise [batch, max_gt,
 *     num_try, 3] and d_rot_noise [batch, max_gt, num_try] fp64 (the draws), context = data_aug_with_context (<= 0: none; > 0 enlarges
 *     w and l).  d_selected [batch, max_gt] i32: the try each valid box takes, -1 when every try collides, for invalid boxes and for
 *     the padding.  max_gt <= SESSD_AUGMENT_MAX_GT, num_try <= SESSD_AUGMENT_MAX_TRY (SESSD_ECAPACITY above); no workspace.
 * ------------------------------------------------------------------------------------------------ */
#define SESSD_AUGMENT_MAX_GT 256
#define SESSD_AUGMENT_MAX_TRY 128
int sessd_box_collision(const double *d_boxes, int n, const double *d_qboxes, int k, uint8_t *d_out, void *stream);
int sessd_noise_per_box(const float *d_gt_boxes, const int *d_num_gt, const uint8_t *d_valid, int batch, int max_gt,
                        const double *d_loc_noise, const double *d_rot_noise, int num_try, double context, int *d_selected,
                        void *stream);
/* sessd_augment_points -- points_transform_ (:545-560) with the membership of points_in_convex_polygon_3d_jit (:634-646), the raw
 *     twin (pipelines/preprocess.py:131), random_flip_v2 / global_rotation_v3 / global_scaling_v3 (:896-941) and the shuffle
 *     (pipelines/preprocess.py:159-161) in one pass.  d_points [*, 4] f32 with d_frame_off [batch + 1] (device); max_frame_points: the
 *     largest frame (sizes the grid); boxes, valid and draws as for sessd_noise_per_box and its d_selected; d_global [batch, 5] f32 =
 *     fp32 cos, fp32 sin of the global angle, fp32 scale, flip (0 / 1), fp32 angle; d_perm [*] i32: frame-local permutation, student
 *     row k of frame f = point d_perm[off + k] of the frame; d_labeled [batch] u8 (nullable: all labelled; an unlabelled frame is
 *     shuffled, flipped, rotated and scaled only, pipelines/preprocess.py:163-167).  A point moves with the first VALID box holding it
 *     (pre-noise boxes).  Outputs: d_points_raw (nullable) = the noised points before the global stages, unshuffled (rows of unlabelled
 *     frames untouched); d_points_out = the student's points.  d_points, d_points_raw and d_points_out are read / written as float4
 *     rows and must be 16-byte aligned (SESSD_EINVAL otherwise).  d_perm must hold a permutation of [0, n_f) per frame; a row whose
 *     entry is out of range is left unwritten (never an out-of-bounds access).
 * sessd_augment_boxes -- box3d_transform_ (:562-567), the valid-box selection, the global stages on the boxes, then the bookkeeping of
 *     Voxelization / AssignTarget (pipelines/preprocess.py:200-205, :290-330): both sets keep the boxes that are valid and in d_target
 *     (u8 [batch, max_gt], nullable: all), the student's set also drops the boxes with no BEV corner strictly inside range_bev (HOST
 *     float[4] x0 y0 x1 y1, filter_gt_box_outside_range); angles -> limit_period(r, 0.5, 2 pi); compacted in index order into
 *     d_boxes_raw / d_boxes_out [batch, max_gt, 7] (zero padded) with d_num_raw / d_num_out [batch]: the layout sessd_assign_targets reads.
 *     d_boxes_global [batch, max_gt, 7] f32 with d_num_global [batch] (nullable, both or neither: one without the other ->
 *     SESSD_EINVAL; d_boxes_global may be null when max_gt is 0): per frame, its class-valid boxes after the noise and the global
 *     stages, in index order, before the range filter and limit_period (the boxes Preprocess hands to pyramid_augment_v0), zero
 *     padded, with their count. */
/* sessd_points_in_boxes -- points_in_rbbox / points_in_convex_polygon_3d_jit over center_to_corner_box3d(origin 0.5) faces, as the
 *     point pass tests membership and as GT-AUG's point removal needs it: d_mask [n, m] u8 = point i (d_points rows of point_stride floats,
 *     x y z first) inside box j of d_boxes [m, 7] f32, w and l enlarged by context when it is positive.  The test is |R^T (p - c)| < dims/2
 *     in fp64: the reference's face-plane test holds the same points except within rounding of a face. */
int sessd_points_in_boxes(const float *d_points, int n, int point_stride, const float *d_boxes, int m, double context, uint8_t *d_mask,
                          void *stream);
int sessd_augment_points(const float *d_points, const int *d_frame_off, int batch, int max_frame_points, const float *d_gt_boxes,
                         const int *d_num_gt, const uint8_t *d_valid, int max_gt, const double *d_loc_noise, const double *d_rot_noise,
                         int num_try, const int *d_selected, double context, const float *d_global, const int *d_perm,
                         const uint8_t *d_labeled, float *d_points_raw, float *d_points_out, void *stream);
int sessd_augment_boxes(const float *d_gt_boxes, const int *d_num_gt, const uint8_t *d_valid, const uint8_t *d_target, int batch,
                        int max_gt, const double *d_loc_noise, const double *d_rot_noise, int num_try, const int *d_selected,
                        const float *d_global, const float *range_bev, float *d_boxes_raw, int *d_num_raw, float *d_boxes_out,
                        int *d_num_out, float *d_boxes_global, int *d_num_global, void *stream);

/* ------------------------------------------------------------------------------------------------
 * GT-database sampling (GT-AUG) of the training frames (csrc/gtaug.cu, csrc/augment.cu).  Replaces DataBaseSamplerV2.sample_class_v2's
 * acceptance (det3d/core/sampler/sample_ops_v2.py:238-276), the point half of sample_all (:133-150) and the paste of Preprocess.__call__
 * (det3d/datasets/pipelines/preprocess.py:96-110).  Which objects each frame draws is decided on the host (sessd_b200/augment.py,
 * det3d/core/sampler): the draws and the sampler's resets depend on every earlier frame.
 * sessd_gtaug_select_host -- HOST buffers, synchronous, no device: h_corners [num_boxes + num_cand, 4, 2] fp64 = the BEV corners of
 *     center_to_corner_box2d of [boxes so far | candidates] (candidates in sampler order); h_accepted [num_cand] u8 out: candidate c is
 *     accepted when its corner set collides (box_collision_test, the predicate of sessd_box_collision) with no box, no accepted
 *     candidate and no later candidate not yet rejected -- the loop of coll_mat[i].any() with rejected rows / columns cleared.  Returns
 *     the number accepted (>= 0), SESSD_EINVAL for null pointers or negative counts.
 * sessd_gtaug_paste -- device.  d_points [num_points, 4] f32 with d_frame_off [batch + 1] (the scene points); d_obj_off [batch + 1] i32 and
 *     d_obj_ids [num_objects] i32: the accepted database objects per frame (CSR, acceptance order); the resident database: d_db_points
 *     [*, 4] f32 (points relative to the box centre, as the database files hold them), d_db_off / d_db_count [db_size] i32 (first row and
 *     row count of each object), d_db_boxes [db_size, 7] f64 (box3d_lidar: the centre added back and the box whose points are removed).
 *     Output d_points_out [capacity, 4] with d_frame_off_out [batch + 1]: per frame, the pasted objects' points (fp32(rel + centre) in
 *     fp64, acceptance order), then the scene points outside every pasted box (points_in_rbbox, origin 0.5: the fp64 membership frame
 *     of sessd_points_in_boxes) in their original order.  max_paste_points: the host-known total row count of the accepted objects;
 *     capacity < num_points + max_paste_points -> SESSD_ECAPACITY, workspace_bytes < sessd_gtaug_paste_workspace_bytes(...) ->
 *     SESSD_EWORKSPACE.  d_points,
 *     d_db_points and d_points_out are float4 rows and must be 16-byte aligned (SESSD_EINVAL otherwise).  An object id outside
 *     [0, db_size) pastes no rows and removes no points (the ids are device memory, so it cannot be reported); no access is ever out of
 *     bounds.  The new frame offsets stay on the device.
 * ------------------------------------------------------------------------------------------------ */
int sessd_gtaug_select_host(const double *h_corners, int num_boxes, int num_cand, uint8_t *h_accepted);
size_t sessd_gtaug_paste_workspace_bytes(int batch, int num_points, int num_objects);
int sessd_gtaug_paste(const float *d_points, const int *d_frame_off, int batch, int num_points, const int *d_obj_off, const int *d_obj_ids,
                      int num_objects, int max_paste_points, const float *d_db_points, const int *d_db_off, const int *d_db_count,
                      const double *d_db_boxes, int db_size, void *d_workspace, size_t workspace_bytes, float *d_points_out, int capacity,
                      int *d_frame_off_out, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Shape-aware data augmentation (SA-DA) of the training frames (csrc/sada.cu).  Replaces pyramid_augment_v0 and its helpers
 * (det3d/datasets/utils/sa_da_v2.py): pyramid dropout, farthest-point sparsify and pyramid swap, one frame per call.  Every draw is made
 * on the host (sessd_b200/sada.py); the entries are pure functions of the points, the pyramids and the lists of pyramids each stage
 * acts on.  Points are [n, 4] f32 float4 rows and must be 16-byte aligned (SESSD_EINVAL otherwise).  All arithmetic is fp32 and
 * individually rounded in the reference's order, except the distances of the farthest-point sampling (fp64).  The boxes SA-DA acts on
 * are sessd_augment_boxes's d_boxes_global.
 * sessd_sada_pyramids -- device.  d_boxes [num_boxes, 7] f32 -> d_pyramids [num_boxes * 6, 15] (get_pyramids: the box centre, then the
 *     four corners of one face of center_to_corner_box3d(origin 0.5), faces box-major) and d_planes [num_boxes * 6, 5, 4] (normal and
 *     offset of each of the 5 surfaces, as surface_equ_3d_jitv2 computes them).  num_boxes <= SESSD_AUGMENT_MAX_GT; the pointers are
 *     required even when num_boxes is 0.
 * sessd_sada_membership -- device.  For the pyramid list d_ids [num_ids] (indices into d_planes [num_pyramids, 5, 4]; num_ids <=
 *     SESSD_SADA_MAX_IDS): d_bits [n, ceil(num_ids / 32)] u32 (optional, may be null) with bit a of point i set when the point lies
 *     strictly inside pyramid d_ids[a] (points_in_convex_polygon_3d_jit: a surface sign >= 0 is outside), and d_counts [num_ids] the
 *     number of points inside each.  An id outside [0, num_pyramids) holds no point.  Integer atomics only: deterministic.
 * sessd_sada_compact -- device.  Writes the rows of d_points that lie in no listed pyramid a with d_counts[a] > min_count (min_count < 0:
 *     every listed pyramid) to d_out in their order, and their number to d_num_out [1] (device).  capacity < n -> SESSD_ECAPACITY;
 *     workspace_bytes < sessd_sada_compact_workspace_bytes(n) -> SESSD_EWORKSPACE.
 * sessd_sada_fps -- device.  For each listed pyramid a with d_counts[a] > min_count, in list order: its points in row order, then k
 *     rows by exact farthest-point sampling (start at its first point; each step the point with the largest fp64 distance
 *     sqrt((dx^2 + dy^2) + dz^2) to its nearest picked point, ties to the first), written in pick order at d_out[*d_num + k * r], r =
 *     the number of such pyramids before a; *d_num (device, in: rows already in d_out) is advanced by k per such pyramid.  Requires
 *     min_count >= k - 1 (SESSD_EINVAL), capacity >= n + k * num_ids (SESSD_ECAPACITY) and sessd_sada_fps_workspace_bytes(n, num_ids)
 *     (SESSD_EWORKSPACE).  A pyramid of up to 4096 points is sampled from shared memory, a larger one from the workspace.
 * sessd_sada_swap -- device.  d_ids [2 * num_pairs]: to_swap pyramids, then their partners; d_bits / d_counts: sessd_sada_membership
 *     of that list over d_points; d_pyramids [num_pyramids, 15].  Pair p writes, from row *d_num_in on (device) and after the pairs
 *     before it, the partner's points in pyramid p's ratio coordinates (get_points_ratio / recover_points_by_ratio) with intensities
 *     through the min / max ratio (clip(max - min, 1e-6, 1)), then pyramid p's points in the partner's coordinates; *d_num_out is
 *     the frame's new size.  max_swap_points: the host-known sum of the listed counts; capacity < n + max_swap_points -> SESSD_ECAPACITY.
 *     A pair with an id outside [0, num_pyramids) writes nothing.
 * sessd_sada_shuffle -- device.  d_out[off_b + k] = d_points[off_b + d_perm[off_b + k]] for each frame b of d_frame_off [batch + 1];
 *     a row whose source is outside its frame is left unwritten.
 * ------------------------------------------------------------------------------------------------ */
#define SESSD_SADA_MAX_IDS (6 * SESSD_AUGMENT_MAX_GT)
int sessd_sada_pyramids(const float *d_boxes, int num_boxes, float *d_pyramids, float *d_planes, void *stream);
int sessd_sada_membership(const float *d_points, int n, const int *d_n, const float *d_planes, int num_pyramids, const int *d_ids, int num_ids,
                          uint32_t *d_bits, int *d_counts, void *stream);
size_t sessd_sada_compact_workspace_bytes(int n);
int sessd_sada_compact(const float *d_points, int n, const int *d_n, const uint32_t *d_bits, int num_ids, const int *d_counts, int min_count,
                       void *d_workspace, size_t workspace_bytes, float *d_out, int capacity, int *d_num_out, void *stream);
size_t sessd_sada_fps_workspace_bytes(int n, int num_ids);
int sessd_sada_fps(const float *d_points, int n, const int *d_n, const uint32_t *d_bits, int num_ids, const int *d_counts, int min_count, int k,
                   void *d_workspace, size_t workspace_bytes, float *d_out, int capacity, int *d_num, void *stream);
int sessd_sada_swap(const float *d_points, int n, const int *d_n, const uint32_t *d_bits, int num_pairs, const int *d_counts, const float *d_pyramids,
                    int num_pyramids, const int *d_ids, int max_swap_points, float *d_out, int capacity, const int *d_num_in,
                    int *d_num_out, void *stream);
int sessd_sada_shuffle(const float *d_points, const int *d_frame_off, int batch, int max_frame_points, const int *d_perm, float *d_out,
                       void *stream);

/* ------------------------------------------------------------------------------------------------
 * KITTI data preparation (csrc/kitti_prep.cu).  Replaces the membership tests of the reference's data preparation: remove_outside_points
 * (det3d/core/bbox/box_np_ops.py:981-992) in _create_reduced_point_cloud / _calculate_num_points_in_gt and points_in_rbbox (:1152-1157)
 * in _calculate_num_points_in_gt / create_groundtruth_database.  Every plane is computed on the host (sessd_b200/kitti_prep.py).  A
 * polyhedron is six planes [6, 4] fp64 (a, b, c, d); a point is inside when (((x*a) + (y*b)) + (z*c)) + d < 0 for all six, x y z the fp32
 * coordinates widened to fp64 and each operation rounded on its own (_points_in_convex_polygon_3d_jit: a sign >= 0 is outside).  Points
 * are [*, 4] f32 float4 rows and must be 16-byte aligned (SESSD_EINVAL otherwise); null pointers and negative counts are SESSD_EINVAL.
 * sessd_prep_frustum_compact -- device.  d_points [num_points, 4] with d_frame_off [batch + 1], d_planes [batch, 6, 4] (one image frustum
 *     per frame).  Writes the rows inside their frame's frustum to d_points_out as bit copies in frame order and the new offsets to
 *     d_frame_off_out [batch + 1] (device).  capacity < num_points -> SESSD_ECAPACITY; workspace_bytes <
 *     sessd_prep_frustum_compact_workspace_bytes(num_points) -> SESSD_EWORKSPACE.
 * sessd_prep_box_count -- device.  d_box_planes [num_boxes, 6, 4] with d_box_off [batch + 1] (CSR boxes per frame): d_counts [num_boxes]
 *     i32 = the points of the box's frame inside the box.  No workspace.
 * sessd_prep_box_gather -- device.  Same boxes plus d_centres [num_boxes, 3] f64 and d_counts from sessd_prep_box_count.  d_obj_off
 *     [num_boxes + 1] = the exclusive scan of the counts (device); box k's points, in frame order, go to rows [d_obj_off[k],
 *     d_obj_off[k + 1]) of d_rows_out as fp32(double(p) - centre) for x y z and the intensity unchanged.  A point inside two boxes is
 *     written for both.  num_rows: the host-known sum of the counts; capacity < num_rows -> SESSD_ECAPACITY; workspace_bytes <
 *     sessd_prep_box_gather_workspace_bytes(num_boxes) -> SESSD_EWORKSPACE.  No write is ever past the capacity.
 * ------------------------------------------------------------------------------------------------ */
size_t sessd_prep_frustum_compact_workspace_bytes(int num_points);
int sessd_prep_frustum_compact(const float *d_points, const int *d_frame_off, int batch, int num_points, const double *d_planes,
                               void *d_workspace, size_t workspace_bytes, float *d_points_out, int capacity, int *d_frame_off_out, void *stream);
int sessd_prep_box_count(const float *d_points, const int *d_frame_off, int batch, int num_points, const double *d_box_planes,
                         const int *d_box_off, int num_boxes, int *d_counts, void *stream);
size_t sessd_prep_box_gather_workspace_bytes(int num_boxes);
int sessd_prep_box_gather(const float *d_points, const int *d_frame_off, int batch, int num_points, const double *d_box_planes,
                          const double *d_centres, const int *d_box_off, int num_boxes, const int *d_counts, int num_rows, void *d_workspace,
                          size_t workspace_bytes, float *d_rows_out, int capacity, int *d_obj_off, void *stream);

/* ------------------------------------------------------------------------------------------------
 * SURVEY.md 8(f) row 1, first slice of the training step: the supervised SSD-head loss terms, value AND gradient in one pass.
 * Replaces (for the terms without the teacher model) det3d/models/bbox_heads/mg_head_sessd.py:706-760:
 * prepare_loss_weights/NormByNumPositives (:525-572), SigmoidFocalLoss (det3d/models/losses/losses.py:345-420, gamma = 2),
 * add_sin_difference + WeightedSmoothL1Loss (mg_head_sessd.py:39-44, losses.py:147-204), get_direction_target +
 * WeightedSoftmaxClassificationLoss (mg_head_sessd.py:62-76, losses.py:489-531) and their autograd backward.
 *   d_head [batch, A/2, head_stride]: the fused head tensor (box 2x7 | cls 2 | dir 2x2 | iou 2 | pad), as sessd_postprocess reads it;
 *   d_labels [batch, A] (1 / 0 / -1) and d_reg_targets [batch, A, 7]: outputs of sessd_assign_targets; d_anchors [A, 7].
 *   d_losses [batch, 8] = per-frame SUMS {cls, loc, dir, cls on positives, cls on negatives, 0, num_pos, num_neg} (the reference
 *   reports loss_weight * batch total / batch); d_grad_head (nullable) [batch, A/2, head_stride] = d/d_head of
 *   (w_cls * sum cls + w_loc * sum loc + w_dir * sum dir) / batch.  Sums are reduced in a fixed order (deterministic).
 * ------------------------------------------------------------------------------------------------ */
size_t sessd_head_loss_workspace_bytes(int batch);
/* IoU-prediction term (mg_head_sessd.py:755-768): smooth-L1 of the head's iou output against 2 * aligned-3D-IoU(decoded prediction,
 * decoded target) - 1 on the positives (det3d/core/iou3d/iou3d_utils.py:197-252 as the constant target).  Run AFTER sessd_head_loss on the
 * same stream: reads num_pos from d_losses[b][6], writes the per-frame sum to d_losses[b][5] and d(w_iou * sum / batch) into the iou
 * channels of d_grad_head.  num_anchors must be a multiple of anchors_per_loc (SESSD_EINVAL otherwise, before any launch). */
/* ODIoU box-regression loss (det3d/models/losses/odious.py:845-900 called from mg_head_sessd.py:770-778; the reference evaluates it with
 * per-box numpy loops on the CPU inside the training step): odiou = 1 - IoU3D + centre distance^2 / (min bounding rectangle diagonal^2 +
 * inter_h^2) + 1.25 (1 - |cos dr|) between the decoded prediction and the decoded target of every positive anchor, weight 1 / num_pos.
 * Run AFTER sessd_head_loss on the same stream (reads num_pos from d_losses[b][6]); d_odiou_sum [batch] receives the per-frame sums,
 * and w_odiou * d(sum over frames) / batch is ADDED to the box channels of d_grad_head (nullable).  The reference's ious_loss is
 * 2.0 * batch total / batch_size: pass w_odiou = 2.0.  Gradients are exact (forward-mode differentiation of the same arithmetic). */
size_t sessd_odiou_loss_workspace_bytes(int batch);
int sessd_odiou_loss(const float *d_head, const float *d_anchors, const int *d_labels, const float *d_reg_targets, int batch,
                     int num_anchors, int anchors_per_loc, int head_stride, float w_odiou, const float *d_losses, float *d_odiou_sum,
                     float *d_grad_head, void *workspace, size_t workspace_bytes, void *stream);
/* HOST evaluation of the identical arithmetic for n (target, prediction) box pairs [n,7]: odiou values [n] and d(odiou)/d(prediction)
 * [n,7] (nullable).  Used to pin the kernel's math to the reference's odiou_3D on the CPU; not a fallback of the device path. */
int sessd_odiou_pairs_host(const float *h_gboxes, const float *h_qboxes, int n, float *h_odiou, float *h_grad_q);
size_t sessd_iou_pred_loss_workspace_bytes(int batch);
int sessd_iou_pred_loss(const float *d_head, const float *d_anchors, const int *d_labels, const float *d_reg_targets, int batch,
                        int num_anchors, int anchors_per_loc, int head_stride, float sigma, float w_iou, float *d_losses,
                        float *d_grad_head, void *workspace, size_t workspace_bytes, void *stream);
int sessd_head_loss(const float *d_head, const float *d_anchors, const int *d_labels, const float *d_reg_targets, int batch,
                    int num_anchors, int anchors_per_loc, int head_stride, float alpha, float sigma, float dir_offset,
                    float pos_cls_weight, float neg_cls_weight, float w_cls, float w_loc, float w_dir, float *d_losses,
                    float *d_grad_head, void *workspace, size_t workspace_bytes, void *stream);

/* ------------------------------------------------------------------------------------------------
 * Training step, optimiser side (SURVEY 8(f) rows 1-2), over flat fp32 arenas (csrc/train.cu):
 * sessd_axpby  -- d_y = a d_y + b d_x: the teacher's exponential moving average of det3d/torchie/trainer/trainer_sessd.py:315-318 in one
 *                 launch (a = alpha, b = 1 - alpha), and the 1 / world_size scaling after the gradient all-reduce
 *                 (det3d/core/utils/dist_utils.py:8-29) with d_x = NULL;
 * sessd_adamw_step -- Adam with decoupled weight decay (the fastai true_wd step of det3d/solver/fastai_optim.py == torch.optim.AdamW).
 * sessd_grad_sqnorm -- the gradient clip of det3d/torchie/trainer/hooks/optimizer.py:35-62 (clip_grad_norm_(params, max_norm=35,
 *                 norm_type=2), optimizer_config of examples/second/configs/config.py:257-260) without a host round trip: d_out[0] =
 *                 total_norm (fp32, sqrt of an fp64 sum, rounded once), d_out[1] = clip_coef = min(1, max_norm / (total_norm + 1e-6)),
 *                 both on the device.  Bitwise deterministic run to run and across SM counts (the chunking depends on n only), so DDP
 *                 ranks holding the same all-reduced arena clip identically.  d_workspace: sessd_grad_sqnorm_workspace_bytes(n) bytes,
 *                 zero-filled once before first use, one stream at a time.
 * sessd_adamw_clip_ema_step -- sessd_adamw_step (the same kernel) with the gradient scaled by *d_clip_coef and stored back, and the
 *                 teacher EMA of det3d/torchie/trainer/trainer_sessd.py:315-318 (ema = alpha ema + (1 - alpha) p_new, with a = (float)alpha,
 *                 b = (float)(1 - alpha) as sessd_axpby takes them) in the same pass; d_clip_coef and d_ema are nullable.  beta1 is the
 *                 one-cycle momentum of the step (det3d/solver/learning_schedules_fastai.py:7-100); bias corrections use it.
 * ------------------------------------------------------------------------------------------------ */
int sessd_axpby(float *d_y, const float *d_x, float a, float b, long long n, void *stream);
int sessd_adamw_step(float *d_param, const float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, long long n, float lr, float beta1,
                     float beta2, float eps, float weight_decay, int step, void *stream);
size_t sessd_grad_sqnorm_workspace_bytes(long long n);
int sessd_grad_sqnorm(const float *d_x, long long n, float max_norm, float *d_out, void *d_workspace, void *stream);
int sessd_adamw_clip_ema_step(float *d_param, float *d_grad, float *d_exp_avg, float *d_exp_avg_sq, long long n, float lr, float beta1,
                              float beta2, float eps, float weight_decay, int step, const float *d_clip_coef, float *d_ema, double ema_alpha,
                              void *stream);

/* ------------------------------------------------------------------------------------------------
 * KITTI object evaluation (csrc/kitti_eval.cu): det3d/datasets/kitti/kitti.py convert_detection_to_kitti_annos and
 * det3d/datasets/kitti/eval.py eval_class_v3 on flat arrays.  The precision of every step is written down in the kernel file.
 *
 * A box record is SESSD_KITTI_REC doubles: bbox x0 y0 x1 y1, alpha, location x y z, dimensions (l h w), rotation_y, then the score
 * (detections) or the truncation (ground truth).  Class codes: the index into the evaluation's class list (car 0, pedestrian 1,
 * bicycle 2, truck 3, bus 4, trailer 5, construction_vehicle 6, motorcycle 7, barrier 8, traffic_cone 9, cyclist 10) of the
 * lower-cased name, SESSD_KITTI_PERSON_SITTING, SESSD_KITTI_VAN (the neighbour classes of pedestrian and car), -1 for any other
 * name.  DontCare boxes (names "DontCare" / "ignore") are passed once more, as 2D boxes, in their own CSR list.
 *
 * sessd_kitti_convert_detections -- one thread per lidar detection (x y z w l h ry, fp32): camera record, image box, alpha; boxes
 *     outside the image are dropped and the rest kept in input order, frame f's kept records at d_rec[d_off[f] ...] (the input's
 *     slots) and their count in d_cnt[f].  d_calib [F, 24] fp64: rows 0-2 of R0_rect . Tr_velo_to_cam, rows 0-2 of P2;
 *     d_image_hw [F, 2] (height, width).  d_code[j] = d_label_code[label] (-1 for labels outside [0, num_labels)).  capacity =
 *     d_off[F].  workspace: sessd_kitti_convert_workspace_bytes(capacity).
 * sessd_kitti_overlaps -- the block-diagonal overlap of one metric (0 2D, 1 BEV, 2 3D): frame f's [dt_cnt[f], n_gt_f] block, row
 *     stride n_gt_f, at d_overlaps + ov_off[f].  z_axis / z_center: (1, 1.0) for KITTI camera boxes, (2, 0.5) for lidar boxes.
 * sessd_kitti_eval -- overlaps, both matching passes, get_thresholds and the curves of one metric for num_configs configs d_cfg
 *     [n, 2] = (class code, difficulty 0-2) with d_min_overlap [n].  Outputs per config: d_thresholds / d_precision / d_aos [n, 41]
 *     (zero past d_num_thresholds[c]), d_map [n, 4] = R11 precision, R40 precision, R11 AOS, R40 AOS (get_mAP / get_mAP_v2, in
 *     percent).  A config with no valid ground truth has no thresholds and AP 0.  max_frame_dt: the largest dt_off[f+1] - dt_off[f]
 *     (SESSD_ECAPACITY above 1024).  This is the frame's capacity, not dt_cnt[f]: a frame of 1025 input detections is refused
 *     even when the conversion kept 1024 or fewer.  total_gt = gt_off[F]; overlap_elems = ov_off[F].  Bitwise deterministic run to run.  The
 *     workspace holds the overlaps, 2 x num_configs x total_gt fp64 scores and, with compute_aos, one fp64 similarity per (config,
 *     threshold, frame) for the frame-ordered sum: num_configs x 41 x F doubles (133 MB for 108 configs over 3769 frames).
 * ------------------------------------------------------------------------------------------------ */
#define SESSD_KITTI_REC 13
#define SESSD_KITTI_PERSON_SITTING 11
#define SESSD_KITTI_VAN 12
typedef struct {
    int num_frames;
    const int *gt_off;        /* [F+1] CSR of ground-truth boxes */
    const double *gt;         /* [n_gt, SESSD_KITTI_REC] */
    const int *gt_code;       /* [n_gt] */
    const int *gt_occluded;   /* [n_gt] */
    const int *dc_off;        /* [F+1] CSR of DontCare boxes */
    const double *dc;         /* [n_dc, 4] (may be NULL when there are none) */
    const int *dt_off;        /* [F+1] CSR capacity of detections */
    const int *dt_cnt;        /* [F] detections held by frame f (<= its capacity) */
    const double *dt;         /* [dt_off[F], SESSD_KITTI_REC] */
    const int *dt_code;       /* [dt_off[F]] */
    const long long *ov_off;  /* [F+1] start of frame f's overlap block; block f holds at least dt_cnt[f] * n_gt_f values */
} SessdKittiFrames;
size_t sessd_kitti_convert_workspace_bytes(long long capacity);
int sessd_kitti_convert_detections(const float *d_boxes7, const float *d_scores, const int *d_labels, const int *d_off, int num_frames,
                                   long long capacity, const double *d_calib, const int *d_image_hw, const int *d_label_code,
                                   int num_labels, double *d_rec, int *d_label, int *d_code, int *d_cnt, void *workspace,
                                   size_t workspace_bytes, void *stream);
int sessd_kitti_overlaps(const SessdKittiFrames *frames, int metric, int z_axis, double z_center, double *d_overlaps, void *stream);
size_t sessd_kitti_eval_workspace_bytes(int num_frames, long long total_gt, long long overlap_elems, int num_configs, int compute_aos);
int sessd_kitti_eval(const SessdKittiFrames *frames, int max_frame_dt, int metric, int z_axis, double z_center, int num_configs,
                     const int *d_cfg, const double *d_min_overlap, int compute_aos, long long total_gt, long long overlap_elems,
                     double *d_thresholds, int *d_num_thresholds, double *d_precision, double *d_aos, double *d_map, void *workspace,
                     size_t workspace_bytes, void *stream);

#ifdef __cplusplus
}
#endif
#endif
