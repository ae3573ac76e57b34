"""Tensor-level wrappers over the C ABI (PyTorch supplies device memory and streams only).

Every function launches asynchronously on ``torch.cuda.current_stream()`` and never synchronises; data-dependent
row counts stay on the device as int32 tensors (``n`` arguments), buffers are capacity sized.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import ConvDesc, DinmsCfg, Grid, PostCfg, VoxelCfg, check, lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _st():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _cuda(t, dtype, name):
    if not (isinstance(t, torch.Tensor) and t.is_cuda and t.dtype == dtype and t.is_contiguous()):
        raise ValueError("%s must be a contiguous CUDA %s tensor" % (name, dtype))
    return t


def _i3(v):
    return (C.c_int * 3)(*[int(x) for x in v])


def make_grid(batch, shape_dhw):
    g = Grid()
    g.batch = int(batch)
    g.shape[0], g.shape[1], g.shape[2] = [int(v) for v in shape_dhw]
    return g


# ------------------------------------------------------------------------------------------------ voxeliser
def make_voxel_cfg(voxel_size, pc_range, max_points, max_voxels, num_feat=4):
    cfg = VoxelCfg()
    vs = np.asarray(voxel_size, np.float32)
    rg = np.asarray(pc_range, np.float32)
    grid = np.round((rg[3:] - rg[:3]) / vs).astype(np.int64)      # voxel_generator.py:15-16
    for j in range(3):
        cfg.voxel_size[j] = float(vs[j])
        cfg.range_min[j] = float(rg[j])
        cfg.range_max[j] = float(rg[3 + j])
        cfg.grid[j] = int(grid[j])
    cfg.max_points, cfg.max_voxels, cfg.num_feat = int(max_points), int(max_voxels), int(num_feat)
    return cfg


class VoxelBuffers:
    """Capacity-sized outputs + workspace of the batched voxeliser (reused across frames / graph replays)."""

    def __init__(self, cfg, batch, max_total_points, device, with_mean=True):
        self.cfg, self.batch, self.max_total_points = cfg, batch, max_total_points
        nv = batch * cfg.max_voxels
        self.voxels = torch.empty((nv, cfg.max_points, cfg.num_feat), dtype=torch.float32, device=device)
        self.coors = torch.empty((nv, 4), dtype=torch.int32, device=device)
        self.num_points = torch.empty((nv,), dtype=torch.int32, device=device)
        self.mean = torch.empty((nv, cfg.num_feat), dtype=torch.float32, device=device) if with_mean else None
        self.num_voxels = torch.zeros((batch + 1,), dtype=torch.int32, device=device)
        ws = lib.sessd_voxelize_workspace_bytes(max_total_points, batch, C.byref(cfg))
        self.ws = torch.empty((ws,), dtype=torch.uint8, device=device)


def voxelize(points, frame_off, buf):
    """points [P,F] f32 cuda (P <= buf.max_total_points), frame_off [B+1] i32 cuda -> fills buf."""
    _cuda(points, torch.float32, "points")
    _cuda(frame_off, torch.int32, "frame_off")
    if points.shape[0] > buf.max_total_points or points.shape[1] != buf.cfg.num_feat or frame_off.numel() != buf.batch + 1:
        raise ValueError("voxelize: shape/capacity mismatch")
    rc = lib.sessd_voxelize(_p(points), _p(frame_off), buf.batch, buf.max_total_points, C.byref(buf.cfg), _p(buf.voxels),
                            _p(buf.coors), _p(buf.num_points), _p(buf.mean), _p(buf.num_voxels), _p(buf.ws), buf.ws.numel(), _st())
    check(rc, "sessd_voxelize")
    return buf


def voxelize_host(points_np, cfg):
    """numpy in / numpy out single-frame path (VoxelGenerator.generate)."""
    pts = np.ascontiguousarray(points_np, np.float32)
    if pts.ndim != 2 or pts.shape[1] != cfg.num_feat:
        raise ValueError("points must be [N,%d]" % cfg.num_feat)
    voxels = np.zeros((cfg.max_voxels, cfg.max_points, cfg.num_feat), np.float32)
    coors = np.zeros((cfg.max_voxels, 3), np.int32)
    num = np.zeros((cfg.max_voxels,), np.int32)
    m = lib.sessd_voxelize_host(pts.ctypes.data_as(C.c_void_p), pts.shape[0], C.byref(cfg), voxels.ctypes.data_as(C.c_void_p),
                                coors.ctypes.data_as(C.c_void_p), num.ctypes.data_as(C.c_void_p))
    if m < 0:
        raise _lib.SessdError("sessd_voxelize_host failed (%d)" % m)
    return voxels[:m].copy(), coors[:m].copy(), num[:m].copy()


# ------------------------------------------------------------------------------------------------ rulebook
def hash_capacity(max_rows):
    cap = C.c_int(0)
    lib.sessd_hash_bytes(int(max_rows), C.byref(cap))
    return cap.value


def hash_build(coors, n, max_rows, grid, table=None):
    cap = hash_capacity(max_rows)
    if table is None:
        table = torch.empty((cap,), dtype=torch.int64, device=coors.device)
    check(lib.sessd_hash_build(_p(coors), _p(n), int(max_rows), grid, _p(table), cap, _st()), "sessd_hash_build")
    return table


def bitmap_alloc(grid, device):
    words = lib.sessd_bitmap_words(grid)
    bitmap = torch.empty((words, 2), dtype=torch.int32, device=device)
    scratch = torch.empty((lib.sessd_scan_scratch_bytes(words),), dtype=torch.uint8, device=device)
    return bitmap, scratch


def subm_rulebook(coors, n, max_rows, grid, ksize, index_kind, index, nbr=None):
    kvol = int(ksize[0] * ksize[1] * ksize[2])
    if nbr is None:
        nbr = torch.empty((max_rows, kvol), dtype=torch.int32, device=coors.device)
    cap = index.numel() if index_kind == 0 else 0
    check(lib.sessd_subm_rulebook(_p(coors), _p(n), int(max_rows), grid, _i3(ksize), int(index_kind), _p(index), cap, _p(nbr), _st()),
          "sessd_subm_rulebook")
    return nbr


def strided_rulebook(in_coors, n_in, max_in, in_grid, in_index_kind, in_index, ksize, stride, padding, out_grid, bitmap,
                     scratch, out_coors, n_out, max_out, nbr, status):
    cap = in_index.numel() if in_index_kind == 0 else 0
    check(lib.sessd_strided_rulebook(_p(in_coors), _p(n_in), int(max_in), in_grid, int(in_index_kind), _p(in_index), cap, _i3(ksize),
                                     _i3(stride), _i3(padding), out_grid, _p(bitmap), _p(scratch), _p(out_coors), _p(n_out),
                                     int(max_out), _p(nbr), _p(status), _st()), "sessd_strided_rulebook")


# ------------------------------------------------------------------------------------------------ sparse conv
def spconv_forward(in_feat, nbr, n_out, max_out, weight, scale, shift, relu, out=None):
    """in_feat [*,Cin]; nbr [max_out,kvol]; weight [kvol,Cin,Cout]; scale/shift [Cout] or None."""
    kvol, cin, cout = weight.shape
    if out is None:
        out = torch.empty((max_out, cout), dtype=torch.float32, device=in_feat.device)
    check(lib.sessd_spconv_forward(_p(in_feat), int(cin), _p(nbr), int(kvol), _p(n_out), int(max_out), _p(weight), int(cout),
                                   _p(scale), _p(shift), int(bool(relu)), _p(out), _st()), "sessd_spconv_forward")
    return out


def spconv_forward_rows(in_feat, nbr, n_out, max_out, weight, scale, shift, relu, out, amax_out=None):
    """Pair-proportional fp32 kernel for the narrow layers (Cin <= 32); same arguments as spconv_forward (+ optional abs-max output)."""
    kvol, cin, cout = weight.shape
    check(lib.sessd_spconv_forward_rows(_p(in_feat), int(cin), _p(nbr), int(kvol), _p(n_out), int(max_out), _p(weight), int(cout),
                                        _p(scale), _p(shift), int(bool(relu)), _p(out), _p(amax_out), _st()), "sessd_spconv_forward_rows")
    return out


def _fp16_split(wt):
    """[taps, Cout, Cin] fp32 -> (hi, lo, 2^-e[Cout]): every output channel is scaled by the power of two 2^e[n] that puts its largest
    |w| into [2^10, 2^11); hi = fp16_rn(2^e w), lo = fp16_rn(2^e w - hi)"""
    amax = wt.abs().amax(dim=(0, 2))
    _, ex = torch.frexp(amax)                       # amax = m * 2^ex, m in [0.5, 1)
    e = torch.where(amax > 0, 11 - ex, torch.zeros_like(ex)).clamp(-100, 100).to(torch.float32)
    ws = wt * torch.exp2(e)[None, :, None]
    hi = ws.to(torch.float16)
    return hi, (ws - hi.to(torch.float32)).to(torch.float16), torch.exp2(-e).contiguous()


def pack_weight_sp_h2(wp, cp):
    """[kvol, Cin, Cout] (spconv layout, flattened offsets) -> (fp16 weight tiles [kvol, 2 (hi, lo), Cout, cp] of
    sessd_spconv_forward_cg, 2^-e[Cout]) at the plane width cp = Cin of the layer's input (32 or 64); the fp16 split of _fp16_split."""
    kvol, cin, cout = wp.shape
    assert cp in (32, 64) and cin == cp
    hi, lo, inv = _fp16_split(wp.permute(0, 2, 1).contiguous().to(torch.float32))
    return torch.stack([hi, lo], 1).contiguous(), inv


def alloc_planes(max_rows, cp, device):
    """fp16 (hi, lo) planes of a sparse feature tensor: [max_rows + 1, 2 * cp]; the extra last row stays zero (missing neighbours)."""
    return torch.zeros((max_rows + 1, 2 * cp), dtype=torch.float16, device=device)


def absmax_rows(feat, n, max_rows, amax):
    check(lib.sessd_absmax_rows(_p(feat), _p(n), int(max_rows), int(feat.shape[1]), _p(amax), _st()), "sessd_absmax_rows")
    return amax


def spconv_forward_rows_planes(in_feat, nbr, n_out, max_out, weight, scale, shift, relu, amax_in, gain, shift_max, out, out_planes, out_info):
    """spconv_forward_rows that also (out nullable: only) writes the output as fp16 (hi, lo) planes [rows, 2 * cpo] with
    out_info = {abs-max (atomicMax), scale}; the scale is derived from the bound amax_in * gain + shift_max."""
    kvol, cin, cout = weight.shape
    check(lib.sessd_spconv_forward_rows_planes(_p(in_feat), int(cin), _p(nbr), int(kvol), _p(n_out), int(max_out), _p(weight), int(cout),
                                               _p(scale), _p(shift), int(bool(relu)), _p(amax_in), float(gain), float(shift_max), _p(out),
                                               _p(out_planes), int(out_planes.shape[1] // 2), _p(out_info), _st()),
          "sessd_spconv_forward_rows_planes")
    return out_planes


def alloc_tile_lists(max_out, kvol, device):
    """buffer of the per-tile pair lists of one rulebook (rulebook_tile_lists)"""
    return torch.zeros((-(-int(max_out) // 128), int(lib.sessd_tile_list_stride(int(kvol)))), dtype=torch.int32, device=device)


def rulebook_tile_lists(nbr, n_out, max_out, tiles):
    """nbr table [max_out, kvol] -> per-tile pair lists (counts, row masks, (input row << 7 | tile row) grouped by kernel offset): the
    rulebook format of spconv_forward_cg.  Once per rulebook build."""
    check(lib.sessd_rulebook_tile_lists(_p(nbr), int(nbr.shape[1]), _p(n_out), int(max_out), _p(tiles), _st()), "sessd_rulebook_tile_lists")
    return tiles


def spconv_forward_cg(in_planes, in_info, tiles, n_out, max_out, weight_h2, scale, shift, relu, gain, shift_max, out, out_planes, out_info):
    """Pair-proportional tensor-core sparse conv (csrc/spconv_cg.cu).  in_planes [rows, 2 * cp] fp16 with in_info = {abs-max, scale};
    tiles from rulebook_tile_lists; weight_h2 / scale from pack_weight_sp_h2 (scale = bn_scale * 2^-e); out (fp32 rows) and / or
    out_planes + out_info."""
    cp = in_planes.shape[1] // 2
    kvol = weight_h2.shape[0]
    cout = weight_h2.shape[2]
    check(lib.sessd_spconv_forward_cg(_p(in_planes), int(cp), int(in_planes.shape[0]), _p(in_info), _p(tiles), int(kvol), _p(n_out), int(max_out),
                                      _p(weight_h2), int(cout), _p(scale), _p(shift), int(bool(relu)), float(gain), float(shift_max), _p(out),
                                      _p(out_planes), _p(out_info), _st()), "sessd_spconv_forward_cg")
    return out if out is not None else out_planes


def set_sp_cg_deep(on):
    """spconv_forward_cg: 1 = deep pipeline, one CTA per SM (launches with fewer tiles than SMs: single frames); 0 = two CTAs per SM"""
    lib.sessd_set_sp_cg_deep(int(on))


def spconv_cg_blocks_per_sm(cp, cout, deep=0):
    """CTAs of spconv_forward_cg's (cp, cout, deep) kernel resident on one SM of the current device"""
    n = int(lib.sessd_spconv_cg_blocks_per_sm(int(cp), int(cout), int(deep)))
    check(min(n, 0), "sessd_spconv_cg_blocks_per_sm")
    return n


# ---- backward of the sparse convs (csrc/spconv_grad.cu) -------------------------------------------------------------------------
def rulebook_transpose(nbr, n_out, max_out, max_in, nbr_t=None):
    """nbr [max_out, kvol] -> nbr_t [max_in, kvol]: nbr_t[i, k] = o where nbr[o, k] = i, else -1 (strided layers' data gradient)"""
    kvol = int(nbr.shape[1])
    if nbr_t is None:
        nbr_t = torch.empty((int(max_in), kvol), dtype=torch.int32, device=nbr.device)
    check(lib.sessd_rulebook_transpose(_p(nbr), kvol, _p(n_out), int(max_out), int(max_in), _p(nbr_t), _st()), "sessd_rulebook_transpose")
    return nbr_t


def sparse_split_planes(x, n, max_rows, info, planes):
    """fp32 rows [max_rows, C] -> fp16 (hi, lo) planes [rows, 2 * cp] at the power-of-two scale of info[0] (abs-max: absmax_rows first);
    info[1] <- the scale"""
    check(lib.sessd_sparse_split_planes(_p(x), _p(n), int(max_rows), int(x.shape[1]), _p(info), _p(planes), int(planes.shape[1] // 2), _st()),
          "sessd_sparse_split_planes")
    return planes


def dense_grad_gather(grad, coors, n, max_rows, grid, channels, out=None):
    """adjoint of sparse_to_dense: grad NHWC [B, H, W, C*D] (contiguous) -> rows [max_rows, C] (rows >= n untouched)"""
    if out is None:
        out = torch.empty((int(max_rows), int(channels)), dtype=torch.float32, device=grad.device)
    check(lib.sessd_dense_grad_gather(_p(grad), _p(coors), _p(n), int(max_rows), int(channels), grid, _p(out), _st()), "sessd_dense_grad_gather")
    return out


def wgrad_items(max_out, kvol):
    """work items of one weight-gradient launch (a function of max_out and kvol only)"""
    return int(lib.sessd_spconv_wgrad_items(int(max_out), int(kvol)))


def wgrad_workspace(max_out, kvol, cin, cout, device):
    return torch.empty((int(lib.sessd_spconv_wgrad_workspace_bytes(int(max_out), int(kvol), int(cin), int(cout))),), dtype=torch.uint8,
                       device=device)


def spconv_wgrad_rows(in_feat, gout, tiles, n_out, max_out, kvol, gw=None, ws=None):
    """fp32 weight gradient [kvol, Cin, Cout] of the narrow layers (Cin <= 16) from the forward rulebook's tile lists"""
    cin, cout = int(in_feat.shape[1]), int(gout.shape[1])
    if gw is None:
        gw = torch.empty((int(kvol), cin, cout), dtype=torch.float32, device=gout.device)
    if ws is None:
        ws = wgrad_workspace(max_out, kvol, cin, cout, gout.device)
    check(lib.sessd_spconv_wgrad_rows(_p(in_feat), cin, _p(gout), cout, _p(tiles), int(kvol), _p(n_out), int(max_out), _p(gw), _p(ws), ws.numel(),
                                      _st()), "sessd_spconv_wgrad_rows")
    return gw


def spconv_wgrad_cg(in_planes, in_info, g_planes, g_info, tiles, n_out, max_out, kvol, gw=None, ws=None):
    """tensor-core weight gradient [kvol, Cp, Cout] from the input planes (+ {abs-max, scale}) and the gradient planes (sparse_split_planes)"""
    cp, cout = int(in_planes.shape[1] // 2), int(g_planes.shape[1] // 2)
    if gw is None:
        gw = torch.empty((int(kvol), cp, cout), dtype=torch.float32, device=g_planes.device)
    if ws is None:
        ws = wgrad_workspace(max_out, kvol, cp, cout, g_planes.device)
    check(lib.sessd_spconv_wgrad_cg(_p(in_planes), cp, _p(in_info), _p(g_planes), cout, _p(g_info), _p(tiles), int(kvol), _p(n_out), int(max_out),
                                    _p(gw), _p(ws), ws.numel(), _st()), "sessd_spconv_wgrad_cg")
    return gw


def sparse_planes_to_float(planes, info, channels):
    """(hi + lo) / S of sparse feature planes [rows, 2 * cp] as fp32 [rows, channels] (tests / debugging)"""
    cp = planes.shape[1] // 2
    return (planes[:, :channels].float() + planes[:, cp:cp + channels].float()) / info[1]


def sparse_to_dense(feat, coors, n, max_rows, grid, out=None):
    c = feat.shape[1]
    d, h, w = grid.shape[0], grid.shape[1], grid.shape[2]
    if out is None:
        out = torch.empty((grid.batch, h, w, c * d), dtype=torch.float32, device=feat.device)
    check(lib.sessd_sparse_to_dense(_p(feat), _p(coors), _p(n), int(max_rows), int(c), grid, _p(out), _st()), "sessd_sparse_to_dense")
    return out


def sparse_to_dense_indexed(feat, bitmap_index, grid, out):
    """dense() in one gather pass through the level's bitmap index (see sessd_sparse_to_dense_indexed)."""
    check(lib.sessd_sparse_to_dense_indexed(_p(feat), int(feat.shape[0]), _p(bitmap_index), int(feat.shape[1]), grid, _p(out), _st()),
          "sessd_sparse_to_dense_indexed")
    return out


# ------------------------------------------------------------------------------------------------ BEV convs
def conv_desc(batch, in_hw, cin, out_hw, cout, grid_hw, taps, in_stride=1, out_stride=1, out_off=(0, 0), relu=True):
    d = ConvDesc()
    d.batch, d.in_h, d.in_w, d.cin = int(batch), int(in_hw[0]), int(in_hw[1]), int(cin)
    d.out_h, d.out_w, d.cout = int(out_hw[0]), int(out_hw[1]), int(cout)
    d.grid_h, d.grid_w = int(grid_hw[0]), int(grid_hw[1])
    d.in_stride, d.out_stride, d.out_off_y, d.out_off_x = int(in_stride), int(out_stride), int(out_off[0]), int(out_off[1])
    d.ntaps = len(taps)
    for t, (dy, dx) in enumerate(taps):
        d.tap_dy[t], d.tap_dx[t] = int(dy), int(dx)
    d.relu = int(bool(relu))
    return d


def pack_weight_h2(wp, cout_pad):
    """[taps, Cin, Cout] (tap-list packing) -> (planes fp16 [2, taps, cout_pad, Cin], exps [cout_pad] fp32 = 2^-e[n]) for sessd_bev_conv_p2 / _h2:
    the fp16 split of _fp16_split over the zero-padded weight.  The returned 2^-e[n] must be folded into the epilogue scale."""
    taps, cin, cout = wp.shape
    wt = torch.zeros((taps, cout_pad, cin), dtype=torch.float32, device=wp.device)
    wt[:, :cout] = wp.permute(0, 2, 1)
    hi, lo, inv = _fp16_split(wt)
    return torch.stack([hi, lo], 0).contiguous(), inv


def bev_conv_h2(x, weight_h2, scale, shift, residual, out, desc, amax_in=None, amax_out=None):
    check(lib.sessd_bev_conv_h2(_p(x), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual), _p(out), C.byref(desc),
                                _p(amax_in), _p(amax_out), _st()), "sessd_bev_conv_h2")
    return out


def bev_deconv_h2(x, weight_h2, scale, shift, residual, out, relu=True, amax_in=None, amax_out=None):
    """ConvTranspose2d(k3,s2,p1,op1)+BN+ReLU(+residual) with the fp16 split in the kernel: x [B,H,W,Cin] -> out [B,2H,2W,Cout];
    weight_h2 from pack_weight_h2(W.permute(2,3,0,1).reshape(9,Cin,Cout), cout_pad)."""
    b, h, w, cin = x.shape
    check(lib.sessd_bev_deconv_h2(_p(x), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual), _p(out),
                                  int(b), int(h), int(w), int(cin), int(out.shape[-1]), int(bool(relu)), _p(amax_in), _p(amax_out), _st()),
          "sessd_bev_deconv_h2")
    return out


# ---- BEV convs from pre-split fp16 planes (csrc/bevconv_p2.cu) ---------------------------------------------------------------
def alloc_bev_planes(batch, h, w, c, device):
    """fp16 (hi, lo) planes [2, B, H, W, C] of one activation tensor"""
    return torch.zeros((2, batch, h, w, c), dtype=torch.float16, device=device)


def conv_gain(wp, scale):
    """max_n sum_{tap,c} |w[tap][c][n] * scale[n]| of a [taps, Cin, Cout] weight: |conv(x) * scale| <= max|x| * gain"""
    g = wp.abs().sum(dim=(0, 1)) * scale.abs().to(wp.device)[: wp.shape[2]]
    return float(g.max()) * (1.0 + 1e-5)


def bev_conv_p2(in_planes, in_info, weight_h2, scale, shift, residual, resid_info, gain, shift_max, out_f32, out_planes, out_info, desc,
                items=None, segs=None):
    """items: optional launch record of a skip plan (BevSkipPlan.record): only the work items it lists run; segs (stride 1, instead of
    items): optional segment record (BevSkipPlan.seg_record): only the segments it lists run"""
    check(lib.sessd_bev_conv_p2(_p(in_planes), _p(in_info), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual),
                                _p(resid_info), float(gain), float(shift_max), _p(out_f32), _p(out_planes), _p(out_info), C.byref(desc),
                                _p(items), _p(segs), _st()), "sessd_bev_conv_p2")


def bev_deconv_p2(in_planes, in_info, weight_h2, scale, shift, residual, resid_info, gain, shift_max, out_f32, out_planes, out_info, relu=True,
                  items=None, segs=None):
    _two, b, h, w, cin = in_planes.shape
    cout = (out_f32 if out_f32 is not None else out_planes).shape[-1]
    check(lib.sessd_bev_deconv_p2(_p(in_planes), _p(in_info), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual),
                                  _p(resid_info), float(gain), float(shift_max), _p(out_f32), _p(out_planes), _p(out_info), int(b), int(h),
                                  int(w), int(cin), int(cout), int(bool(relu)), _p(items), _p(segs), _st()), "sessd_bev_deconv_p2")


class BevSkipPlan:
    """Device buffer of the SSFA neck's constant-region skip plan (sessd_bev_skip_plan): one int32 record per neck launch, in the
    order of runners.SSFAPlanesRunner.SKIP_LAUNCHES.  Record layout (csrc/bevskip.cu): header of 32 words (0: items to run, 1: skipped
    tiles, then the launch geometry), the work items to run, the skipped (class, tile) entries, the per-(class, tile) flags.
    Segment records (seg_buf, every launch but the stride-2 conv): header of 32 words (0: items to run, 1: skipped segments, 2: groups,
    then the geometry and the representatives), groups of 16 segment entries, the skipped (class, segment) entries, the flags."""

    LAUNCHES = 13

    def __init__(self, batch, h, w, device):
        offs, seg_offs = (C.c_int * self.LAUNCHES)(), (C.c_int * self.LAUNCHES)()
        words = lib.sessd_bev_skip_plan_words(int(batch), int(h), int(w), offs)
        seg_words = lib.sessd_bev_skip_seg_words(int(batch), int(h), int(w), seg_offs)
        if words <= 0 or seg_words <= 0:
            raise ValueError("no skip plan for a [%d, %d, %d] neck" % (batch, h, w))
        self.offsets, self.seg_offsets = list(offs), list(seg_offs)
        self.buf = torch.zeros((int(words),), dtype=torch.int32, device=device)
        self.seg_buf = torch.zeros((int(seg_words),), dtype=torch.int32, device=device)

    def record(self, i):
        return self.buf[self.offsets[i]:]

    def seg_record(self, i):
        """launch i's segment record, or None (the stride-2 conv runs tiles)"""
        return self.seg_buf[self.seg_offsets[i]:] if self.seg_offsets[i] >= 0 else None

    def build(self, bitmap_index, grid):
        """bitmap_index / grid: the last sparse level's index (SpMiddleRunner.levels[-1]) -- grid.shape = (D, h, w)"""
        check(lib.sessd_bev_skip_plan(_p(bitmap_index), grid, _p(self.buf), _p(self.seg_buf), _st()), "sessd_bev_skip_plan")

    def fill(self, i, out_f32, out_planes, cout):
        check(lib.sessd_bev_skip_fill(_p(self.record(i)), _p(out_f32), _p(out_planes), int(cout), _st()), "sessd_bev_skip_fill")

    def fill_segs(self, i, out_f32, out_planes, cout):
        check(lib.sessd_bev_skip_fill_segs(_p(self.seg_record(i)), _p(out_f32), _p(out_planes), int(cout), _st()),
              "sessd_bev_skip_fill_segs")


def bev_split_planes(x, info, planes):
    """fp32 tensor -> planes with the scale from info[0] (its abs-max: call absmax(x, info[0:1]) first); info[1] <- scale"""
    check(lib.sessd_bev_split_planes(_p(x), int(x.numel()), _p(info), _p(planes), _st()), "sessd_bev_split_planes")
    return planes


def bev_wgrad_workspace(desc, device):
    n = int(lib.sessd_bev_wgrad_workspace_bytes(C.byref(desc)))
    if n == 0:
        raise ValueError("sessd_bev_wgrad: no weight gradient for this descriptor")
    return torch.empty((n,), dtype=torch.uint8, device=device)


def bev_wgrad(in_planes, in_info, g_planes, g_info, desc, gw=None, ws=None):
    """weight gradient [ntaps, Cin, Cout] fp32 of the conv of ``desc`` (csrc/bevgrad.cu) from the input planes the forward read and the
    planes of the output gradient (absmax + bev_split_planes)"""
    if gw is None:
        gw = torch.empty((desc.ntaps, desc.cin, desc.cout), dtype=torch.float32, device=g_planes.device)
    if ws is None:
        ws = bev_wgrad_workspace(desc, g_planes.device)
    check(lib.sessd_bev_wgrad(_p(in_planes), _p(in_info), _p(g_planes), _p(g_info), C.byref(desc), _p(gw), _p(ws), ws.numel(), _st()),
          "sessd_bev_wgrad")
    return gw


def planes_to_float(planes, info):
    """(hi + lo) / S as fp32 (tests / debugging)"""
    return (planes[0].float() + planes[1].float()) / info[1]


def sparse_to_dense_planes(feat, bitmap_index, grid, amax, info, planes):
    check(lib.sessd_sparse_to_dense_planes(_p(feat), int(feat.shape[0]), _p(bitmap_index), int(feat.shape[1]), grid, _p(amax), _p(info),
                                           _p(planes), _st()), "sessd_sparse_to_dense_planes")
    return planes


def ssfa_fuse_planes(x0, x1, w0, w1, s0, t0, s1, t1, out, info0, info1, out_info, planes):
    npix = x0.numel() // x0.shape[-1]
    check(lib.sessd_ssfa_fuse_planes(_p(x0), _p(x1), _p(w0), _p(w1), float(s0), float(t0), float(s1), float(t1), int(npix), int(x0.shape[-1]),
                                     _p(out), _p(info0), _p(info1), _p(out_info), _p(planes), _st()), "sessd_ssfa_fuse_planes")
    return out


def absmax(x, amax):
    """amax[0] = max(amax[0], max|x|) on the current stream."""
    check(lib.sessd_absmax(_p(x), int(x.numel()), _p(amax), _st()), "sessd_absmax")
    return amax


# ------------------------------------------------------------------------------------------------ post-processing
NMS_TYPES = ("rotate_nms", "rotate_weighted_nms")
DINMS_MAX_PRE = 4096          # SESSD_DINMS_MAX_PRE


def make_dinms_cfg(nms_cnt_thresh=2.6, nms_sigma_dist_interval=(0, 20, 40, 60), nms_sigma_square=(0.0009, 0.009, 0.1, 1),
                   suppressed_thresh=0.3, centerness_pow=2, enable_centerness=True):
    """DI-NMS constants; the defaults are the values get_task_detections passes (mg_head_sessd.py:1001-1018).  The fourth sigma^2
    of the reference's tuple belongs to no band and is never read."""
    if len(nms_sigma_dist_interval) != 4 or len(nms_sigma_square) < 3:
        raise ValueError("DI-NMS takes four distance edges (three bands) and their three sigma^2")
    d = DinmsCfg()
    d.cnt_thresh, d.suppressed_thresh, d.centerness_pow = float(nms_cnt_thresh), float(suppressed_thresh), float(centerness_pow)
    for j in range(4):
        d.dist_edge[j] = float(nms_sigma_dist_interval[j])
    for j in range(3):
        d.sigma2[j] = float(nms_sigma_square[j])
    d.centerness = int(bool(enable_centerness))
    return d


def make_post_cfg(batch, num_anchors=70400, anchors_per_loc=2, head_stride=24, score_thresh=0.3, nms_pre_max=1000, nms_post_max=100,
                  nms_iou_thresh=0.01, nms_ge=True, post_range=(0, -40.0, -5.0, 70.4, 40.0, 5.0), direction_offset=0.0,
                  use_frustum=False, nms_type="rotate_nms"):
    """nms_type "rotate_nms" (greedy rotated NMS) or "rotate_weighted_nms" (DI-NMS with the head's constants, make_dinms_cfg();
    it keeps up to nms_pre_max detections and ignores nms_post_max, nms_iou_thresh and nms_ge, as the reference does)"""
    if nms_type not in NMS_TYPES:
        raise ValueError("nms_type must be one of %s, not %r" % (NMS_TYPES, nms_type))
    c = PostCfg()
    c.batch, c.num_anchors, c.anchors_per_loc, c.head_stride = int(batch), int(num_anchors), int(anchors_per_loc), int(head_stride)
    c.score_thresh, c.nms_pre_max, c.nms_post_max = float(score_thresh), int(nms_pre_max), int(nms_post_max)
    c.nms_iou_thresh, c.nms_ge = float(nms_iou_thresh), int(bool(nms_ge))
    for j in range(6):
        c.post_range[j] = float(post_range[j])
    c.direction_offset, c.use_frustum = float(direction_offset), int(bool(use_frustum))
    if nms_type == "rotate_weighted_nms":
        c.nms_mode, c.dinms = 1, make_dinms_cfg()
    return c


def post_capacity(cfg):
    """detections per frame the post-processing outputs hold: nms_post_max, or nms_pre_max under DI-NMS"""
    return cfg.nms_pre_max if cfg.nms_mode == 1 else cfg.nms_post_max


class PostBuffers:
    def __init__(self, cfg, device):
        self.cfg = cfg
        b, p = cfg.batch, post_capacity(cfg)
        self.boxes = torch.zeros((b, p, 7), dtype=torch.float32, device=device)
        self.scores = torch.zeros((b, p), dtype=torch.float32, device=device)
        self.labels = torch.zeros((b, p), dtype=torch.int32, device=device)
        self.count = torch.zeros((b,), dtype=torch.int32, device=device)
        self.aux = torch.zeros((b, 4), dtype=torch.int32, device=device)
        self.sel_anchor = torch.zeros((b, p), dtype=torch.int32, device=device)
        self.ws = torch.empty((lib.sessd_postprocess_workspace_bytes(C.byref(cfg)),), dtype=torch.uint8, device=device)


def postprocess(head, anchors, frustum_planes, buf):
    check(lib.sessd_postprocess(_p(head), _p(anchors), _p(frustum_planes), C.byref(buf.cfg), _p(buf.boxes), _p(buf.scores), _p(buf.labels),
                                _p(buf.count), _p(buf.aux), _p(buf.sel_anchor), _p(buf.ws), buf.ws.numel(), _st()), "sessd_postprocess")
    return buf


def postprocess_packed(head, anchors, frustum_planes, buf, packed, meta, num_voxels=None, status=None):
    """postprocess + a packed copy [B,P,8] / meta [B,8+P] of the results (one D2H per batch; see sessd_postprocess_packed)."""
    check(lib.sessd_postprocess_packed(_p(head), _p(anchors), _p(frustum_planes), C.byref(buf.cfg), _p(buf.boxes), _p(buf.scores),
                                       _p(buf.labels), _p(buf.count), _p(buf.aux), _p(buf.sel_anchor), _p(packed), _p(meta),
                                       _p(num_voxels), _p(status), _p(buf.ws), buf.ws.numel(), _st()), "sessd_postprocess_packed")
    return buf


def rotate_nms(boxes5, scores, n, max_boxes, pre_max, post_max, iou_thresh, ge=True):
    dev = boxes5.device
    keep = torch.empty((post_max,), dtype=torch.int32, device=dev)
    num = torch.zeros((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((lib.sessd_rotate_nms_workspace_bytes(int(max_boxes), int(pre_max)),), dtype=torch.uint8, device=dev)
    check(lib.sessd_rotate_nms(_p(boxes5), _p(scores), _p(n), int(max_boxes), int(pre_max), int(post_max), float(iou_thresh),
                               int(bool(ge)), _p(keep), _p(num), _p(ws), ws.numel(), _st()), "sessd_rotate_nms")
    return keep, num


def rotate_weighted_nms(boxes7, boxes5, scores, iou_preds, labels, dirs, anchors, n, max_boxes, pre_max, dinms_cfg, ws=None):
    """Stand-alone DI-NMS (sessd_rotate_weighted_nms).  boxes7 [N,7], boxes5 [N,5], scores [N], iou_preds [N] (rectified q) f32,
    labels / dirs [N] i32, anchors [N,7] f32 (or None without centerness), n [1] i32 on the device.  Returns (boxes [pre_max,7],
    scores, labels, dirs, keep = top-k position of each pick, selected = its input index, count [2] = emitted clusters, picks);
    rows beyond count[0] are unspecified.  ws: a uint8 CUDA workspace of at least
    sessd_rotate_weighted_nms_workspace_bytes(max_boxes, pre_max) bytes to reuse across calls (allocated per call when None)."""
    dev = scores.device
    for t, dt, name in ((boxes7, torch.float32, "boxes7"), (boxes5, torch.float32, "boxes5"), (scores, torch.float32, "scores"),
                        (iou_preds, torch.float32, "iou_preds"), (labels, torch.int32, "labels"), (dirs, torch.int32, "dirs"),
                        (n, torch.int32, "n")):
        _cuda(t, dt, name)
    if anchors is not None:
        _cuda(anchors, torch.float32, "anchors")
    p = int(pre_max)
    out = dict(boxes=torch.empty((p, 7), dtype=torch.float32, device=dev), scores=torch.empty((p,), dtype=torch.float32, device=dev),
               labels=torch.empty((p,), dtype=torch.int32, device=dev), dirs=torch.empty((p,), dtype=torch.int32, device=dev),
               keep=torch.empty((p,), dtype=torch.int32, device=dev), selected=torch.empty((p,), dtype=torch.int32, device=dev),
               count=torch.zeros((2,), dtype=torch.int32, device=dev))
    if ws is None:
        ws = torch.empty((max(lib.sessd_rotate_weighted_nms_workspace_bytes(int(max_boxes), p), 1),), dtype=torch.uint8, device=dev)
    check(lib.sessd_rotate_weighted_nms(_p(boxes7), _p(boxes5), _p(scores), _p(iou_preds), _p(labels), _p(dirs), _p(anchors), _p(n),
                                        int(max_boxes), p, C.byref(dinms_cfg), _p(out["boxes"]), _p(out["scores"]), _p(out["labels"]),
                                        _p(out["dirs"]), _p(out["keep"]), _p(out["selected"]), _p(out["count"]), _p(ws), ws.numel(),
                                        _st()), "sessd_rotate_weighted_nms")
    return out


# ------------------------------------------------------------------------------------------------ iou3d family
def boxes_overlap_bev(a, b, out):
    check(lib.sessd_boxes_overlap_bev(_p(a), a.shape[0], _p(b), b.shape[0], _p(out), _st()), "sessd_boxes_overlap_bev")
    return out


def boxes_aligned_overlap_bev(a, b, out):
    check(lib.sessd_boxes_aligned_overlap_bev(_p(a), _p(b), a.shape[0], _p(out), _st()), "sessd_boxes_aligned_overlap_bev")
    return out


def boxes_iou_bev(a, b, out):
    check(lib.sessd_boxes_iou_bev(_p(a), a.shape[0], _p(b), b.shape[0], _p(out), _st()), "sessd_boxes_iou_bev")
    return out


def boxes_iou3d(a, b, out):
    check(lib.sessd_boxes_iou3d(_p(a), a.shape[0], _p(b), b.shape[0], _p(out), _st()), "sessd_boxes_iou3d")
    return out


def nms_sorted(boxes, thresh, mode):
    n = boxes.shape[0]
    dev = boxes.device
    keep = torch.empty((max(n, 1),), dtype=torch.int64, device=dev)
    num = torch.zeros((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((lib.sessd_nms_workspace_bytes(n),), dtype=torch.uint8, device=dev)
    check(lib.sessd_nms_sorted(_p(boxes), n, float(thresh), int(mode), _p(keep), _p(num), _p(ws), ws.numel(), _st()), "sessd_nms_sorted")
    return keep, num


# ------------------------------------------------------------------------------------------------ target assignment (T1)
class AssignBuffers:
    """Device outputs + workspace of sessd_assign_targets for `batch` frames of `num_anchors` anchors, up to `max_gt` GT boxes."""

    def __init__(self, num_anchors, batch, max_gt, device):
        self.num_anchors, self.batch, self.max_gt = int(num_anchors), int(batch), int(max_gt)
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=device)   # noqa: E731
        self.labels = z((batch, num_anchors), torch.int32)
        self.bbox_targets = z((batch, num_anchors, 7), torch.float32)
        self.bbox_outside_weights = z((batch, num_anchors), torch.float32)
        self.pos_anchor = z((batch, num_anchors), torch.int32)
        self.pos_gt_id = z((batch, num_anchors), torch.int32)
        self.num_pos = z((batch,), torch.int32)
        self.ws = torch.empty((lib.sessd_assign_workspace_bytes(self.num_anchors, self.batch, self.max_gt),), dtype=torch.uint8,
                              device=device)


def assign_targets(anchors, gt_boxes, num_gt, buf, matched_thr=0.6, unmatched_thr=0.45):
    """anchors [A,7] f32, gt_boxes [B,max_gt,7] f32 (padded), num_gt [B] i32 -- all on the device; fills `buf` on the current stream."""
    _cuda(anchors, torch.float32, "anchors"); _cuda(gt_boxes, torch.float32, "gt_boxes"); _cuda(num_gt, torch.int32, "num_gt")
    assert anchors.shape == (buf.num_anchors, 7) and tuple(gt_boxes.shape) == (buf.batch, buf.max_gt, 7) and num_gt.numel() == buf.batch
    check(lib.sessd_assign_targets(_p(anchors), buf.num_anchors, _p(gt_boxes), _p(num_gt), buf.batch, buf.max_gt, float(matched_thr),
                                   float(unmatched_thr), _p(buf.labels), _p(buf.bbox_targets), _p(buf.bbox_outside_weights),
                                   _p(buf.pos_anchor), _p(buf.pos_gt_id), _p(buf.num_pos), _p(buf.ws), buf.ws.numel(), _st()),
          "sessd_assign_targets")
    return buf


# ------------------------------------------------------------------------------------------------ supervised head loss (training, first slice)
def head_loss(head, anchors, labels, reg_targets, alpha=0.25, sigma=3.0, dir_offset=0.0, pos_cls_weight=1.0, neg_cls_weight=1.0,
              w_cls=1.0, w_loc=2.0, w_dir=0.2, w_iou=None, with_grad=True):
    """head [B, A/2, stride] f32 (fused head tensor), anchors [A,7], labels [B,A] i32, reg_targets [B,A,7] -- device tensors.
    w_iou: None = skip the IoU-prediction term; a float = also run sessd_iou_pred_loss (smooth-L1 of the iou head vs 2*IoU3D-1 on positives).
    Returns (losses [B,8] = per-frame sums {cls, loc, dir, cls_pos, cls_neg, iou_pred, num_pos, num_neg}, grad_head or None)."""
    _cuda(head, torch.float32, "head"); _cuda(anchors, torch.float32, "anchors"); _cuda(labels, torch.int32, "labels")
    _cuda(reg_targets, torch.float32, "reg_targets")
    B, A = labels.shape
    assert head.shape[0] == B and head.shape[1] * 2 == A and anchors.shape == (A, 7) and tuple(reg_targets.shape) == (B, A, 7)
    losses = torch.empty((B, 8), dtype=torch.float32, device=head.device)
    grad = torch.empty_like(head) if with_grad else None
    ws = torch.empty((lib.sessd_head_loss_workspace_bytes(int(B)),), dtype=torch.uint8, device=head.device)
    check(lib.sessd_head_loss(_p(head), _p(anchors), _p(labels), _p(reg_targets), int(B), int(A), 2, int(head.shape[2]), float(alpha), float(sigma),
                              float(dir_offset), float(pos_cls_weight), float(neg_cls_weight), float(w_cls), float(w_loc), float(w_dir),
                              _p(losses), _p(grad), _p(ws), ws.numel(), _st()), "sessd_head_loss")
    if w_iou is not None:
        ws2 = torch.empty((lib.sessd_iou_pred_loss_workspace_bytes(int(B)),), dtype=torch.uint8, device=head.device)
        check(lib.sessd_iou_pred_loss(_p(head), _p(anchors), _p(labels), _p(reg_targets), int(B), int(A), 2, int(head.shape[2]), float(sigma),
                                      float(w_iou), _p(losses), _p(grad), _p(ws2), ws2.numel(), _st()), "sessd_iou_pred_loss")
    return losses, grad


def odiou_pairs_host(gboxes, qboxes, with_grad=True):
    """HOST evaluation (numpy in / out) of the ODIoU arithmetic the device kernel uses: (odiou [n], d odiou / d qboxes [n,7])."""
    g = np.ascontiguousarray(gboxes, np.float32).reshape(-1, 7)
    q = np.ascontiguousarray(qboxes, np.float32).reshape(-1, 7)
    assert g.shape == q.shape
    out = np.zeros((g.shape[0],), np.float32)
    grad = np.zeros_like(q) if with_grad else None
    check(lib.sessd_odiou_pairs_host(g.ctypes.data_as(C.c_void_p), q.ctypes.data_as(C.c_void_p), int(g.shape[0]), out.ctypes.data_as(C.c_void_p),
                                     grad.ctypes.data_as(C.c_void_p) if with_grad else C.c_void_p(0)), "sessd_odiou_pairs_host")
    return out, grad


def odiou_loss(head, anchors, labels, reg_targets, losses, grad_head=None, w_odiou=2.0):
    """ODIoU term on the device; `losses` / `grad_head` are the outputs of head_loss() on the same stream (grad_head is updated in place).
    Returns the per-frame sums [B] of odiou / num_pos over the positives."""
    B, A = labels.shape
    out = torch.empty((B,), dtype=torch.float32, device=head.device)
    ws = torch.empty((lib.sessd_odiou_loss_workspace_bytes(int(B)),), dtype=torch.uint8, device=head.device)
    check(lib.sessd_odiou_loss(_p(head), _p(anchors), _p(labels), _p(reg_targets), int(B), int(A), 2, int(head.shape[2]), float(w_odiou),
                               _p(losses), _p(out), _p(grad_head), _p(ws), ws.numel(), _st()), "sessd_odiou_loss")
    return out


# ------------------------------------------------------------------------------------------------ training augmentation (csrc/augment.cu)
def box_collision(boxes, qboxes, out=None):
    """box_collision_test: boxes [N,4,2], qboxes [K,4,2] fp64 corner sets (device) -> [N,K] uint8 (1 = collide)."""
    _cuda(boxes, torch.float64, "boxes"); _cuda(qboxes, torch.float64, "qboxes")
    n, k = boxes.shape[0], qboxes.shape[0]
    if out is None:
        out = torch.empty((n, k), dtype=torch.uint8, device=boxes.device)
    check(lib.sessd_box_collision(_p(boxes), int(n), _p(qboxes), int(k), _p(out), _st()), "sessd_box_collision")
    return out


def _aug_inputs(gt_boxes, num_gt, valid, loc_noise, rot_noise, selected=None):
    """checks the padded box batch and its draws: gt_boxes [B,M,7] f32, num_gt [B] i32, valid [B,M] u8, loc_noise [B,M,T,3] and
    rot_noise [B,M,T] f64, selected [B,M] i32 -- contiguous CUDA tensors; returns (B, M, T)"""
    _cuda(gt_boxes, torch.float32, "gt_boxes"); _cuda(num_gt, torch.int32, "num_gt"); _cuda(valid, torch.uint8, "valid")
    _cuda(loc_noise, torch.float64, "loc_noise"); _cuda(rot_noise, torch.float64, "rot_noise")
    B, M = valid.shape
    T = rot_noise.shape[2]
    if (tuple(gt_boxes.shape) != (B, M, 7) or num_gt.numel() != B or tuple(loc_noise.shape) != (B, M, T, 3)
            or tuple(rot_noise.shape) != (B, M, T)):
        raise ValueError("augmentation inputs: shape mismatch")
    if selected is not None:
        _cuda(selected, torch.int32, "selected")
        if tuple(selected.shape) != (B, M):
            raise ValueError("selected must be [B, M]")
    return B, M, T


def points_in_boxes(points, boxes, context=-1.0, mask=None):
    """points [N, >=3] f32, boxes [M, 7] f32 (device) -> [N, M] uint8 membership mask (sessd_points_in_boxes)."""
    _cuda(points, torch.float32, "points"); _cuda(boxes, torch.float32, "boxes")
    if points.dim() != 2 or points.shape[1] < 3 or boxes.dim() != 2 or boxes.shape[1] != 7:
        raise ValueError("points_in_boxes: points [N, >=3], boxes [M, 7]")
    n, m = points.shape[0], boxes.shape[0]
    if mask is None:
        mask = torch.empty((n, m), dtype=torch.uint8, device=points.device)
    check(lib.sessd_points_in_boxes(_p(points), int(n), int(points.shape[1]), _p(boxes), int(m), float(context), _p(mask), _st()),
          "sessd_points_in_boxes")
    return mask


def noise_per_box(gt_boxes, num_gt, valid, loc_noise, rot_noise, context=-1.0, selected=None):
    """noise_per_box over a padded batch: gt_boxes [B,M,7] f32, num_gt [B] i32, valid [B,M] u8, loc_noise [B,M,T,3] / rot_noise [B,M,T]
    f64 (device) -> selected try per box [B,M] i32 (-1: none)."""
    B, M, T = _aug_inputs(gt_boxes, num_gt, valid, loc_noise, rot_noise)
    if selected is None:
        selected = torch.empty((B, M), dtype=torch.int32, device=gt_boxes.device)
    _cuda(selected, torch.int32, "selected")
    check(lib.sessd_noise_per_box(_p(gt_boxes), _p(num_gt), _p(valid), int(B), int(M), _p(loc_noise), _p(rot_noise), int(T),
                                  float(context), _p(selected), _st()), "sessd_noise_per_box")
    return selected


def augment_points(points, frame_off, max_frame_points, gt_boxes, num_gt, valid, loc_noise, rot_noise, selected, glob, perm, labeled=None,
                   context=-1.0, points_raw=None, points_out=None, with_raw=True):
    """per-object transform, raw twin, global flip / rotation / scaling and shuffle of a batch of frames (sessd_augment_points).
    points [P,4] f32 (16-byte aligned rows), frame_off [B+1] i32, glob [B,5] f32 (cos, sin, scale, flip, angle), perm [P] i32 holding a
    permutation of each frame's rows, labeled [B] u8 or None.  Returns (points_raw, points_out) [P,4] f32; with_raw=False writes no twin
    and returns (None, points_out)."""
    B, M, T = _aug_inputs(gt_boxes, num_gt, valid, loc_noise, rot_noise, selected)
    _cuda(points, torch.float32, "points"); _cuda(frame_off, torch.int32, "frame_off"); _cuda(glob, torch.float32, "glob")
    _cuda(perm, torch.int32, "perm")
    if labeled is not None:
        _cuda(labeled, torch.uint8, "labeled")
        if labeled.numel() != B:
            raise ValueError("labeled must be [B]")
    if points.dim() != 2 or points.shape[1] != 4 or frame_off.numel() != B + 1 or perm.numel() != points.shape[0] or tuple(glob.shape) != (B, 5):
        raise ValueError("augment_points: shape mismatch")
    if not with_raw:
        points_raw = None
    elif points_raw is None:
        points_raw = torch.empty_like(points)
    if points_out is None:
        points_out = torch.empty_like(points)
    written = (("points_raw", points_raw), ("points_out", points_out)) if with_raw else (("points_out", points_out),)
    for name, t in written:
        _cuda(t, torch.float32, name)
        if t.shape != points.shape:
            raise ValueError("%s must be shaped like points" % name)
    if any(t.data_ptr() % 16 for t in (points, points_out) + ((points_raw,) if with_raw else ())):
        raise ValueError("augment_points: point rows are read and written as float4 and must be 16-byte aligned")
    check(lib.sessd_augment_points(_p(points), _p(frame_off), int(B), int(max_frame_points), _p(gt_boxes), _p(num_gt), _p(valid), int(M),
                                   _p(loc_noise), _p(rot_noise), int(T), _p(selected), float(context), _p(glob), _p(perm), _p(labeled),
                                   _p(points_raw), _p(points_out), _st()), "sessd_augment_points")
    return points_raw, points_out


def augment_boxes(gt_boxes, num_gt, valid, target, loc_noise, rot_noise, selected, glob, range_bev, global_boxes=False):
    """box3d_transform_, valid-box selection, global stages and the Voxelization / AssignTarget bookkeeping (sessd_augment_boxes).
    target: [B,M] u8 target-class mask or None (all); range_bev: host (x0, y0, x1, y1).  Returns (boxes_raw [B,M,7], num_raw [B],
    boxes [B,M,7], num [B]) on the device; global_boxes=True appends (boxes_global [B,M,7], num_global [B]): the class-valid boxes after
    the global stages, before the range filter and limit_period (the boxes SA-DA takes)."""
    B, M, T = _aug_inputs(gt_boxes, num_gt, valid, loc_noise, rot_noise, selected)
    _cuda(glob, torch.float32, "glob")
    if tuple(glob.shape) != (B, 5):
        raise ValueError("glob must be [B, 5]")
    if target is not None:
        _cuda(target, torch.uint8, "target")
        if tuple(target.shape) != (B, M):
            raise ValueError("target must be [B, M]")
    dev = gt_boxes.device
    boxes_raw = torch.empty((B, M, 7), dtype=torch.float32, device=dev)
    boxes_out = torch.empty((B, M, 7), dtype=torch.float32, device=dev)
    num_raw = torch.empty((B,), dtype=torch.int32, device=dev)
    num_out = torch.empty((B,), dtype=torch.int32, device=dev)
    boxes_glob = torch.empty((B, M, 7), dtype=torch.float32, device=dev) if global_boxes else None
    num_glob = torch.empty((B,), dtype=torch.int32, device=dev) if global_boxes else None
    rg = (C.c_float * 4)(*[float(v) for v in range_bev])
    check(lib.sessd_augment_boxes(_p(gt_boxes), _p(num_gt), _p(valid), _p(target), int(B), int(M), _p(loc_noise), _p(rot_noise), int(T),
                                  _p(selected), _p(glob), rg, _p(boxes_raw), _p(num_raw), _p(boxes_out), _p(num_out), _p(boxes_glob),
                                  _p(num_glob), _st()), "sessd_augment_boxes")
    res = (boxes_raw, num_raw, boxes_out, num_out)
    return res + (boxes_glob, num_glob) if global_boxes else res


def gtaug_select_host(corners, num_boxes):
    """sample_class_v2's acceptance (sessd_gtaug_select_host): corners [num_boxes + K, 4, 2] fp64 (host, center_to_corner_box2d of
    [boxes so far | candidates]) -> accepted mask [K] bool."""
    corners = np.ascontiguousarray(corners, np.float64)
    if corners.ndim != 3 or corners.shape[1:] != (4, 2) or not 0 <= num_boxes <= corners.shape[0]:
        raise ValueError("gtaug_select_host: corners [num_boxes + K, 4, 2], 0 <= num_boxes <= rows")
    k = corners.shape[0] - int(num_boxes)
    acc = np.zeros(max(k, 1), np.uint8)
    rc = lib.sessd_gtaug_select_host(corners.ctypes.data_as(C.c_void_p), int(num_boxes), int(k), acc.ctypes.data_as(C.c_void_p))
    if rc < 0:
        check(rc, "sessd_gtaug_select_host")
    return acc[:k].astype(bool)


def gtaug_paste(points, frame_off, obj_off, obj_ids, db_points, db_off, db_count, db_boxes, max_paste_points, out=None,
                frame_off_out=None):
    """Paste the accepted database objects into a batch of frames and drop the scene points inside them (sessd_gtaug_paste).
    points [P,4] f32 with frame_off [B+1] i32; obj_off [B+1] / obj_ids [K] i32 (CSR, acceptance order); the resident database:
    db_points [*,4] f32 (relative to the centre), db_off / db_count [N] i32, db_boxes [N,7] f64; max_paste_points: the host-known row
    total of the accepted objects (sizes the output).  Returns (points_out [P + max_paste_points, 4] f32, frame_off_out [B+1] i32); the
    rows past frame_off_out[B] are unused.  obj_off / obj_ids given as host numpy arrays are checked here (every id in [0, N), offsets
    non-decreasing from 0 to K) and uploaded; given as device tensors they are not (an out-of-range id then pastes nothing and removes
    nothing: the C entry cannot see it)."""
    _cuda(points, torch.float32, "points"); _cuda(frame_off, torch.int32, "frame_off"); _cuda(db_points, torch.float32, "db_points")
    _cuda(db_off, torch.int32, "db_off"); _cuda(db_count, torch.int32, "db_count"); _cuda(db_boxes, torch.float64, "db_boxes")
    B = frame_off.numel() - 1
    N = db_count.numel()
    if isinstance(obj_ids, np.ndarray) or isinstance(obj_off, np.ndarray):
        ids = np.asarray(obj_ids).reshape(-1); off = np.asarray(obj_off).reshape(-1)
        if ids.size and (ids.min() < 0 or ids.max() >= N):
            raise ValueError("gtaug_paste: object id out of range [0, %d)" % N)
        if off.size != B + 1 or off[0] != 0 or off[-1] != ids.size or (np.diff(off) < 0).any():
            raise ValueError("gtaug_paste: obj_off must be a CSR offset array [B+1] over the ids")
        host = np.concatenate([off.astype(np.int32), ids.astype(np.int32)])
        dev_ids = torch.from_numpy(host).to(points.device)
        obj_off, obj_ids = dev_ids[:B + 1], dev_ids[B + 1:]
    _cuda(obj_off, torch.int32, "obj_off"); _cuda(obj_ids, torch.int32, "obj_ids")
    if (B < 1 or points.dim() != 2 or points.shape[1] != 4 or obj_off.numel() != B + 1 or db_points.dim() != 2 or db_points.shape[1] != 4
            or db_off.numel() != N or tuple(db_boxes.shape) != (N, 7)):
        raise ValueError("gtaug_paste: shape mismatch")
    cap = int(points.shape[0]) + int(max_paste_points)
    dev = points.device
    if out is None:
        out = torch.empty((max(cap, 1), 4), dtype=torch.float32, device=dev)
    if frame_off_out is None:
        frame_off_out = torch.empty((B + 1,), dtype=torch.int32, device=dev)
    _cuda(out, torch.float32, "out"); _cuda(frame_off_out, torch.int32, "frame_off_out")
    if out.dim() != 2 or out.shape[1] != 4 or frame_off_out.numel() != B + 1:
        raise ValueError("gtaug_paste: out [capacity, 4], frame_off_out [B+1]")
    if any(t.data_ptr() % 16 for t in (points, db_points, out)):
        raise ValueError("gtaug_paste: point rows are read and written as float4 and must be 16-byte aligned")
    K = obj_ids.numel()
    ws = torch.empty((int(lib.sessd_gtaug_paste_workspace_bytes(B, int(points.shape[0]), K)),), dtype=torch.uint8, device=dev)
    check(lib.sessd_gtaug_paste(_p(points), _p(frame_off), int(B), int(points.shape[0]), _p(obj_off), _p(obj_ids), int(K),
                                int(max_paste_points), _p(db_points), _p(db_off), _p(db_count), _p(db_boxes), int(N), _p(ws),
                                ws.numel(), _p(out), int(out.shape[0]), _p(frame_off_out), _st()), "sessd_gtaug_paste")
    return out, frame_off_out


# ------------------------------------------------------------------------------------------------ shape-aware augmentation (SA-DA)
SADA_MAX_IDS = 6 * 256                 # SESSD_SADA_MAX_IDS


def _rows4(points, name):
    _cuda(points, torch.float32, name)
    if points.dim() != 2 or points.shape[1] != 4:
        raise ValueError("%s must be [N, 4]" % name)
    if points.data_ptr() % 16:
        raise ValueError("%s: point rows are read and written as float4 and must be 16-byte aligned" % name)
    return points


def _count(d_n, name="n"):
    if d_n is not None:
        _cuda(d_n, torch.int32, name)
        if d_n.numel() < 1:
            raise ValueError("%s must hold one count" % name)
    return d_n


def _ids(ids, num_pyramids, device):
    """a pyramid list: host ids are checked against [0, num_pyramids) and uploaded; device ids are taken as they are"""
    if not isinstance(ids, torch.Tensor):
        ids = np.asarray(ids, np.int64).reshape(-1)
        if ids.size and (ids.min() < 0 or ids.max() >= num_pyramids):
            raise ValueError("pyramid id out of range [0, %d)" % num_pyramids)
        if ids.size > SADA_MAX_IDS:
            raise ValueError("at most %d listed pyramids" % SADA_MAX_IDS)
        ids = torch.from_numpy(ids.astype(np.int32)).to(device)
    return _cuda(ids, torch.int32, "ids")


def sada_pyramids(boxes):
    """get_pyramids and their face planes (sessd_sada_pyramids): boxes [K,7] f32 -> (pyramids [6K,15], planes [6K,5,4]) f32"""
    _cuda(boxes, torch.float32, "boxes")
    if boxes.dim() != 2 or boxes.shape[1] != 7:
        raise ValueError("sada_pyramids: boxes [K, 7]")
    K = boxes.shape[0]
    pyr = torch.empty((6 * K, 15), dtype=torch.float32, device=boxes.device)
    planes = torch.empty((6 * K, 5, 4), dtype=torch.float32, device=boxes.device)
    if K == 0:
        return pyr, planes
    check(lib.sessd_sada_pyramids(_p(boxes), int(K), _p(pyr), _p(planes), _st()), "sessd_sada_pyramids")
    return pyr, planes


def sada_membership(points, planes, ids, n=None, with_bits=True):
    """points_in_pyramids_mask over a pyramid list (sessd_sada_membership): points [N,4] f32, planes [P,5,4] f32, ids [A] (host ids are
    range-checked), n: optional device row count.  Returns (bits [N, ceil(A/32)] i32 or None, counts [A] i32, ids on the device)."""
    _rows4(points, "points"); _cuda(planes, torch.float32, "planes"); _count(n)
    if planes.dim() != 3 or tuple(planes.shape[1:]) != (5, 4):
        raise ValueError("planes must be [P, 5, 4]")
    dev = points.device
    ids = _ids(ids, planes.shape[0], dev)
    A, N = ids.numel(), points.shape[0]
    bits = torch.empty((N, max(-(-A // 32), 1)), dtype=torch.int32, device=dev) if with_bits else None
    counts = torch.zeros((max(A, 1),), dtype=torch.int32, device=dev)
    check(lib.sessd_sada_membership(_p(points), int(N), _p(n), _p(planes), int(planes.shape[0]), _p(ids), int(A), _p(bits), _p(counts),
                                    _st()), "sessd_sada_membership")
    return bits, counts[:A], ids


def sada_compact(points, bits, counts, min_count=-1, n=None, out=None):
    """the rows of points in no listed pyramid whose count exceeds min_count, in order (sessd_sada_compact).  Returns (out [N,4],
    num [1] i32 on the device)."""
    _rows4(points, "points"); _cuda(bits, torch.int32, "bits"); _cuda(counts, torch.int32, "counts"); _count(n)
    N, A = points.shape[0], counts.numel()
    if bits.shape[0] != N or bits.shape[1] * 32 < A:
        raise ValueError("sada_compact: bits [N, ceil(A / 32)]")
    dev = points.device
    out = _rows4(torch.empty((max(N, 1), 4), dtype=torch.float32, device=dev) if out is None else out, "out")
    num = torch.empty((1,), dtype=torch.int32, device=dev)
    ws = torch.empty((max(int(lib.sessd_sada_compact_workspace_bytes(int(N))), 16),), dtype=torch.uint8, device=dev)
    check(lib.sessd_sada_compact(_p(points), int(N), _p(n), _p(bits), int(A), _p(counts), int(min_count), _p(ws), ws.numel(), _p(out),
                                 int(out.shape[0]), _p(num), _st()), "sessd_sada_compact")
    return out, num


def sada_fps(points, bits, counts, min_count, k, out, num, n=None):
    """farthest-point sampling of every listed pyramid whose count exceeds min_count (sessd_sada_fps): k rows each, written after the
    num[0] rows already in out (capacity >= N + k * A); num is advanced on the device."""
    _rows4(points, "points"); _cuda(bits, torch.int32, "bits"); _cuda(counts, torch.int32, "counts"); _rows4(out, "out")
    _count(num, "num"); _count(n)
    N, A = points.shape[0], counts.numel()
    if bits.shape[0] != N or bits.shape[1] * 32 < A:
        raise ValueError("sada_fps: bits [N, ceil(A / 32)]")
    ws = torch.empty((max(int(lib.sessd_sada_fps_workspace_bytes(int(N), int(A))), 16),), dtype=torch.uint8, device=points.device)
    check(lib.sessd_sada_fps(_p(points), int(N), _p(n), _p(bits), int(A), _p(counts), int(min_count), int(k), _p(ws), ws.numel(), _p(out),
                             int(out.shape[0]), _p(num), _st()), "sessd_sada_fps")
    return out, num


def sada_swap(points, bits, counts, pyramids, ids, max_swap_points, out, num_in, n=None):
    """the pyramid swap of sessd_sada_swap: ids [2 * pairs] (to_swap, then partners) with bits / counts from sada_membership of that
    list; out already holds num_in[0] kept rows and has room for N + max_swap_points.  Returns (out, num_out [1] i32)."""
    _rows4(points, "points"); _cuda(bits, torch.int32, "bits"); _cuda(counts, torch.int32, "counts"); _rows4(out, "out")
    _cuda(pyramids, torch.float32, "pyramids"); _cuda(ids, torch.int32, "ids"); _count(num_in, "num_in"); _count(n)
    N, A = points.shape[0], ids.numel()
    if A % 2 or counts.numel() != A or bits.shape[0] != N or bits.shape[1] * 32 < A or pyramids.dim() != 2 or pyramids.shape[1] != 15:
        raise ValueError("sada_swap: shape mismatch")
    num_out = torch.empty((1,), dtype=torch.int32, device=points.device)
    check(lib.sessd_sada_swap(_p(points), int(N), _p(n), _p(bits), int(A // 2), _p(counts), _p(pyramids), int(pyramids.shape[0]), _p(ids),
                              int(max_swap_points), _p(out), int(out.shape[0]), _p(num_in), _p(num_out), _st()), "sessd_sada_swap")
    return out, num_out


def sada_shuffle(points, frame_off, max_frame_points, perm, out=None):
    """out[off_b + k] = points[off_b + perm[off_b + k]] per frame (sessd_sada_shuffle); perm [P] i32 frame-local"""
    _rows4(points, "points"); _cuda(frame_off, torch.int32, "frame_off"); _cuda(perm, torch.int32, "perm")
    if perm.numel() != points.shape[0]:
        raise ValueError("sada_shuffle: perm [P]")
    out = _rows4(torch.empty_like(points) if out is None else out, "out")
    if out.shape != points.shape:
        raise ValueError("sada_shuffle: out must be shaped like points")
    check(lib.sessd_sada_shuffle(_p(points), _p(frame_off), int(frame_off.numel() - 1), int(max_frame_points), _p(perm), _p(out), _st()),
          "sessd_sada_shuffle")
    return out


# ------------------------------------------------------------------------------------------------ KITTI data preparation
def _rows16(name, *ts):
    if any(t is not None and t.data_ptr() % 16 for t in ts):
        raise ValueError("%s: point rows are read and written as float4 and must be 16-byte aligned" % name)


def prep_frustum_compact(points, frame_off, planes, out=None, frame_off_out=None):
    """The rows of each frame inside its image frustum, bit copies in frame order (sessd_prep_frustum_compact).  points [P,4] f32 with
    frame_off [B+1] i32, planes [B,6,4] f64.  Returns (out [P,4] f32, frame_off_out [B+1] i32); rows past frame_off_out[B] are unused."""
    _cuda(points, torch.float32, "points"); _cuda(frame_off, torch.int32, "frame_off"); _cuda(planes, torch.float64, "planes")
    B = frame_off.numel() - 1
    P = int(points.shape[0])
    if B < 1 or points.dim() != 2 or points.shape[1] != 4 or tuple(planes.shape) != (B, 6, 4):
        raise ValueError("prep_frustum_compact: points [P, 4], frame_off [B+1], planes [B, 6, 4]")
    dev = points.device
    if out is None:
        out = torch.empty((max(P, 1), 4), dtype=torch.float32, device=dev)
    if frame_off_out is None:
        frame_off_out = torch.empty((B + 1,), dtype=torch.int32, device=dev)
    _cuda(out, torch.float32, "out"); _cuda(frame_off_out, torch.int32, "frame_off_out")
    _rows16("prep_frustum_compact", points, out)
    ws = torch.empty((max(int(lib.sessd_prep_frustum_compact_workspace_bytes(P)), 16),), dtype=torch.uint8, device=dev)
    check(lib.sessd_prep_frustum_compact(_p(points), _p(frame_off), int(B), P, _p(planes), _p(ws), ws.numel(), _p(out), int(out.shape[0]),
                                         _p(frame_off_out), _st()), "sessd_prep_frustum_compact")
    return out, frame_off_out


def prep_box_count(points, frame_off, box_planes, box_off, counts=None):
    """Points of each box's frame inside the box (sessd_prep_box_count): box_planes [K,6,4] f64, box_off [B+1] i32 (CSR boxes per
    frame).  Returns counts [K] i32 (device)."""
    _cuda(points, torch.float32, "points"); _cuda(frame_off, torch.int32, "frame_off"); _cuda(box_planes, torch.float64, "box_planes")
    _cuda(box_off, torch.int32, "box_off")
    B = frame_off.numel() - 1
    K = int(box_planes.shape[0])
    if B < 1 or points.dim() != 2 or points.shape[1] != 4 or tuple(box_planes.shape[1:]) != (6, 4) or box_off.numel() != B + 1:
        raise ValueError("prep_box_count: points [P, 4], frame_off [B+1], box_planes [K, 6, 4], box_off [B+1]")
    if counts is None:
        counts = torch.empty((max(K, 1),), dtype=torch.int32, device=points.device)
    _cuda(counts, torch.int32, "counts")
    _rows16("prep_box_count", points)
    check(lib.sessd_prep_box_count(_p(points), _p(frame_off), int(B), int(points.shape[0]), _p(box_planes), _p(box_off), K, _p(counts),
                                   _st()), "sessd_prep_box_count")
    return counts[:K]


def prep_box_gather(points, frame_off, box_planes, centres, box_off, counts, num_rows, out=None, obj_off=None):
    """Each box's points in frame order as fp32(double(p) - centre) for x y z (sessd_prep_box_gather).  counts: prep_box_count's;
    num_rows: their host-known sum.  Returns (rows [num_rows, 4] f32, obj_off [K+1] i32 = the exclusive scan of the counts)."""
    _cuda(points, torch.float32, "points"); _cuda(frame_off, torch.int32, "frame_off"); _cuda(box_planes, torch.float64, "box_planes")
    _cuda(centres, torch.float64, "centres"); _cuda(box_off, torch.int32, "box_off"); _cuda(counts, torch.int32, "counts")
    B = frame_off.numel() - 1
    K = int(box_planes.shape[0])
    if (B < 1 or points.dim() != 2 or points.shape[1] != 4 or tuple(box_planes.shape[1:]) != (6, 4) or tuple(centres.shape) != (K, 3)
            or box_off.numel() != B + 1 or counts.numel() < K):
        raise ValueError("prep_box_gather: shape mismatch")
    dev = points.device
    if out is None:
        out = torch.empty((max(int(num_rows), 1), 4), dtype=torch.float32, device=dev)
    if obj_off is None:
        obj_off = torch.empty((K + 1,), dtype=torch.int32, device=dev)
    _cuda(out, torch.float32, "out"); _cuda(obj_off, torch.int32, "obj_off")
    _rows16("prep_box_gather", points, out)
    ws = torch.empty((max(int(lib.sessd_prep_box_gather_workspace_bytes(K)), 16),), dtype=torch.uint8, device=dev)
    check(lib.sessd_prep_box_gather(_p(points), _p(frame_off), int(B), int(points.shape[0]), _p(box_planes), _p(centres), _p(box_off), K,
                                    _p(counts), int(num_rows), _p(ws), ws.numel(), _p(out), int(out.shape[0]), _p(obj_off), _st()),
          "sessd_prep_box_gather")
    return out[:int(num_rows)], obj_off
