"""Tensor-level wrappers over the C ABI (PyTorch supplies device memory and streams only).

Every function launches asynchronously on ``torch.cuda.current_stream()`` and never synchronises; data-dependent
row counts stay on the device as int32 tensors (``n`` arguments), buffers are capacity sized.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib
from ._lib import ConvDesc, Grid, PostCfg, VoxelCfg, check, lib


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


def rulebook_pairs(nbr, n, max_rows, kvol):
    dev = nbr.device
    pin = torch.full((kvol, max_rows), -1, dtype=torch.int32, device=dev)
    pout = torch.full((kvol, max_rows), -1, dtype=torch.int32, device=dev)
    num = torch.zeros((kvol,), dtype=torch.int32, device=dev)
    ws = torch.empty((lib.sessd_rulebook_pairs_workspace_bytes(int(max_rows), int(kvol)),), dtype=torch.uint8, device=dev)
    check(lib.sessd_rulebook_pairs(_p(nbr), _p(n), int(max_rows), int(kvol), _p(pin), _p(pout), _p(num), _p(ws), ws.numel(), _st()),
          "sessd_rulebook_pairs")
    return pin, pout, num


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


def pack_weight_sp_h2(wp, cp, layout="cg"):
    """[kvol, Cin, Cout] (spconv layout, flattened offsets) -> (fp16 weight tiles of the tensor-core sparse convs, 2^-e[Cout]).
    Every output channel is scaled by the power of two that puts its largest |w| into [2^10, 2^11); hi = fp16_rn(2^e w),
    lo = fp16_rn(2^e w - hi).  cp = 64: [kvol, 2, Cout, 64]; cp = 32: layout "cg" (sessd_spconv_forward_cg): [kvol, 2, Cout, 32] (hi rows, then
    lo rows), layout "h2": [kvol, Cout, 64] with hi in columns [0, Cin), lo in [32, 32+Cin)."""
    kvol, cin, cout = wp.shape
    assert cp in (32, 64) and cin <= cp and (cp == 32 or cin == 64)
    wt = wp.permute(0, 2, 1).contiguous().to(torch.float32)                      # [kvol, Cout, Cin]
    amax = wt.abs().amax(dim=(0, 2))
    _, ex = torch.frexp(amax)
    e = torch.where(amax > 0, 11 - ex, torch.zeros_like(ex)).clamp(-100, 100).to(torch.float32)
    ws = wt * torch.exp2(e)[None, :, None]
    hi = ws.to(torch.float16)
    lo = (ws - hi.to(torch.float32)).to(torch.float16)
    if cp == 64:
        tiles = torch.stack([hi, lo], 1).contiguous()                            # [kvol, 2, Cout, 64]
    elif layout == "cg":
        assert cin == 32
        tiles = torch.stack([hi, lo], 1).contiguous()                            # [kvol, 2, Cout, 32]
    else:
        tiles = torch.zeros((kvol, cout, 64), dtype=torch.float16, device=wp.device)
        tiles[:, :, :cin] = hi
        tiles[:, :, 32:32 + cin] = lo
    return tiles, torch.exp2(-e).contiguous()


def alloc_planes(max_rows, cp, device):
    """fp16 (hi, lo) planes of a sparse feature tensor: [max_rows + 1, 2 * cp]; the extra last row stays zero (missing neighbours)."""
    return torch.zeros((max_rows + 1, 2 * cp), dtype=torch.float16, device=device)


def absmax_rows(feat, n, max_rows, amax):
    check(lib.sessd_absmax_rows(_p(feat), _p(n), int(max_rows), int(feat.shape[1]), _p(amax), _st()), "sessd_absmax_rows")
    return amax


SP_H2_ZERO_MODE = 1      # missing neighbours: 0 = read the all-zero last row, 1 = row index -1 (TMA OOB fill), 2 = row index rows (OOB)


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


def bev_conv(x, weight, scale, shift, residual, out, desc):
    check(lib.sessd_bev_conv(_p(x), _p(weight), _p(scale), _p(shift), _p(residual), _p(out), C.byref(desc), _st()), "sessd_bev_conv")
    return out


def split_tf32(w):
    """w -> (hi, lo): hi = w truncated to tf32 (13 low mantissa bits cleared), lo = w - hi (exact in fp32)."""
    hi = (w.contiguous().view(torch.int32) & -8192).view(torch.float32)
    return hi, w - hi


def pack_weight_tc(wp, cout_pad):
    """[taps, Cin, Cout] (SIMT packing) -> [2, taps, cout_pad, Cin] K-major hi/lo planes for sessd_bev_conv_tc."""
    taps, cin, cout = wp.shape
    wt = torch.zeros((taps, cout_pad, cin), dtype=torch.float32, device=wp.device)
    wt[:, :cout] = wp.permute(0, 2, 1)
    hi, lo = split_tf32(wt)
    return torch.stack([hi, lo], 0).contiguous()


def bev_conv_tc(x, weight_split, scale, shift, residual, out, desc):
    check(lib.sessd_bev_conv_tc(_p(x), _p(weight_split), int(weight_split.shape[2]), _p(scale), _p(shift), _p(residual), _p(out),
                                C.byref(desc), _st()), "sessd_bev_conv_tc")
    return out


def bev_deconv_tc(x, weight_split, scale, shift, residual, out, relu=True):
    """ConvTranspose2d(k3,s2,p1,op1)+BN+ReLU(+residual): x [B,H,W,Cin] -> out [B,2H,2W,Cout]; weight_split from
    pack_weight_tc(W.permute(2,3,0,1).reshape(9,Cin,Cout), cout_pad)."""
    b, h, w, cin = x.shape
    check(lib.sessd_bev_deconv_tc(_p(x), _p(weight_split), int(weight_split.shape[2]), _p(scale), _p(shift), _p(residual), _p(out),
                                  int(b), int(h), int(w), int(cin), int(out.shape[-1]), int(bool(relu)), _st()), "sessd_bev_deconv_tc")
    return out


def pack_weight_h2(wp, cout_pad):
    """[taps, Cin, Cout] (SIMT packing) -> (planes fp16 [2, taps, cout_pad, Cin], exps [cout_pad] fp32 = 2^-e[n]) for sessd_bev_conv_p2 / _h2:
    every output channel is scaled by the power of two 2^e[n] that puts its largest |w| into [2^10, 2^11); hi = fp16_rn(2^e w),
    lo = fp16_rn(2^e w - hi).  The returned 2^-e[n] must be folded into the epilogue scale."""
    taps, cin, cout = wp.shape
    wt = torch.zeros((taps, cout_pad, cin), dtype=torch.float32, device=wp.device)
    wt[:, :cout] = wp.permute(0, 2, 1)
    amax = wt.abs().amax(dim=(0, 2))
    _, ex = torch.frexp(amax)                       # amax = m * 2^ex, m in [0.5, 1)
    e = torch.where(amax > 0, 11 - ex, torch.zeros_like(ex)).clamp(-100, 100).to(torch.float32)
    ws = wt * torch.exp2(e)[None, :, None]
    hi = ws.to(torch.float16)
    lo = (ws - hi.to(torch.float32)).to(torch.float16)
    return torch.stack([hi, lo], 0).contiguous(), torch.exp2(-e).contiguous()


def bev_conv_h2(x, weight_h2, scale, shift, residual, out, desc, amax_in=None, amax_out=None):
    check(lib.sessd_bev_conv_h2(_p(x), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual), _p(out), C.byref(desc),
                                _p(amax_in), _p(amax_out), _st()), "sessd_bev_conv_h2")
    return out


def bev_deconv_h2(x, weight_h2, scale, shift, residual, out, relu=True, amax_in=None, amax_out=None):
    """fp16-split twin of bev_deconv_tc; weight_h2 from pack_weight_h2(W.permute(2,3,0,1).reshape(9,Cin,Cout), cout_pad)."""
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


def bev_conv_p2(in_planes, in_info, weight_h2, scale, shift, residual, resid_info, gain, shift_max, out_f32, out_planes, out_info, desc):
    check(lib.sessd_bev_conv_p2(_p(in_planes), _p(in_info), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual),
                                _p(resid_info), float(gain), float(shift_max), _p(out_f32), _p(out_planes), _p(out_info), C.byref(desc),
                                _st()), "sessd_bev_conv_p2")


def bev_deconv_p2(in_planes, in_info, weight_h2, scale, shift, residual, resid_info, gain, shift_max, out_f32, out_planes, out_info, relu=True):
    _two, b, h, w, cin = in_planes.shape
    cout = (out_f32 if out_f32 is not None else out_planes).shape[-1]
    check(lib.sessd_bev_deconv_p2(_p(in_planes), _p(in_info), _p(weight_h2), int(weight_h2.shape[2]), _p(scale), _p(shift), _p(residual),
                                  _p(resid_info), float(gain), float(shift_max), _p(out_f32), _p(out_planes), _p(out_info), int(b), int(h),
                                  int(w), int(cin), int(cout), int(bool(relu)), _st()), "sessd_bev_deconv_p2")


def bev_split_planes(x, info, planes):
    """fp32 tensor -> planes with the scale from info[0] (its abs-max: call absmax(x, info[0:1]) first); info[1] <- scale"""
    check(lib.sessd_bev_split_planes(_p(x), int(x.numel()), _p(info), _p(planes), _st()), "sessd_bev_split_planes")
    return planes


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


def ssfa_fuse(x0, x1, w0, w1, s0, t0, s1, t1, out):
    npix = x0.numel() // x0.shape[-1]
    check(lib.sessd_ssfa_fuse(_p(x0), _p(x1), _p(w0), _p(w1), float(s0), float(t0), float(s1), float(t1), int(npix), int(x0.shape[-1]),
                              _p(out), _st()), "sessd_ssfa_fuse")
    return out


# ------------------------------------------------------------------------------------------------ post-processing
def make_post_cfg(batch, num_anchors=70400, anchors_per_loc=2, head_stride=24, score_thresh=0.3, nms_pre_max=1000, nms_post_max=100,
                  nms_iou_thresh=0.01, nms_ge=True, post_range=(0, -40.0, -5.0, 70.4, 40.0, 5.0), direction_offset=0.0,
                  use_frustum=False):
    c = PostCfg()
    c.batch, c.num_anchors, c.anchors_per_loc, c.head_stride = int(batch), int(num_anchors), int(anchors_per_loc), int(head_stride)
    c.score_thresh, c.nms_pre_max, c.nms_post_max = float(score_thresh), int(nms_pre_max), int(nms_post_max)
    c.nms_iou_thresh, c.nms_ge = float(nms_iou_thresh), int(bool(nms_ge))
    for j in range(6):
        c.post_range[j] = float(post_range[j])
    c.direction_offset, c.use_frustum = float(direction_offset), int(bool(use_frustum))
    return c


class PostBuffers:
    def __init__(self, cfg, device):
        self.cfg = cfg
        b, p = cfg.batch, cfg.nms_post_max
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
