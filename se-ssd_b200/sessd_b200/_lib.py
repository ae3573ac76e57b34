"""ctypes binding of libsessd_b200.so (the C ABI declared in include/sessd_b200.h).

The product path has NO fallback: if the CUDA library has not been built this module raises at import time
(``python se-ssd_b200/build.py`` builds it in-tree; ``__graft_entry__.build()`` does the same).
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(os.path.dirname(_HERE), "libsessd_b200.so")
LAB_PATH = os.path.join(os.path.dirname(_HERE), "libsessd_b200_lab.so")


class SessdError(RuntimeError):
    pass


class VoxelCfg(C.Structure):
    _fields_ = [("voxel_size", C.c_float * 3), ("range_min", C.c_float * 3), ("range_max", C.c_float * 3),
                ("grid", C.c_int * 3), ("max_points", C.c_int), ("max_voxels", C.c_int), ("num_feat", C.c_int)]


class Grid(C.Structure):
    _fields_ = [("batch", C.c_int), ("shape", C.c_int * 3)]


class ConvDesc(C.Structure):
    _fields_ = [("batch", C.c_int), ("in_h", C.c_int), ("in_w", C.c_int), ("cin", C.c_int),
                ("out_h", C.c_int), ("out_w", C.c_int), ("cout", C.c_int),
                ("grid_h", C.c_int), ("grid_w", C.c_int), ("in_stride", C.c_int),
                ("out_stride", C.c_int), ("out_off_y", C.c_int), ("out_off_x", C.c_int),
                ("ntaps", C.c_int), ("tap_dy", C.c_int * 16), ("tap_dx", C.c_int * 16), ("relu", C.c_int)]


class DinmsCfg(C.Structure):
    _fields_ = [("cnt_thresh", C.c_float), ("dist_edge", C.c_float * 4), ("sigma2", C.c_float * 3), ("suppressed_thresh", C.c_float),
                ("centerness_pow", C.c_float), ("centerness", C.c_int)]


class PostCfg(C.Structure):
    _fields_ = [("batch", C.c_int), ("num_anchors", C.c_int), ("anchors_per_loc", C.c_int), ("head_stride", C.c_int),
                ("score_thresh", C.c_float), ("nms_pre_max", C.c_int), ("nms_post_max", C.c_int),
                ("nms_iou_thresh", C.c_float), ("nms_ge", C.c_int), ("post_range", C.c_float * 6),
                ("direction_offset", C.c_float), ("use_frustum", C.c_int), ("nms_mode", C.c_int), ("dinms", DinmsCfg)]


class KittiFrames(C.Structure):
    _fields_ = [("num_frames", C.c_int), ("gt_off", C.c_void_p), ("gt", C.c_void_p), ("gt_code", C.c_void_p),
                ("gt_occluded", C.c_void_p), ("dc_off", C.c_void_p), ("dc", C.c_void_p), ("dt_off", C.c_void_p),
                ("dt_cnt", C.c_void_p), ("dt", C.c_void_p), ("dt_code", C.c_void_p), ("ov_off", C.c_void_p)]


_vp, _i, _f, _sz, _ll = C.c_void_p, C.c_int, C.c_float, C.c_size_t, C.c_longlong
_I3 = C.POINTER(C.c_int)

# name -> (restype, argtypes); must list every symbol declared in include/sessd_b200.h (tests check this)
SIGNATURES = {
    "sessd_version": (C.c_char_p, []),
    "sessd_launch_count": (_ll, []),
    "sessd_voxelize_workspace_bytes": (_sz, [_i, _i, C.POINTER(VoxelCfg)]),
    "sessd_voxelize": (_i, [_vp, _vp, _i, _i, C.POINTER(VoxelCfg), _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sessd_voxelize_host": (_i, [_vp, _i, C.POINTER(VoxelCfg), _vp, _vp, _vp]),
    "sessd_hash_bytes": (_sz, [_i, _I3]),
    "sessd_hash_build": (_i, [_vp, _vp, _i, Grid, _vp, _i, _vp]),
    "sessd_bitmap_words": (_sz, [Grid]),
    "sessd_scan_scratch_bytes": (_sz, [_sz]),
    "sessd_subm_rulebook": (_i, [_vp, _vp, _i, Grid, _I3, _i, _vp, _i, _vp, _vp]),
    "sessd_strided_rulebook": (_i, [_vp, _vp, _i, Grid, _i, _vp, _i, _I3, _I3, _I3, Grid, _vp, _vp, _vp, _vp, _i, _vp, _vp, _vp]),
    "sessd_tile_list_stride": (_i, [_i]),
    "sessd_rulebook_tile_lists": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "sessd_spconv_forward": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _vp, _vp]),
    "sessd_spconv_forward_rows": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _vp, _vp, _vp]),
    "sessd_spconv_forward_rows_planes": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _vp, _f, _f, _vp, _vp, _i, _vp, _vp]),
    "sessd_spconv_forward_cg": (_i, [_vp, _i, _i, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _i, _f, _f, _vp, _vp, _vp, _vp]),
    "sessd_set_sp_cg_deep": (None, [_i]),
    "sessd_spconv_cg_blocks_per_sm": (_i, [_i, _i, _i]),
    "sessd_absmax_rows": (_i, [_vp, _vp, _i, _i, _vp, _vp]),
    "sessd_rulebook_transpose": (_i, [_vp, _i, _vp, _i, _i, _vp, _vp]),
    "sessd_sparse_split_planes": (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _vp]),
    "sessd_dense_grad_gather": (_i, [_vp, _vp, _vp, _i, _i, Grid, _vp, _vp]),
    "sessd_spconv_wgrad_items": (_i, [_i, _i]),
    "sessd_spconv_wgrad_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "sessd_spconv_wgrad_rows": (_i, [_vp, _i, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "sessd_spconv_wgrad_cg": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _sz, _vp]),
    "sessd_sparse_to_dense_indexed": (_i, [_vp, _i, _vp, _i, Grid, _vp, _vp]),
    "sessd_sparse_to_dense": (_i, [_vp, _vp, _vp, _i, _i, Grid, _vp, _vp]),
    "sessd_bev_conv_p2": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, C.POINTER(ConvDesc), _vp, _vp, _vp]),
    "sessd_bev_deconv_p2": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "sessd_bev_skip_plan_words": (_ll, [_i, _i, _i, _I3]),
    "sessd_bev_skip_seg_words": (_ll, [_i, _i, _i, _I3]),
    "sessd_bev_skip_plan": (_i, [_vp, Grid, _vp, _vp, _vp]),
    "sessd_bev_skip_fill": (_i, [_vp, _vp, _vp, _i, _vp]),
    "sessd_bev_skip_fill_segs": (_i, [_vp, _vp, _vp, _i, _vp]),
    "sessd_bev_wgrad_items": (_i, [C.POINTER(ConvDesc)]),
    "sessd_bev_wgrad_workspace_bytes": (_sz, [C.POINTER(ConvDesc)]),
    "sessd_bev_wgrad": (_i, [_vp, _vp, _vp, _vp, C.POINTER(ConvDesc), _vp, _vp, _sz, _vp]),
    "sessd_bev_split_planes": (_i, [_vp, _ll, _vp, _vp, _vp]),
    "sessd_sparse_to_dense_planes": (_i, [_vp, _i, _vp, _i, Grid, _vp, _vp, _vp, _vp]),
    "sessd_ssfa_fuse_planes": (_i, [_vp, _vp, _vp, _vp, _f, _f, _f, _f, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sessd_absmax": (_i, [_vp, C.c_longlong, _vp, _vp]),
    "sessd_postprocess_workspace_bytes": (_sz, [C.POINTER(PostCfg)]),
    "sessd_postprocess": (_i, [_vp, _vp, _vp, C.POINTER(PostCfg), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sessd_postprocess_packed": (_i, [_vp, _vp, _vp, C.POINTER(PostCfg), _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sessd_rotate_nms_workspace_bytes": (_sz, [_i, _i]),
    "sessd_rotate_nms": (_i, [_vp, _vp, _vp, _i, _i, _i, _f, _i, _vp, _vp, _vp, _sz, _vp]),
    "sessd_rotate_weighted_nms_workspace_bytes": (_sz, [_i, _i]),
    "sessd_rotate_weighted_nms": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, C.POINTER(DinmsCfg), _vp, _vp, _vp, _vp, _vp, _vp, _vp,
                                       _vp, _sz, _vp]),
    "sessd_boxes_overlap_bev": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "sessd_boxes_aligned_overlap_bev": (_i, [_vp, _vp, _i, _vp, _vp]),
    "sessd_boxes_iou_bev": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "sessd_boxes_iou3d": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "sessd_nms_workspace_bytes": (_sz, [_i]),
    "sessd_nms_sorted": (_i, [_vp, _i, _f, _i, _vp, _vp, _vp, _sz, _vp]),
    "sessd_head_loss_workspace_bytes": (_sz, [_i]),
    "sessd_head_loss": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _f, _f, _f, _f, _f, _f, _vp, _vp, _vp, _sz, _vp]),
    "sessd_odiou_loss_workspace_bytes": (_sz, [_i]),
    "sessd_odiou_loss": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sessd_odiou_pairs_host": (_i, [_vp, _vp, _i, _vp, _vp]),
    "sessd_iou_pred_loss_workspace_bytes": (_sz, [_i]),
    "sessd_iou_pred_loss": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _f, _vp, _vp, _vp, _sz, _vp]),
    "sessd_axpby": (_i, [_vp, _vp, _f, _f, _ll, _vp]),
    "sessd_adamw_step": (_i, [_vp, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _f, _i, _vp]),
    "sessd_grad_sqnorm_workspace_bytes": (_sz, [_ll]),
    "sessd_grad_sqnorm": (_i, [_vp, _ll, _f, _vp, _vp, _vp]),
    "sessd_adamw_clip_ema_step": (_i, [_vp, _vp, _vp, _vp, _ll, _f, _f, _f, _f, _f, _i, _vp, _vp, C.c_double, _vp]),
    "sessd_assign_workspace_bytes": (_sz, [_i, _i, _i]),
    "sessd_assign_targets": (_i, [_vp, _i, _vp, _vp, _i, _i, _f, _f, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sessd_box_collision": (_i, [_vp, _i, _vp, _i, _vp, _vp]),
    "sessd_noise_per_box": (_i, [_vp, _vp, _vp, _i, _i, _vp, _vp, _i, C.c_double, _vp, _vp]),
    "sessd_points_in_boxes": (_i, [_vp, _i, _i, _vp, _i, C.c_double, _vp, _vp]),
    "sessd_augment_points": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _vp, _i, _vp, C.c_double, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sessd_augment_boxes": (_i, [_vp, _vp, _vp, _vp, _i, _i, _vp, _vp, _i, _vp, _vp, C.POINTER(C.c_float), _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    "sessd_gtaug_select_host": (_i, [_vp, _i, _i, _vp]),
    "sessd_gtaug_paste_workspace_bytes": (_sz, [_i, _i, _i]),
    "sessd_gtaug_paste": (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _i, _vp, _sz, _vp, _i, _vp, _vp]),
    "sessd_sada_pyramids": (_i, [_vp, _i, _vp, _vp, _vp]),
    "sessd_sada_membership": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "sessd_sada_compact_workspace_bytes": (_sz, [_i]),
    "sessd_sada_compact": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _vp, _sz, _vp, _i, _vp, _vp]),
    "sessd_sada_fps_workspace_bytes": (_sz, [_i, _i]),
    "sessd_sada_fps": (_i, [_vp, _i, _vp, _vp, _i, _vp, _i, _i, _vp, _sz, _vp, _i, _vp, _vp]),
    "sessd_sada_swap": (_i, [_vp, _i, _vp, _vp, _i, _vp, _vp, _i, _vp, _i, _vp, _i, _vp, _vp, _vp]),
    "sessd_sada_shuffle": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp]),
    "sessd_prep_frustum_compact_workspace_bytes": (_sz, [_i]),
    "sessd_prep_frustum_compact": (_i, [_vp, _vp, _i, _i, _vp, _vp, _sz, _vp, _i, _vp, _vp]),
    "sessd_prep_box_count": (_i, [_vp, _vp, _i, _i, _vp, _vp, _i, _vp, _vp]),
    "sessd_prep_box_gather_workspace_bytes": (_sz, [_i]),
    "sessd_prep_box_gather": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _i, _vp, _i, _vp, _sz, _vp, _i, _vp, _vp]),
    "sessd_kitti_convert_workspace_bytes": (_sz, [_ll]),
    "sessd_kitti_convert_detections": (_i, [_vp, _vp, _vp, _vp, _i, _ll, _vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "sessd_kitti_overlaps": (_i, [C.POINTER(KittiFrames), _i, _i, C.c_double, _vp, _vp]),
    "sessd_kitti_eval_workspace_bytes": (_sz, [_i, _ll, _ll, _i, _i]),
    "sessd_kitti_eval": (_i, [C.POINTER(KittiFrames), _i, _i, _i, C.c_double, _i, _vp, _vp, _i, _ll, _ll, _vp, _vp, _vp, _vp, _vp, _vp,
                              _sz, _vp]),
}


# include/sessd_b200_lab.h: the in-kernel fp16 split, the probes and the launch plan of the BEV conv (libsessd_b200_lab.so; loaded on first
# use, by tests and scripts only)
LAB_SIGNATURES = {
    "sessd_bev_conv_h2": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, C.POINTER(ConvDesc), _vp, _vp, _vp]),
    "sessd_bev_deconv_h2": (_i, [_vp, _vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp, _vp]),
    "sessd_bev_conv_p2_profile": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, C.POINTER(ConvDesc), _vp, _vp, _vp,
                                       _vp]),
    "sessd_bev_deconv_p2_profile": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp, _vp,
                                         _vp, _vp]),
    "sessd_bev_conv_p2_loads": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, C.POINTER(ConvDesc), _vp, _i, _vp, _vp]),
    "sessd_bev_conv_p2_seg_loads": (_i, [_vp, _vp, _vp, _i, _vp, _vp, _vp, _vp, _f, _f, _vp, _vp, _vp, C.POINTER(ConvDesc), _vp, _vp,
                                         _vp]),
    "sessd_bev_p2_plan": (_i, [C.POINTER(ConvDesc), _i, _i, _i, _i, _I3]),
}


def _load(path, signatures, mode=C.DEFAULT_MODE):
    if not os.path.exists(path):
        raise ImportError(
            "sessd_b200: %s is missing -- the CUDA library has not been built (run `python se-ssd_b200/build.py`). "
            "There is no CPU fallback." % path)
    lib = C.CDLL(path, mode=mode)
    for name, (res, args) in signatures.items():
        fn = getattr(lib, name)
        fn.restype = res
        fn.argtypes = args
    return lib


class _Libs:
    """`lib.sessd_xxx` resolves in libsessd_b200.so (the product, loaded at import time); the names of LAB_SIGNATURES resolve in
    libsessd_b200_lab.so, which is loaded the first time one of them is touched (the product path never does)."""

    def __init__(self):
        self._prod = _load(LIB_PATH, SIGNATURES, C.RTLD_GLOBAL)
        self._lab = None

    def lab(self):
        if self._lab is None:
            self._lab = _load(LAB_PATH, LAB_SIGNATURES)
        return self._lab

    @property
    def lab_loaded(self):
        return self._lab is not None

    def __getattr__(self, name):
        if name in LAB_SIGNATURES:
            return getattr(self.lab(), name)
        return getattr(self._prod, name)


lib = _Libs()


def check(rc, what):
    if rc != 0:
        kind = {-1: "invalid argument", -2: "capacity exceeded", -3: "workspace too small"}.get(rc, "cudaError %d" % rc)
        raise SessdError("%s failed: %s" % (what, kind))


def version():
    return lib.sessd_version().decode()


def launch_count():
    return int(lib.sessd_launch_count())
