"""KITTI data preparation: info files, image-FOV point clouds (velodyne_reduced) and the GT database, in the reference's formats.

    python -m sessd_b200.kitti_prep ROOT [--imageset-dir DIR]

Does what the reference's tools/create_data.py (kitti_data_prep) does with create_kitti_info_file, create_reduced_point_cloud and
create_groundtruth_database (det3d/datasets/kitti/kitti_common.py, det3d/datasets/utils/create_gt_database.py), in one pass that reads
each raw `.bin` once: per batch of frames, the image-frustum compaction, then (train and val frames) the point count of every label box,
then (train frames) the database objects' points, all on the device over the resident reduced frames.  Files are read by a host thread
pool into pinned memory while the device works on the previous batch; each batch is one upload, one read-back of the row counts and one
fetch of the outputs.

Every plane is computed here on the host in fp64 (`surface_planes`: surface_equ_3d_jitv2's arithmetic, operation for operation); the
device evaluates the sign tests (csrc/kitti_prep.cu).  The reference-named functions of det3d.datasets.kitti.kitti_common,
det3d.datasets.utils.create_gt_database and det3d.core.bbox.box_np_ops are thin calls into `run_frames` with the passes they need.

Deviations from the reference:
- the split files ImageSets/{train,val,test}.txt are read from `imageset_dir` (default <root>/ImageSets);
- image_shape is (height, width) from the PNG IHDR chunk, without decoding the image;
- gt_aug_with_context > 0 and with_back=True raise NotImplementedError; add_rgb, lidar_only, bev_only and coors_range are ignored, as
  in the reference;
- box-angle sin / cos are the correctly rounded fp64 values (math.sin / math.cos), not numpy's vector functions.
"""
import math
import os
import pickle
import struct
import sys
from concurrent.futures import ThreadPoolExecutor
from pathlib import Path

import numpy as np
import torch

from . import ops

PNG_SIGNATURE = b"\x89PNG\r\n\x1a\n"
# corner_to_surfaces_3d's corner order: six faces with inward normals
SURFACE_CORNERS = np.array([0, 1, 2, 3, 7, 6, 5, 4, 0, 3, 7, 4, 1, 5, 6, 2, 0, 4, 5, 1, 3, 2, 6, 7]).reshape(6, 4)
# planes every point with a non-NaN sign satisfies: (((x*0) + (y*0)) + (z*0)) - 1 < 0 -- the frustum of "keep every point"
ALL_PASS = np.array([[0.0, 0.0, 0.0, -1.0]] * 6)


# ------------------------------------------------------------------------------------------------ host parsing
def read_imageset(path):
    with open(path, "r") as f:
        return [int(line) for line in f.readlines()]


def imageset_ids(imageset_dir, split):
    path = Path(imageset_dir) / ("%s.txt" % split)
    if not path.exists():
        raise FileNotFoundError("KITTI split file %s not found: put the split files train.txt, val.txt and test.txt (one frame number "
                                "per line, e.g. the SECOND / det3d ImageSets) into %s, or pass imageset_dir" % (path, imageset_dir))
    return read_imageset(path)


def png_shape(path):
    """(height, width) int32 from a PNG's IHDR chunk; ValueError for a file that is not a PNG."""
    with open(path, "rb") as f:
        head = f.read(24)
    if len(head) < 24 or head[:8] != PNG_SIGNATURE or head[12:16] != b"IHDR":
        raise ValueError("not a PNG image: %s" % path)
    w, h = struct.unpack(">II", head[16:24])
    return np.array([h, w], dtype=np.int32)


def get_label_anno(label_path):
    """A KITTI label file as the reference's annotation dict: dimensions reordered hwl -> lhw, `score` from 16-field lines (zeros
    otherwise), `index` / `group_ids` assigned by position."""
    with open(label_path, "r") as f:
        rows = [line.strip().split(" ") for line in f.readlines()]
    num_objects = len([r[0] for r in rows if r[0] != "DontCare"])
    num_gt = len(rows)
    anno = {"name": np.array([r[0] for r in rows]),
            "truncated": np.array([float(r[1]) for r in rows]),
            "occluded": np.array([int(r[2]) for r in rows]),
            "alpha": np.array([float(r[3]) for r in rows]),
            "bbox": np.array([[float(v) for v in r[4:8]] for r in rows]).reshape(-1, 4),
            "dimensions": np.array([[float(v) for v in r[8:11]] for r in rows]).reshape(-1, 3)[:, [2, 0, 1]],
            "location": np.array([[float(v) for v in r[11:14]] for r in rows]).reshape(-1, 3),
            "rotation_y": np.array([float(r[14]) for r in rows]).reshape(-1)}
    if num_gt and len(rows[0]) == 16:
        anno["score"] = np.array([float(r[15]) for r in rows])
    else:
        anno["score"] = np.zeros((anno["bbox"].shape[0],))
    anno["index"] = np.array(list(range(num_objects)) + [-1] * (num_gt - num_objects), dtype=np.int32)
    anno["group_ids"] = np.arange(num_gt, dtype=np.int32)
    return anno


def _extend(mat):
    return np.concatenate([mat, np.array([[0.0, 0.0, 0.0, 1.0]])], axis=0)


def read_calib(path, extend_matrix=True):
    """P0-P3, R0_rect, Tr_velo_to_cam and Tr_imu_to_velo of a KITTI calibration file, extended to 4x4 when extend_matrix."""
    with open(path, "r") as f:
        lines = f.readlines()

    def mat(k, n, shape):
        return np.array([float(v) for v in lines[k].split(" ")[1:1 + n]]).reshape(shape)
    P = [mat(k, 12, [3, 4]) for k in range(4)]
    rect = mat(4, 9, [3, 3])
    velo, imu = mat(5, 12, [3, 4]), mat(6, 12, [3, 4])
    if extend_matrix:
        P = [_extend(p) for p in P]
        r4 = np.zeros([4, 4], dtype=rect.dtype)
        r4[3, 3] = 1.0
        r4[:3, :3] = rect
        rect = r4
        velo, imu = _extend(velo), _extend(imu)
    return {"P0": P[0], "P1": P[1], "P2": P[2], "P3": P[3], "R0_rect": rect, "Tr_velo_to_cam": velo, "Tr_imu_to_velo": imu}


def add_difficulty_to_annos(info):
    """KITTI difficulty per object: 0 easy, 1 moderate, 2 hard, -1 none (a height <= the minimum fails a level)."""
    annos = info["annos"]
    height = annos["bbox"][:, 3] - annos["bbox"][:, 1]
    occ, trunc = annos["occluded"], annos["truncated"]
    n = len(annos["dimensions"])
    masks = [np.ones((n,), dtype=bool) & ~((occ > mo) | (height <= mh) | (trunc > mt))
             for mh, mo, mt in ((40, 0, 0.15), (25, 1, 0.3), (25, 2, 0.5))]
    easy, moderate = masks[0], np.logical_xor(masks[0], masks[1])
    hard = np.logical_xor(masks[2], masks[1])
    diff = [0 if easy[i] else 1 if moderate[i] else 2 if hard[i] else -1 for i in range(n)]
    annos["difficulty"] = np.array(diff, np.int32)
    return diff


def _kitti_path(idx, root, kind, tail, training, relative_path, exist_check=True):
    rel = Path("training" if training else "testing") / kind / ("%06d%s" % (idx, tail))
    if exist_check and not (Path(root) / rel).exists():
        raise ValueError("file not exist: {}".format(rel))
    return str(rel) if relative_path else str(Path(root) / rel)


def image_info(root, idx, training=True, label_info=True, velodyne=False, calib=False, extend_matrix=True, relative_path=True,
               with_imageshape=True):
    """One frame's info record, as get_kitti_image_info writes it (without num_points_in_gt)."""
    root = Path(root)
    info, pc_info, img = {}, {"num_features": 4}, {"image_idx": idx}
    if velodyne:
        pc_info["velodyne_path"] = _kitti_path(idx, root, "velodyne", ".bin", training, relative_path)
    img["image_path"] = _kitti_path(idx, root, "image_2", ".png", training, relative_path)
    if with_imageshape:
        p = img["image_path"]
        img["image_shape"] = png_shape(str(root / p) if relative_path else p)
    annos = None
    if label_info:
        p = _kitti_path(idx, root, "label_2", ".txt", training, relative_path)
        annos = get_label_anno(str(root / p) if relative_path else p)
    info["image"] = img
    info["point_cloud"] = pc_info
    if calib:
        info["calib"] = read_calib(_kitti_path(idx, root, "calib", ".txt", training, relative_path=False), extend_matrix)
    if annos is not None:
        info["annos"] = annos
        add_difficulty_to_annos(info)
    return info


# ------------------------------------------------------------------------------------------------ planes (host, fp64)
def surface_planes(surfaces):
    """[N, S, >=3, 3] surfaces -> [N, S, 4] fp64 (a, b, c, d): surface_equ_3d_jitv2's arithmetic, operation for operation."""
    s = np.asarray(surfaces, np.float64)
    s0, s1, s2 = s[:, :, 0], s[:, :, 1], s[:, :, 2]
    sv0, sv1 = s0 - s1, s1 - s2
    a = sv0[..., 1] * sv1[..., 2] - sv0[..., 2] * sv1[..., 1]
    b = sv0[..., 2] * sv1[..., 0] - sv0[..., 0] * sv1[..., 2]
    c = sv0[..., 0] * sv1[..., 1] - sv0[..., 1] * sv1[..., 0]
    d = ((-s0[..., 0]) * a - s0[..., 1] * b) - s0[..., 2] * c
    return np.stack([a, b, c, d], axis=-1)


def frustum_planes(rect, Trv2c, P2, image_shape):
    """[6, 4] planes of the image frustum in velodyne coordinates (remove_outside_points' polyhedron)."""
    from det3d.core.bbox import box_np_ops
    return surface_planes(box_np_ops.get_valid_frustum(rect, Trv2c, P2, image_shape)[:, :, :3])[0]


def center_to_corner_box3d(centers, dims, angles=None, origin=(0.5, 0.5, 0.5), axis=2):
    """[N, 8, 3] fp64 corners of boxes rotated about z (corners_nd order), with correctly rounded sin / cos of the angles."""
    if axis not in (2, -1):
        raise NotImplementedError("center_to_corner_box3d: only rotation about the z axis (axis=2) is supported")
    centers, dims = np.asarray(centers), np.asarray(dims)
    unit = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]], dtype=dims.dtype)
    corners = dims.reshape([-1, 1, 3]) * (unit - np.array(origin, dtype=dims.dtype)).reshape([1, 8, 3])
    if angles is not None:
        ang = np.asarray(angles).reshape(-1)
        sin = np.array([math.sin(a) for a in ang], dtype=corners.dtype)[:, None]
        cos = np.array([math.cos(a) for a in ang], dtype=corners.dtype)[:, None]
        x, y, z = corners[..., 0], corners[..., 1], corners[..., 2]
        corners = np.stack([x * cos + y * sin, -(x * sin) + y * cos, z], axis=-1)
    return corners + centers.reshape([-1, 1, 3])


def box_planes(boxes, origin=(0.5, 0.5, 0.5)):
    """[K, 7] (x, y, z, w, l, h, ry) lidar boxes -> [K, 6, 4] fp64 face planes (points_in_rbbox's polyhedra)."""
    boxes = np.asarray(boxes).reshape(-1, 7)
    if len(boxes) == 0:
        return np.zeros((0, 6, 4))
    corners = center_to_corner_box3d(boxes[:, :3], boxes[:, 3:6], boxes[:, 6], origin=origin)
    return surface_planes(corners[:, SURFACE_CORNERS][:, :, :3])


def info_boxes(info):
    """_calculate_num_points_in_gt's boxes: the first num_obj label rows (num_obj = the non-DontCare count; the reference assumes the
    DontCare lines come last), fp64, through box_camera_to_lidar WITHOUT change_box3d_center_ -- counted as if the box sat h/2 lower."""
    from det3d.core.bbox import box_np_ops
    annos, calib = info["annos"], info["calib"]
    n = len([x for x in annos["name"] if x != "DontCare"])
    cam = np.concatenate([annos["location"][:n], annos["dimensions"][:n], annos["rotation_y"][:n][..., np.newaxis]], axis=1)
    return box_np_ops.box_camera_to_lidar(cam, calib["R0_rect"], calib["Tr_velo_to_cam"])


def db_boxes(info):
    """create_groundtruth_database's boxes and names: LoadPointCloudAnnotations' fp32 cast, fp64 box_camera_to_lidar and
    change_box3d_center_, DontCare removed; plus the annotations the database reads (difficulty)."""
    from det3d.core.bbox import box_np_ops
    from det3d.datasets.pipelines.loading import remove_dontcare
    annos, calib = remove_dontcare(info["annos"]), info["calib"]
    b = np.concatenate([annos["location"], annos["dimensions"], annos["rotation_y"][..., np.newaxis]], axis=1).astype(np.float32)
    b = box_np_ops.box_camera_to_lidar(b, calib["R0_rect"], calib["Tr_velo_to_cam"])
    box_np_ops.change_box3d_center_(b, [0.5, 0.5, 0], [0.5, 0.5, 0.5])
    return b, annos


# ------------------------------------------------------------------------------------------------ device passes
class Frame:
    """One frame of a batch: its points (a .bin path, or an [N, 4] f32 array), the frustum planes [6, 4], the count boxes' planes
    [Kc, 6, 4] and the database boxes' planes [Kd, 6, 4] with their centres [Kd, 3]."""

    def __init__(self, src, frustum=ALL_PASS, count_planes=None, db_planes=None, db_centres=None, tag=None):
        self.src, self.frustum, self.tag = src, np.asarray(frustum, np.float64), tag
        self.count_planes = np.zeros((0, 6, 4)) if count_planes is None else np.asarray(count_planes, np.float64)
        self.db_planes = np.zeros((0, 6, 4)) if db_planes is None else np.asarray(db_planes, np.float64)
        self.db_centres = np.zeros((0, 3)) if db_centres is None else np.asarray(db_centres, np.float64).reshape(-1, 3)

    def rows(self):
        return os.path.getsize(self.src) // 16 if isinstance(self.src, (str, Path)) else len(self.src)


class Result:
    """A frame's outputs: reduced [R, 4] f32, counts [Kc] i32, db_counts [Kd] i32, db_rows: one [n_k, 4] f32 array per database box."""

    def __init__(self, frame, reduced, counts, db_counts, db_rows):
        self.frame, self.reduced, self.counts, self.db_counts, self.db_rows = frame, reduced, counts, db_counts, db_rows


def _align(n):
    return (n + 15) & ~15


class _Layout:
    """byte offsets of one batch's upload: points, then the int32 offsets, then the fp64 planes and centres (16-byte aligned each)"""

    def __init__(self, frames):
        self.B = len(frames)
        self.sizes = [f.rows() for f in frames]
        self.P = int(sum(self.sizes))
        self.kc = [len(f.count_planes) for f in frames]
        self.kd = [len(f.db_planes) for f in frames]
        self.Kc, self.Kd = int(sum(self.kc)), int(sum(self.kd))
        off = 0
        spans = {}
        for name, nbytes in (("points", 16 * self.P), ("frame_off", 4 * (self.B + 1)), ("count_off", 4 * (self.B + 1)),
                             ("db_off", 4 * (self.B + 1)), ("frustum", 8 * 24 * self.B), ("count_planes", 8 * 24 * self.Kc),
                             ("db_planes", 8 * 24 * self.Kd), ("db_centres", 8 * 3 * self.Kd)):
            spans[name] = (off, nbytes)
            off = _align(off + nbytes)
        self.spans, self.nbytes = spans, max(off, 16)


def _fill(buf, lay, frames, pool):
    """the batch's upload in pinned host memory; the point files are read by the pool straight into it"""
    host = buf.numpy()

    def view(name, dtype):
        o, n = lay.spans[name]
        return host[o:o + n].view(dtype)
    pts = view("points", np.float32).reshape(-1, 4)
    fo = np.concatenate([[0], np.cumsum(lay.sizes)]).astype(np.int32)
    view("frame_off", np.int32)[:] = fo
    view("count_off", np.int32)[:] = np.concatenate([[0], np.cumsum(lay.kc)]).astype(np.int32)
    view("db_off", np.int32)[:] = np.concatenate([[0], np.cumsum(lay.kd)]).astype(np.int32)
    view("frustum", np.float64)[:] = np.concatenate([f.frustum.reshape(-1) for f in frames]) if frames else []
    if lay.Kc:
        view("count_planes", np.float64)[:] = np.concatenate([f.count_planes.reshape(-1) for f in frames])
    if lay.Kd:
        view("db_planes", np.float64)[:] = np.concatenate([f.db_planes.reshape(-1) for f in frames])
        view("db_centres", np.float64)[:] = np.concatenate([f.db_centres.reshape(-1) for f in frames])

    def read(b):
        dst = pts[fo[b]:fo[b + 1]]
        src = frames[b].src
        if isinstance(src, (str, Path)):
            with open(src, "rb") as f:
                got = f.readinto(memoryview(dst).cast("B"))
            if got != dst.nbytes:
                raise IOError("short read of %s" % src)
        else:
            dst[:] = np.asarray(src, np.float32).reshape(-1, 4)
    list(pool.map(read, range(lay.B)))


class Runner:
    """The device half of the preparation: batches of frames through frustum compaction, box counts and the object gather."""

    def __init__(self, device="cuda", batch_frames=16, workers=8):
        self.device = torch.device(device)
        self.batch_frames, self.workers = int(batch_frames), int(workers)
        self.event_ms = 0.0      # device time of the stages (CUDA events), summed over batches

    def _device_batch(self, up_host, lay, dev_buf, evs):
        dev = self.device
        dev_buf[:lay.nbytes].copy_(up_host[:lay.nbytes], non_blocking=True)

        def view(name, dtype, shape):
            o, n = lay.spans[name]
            return dev_buf[o:o + n].view(dtype).view(shape)
        pts = view("points", torch.float32, (-1, 4)) if lay.P else torch.empty((0, 4), dtype=torch.float32, device=dev)
        frame_off = view("frame_off", torch.int32, (-1,))
        count_off, db_off = view("count_off", torch.int32, (-1,)), view("db_off", torch.int32, (-1,))
        frustum = view("frustum", torch.float64, (lay.B, 6, 4))
        cpl = view("count_planes", torch.float64, (lay.Kc, 6, 4)) if lay.Kc else torch.empty((0, 6, 4), dtype=torch.float64, device=dev)
        dpl = view("db_planes", torch.float64, (lay.Kd, 6, 4)) if lay.Kd else torch.empty((0, 6, 4), dtype=torch.float64, device=dev)
        dce = view("db_centres", torch.float64, (lay.Kd, 3)) if lay.Kd else torch.empty((0, 3), dtype=torch.float64, device=dev)
        # [frame_off_out | counts | db_counts]: the one read-back between the count and the gather
        ints = torch.empty((lay.B + 1 + lay.Kc + lay.Kd + 1,), dtype=torch.int32, device=dev)
        fo_out = ints[:lay.B + 1]
        evs[0].record()
        out, _ = ops.prep_frustum_compact(pts, frame_off, frustum, frame_off_out=fo_out)
        if lay.Kc:
            ops.prep_box_count(out, fo_out, cpl, count_off, counts=ints[lay.B + 1:lay.B + 1 + lay.Kc])
        if lay.Kd:
            ops.prep_box_count(out, fo_out, dpl, db_off, counts=ints[lay.B + 1 + lay.Kc:lay.B + 1 + lay.Kc + lay.Kd])
        evs[1].record()
        h_ints = ints.cpu().numpy()
        fo = h_ints[:lay.B + 1].astype(np.int64)
        counts = h_ints[lay.B + 1:lay.B + 1 + lay.Kc].copy()
        dcounts = h_ints[lay.B + 1 + lay.Kc:lay.B + 1 + lay.Kc + lay.Kd].copy()
        R, T = int(fo[-1]), int(dcounts.sum())
        if R + T > out.shape[0]:
            grown = torch.empty((R + T, 4), dtype=torch.float32, device=dev)
            grown[:R].copy_(out[:R])
            out = grown
        evs[2].record()
        if lay.Kd:
            ops.prep_box_gather(out, fo_out, dpl, dce, db_off, ints[lay.B + 1 + lay.Kc:lay.B + 1 + lay.Kc + lay.Kd], T, out=out[R:],
                                obj_off=torch.empty((lay.Kd + 1,), dtype=torch.int32, device=dev))
        evs[3].record()
        host = out[:R + T].cpu().numpy() if R + T else np.zeros((0, 4), np.float32)
        self.event_ms += evs[0].elapsed_time(evs[1]) + evs[2].elapsed_time(evs[3])
        return host, fo, counts, dcounts

    def run(self, frames, on_result):
        """Calls on_result(Result) for every frame, in order.  Reads the next batch while the device works on this one."""
        frames = list(frames)
        batches = [frames[i:i + self.batch_frames] for i in range(0, len(frames), self.batch_frames)]
        if not batches:
            return
        pool = ThreadPoolExecutor(max_workers=self.workers)
        reader = ThreadPoolExecutor(max_workers=1)
        try:
            lays = [_Layout(b) for b in batches]
            cap = max(lay.nbytes for lay in lays)
            ups = [torch.empty((cap,), dtype=torch.uint8, pin_memory=True) for _ in range(2)]
            dev_buf = torch.empty((cap,), dtype=torch.uint8, device=self.device)
            evs = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
            nxt = reader.submit(_fill, ups[0], lays[0], batches[0], pool)
            for i, (batch, lay) in enumerate(zip(batches, lays)):
                nxt.result()
                if i + 1 < len(batches):
                    # batch i + 1 is read into the other pinned buffer while the device works on batch i; that buffer's last upload
                    # (batch i - 1) completed before batch i - 1's read-back returned
                    nxt = reader.submit(_fill, ups[(i + 1) % 2], lays[i + 1], batches[i + 1], pool)
                host, fo, counts, dcounts = self._device_batch(ups[i % 2], lay, dev_buf, evs)
                R = int(fo[-1])
                doff = R + np.concatenate([[0], np.cumsum(dcounts)]).astype(np.int64)
                c0 = d0 = 0
                for b, f in enumerate(batch):
                    kc, kd = lay.kc[b], lay.kd[b]
                    rows = [host[doff[d0 + k]:doff[d0 + k + 1]] for k in range(kd)]
                    on_result(Result(f, host[fo[b]:fo[b + 1]], counts[c0:c0 + kc], dcounts[d0:d0 + kd], rows))
                    c0, d0 = c0 + kc, d0 + kd
        finally:
            reader.shutdown()
            pool.shutdown()


def run_frames(frames, batch_frames=16, workers=8, device="cuda"):
    """[Result] of every frame, in order (see Runner)."""
    out = []
    Runner(device, batch_frames, workers).run(frames, out.append)
    return out


def _index_rows(points):
    """[N, 4] f32 rows x, y, z and the row index as the bits of the fourth float (the gather and the compaction copy it unchanged)"""
    p = np.asarray(points)
    rows = np.empty((len(p), 4), np.float32)
    rows[:, :3] = p[:, :3]
    rows[:, 3] = np.arange(len(p), dtype=np.int32).view(np.float32)
    return rows


def _row_index(rows):
    return np.ascontiguousarray(rows[:, 3]).view(np.int32)


def remove_outside_points(points, rect, Trv2c, P2, image_shape):
    """The rows of points inside the image frustum, in order (box_np_ops.remove_outside_points; membership on the device)."""
    r = run_frames([Frame(_index_rows(points), frustum_planes(rect, Trv2c, P2, image_shape))])[0]
    return points[_row_index(r.reduced)]


def points_in_rbbox(points, rbbox, z_axis=2, origin=(0.5, 0.5, 0.5)):
    """[N, K] bool: point i inside box k (box_np_ops.points_in_rbbox; membership on the device)."""
    if z_axis != 2:
        raise NotImplementedError("points_in_rbbox: only z_axis=2 is supported")
    rbbox = np.asarray(rbbox)
    planes = box_planes(rbbox, origin)
    r = run_frames([Frame(_index_rows(points), db_planes=planes, db_centres=np.zeros((len(rbbox), 3)))])[0]
    mask = np.zeros((len(points), len(rbbox)), dtype=bool)
    for k, rows in enumerate(r.db_rows):
        mask[_row_index(rows), k] = True
    return mask


# ------------------------------------------------------------------------------------------------ the driver
def _velo_path(root, info, relative_path=True):
    p = info["point_cloud"]["velodyne_path"]
    return str(Path(root) / p) if relative_path else p


def _reduced_path(v_path, save_path=None):
    v_path = Path(v_path)
    if save_path is None:
        return str(v_path.parent.parent / (v_path.parent.stem + "_reduced") / v_path.name)
    return str(Path(save_path) / v_path.name)


def _frame_for(root, info, relative_path, reduce, count, db, used=None):
    calib = info["calib"]
    frustum = frustum_planes(calib["R0_rect"], calib["Tr_velo_to_cam"], calib["P2"], info["image"]["image_shape"]) if reduce else ALL_PASS
    f = Frame(_velo_path(root, info, relative_path), frustum, tag=info)
    if count and "annos" in info:
        f.count_planes = box_planes(info_boxes(info))
    if db and "annos" in info:
        boxes, annos = db_boxes(info)
        f.db_planes, f.db_centres, f.db = box_planes(boxes), boxes[:, :3], (boxes, annos)
    return f


class _DbWriter:
    """create_groundtruth_database's loop over the gathered rows: one .bin per object, dbinfos for used_classes, the group counter"""

    def __init__(self, db_path, used_classes=None, relative_path=True):
        self.db_path, self.used, self.relative = Path(db_path), used_classes, relative_path
        self.db_path.mkdir(parents=True, exist_ok=True)
        self.infos, self.group_counter = {}, 0

    def add(self, info, boxes, annos, counts, rows):
        image_idx = info["image"]["image_idx"]
        names = annos["name"]
        difficulty = annos["difficulty"] if "difficulty" in annos else np.zeros(boxes.shape[0], dtype=np.int32)
        group_ids = np.arange(boxes.shape[0], dtype=np.int64)
        group = {}
        for i in range(boxes.shape[0]):
            filename = f"{image_idx}_{names[i]}_{i}.bin"
            with open(self.db_path / filename, "w") as f:
                rows[i].tofile(f)
            if self.used is None or names[i] in self.used:
                entry = {"name": names[i], "path": str(self.db_path.stem + "/" + filename) if self.relative else str(self.db_path / filename),
                         "image_idx": image_idx, "gt_idx": i, "box3d_lidar": boxes[i], "num_points_in_gt": np.int64(counts[i]),
                         "difficulty": difficulty[i]}
                if group_ids[i] not in group:
                    group[group_ids[i]] = self.group_counter
                    self.group_counter += 1
                entry["group_id"] = group[group_ids[i]]
                self.infos.setdefault(names[i], []).append(entry)

    def dump(self, path):
        with open(path, "wb") as f:
            pickle.dump(self.infos, f)


def prepare(root, infos, relative_path=True, reduce=False, count=False, remove_outside=True, db=None, reduced_save_path=None,
            batch_frames=16, workers=8):
    """The fused pass over `infos` (list of info records): write each frame's reduced file when `reduce`, set annos["num_points_in_gt"]
    when `count` (on the frustum-reduced points when remove_outside), feed the database writer `db` (a _DbWriter) when given."""
    frames = [_frame_for(root, info, relative_path, reduce or remove_outside, count, db is not None) for info in infos]
    writer = ThreadPoolExecutor(max_workers=max(1, workers // 2))
    pending = []

    def done(r):
        info = r.frame.tag
        if reduce:
            pending.append(writer.submit(r.reduced.tofile, _reduced_path(r.frame.src, reduced_save_path)))
        if count and "annos" in info:
            n_ign = len(info["annos"]["dimensions"]) - len(r.counts)
            info["annos"]["num_points_in_gt"] = np.concatenate([r.counts.astype(np.int64), -np.ones([n_ign])]).astype(np.int32)
        if db is not None and hasattr(r.frame, "db"):
            boxes, annos = r.frame.db
            db.add(info, boxes, annos, r.db_counts, r.db_rows)
    try:
        if reduce:
            for f in frames:
                Path(_reduced_path(f.src, reduced_save_path)).parent.mkdir(parents=True, exist_ok=True)
        Runner("cuda", batch_frames, workers).run(frames, done)
        for p in pending:
            p.result()
    finally:
        writer.shutdown()


def kitti_data_prep(root_path, imageset_dir=None, save_path=None, relative_path=True, used_classes=None, batch_frames=16, workers=8,
                    gt_aug_with_context=-1.0, with_back=False):
    """KITTI infos (train / val / trainval / test), reduced point clouds and the train GT database (gt_database/ + dbinfos_train.pkl),
    reading each raw sweep once.  Returns the four info lists."""
    if gt_aug_with_context > 0:
        raise NotImplementedError("the enlarged GT database (gt_aug_with_context > 0) is not supported")
    if with_back:
        raise NotImplementedError("the mirrored (with_back) reduced point clouds are not supported")
    root = Path(root_path)
    imageset_dir = Path(imageset_dir) if imageset_dir is not None else root / "ImageSets"
    ids = {s: imageset_ids(imageset_dir, s) for s in ("train", "val", "test")}
    save = Path(save_path) if save_path is not None else root

    def infos_of(split):
        training = split != "test"
        return [image_info(root, i, training=training, label_info=training, velodyne=True, calib=True, relative_path=relative_path)
                for i in ids[split]]
    train, val, test = infos_of("train"), infos_of("val"), infos_of("test")
    db = _DbWriter(root / "gt_database", used_classes, relative_path)
    prepare(root, train, relative_path, reduce=True, count=True, db=db, batch_frames=batch_frames, workers=workers)
    prepare(root, val, relative_path, reduce=True, count=True, batch_frames=batch_frames, workers=workers)
    prepare(root, test, relative_path, reduce=True, batch_frames=batch_frames, workers=workers)
    for name, obj in (("kitti_infos_train.pkl", train), ("kitti_infos_val.pkl", val), ("kitti_infos_trainval.pkl", train + val),
                      ("kitti_infos_test.pkl", test)):
        with open(save / name, "wb") as f:
            pickle.dump(obj, f)
    db.dump(root / "dbinfos_train.pkl")
    return {"train": train, "val": val, "trainval": train + val, "test": test}


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("root")
    ap.add_argument("--imageset-dir", default=None)
    ap.add_argument("--batch-frames", type=int, default=16)
    ap.add_argument("--workers", type=int, default=8)
    a = ap.parse_args(argv)
    kitti_data_prep(a.root, imageset_dir=a.imageset_dir, batch_frames=a.batch_frames, workers=a.workers)


if __name__ == "__main__":
    sys.exit(main())
