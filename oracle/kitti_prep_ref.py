"""numpy restatement of the KITTI data preparation's geometry (kitti_common.py _calculate_num_points_in_gt / _create_reduced_point_cloud,
create_gt_database.py), for the CPU tests and the benchmark's CPU column.

Planes follow surface_equ_3d_jitv2 (geometry.py:351-377) operation for operation in fp64; membership is _points_in_convex_polygon_3d_jit
(geometry.py:241-276): inside when (((x*a) + (y*b)) + (z*c)) + d < 0 for every plane, fp32 coordinates widened to fp64.  numpy rounds
each elementwise operation on its own, so the result is bit-exact with the numba loops.  Box corners use math.sin / math.cos.
"""
import math

import numpy as np

FACES = np.array([0, 1, 2, 3, 7, 6, 5, 4, 0, 3, 7, 4, 1, 5, 6, 2, 0, 4, 5, 1, 3, 2, 6, 7]).reshape(6, 4)
UNIT = np.array([[0, 0, 0], [0, 0, 1], [0, 1, 1], [0, 1, 0], [1, 0, 0], [1, 0, 1], [1, 1, 1], [1, 1, 0]], np.float64)


def planes(surfaces):
    """[N, S, >=3, 3] -> [N, S, 4] (a, b, c, d)"""
    s = np.asarray(surfaces, np.float64)
    out = np.zeros(s.shape[:2] + (4,))
    for i in range(s.shape[0]):
        for j in range(s.shape[1]):
            p0, p1, p2 = s[i, j, 0], s[i, j, 1], s[i, j, 2]
            v0, v1 = p0 - p1, p1 - p2
            a = v0[1] * v1[2] - v0[2] * v1[1]
            b = v0[2] * v1[0] - v0[0] * v1[2]
            c = v0[0] * v1[1] - v0[1] * v1[0]
            out[i, j] = (a, b, c, ((-p0[0]) * a - p0[1] * b) - p0[2] * c)
    return out


def inside(points, pl):
    """[N, K] bool: points [N, >=3] (fp32) inside each polyhedron of pl [K, 6, 4]"""
    p = np.asarray(points)[:, :3].astype(np.float64)
    pl = np.asarray(pl, np.float64)
    x, y, z = p[:, 0:1], p[:, 1:2], p[:, 2:3]
    ok = np.ones((len(p), len(pl)), bool)
    for k in range(6):
        s = ((x * pl[None, :, k, 0] + y * pl[None, :, k, 1]) + z * pl[None, :, k, 2]) + pl[None, :, k, 3]
        ok &= ~(s >= 0)
    return ok


def corners(boxes, origin=0.5):
    boxes = np.asarray(boxes, np.float64).reshape(-1, 7)
    c = boxes[:, None, 3:6] * (UNIT - origin)[None]
    sn = np.array([math.sin(a) for a in boxes[:, 6]])[:, None]
    cs = np.array([math.cos(a) for a in boxes[:, 6]])[:, None]
    x, y = c[..., 0], c[..., 1]
    return np.stack([x * cs + y * sn, -(x * sn) + y * cs, c[..., 2]], -1) + boxes[:, None, :3]


def box_planes(boxes):
    boxes = np.asarray(boxes, np.float64).reshape(-1, 7)
    if len(boxes) == 0:
        return np.zeros((0, 6, 4))
    return planes(corners(boxes)[:, FACES])


def frustum_planes(rect, Trv2c, P2, image_shape):
    """the image frustum's six planes [6, 4] (remove_outside_points: get_frustum of the image box, camera -> velodyne)"""
    cr, ct = P2[0:3, 0:3], P2[0:3, 3]
    rinv, cinv = np.linalg.qr(np.linalg.inv(cr))
    C, R, T = np.linalg.inv(cinv), np.linalg.inv(rinv), cinv @ ct
    fku, fkv = C[0, 0], -C[1, 1]
    u0v0 = C[0:2, 2]
    near_clip, far_clip = 0.001, 100
    z = np.array([near_clip] * 4 + [far_clip] * 4, dtype=C.dtype)[:, np.newaxis]
    b = [0, 0, image_shape[1], image_shape[0]]
    box_corners = np.array([[b[0], b[1]], [b[0], b[3]], [b[2], b[3]], [b[2], b[1]]], dtype=C.dtype)
    near = (box_corners - u0v0) / np.array([fku / near_clip, -fkv / near_clip], dtype=C.dtype)
    far = (box_corners - u0v0) / np.array([fku / far_clip, -fkv / far_clip], dtype=C.dtype)
    fr = np.concatenate([np.concatenate([near, far], axis=0), z], axis=1)
    fr -= T
    fr = (np.linalg.inv(R) @ fr.T).T
    fr = np.concatenate([fr, np.ones([8, 1])], axis=-1)
    fr = (fr @ np.linalg.inv((rect @ Trv2c).T))[..., :3]
    return planes(fr[None][:, FACES])[0]


def reduce_frame(points, rect, Trv2c, P2, image_shape):
    return points[inside(points, frustum_planes(rect, Trv2c, P2, image_shape)[None])[:, 0]]


def count_boxes(info):
    """_calculate_num_points_in_gt's boxes: the first num_obj rows, camera -> velodyne, no centre change"""
    a, cal = info["annos"], info["calib"]
    n = int(sum(1 for x in a["name"] if x != "DontCare"))
    cam = np.concatenate([a["location"][:n], a["dimensions"][:n], a["rotation_y"][:n, None]], axis=1)
    return _cam_to_lidar(cam, cal)


def _cam_to_lidar(cam, cal):
    xyz = np.concatenate([cam[:, 0:3], np.ones([len(cam), 1])], axis=-1)
    xyz = (xyz @ np.linalg.inv((cal["R0_rect"] @ cal["Tr_velo_to_cam"]).T))[..., :3]
    return np.concatenate([xyz, cam[:, 5:6], cam[:, 3:4], cam[:, 4:5], cam[:, 6:7]], axis=1)


def db_boxes(info):
    """LoadPointCloudAnnotations' boxes: DontCare removed, fp32 cast, camera -> velodyne in fp64, moved to the box centre"""
    a, cal = info["annos"], info["calib"]
    keep = [i for i, x in enumerate(a["name"]) if x != "DontCare"]
    cam = np.concatenate([a["location"][keep], a["dimensions"][keep], a["rotation_y"][keep][:, None]], axis=1).astype(np.float32)
    b = _cam_to_lidar(cam, cal)
    b[:, :3] += b[:, 3:6] * (np.array([0.5, 0.5, 0.5]) - np.array([0.5, 0.5, 0.0]))
    return b, a["name"][keep], a["difficulty"][keep]


def num_points_in_gt(reduced, info):
    m = inside(reduced, box_planes(count_boxes(info)))
    n_ign = len(info["annos"]["dimensions"]) - m.shape[1]
    return np.concatenate([m.sum(0), -np.ones([n_ign])]).astype(np.int32)


def db_objects(reduced, info):
    """per object (DontCare removed): (name, relative rows fp32, count, box fp64, difficulty)"""
    boxes, names, diff = db_boxes(info)
    m = inside(reduced, box_planes(boxes))
    out = []
    for i in range(len(boxes)):
        rows = reduced[m[:, i]].copy()
        rows[:, :3] -= boxes[i, :3]
        out.append((names[i], rows, int(m[:, i].sum()), boxes[i], diff[i]))
    return out
