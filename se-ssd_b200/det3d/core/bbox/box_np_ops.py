"""numpy box math used on the hot path and by the anchor target assigner (subset of det3d/core/bbox/box_np_ops.py; the
camera / frustum / legacy helpers of the reference are out of scope).  Host-side, one-off or per-GT work."""
import numpy as np


def second_box_encode(boxes, anchors, encode_angle_to_vector=False, smooth_dim=False, cylindrical=False, norm_velo=False):
    """Residual encoding of (x,y,z,w,l,h,r) boxes against anchors (reference :52-113, 7-dim, log sizes)."""
    if anchors.shape[-1] != 7 or encode_angle_to_vector or smooth_dim:
        raise NotImplementedError("only the 7-dim log-size encoding of the SE-SSD config is supported")
    xa, ya, za, wa, la, ha, ra = np.split(anchors, 7, axis=1)
    xg, yg, zg, wg, lg, hg, rg = np.split(boxes, 7, axis=1)
    diag = np.sqrt(la ** 2 + wa ** 2)
    return np.concatenate([(xg - xa) / diag, (yg - ya) / diag, (zg - za) / ha, np.log(wg / wa), np.log(lg / la),
                           np.log(hg / ha), rg - ra], axis=1)


def second_box_decode(box_encodings, anchors, encode_angle_to_vector=False, smooth_dim=False, norm_velo=False):
    if anchors.shape[-1] != 7 or encode_angle_to_vector or smooth_dim:
        raise NotImplementedError("only the 7-dim log-size encoding of the SE-SSD config is supported")
    xa, ya, za, wa, la, ha, ra = np.split(anchors, 7, axis=-1)
    xt, yt, zt, wt, lt, ht, rt = np.split(box_encodings, 7, axis=-1)
    diag = np.sqrt(la ** 2 + wa ** 2)
    return np.concatenate([xt * diag + xa, yt * diag + ya, zt * ha + za, np.exp(wt) * wa, np.exp(lt) * la, np.exp(ht) * ha,
                           rt + ra], axis=-1)


def limit_period(val, offset=0.5, period=2 * np.pi):
    return val - np.floor(val / period + offset) * period


def center_to_minmax_2d(centers, dims, origin=0.5):
    if origin != 0.5:
        raise NotImplementedError
    return np.concatenate([centers - dims / 2, centers + dims / 2], axis=-1)


def rbbox2d_to_near_bbox(rbboxes):
    """Rotated (x,y,w,l,r) -> nearest axis-aligned box; w/l swapped when |r mod pi| > pi/4 (reference :354-366)."""
    rot = np.abs(limit_period(rbboxes[..., -1], 0.5, np.pi))
    swap = (rot > np.pi / 4)[..., np.newaxis]
    c = np.where(swap, rbboxes[:, [0, 1, 3, 2]], rbboxes[:, :4])
    return center_to_minmax_2d(c[:, :2], c[:, 2:])


def iou_jit(boxes, query_boxes, eps=1.0):
    """Axis-aligned IoU matrix [N,K] (reference :1007-1046), vectorised; zero where the boxes do not overlap.
    Rounding follows the reference under numba: differences in the input dtype, then `+ eps` (a Python float = float64)
    promotes the remaining arithmetic to fp64 and the quotient is rounded once into the output dtype."""
    b = boxes[:, None, :]
    q = query_boxes[None, :, :]
    f8 = np.float64
    area_q = ((q[..., 2] - q[..., 0]).astype(f8) + eps) * ((q[..., 3] - q[..., 1]).astype(f8) + eps)
    iw = (np.minimum(b[..., 2], q[..., 2]) - np.maximum(b[..., 0], q[..., 0])).astype(f8) + eps
    ih = (np.minimum(b[..., 3], q[..., 3]) - np.maximum(b[..., 1], q[..., 1])).astype(f8) + eps
    ua = ((b[..., 2] - b[..., 0]).astype(f8) + eps) * ((b[..., 3] - b[..., 1]).astype(f8) + eps) + area_q - iw * ih
    with np.errstate(divide="ignore", invalid="ignore"):
        ov = iw * ih / ua
    return np.where((iw > 0) & (ih > 0), ov, 0).astype(boxes.dtype)


def center_to_corner_box2d(centers, dims, angles=None, origin=0.5):
    """[N,4,2] corners, clockwise from the minimum corner, rotated clockwise for positive angles (reference :512-532)."""
    norm = np.array([[0, 0], [0, 1], [1, 1], [1, 0]], dtype=dims.dtype) - np.array(origin, dtype=dims.dtype)
    corners = dims.reshape(-1, 1, 2) * norm.reshape(1, 4, 2)
    if angles is not None:
        s, c = np.sin(angles), np.cos(angles)
        x, y = corners[..., 0].copy(), corners[..., 1].copy()
        corners = np.stack([x * c[:, None] + y * s[:, None], -x * s[:, None] + y * c[:, None]], axis=-1)
    return corners + centers.reshape(-1, 1, 2)


def corner_to_standup_nd(boxes_corner):
    return np.concatenate([boxes_corner.min(axis=1), boxes_corner.max(axis=1)], axis=-1)


def create_anchors_3d_range(feature_size, anchor_range, sizes=(1.6, 3.9, 1.56), rotations=(0, np.pi / 2), velocities=None,
                            dtype=np.float32):
    """Anchor grid [D, H, W, num_sizes, num_rots, 7] (reference :780-833); centres at cell centres of the range."""
    if velocities is not None:
        raise NotImplementedError("velocity anchors are not part of the SE-SSD KITTI config")
    from sessd_b200.weights import kitti_car_anchors
    flat = kitti_car_anchors(tuple(feature_size), tuple(anchor_range), tuple(np.ravel(sizes)), tuple(rotations), dtype)
    ns = int(np.array(sizes).reshape(-1, 3).shape[0])
    return flat.reshape(feature_size[0], feature_size[1], feature_size[2], ns, len(rotations), 7)


# ------------------------------------------------------------------------------------------------ KITTI wire format (SURVEY 8(f) row 4)
def camera_to_lidar(points, r_rect, velo2cam):
    """Camera-rect coordinates -> velodyne coordinates (reference :937-942)."""
    shape = list(points.shape[:-1])
    if points.shape[-1] == 3:
        points = np.concatenate([points, np.ones(shape + [1])], axis=-1)
    return (points @ np.linalg.inv((r_rect @ velo2cam).T))[..., :3]


def lidar_to_camera(points, r_rect, velo2cam):
    shape = list(points.shape[:-1])
    if points.shape[-1] == 3:
        points = np.concatenate([points, np.ones(shape + [1])], axis=-1)
    return (points @ (r_rect @ velo2cam).T)[..., :3]


def box_camera_to_lidar(data, r_rect, velo2cam):
    """(x, y, z)cam, l, h, w, ry -> (x, y, z)velo, w, l, h, ry (reference :965-970)."""
    xyz_lidar = camera_to_lidar(data[:, 0:3], r_rect, velo2cam)
    l, h, w, r = data[:, 3:4], data[:, 4:5], data[:, 5:6], data[:, 6:7]
    return np.concatenate([xyz_lidar, w, l, h, r], axis=1)


def box_lidar_to_camera(data, r_rect, velo2cam):
    xyz = lidar_to_camera(data[:, 0:3], r_rect, velo2cam)
    w, l, h, r = data[:, 3:4], data[:, 4:5], data[:, 5:6], data[:, 6:7]
    return np.concatenate([xyz, l, h, w, r], axis=1)


def change_box3d_center_(box3d, src, dst):
    """In place: move the box origin from the relative position `src` to `dst` (reference :1406-1409)."""
    dst = np.array(dst, dtype=box3d.dtype)
    src = np.array(src, dtype=box3d.dtype)
    box3d[..., :3] += box3d[..., 3:6] * (dst - src)


def projection_matrix_to_CRT_kitti(proj):
    """P = C @ [R|T] with C upper triangular (reference :623-634)."""
    cr, ct = proj[0:3, 0:3], proj[0:3, 3]
    rinv, cinv = np.linalg.qr(np.linalg.inv(cr))
    return np.linalg.inv(cinv), np.linalg.inv(rinv), cinv @ ct


def get_frustum(bbox_image, C, near_clip=0.001, far_clip=100):
    """8 corners (camera coordinates) of the viewing frustum behind an image box (reference :637-654)."""
    fku, fkv = C[0, 0], -C[1, 1]
    u0v0 = C[0:2, 2]
    z = np.array([near_clip] * 4 + [far_clip] * 4, dtype=C.dtype)[:, np.newaxis]
    b = bbox_image
    corners = np.array([[b[0], b[1]], [b[0], b[3]], [b[2], b[3]], [b[2], b[1]]], dtype=C.dtype)
    near = (corners - u0v0) / np.array([fku / near_clip, -fkv / near_clip], dtype=C.dtype)
    far = (corners - u0v0) / np.array([fku / far_clip, -fkv / far_clip], dtype=C.dtype)
    return np.concatenate([np.concatenate([near, far], axis=0), z], axis=1)


def corner_to_surfaces_3d(corners):
    """[N, 8, 3] box corners -> [N, 6, 4, 3] surfaces with inward normals (reference :1193-1212)."""
    idx = np.array([0, 1, 2, 3, 7, 6, 5, 4, 0, 3, 7, 4, 1, 5, 6, 2, 0, 4, 5, 1, 3, 2, 6, 7]).reshape(6, 4)
    return corners[:, idx]


corner_to_surfaces_3d_jit = corner_to_surfaces_3d


def get_valid_frustum(rect, Trv2c, P2, image_shape):
    """Image frustum in velodyne coordinates as 6 surfaces [1, 6, 4, 3] (reference :995-1003): `calib["frustum"]` of the detector's
    post-processing filter (mg_head_sessd.py:1024-1030)."""
    C, R, T = projection_matrix_to_CRT_kitti(P2)
    frustum = get_frustum([0, 0, image_shape[1], image_shape[0]], C)
    frustum -= T
    frustum = np.linalg.inv(R) @ frustum.T
    frustum = camera_to_lidar(frustum.T, rect, Trv2c)
    return corner_to_surfaces_3d(frustum[np.newaxis, ...])


# ------------------------------------------------------------------------------------------------ KITTI data preparation: numpy in and out,
# membership on the device (sessd_b200.kitti_prep)
def center_to_corner_box3d(centers, dims, angles=None, origin=(0.5, 0.5, 0.5), axis=2):
    """[N, 8, 3] box corners (reference :467-509); rotation about z with correctly rounded sin / cos."""
    from sessd_b200 import kitti_prep
    return kitti_prep.center_to_corner_box3d(centers, dims, angles, origin, axis)


def remove_outside_points(points, rect, Trv2c, P2, image_shape):
    """The rows of points inside the image frustum, in order (reference :981-992)."""
    from sessd_b200 import kitti_prep
    return kitti_prep.remove_outside_points(points, rect, Trv2c, P2, image_shape)


def points_in_rbbox(points, rbbox, z_axis=2, origin=(0.5, 0.5, 0.5)):
    """[N, K] bool membership of points in rotated boxes (reference :1152-1157)."""
    from sessd_b200 import kitti_prep
    return kitti_prep.points_in_rbbox(points, rbbox, z_axis, origin)
