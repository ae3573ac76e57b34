"""numpy restatement of GT-database sampling (GT-AUG) for SE-SSD's training frames, as the reference runs it.

Stages (det3d/core/sampler/sample_ops_v2.py, det3d/core/sampler/preprocess.py:20-110, det3d/datasets/pipelines/preprocess.py:83-110):
  filter_db        DBFilterByMinNumPoint (listed classes, min > 0) then DBFilterByDifficulty (every class), in config order
  Sampler          one index stream per class in the infos' dict order, each shuffled at construction from the same RandomState (plus
                   the Car + Van stream with gt_aug_similar_type); `take(num)` returns the remainder when idx + num >= N, then
                   reshuffles
  accept           sample_class_v2's loop: candidate i is rejected when it collides with a box, an accepted candidate or a later
                   undecided one; a rejected candidate blocks nothing (augment_ref.collide over fp64 BEV corners)
  sample_frame     sample_all: round(rate * (max_num - #names == group)), at most two rounds
  paste            [sampled points (fp32(rel + fp64 centre)), scene points outside every sampled box] and the concatenated boxes
  preprocess_frame GT-AUG chained into augment_ref.augment_frame: Preprocess.__call__ without SA-DA, one frame

Dtypes: box3d_lidar is float64 (see csrc/gtaug.cu), so the sampled boxes and their corners are fp64; a frame's own boxes keep their
dtype for their corners.  Corners follow center_to_corner_box2d operation for operation (corners_nd, the einsum rotation, then + centre).
Point removal is the box-frame membership test of augment_ref (points at least 1e-3 from every face in the fixtures).
"""
import numpy as np

from . import augment_ref


def filter_db(db_infos, min_points, removed_difficulties):
    out = {k: list(v) for k, v in db_infos.items()}
    for name, m in min_points.items():
        if m > 0:
            out[name] = [i for i in out[name] if i["num_points_in_gt"] >= m]
    return {k: [i for i in v if i["difficulty"] not in removed_difficulties] for k, v in out.items()}


class Sampler:
    def __init__(self, n, rs):
        self.rs, self.idx = rs, 0
        self.ind = np.arange(n)
        rs.shuffle(self.ind)

    def take(self, num):
        if self.idx + num >= len(self.ind):
            ret = self.ind[self.idx:].copy()
            self.rs.shuffle(self.ind)
            self.idx = 0
        else:
            ret = self.ind[self.idx:self.idx + num].copy()
            self.idx += num
        return ret


def corners(boxes, add_zero_offset=False):
    """BEV corners of center_to_corner_box2d in the boxes' dtype (the sampled boxes get `dims + [0.0, 0.0]`: fp64)"""
    dims = boxes[:, 3:5] + [0.0, 0.0] if add_zero_offset else boxes[:, 3:5]
    norm = np.array([[-0.5, -0.5], [-0.5, 0.5], [0.5, 0.5], [0.5, -0.5]], dtype=dims.dtype)
    c = dims.reshape(-1, 1, 2) * norm.reshape(1, 4, 2)
    s, co = np.sin(boxes[:, -1]), np.cos(boxes[:, -1])
    x = c[..., 0] * co[:, None] + c[..., 1] * s[:, None]
    y = c[..., 0] * -s[:, None] + c[..., 1] * co[:, None]
    out = np.stack([x, y], -1)
    out += boxes[:, 0:2].reshape(-1, 1, 2)
    return out


def accept(box_corners, cand_corners):
    """[K] bool: sample_class_v2's acceptance"""
    allc = np.concatenate([box_corners, cand_corners]).astype(np.float64)
    nb, k = len(box_corners), len(cand_corners)
    alive = np.ones(k, bool)
    for c in range(k):
        i = nb + c
        hit = any(augment_ref.collide(allc[i], allc[j]) for j in range(nb + k) if j != i and (j < nb or alive[j - nb]))
        alive[c] = not hit
    return alive


class GtAug:
    """the sampler state of DataBaseSamplerV2 for the groups [(name, max_num)]; infos: the filtered dict; similar: gt_aug_similar_type"""

    def __init__(self, infos, groups, rs, rate=1.0, similar=False):
        self.groups, self.rate = groups, rate
        self.infos = [i for v in infos.values() for i in v]
        gid = {id(i): n for n, i in enumerate(self.infos)}
        self.streams = {}
        for k, v in infos.items():
            self.streams[k] = (np.array([gid[id(i)] for i in v], np.int64), Sampler(len(v), rs))
        if similar:
            v = infos["Car"] + infos["Van"]
            self.streams["Car"] = (np.array([gid[id(i)] for i in v], np.int64), Sampler(len(v), rs))
        self.boxes = np.stack([np.asarray(i["box3d_lidar"]) for i in self.infos]) if self.infos else np.zeros((0, 7))

    def sample_frame(self, gt_boxes, gt_names):
        """accepted global ids of one frame, in acceptance order, and the per-round log [(asked, candidates, accepted mask)]"""
        out, log, all_gt = [], [], np.asarray(gt_boxes)
        nums = [np.round(self.rate * int(m - np.sum([n == name for n in gt_names]))).astype(np.int64) for name, m in self.groups]
        for (name, _), num in zip(self.groups, nums):
            times = 0
            while num > 0 and times < 2:
                ids_map, s = self.streams[name]
                cand = ids_map[s.take(num)]
                acc = accept(corners(all_gt), corners(self.boxes[cand], add_zero_offset=True))
                log.append((int(num), cand, acc))
                out += list(cand[acc])
                if acc.any():
                    all_gt = np.concatenate([all_gt, self.boxes[cand[acc]]])
                num -= int(acc.sum())
                times += 1
        return np.array(out, np.int64), log


def point_masks64(points, boxes):
    """[N, M] bool: augment_ref.point_masks on boxes kept in fp64 (points_in_rbbox of the sampled box3d_lidar)"""
    p = np.asarray(points, np.float32)[:, :3].astype(np.float64)
    b = np.asarray(boxes, np.float64)
    if b.shape[0] == 0 or p.shape[0] == 0:
        return np.zeros((p.shape[0], b.shape[0]), bool)
    c = np.cos(b[:, 6]); s = np.sin(b[:, 6])
    dx = p[:, None, 0] - b[None, :, 0]; dy = p[:, None, 1] - b[None, :, 1]; dz = p[:, None, 2] - b[None, :, 2]
    lx = dx * c - dy * s
    ly = dx * s + dy * c
    return (np.abs(lx) < b[:, 3] * 0.5) & (np.abs(ly) < b[:, 4] * 0.5) & (np.abs(dz) < b[:, 5] * 0.5)


def object_points(rel, centre):
    """s_points[:, :3] += box3d_lidar[:3]: fp32(double(rel) + centre)"""
    p = np.array(rel, np.float32, copy=True)
    p[:, :3] = (p[:, :3].astype(np.float64) + np.asarray(centre, np.float64)[:3]).astype(np.float32)
    return p


def paste(points, gt_boxes, gt_names, ids, db_rel_points, db_boxes, db_names):
    """Preprocess.__call__:96-110 for one frame: returns (points, boxes, names, gt_masks of the sampled part)"""
    points = np.asarray(points, np.float32)
    if len(ids) == 0:
        return points, np.asarray(gt_boxes), np.asarray(gt_names), np.zeros(0, bool)
    sb = db_boxes[ids]
    sp = np.concatenate([object_points(db_rel_points[i], db_boxes[i]) for i in ids] + [np.zeros((0, points.shape[1]), np.float32)])
    inside = point_masks64(points, sb).any(1)
    return (np.concatenate([sp, points[~inside]]), np.concatenate([np.asarray(gt_boxes), sb]),
            np.concatenate([np.asarray(gt_names), db_names[ids]]), np.ones(len(ids), bool))


def preprocess_frame(points, gt_boxes, gt_names, ids, db_rel_points, db_boxes, db_names, class_names, draws, context=-1.0):
    """GT-AUG then augment_ref.augment_frame (the boxes as fp32, as the device stages take them): Preprocess without SA-DA"""
    pts, bx, names, _ = paste(points, gt_boxes, gt_names, ids, db_rel_points, db_boxes, db_names)
    valid = np.array([n in class_names for n in names], bool)
    return dict(points_pasted=pts, boxes_pasted=bx, names_pasted=names,
                **augment_ref.augment_frame(pts, np.asarray(bx, np.float32), valid, draws, context))
