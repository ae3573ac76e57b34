"""SE-SSD training-frame augmentation on the device: per-object box noise with collision tests, global flip / rotation / scaling, the
point shuffle and the teacher's un-augmented twin (reference: det3d/datasets/pipelines/preprocess.py:68-175, Preprocess.__call__, and the
numba loops of det3d/core/sampler/preprocess.py it calls).

Every random number is drawn on the host by ``draw_augmentation`` with a numpy ``RandomState``, with the reference's calls in the
reference's order; the kernels of csrc/augment.cu are pure functions of the points, the boxes and those draws, so each stage is
comparable with the reference's own function run on the same seed.

GT-database sampling (GT-AUG, before the per-object noise) runs when ``build_train_batch`` is given a ``db_sampler``
(det3d.core.sampler, csrc/gtaug.cu): selection on the host, the paste on the device.  Shape-aware augmentation (SA-DA,
``pyramid_augment_v0``, between the global scaling and the shuffle) runs when it is given ``sa_da`` (sessd_b200.sada, csrc/sada.cu).  No
``Preprocess`` pipeline is registered; ``build_train_batch`` (the collated batch) and ``augment_batch`` (the augmented points and boxes)
are their own entry points.
"""
from dataclasses import dataclass, field

import numpy as np
import torch

from . import ops

NUM_TRY = 100                                   # noise_per_object_v4_(num_try=100), pipelines/preprocess.py:118
MAX_GT = 256                                    # SESSD_AUGMENT_MAX_GT (include/sessd_b200.h)


@dataclass
class AugmentConfig:
    """the train_preprocessor values the augmentation reads (examples/second/configs/config.py train_preprocessor)"""
    gt_loc_noise: tuple = (1.0, 1.0, 0.5)
    gt_rot_noise: tuple = (-0.785, 0.785)
    global_rot_noise: tuple = (-0.785, 0.785)
    global_scale_noise: tuple = (0.95, 1.05)
    data_aug_with_context: float = -1.0
    class_names: tuple = ("Car", "Van")
    shuffle_points: bool = True
    target_class_ids: tuple = (1, 2)            # AssignTarget: [1, 2] with enable_similar_type, else [1]
    range_bev: tuple = (0.0, -40.0, 70.4, 40.0)  # filter_gt_box_outside_range over pc_range[[0, 1, 3, 4]] (Voxelization)

    @classmethod
    def from_config(cls, cfg):
        """from a loaded det3d Config: cfg.train_preprocessor, cfg.voxel_generator.range, cfg.train_cfg.assigner"""
        tp = cfg.train_preprocessor
        names = list(tp.class_names)                # the reference appends 'Van' to the config's own list; this copies it
        similar = bool(tp.get("enable_similar_type", False))
        if similar and "Car" in names:
            names.append("Van")
        rg = [float(v) for v in cfg.voxel_generator.range]
        similar_assign = bool(cfg.train_cfg.assigner.get("enable_similar_type", False))
        ctx = tp.get("data_aug_with_context", -1)
        return cls(gt_loc_noise=tuple(float(v) for v in tp.gt_loc_noise), gt_rot_noise=tuple(float(v) for v in tp.gt_rot_noise),
                   global_rot_noise=_pair(tp.global_rot_noise), global_scale_noise=tuple(float(v) for v in tp.global_scale_noise),
                   data_aug_with_context=float(ctx), class_names=tuple(names), shuffle_points=bool(tp.get("shuffle_points", False)),
                   target_class_ids=(1, 2) if similar_assign else (1,), range_bev=(rg[0], rg[1], rg[3], rg[4]))


def _pair(r):
    """global_rotation_v3: a scalar r means [-r, r]"""
    if isinstance(r, (list, tuple)):
        return float(r[0]), float(r[1])
    return -float(r), float(r)


@dataclass
class FrameDraws:
    loc: np.ndarray          # [M, NUM_TRY, 3] fp64
    rot: np.ndarray          # [M, NUM_TRY] fp64
    flip: bool
    rotation: float
    scale: float
    perm: np.ndarray         # [N] int64


@dataclass
class Draws:
    frames: list = field(default_factory=list)

    def transformation(self):
        """the per-frame ``transformation`` dicts of Preprocess (pipelines/preprocess.py:140) that consistency_loss undoes"""
        return [dict(flipped=f.flip, noise_rotation=f.rotation, noise_scale=f.scale) for f in self.frames]


def draw_augmentation(rs, frames, cfg):
    """Draw every random number of the augmentation on the host, per frame, with the reference's calls in the reference's order.

    frames: per frame (num_points, num_boxes, labeled).  Labelled frames: ``normal(scale=gt_loc_noise, size=[M, 100, 3])`` and
    ``uniform(*gt_rot_noise, size=[M, 100])`` (noise_per_object_v4_), ``choice([False, True], replace=False, p=[0.5, 0.5])``
    (random_flip_v2), ``uniform`` for the global rotation and for the scale, then ``choice(arange(n), n, replace=False)`` (the shuffle,
    when shuffle_points).  Unlabelled frames: the shuffle first, then flip, rotation and scale.

    GT-AUG's draws (before the noise) come from the sampler (gtaug_batch interleaves them per frame).  SA-DA's draws (between the
    scaling and the shuffle) depend on the frame's device results, so they are not made here: this is the reference's Preprocess
    stream without SA-DA; launch_train_batch(sa_da=SadaConfig()) interleaves them frame by frame (sessd_b200.sada)."""
    out = Draws()
    for n, m, labeled in frames:
        n, m = int(n), int(m)
        if labeled:
            loc, rot, flip, rotation, scale = _labeled_draws(rs, m, cfg)
            perm = _shuffle(rs, n, cfg)
        else:
            loc, rot = np.zeros((0, NUM_TRY, 3)), np.zeros((0, NUM_TRY))
            perm = _shuffle(rs, n, cfg)
            flip, rotation, scale = _global_draws(rs, cfg)
        out.frames.append(FrameDraws(loc, rot, flip, rotation, scale, perm))
    return out


def _labeled_draws(rs, m, cfg):
    """a labelled frame's draws before SA-DA and the shuffle: the per-object noise, then flip, rotation and scale"""
    loc_std = np.array(cfg.gt_loc_noise, dtype=np.float32)          # noise_per_object_v4_: np.array(center_noise_std, gt_boxes.dtype)
    loc = rs.normal(scale=loc_std, size=[m, NUM_TRY, 3])
    rot = rs.uniform(cfg.gt_rot_noise[0], cfg.gt_rot_noise[1], size=[m, NUM_TRY])
    return (loc, rot) + _global_draws(rs, cfg)


def _global_draws(rs, cfg):
    flip = bool(rs.choice([False, True], replace=False, p=[0.5, 0.5]))
    rotation = float(rs.uniform(cfg.global_rot_noise[0], cfg.global_rot_noise[1]))
    scale = float(rs.uniform(cfg.global_scale_noise[0], cfg.global_scale_noise[1]))
    return flip, rotation, scale


def _shuffle(rs, n, cfg):
    if not cfg.shuffle_points:
        return np.arange(n)
    return rs.choice(np.arange(n), n, replace=False)


def global_row(d):
    """fp32 (cos, sin, scale, flip, angle) as rotation_points_single_angle / global_scaling_v3 / random_flip_v2 round them"""
    return np.array([np.float32(np.cos(d.rotation)), np.float32(np.sin(d.rotation)), np.float32(d.scale), 1.0 if d.flip else 0.0,
                     np.float32(d.rotation)], np.float32)


def _pack(arrays):
    """one host buffer for all inputs (one host-to-device copy per batch); returns (bytes, [(offset, dtype, shape)])"""
    layout, off = [], 0
    for a in arrays:
        layout.append((off, a.dtype, a.shape))
        off += -(-a.nbytes // 16) * 16
    buf = np.zeros(max(off, 16), np.uint8)
    for (o, _, _), a in zip(layout, arrays):
        buf[o:o + a.nbytes] = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    return buf, layout


def _unpack(dev, layout):
    out = []
    for o, dt, shape in layout:
        n = int(np.prod(shape)) * np.dtype(dt).itemsize
        out.append(dev[o:o + n].view(getattr(torch, np.dtype(dt).name)).view(*shape) if n else
                   torch.empty(shape, dtype=getattr(torch, np.dtype(dt).name), device=dev.device))
    return out


def _host_inputs(cfg, frame_sizes, gt_boxes, gt_names, draws, labeled):
    """the host arrays of the augmentation: (None, frame_off), (boxes, num_gt, valid, target, loc, rot, glob, perm, labeled), sizes"""
    B = len(frame_sizes)
    labeled = [True] * B if labeled is None else [bool(v) for v in labeled]
    ms = [len(b) if lab else 0 for b, lab in zip(gt_boxes, labeled)]
    max_gt = max([1] + ms)
    if max_gt > MAX_GT:
        raise ValueError("a frame has %d GT boxes > %d" % (max_gt, MAX_GT))
    ns = [int(n) for n in frame_sizes]
    off = np.zeros(B + 1, np.int32)
    off[1:] = np.cumsum(ns)
    boxes = np.zeros((B, max_gt, 7), np.float32)
    valid = np.zeros((B, max_gt), np.uint8)
    target = np.zeros((B, max_gt), np.uint8)
    loc = np.zeros((B, max_gt, NUM_TRY, 3))
    rot = np.zeros((B, max_gt, NUM_TRY))
    glob = np.zeros((B, 5), np.float32)
    perm = np.zeros(int(off[-1]), np.int32)
    for b in range(B):
        d = draws.frames[b]
        if len(d.perm) != ns[b] or d.loc.shape[0] != ms[b]:
            raise ValueError("frame %d: the draws were made for another frame size" % b)
        if ns[b] and not (np.bincount(np.asarray(d.perm), minlength=ns[b])[:ns[b]] == 1).all():
            raise ValueError("frame %d: perm is not a permutation of the frame's points" % b)
        m = ms[b]
        if m:
            boxes[b, :m] = np.asarray(gt_boxes[b], np.float32)
            names = list(gt_names[b])
            valid[b, :m] = [n in cfg.class_names for n in names]
            target[b, :m] = [n in cfg.class_names and cfg.class_names.index(n) + 1 in cfg.target_class_ids for n in names]
            loc[b, :m], rot[b, :m] = d.loc, d.rot
        glob[b] = global_row(d)
        perm[off[b]:off[b + 1]] = d.perm
    num_gt = np.array(ms, np.int32)
    lab = np.array(labeled, np.uint8)
    return (None, off), (boxes, num_gt, valid, target, loc, rot, glob, perm, lab), ns


def augment_batch(cfg, clouds, gt_boxes, gt_names, draws, labeled=None, device="cuda", twin=True):
    """Augment a batch of frames on the device.  clouds: per frame [N, 4] f32; gt_boxes: per frame [M, 7] (x y z w l h r); gt_names: per
    frame [M] class names (DontCare / ignore already dropped, as Preprocess does first); draws: draw_augmentation's output for
    (len(cloud), len(boxes), labeled) of every frame; labeled: per frame, None = all labelled.

    Returns a dict of device tensors: ``points`` (the student's [P, 4]: noised, flipped, rotated, scaled, shuffled), ``points_raw``
    (the teacher's twin: noised, unshuffled; an unlabelled frame's rows are its input), ``frame_off`` [B+1], ``gt_boxes`` / ``num_gt`` (the student's boxes after the range
    filter) and ``gt_boxes_raw`` / ``num_gt_raw`` (the teacher's), both padded [B, max_gt, 7] with limit_period angles -- the layout
    sessd_assign_targets reads --, ``selected`` [B, max_gt] (the try each box took, -1 none); and ``transformation`` (host list of dicts).
    twin=False (labelled frames): no teacher copy of the points is written and ``points_raw`` is None.
    Launches on the current stream and never waits on the device."""
    (_, off), rest, ns = _host_inputs(cfg, [len(c) for c in clouds], gt_boxes, gt_names, draws, labeled)
    pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, 4) for c in clouds] + [np.zeros((0, 4), np.float32)])
    buf, layout = _pack([pts, off] + list(rest))
    dev = torch.from_numpy(buf).pin_memory().to(device, non_blocking=True)
    d = _unpack(dev, layout)
    return _augment_device(cfg, d[0], d[1], ns, d[2:], draws, labeled, twin=twin)


def augment_resident(cfg, d_points, d_frame_off, frame_sizes, gt_boxes, gt_names, draws, device="cuda", student_boxes=False, twin=True):
    """augment_batch on points already on the device (labelled frames): d_points [P, 4] f32 (16-byte aligned rows) with d_frame_off
    [B+1] i32, frame_sizes the host's copy of the frame sizes.  Only the boxes and the draws are uploaded (one copy).  student_boxes:
    also return ``sada_boxes`` [B, max_gt, 7], each frame's class-valid boxes after the global stages (sessd_augment_boxes).
    twin=False: no teacher copy of the points is written (``points_raw`` is None)."""
    _, rest, ns = _host_inputs(cfg, frame_sizes, gt_boxes, gt_names, draws, None)
    buf, layout = _pack(list(rest))
    dev = torch.from_numpy(buf).pin_memory().to(device, non_blocking=True)
    return _augment_device(cfg, d_points, d_frame_off, ns, _unpack(dev, layout), draws, None, student_boxes, twin)


def _augment_device(cfg, d_pts, d_off, ns, rest, draws, labeled, student_boxes=False, twin=True):
    d_boxes, d_num, d_valid, d_target, d_loc, d_rot, d_glob, d_perm, d_lab = rest
    B = len(ns)
    labeled = [True] * B if labeled is None else [bool(v) for v in labeled]
    ctx = cfg.data_aug_with_context
    sel = ops.noise_per_box(d_boxes, d_num, d_valid, d_loc, d_rot, ctx)
    # an unlabelled frame has no twin in the reference: its rows keep the input
    raw = None if not twin or all(labeled) else d_pts.clone()
    raw, out = ops.augment_points(d_pts, d_off, max(ns + [0]), d_boxes, d_num, d_valid, d_loc, d_rot, sel, d_glob, d_perm, d_lab, ctx,
                                  points_raw=raw, with_raw=twin)
    boxes = ops.augment_boxes(d_boxes, d_num, d_valid, d_target, d_loc, d_rot, sel, d_glob, cfg.range_bev, global_boxes=student_boxes)
    boxes_raw, num_raw, boxes_out, num_out = boxes[:4]
    res = dict(points=out, points_raw=raw, frame_off=d_off, gt_boxes=boxes_out, num_gt=num_out, gt_boxes_raw=boxes_raw,
               num_gt_raw=num_raw, selected=sel, transformation=draws.transformation())
    if student_boxes:                                       # the boxes SA-DA takes (sessd_b200.sada)
        res["sada_boxes"] = boxes[4]
    return res


# ------------------------------------------------------------------------------------------------ collated training batch
_STATIC = {}


def _device_anchors(a, device):
    return torch.from_numpy(np.ascontiguousarray(a.reshape(-1, 7), np.float32)).pin_memory().to(device, non_blocking=True)


def _static_eval(cfg, device):
    """per-config constants of an evaluation batch: the voxeliser config and grid, the assigner and every task's anchors on the device
    (AssignTarget's, in task order; any number of one-class tasks).  Built once per config object and device."""
    key = ("eval", id(cfg), str(device))
    if key not in _STATIC:
        from det3d.datasets.pipelines import AssignTarget, Voxelization
        vg = cfg.voxel_generator
        vox = Voxelization(cfg=vg).voxel_generator
        at = AssignTarget(cfg=cfg.train_cfg.assigner)
        if any(len(d) != 1 for d in at.anchor_dicts_by_task):
            raise NotImplementedError("evaluation batches take one class per task")
        anchors = [_device_anchors(d[at.target_class_names[t]]["anchors"], device) for t, d in enumerate(at.anchor_dicts_by_task)]
        _STATIC[key] = dict(cfg=cfg, vcfg=ops.make_voxel_cfg(vg.voxel_size, vg.range, vg.max_points_in_voxel, vg.max_voxel_num),
                            grid=np.asarray(vox.grid_size), assigner=at, task_anchors=anchors)
    return _STATIC[key]


def _static(cfg, device):
    """per-config constants of the training batch builder: _static_eval's, the augmentation values, the one task's anchors and the
    assigner's thresholds (built once per config object and device).  Training is single-task, single-class."""
    key = (id(cfg), str(device))
    if key not in _STATIC:
        tasks = cfg.train_cfg.assigner.target_assigner.tasks
        if len(tasks) != 1 or int(tasks[0]["num_class"]) != 1:
            raise NotImplementedError("build_train_batch supports the single-class SE-SSD KITTI config (training is single-task)")
        ev = _static_eval(cfg, device)
        gen = ev["assigner"].target_assigners[0]._anchor_generators[0]
        _STATIC[key] = dict(ev, aug=AugmentConfig.from_config(cfg), anchors=ev["task_anchors"][0],
                            thr=(float(gen.match_threshold), float(gen.unmatch_threshold)))
    return _STATIC[key]


def voxel_example(st, vb, batch, total, sfx=""):
    """the model-input keys of one voxelised branch (``sfx`` "" or "_raw"): the exact-count voxels / num_points / coordinates (the first
    ``total`` rows of the VoxelBuffers ``vb``, read back by the caller), num_voxels, shape and the per-task anchors"""
    return {"voxels" + sfx: vb.voxels[:total], "num_points" + sfx: vb.num_points[:total], "coordinates" + sfx: vb.coors[:total],
            "num_voxels" + sfx: vb.num_voxels[:batch].long(), "shape" + sfx: np.stack([st["grid"]] * batch),
            "anchors" + sfx: [a.unsqueeze(0).expand(batch, -1, -1).contiguous() for a in st["task_anchors"]]}


class PendingBatch:
    """A training batch whose device work has been launched (augmentation, both voxelisations, both target assignments; the student's
    only when ``vox_raw`` is None) and whose collated dict is not formed yet.  ``example()`` forms it: the one device-to-host read of the
    batch (the branches' voxel totals, which size the exact-count voxel tensors the model reads)."""

    def __init__(self, st, aug, vox, vox_raw, asg, asg_raw, batch, frame_off, num_points_total):
        self._st, self._aug, self._vox, self._vox_raw, self._asg, self._asg_raw = st, aug, vox, vox_raw, asg, asg_raw
        self._batch, self._off, self._total = batch, frame_off, num_points_total

    def example(self):
        B = self._batch
        branches = [("", self._vox, self._asg)] + ([("_raw", self._vox_raw, self._asg_raw)] if self._vox_raw is not None else [])
        totals = torch.stack([vb.num_voxels[B] for _, vb, _ in branches]).cpu().tolist()                 # the one read-back
        dev = self._off.device
        counts = self._off[1:] - self._off[:-1]
        bidx = torch.repeat_interleave(torch.arange(B, dtype=torch.float32, device=dev), counts, output_size=self._total)
        ex = dict(metadata=[dict(token=i) for i in range(B)], points=torch.cat([bidx[:, None], self._aug["points"]], 1))
        for (sfx, vb, ab), n in zip(branches, totals):
            ex.update(voxel_example(self._st, vb, B, n, sfx))
            ex["labels" + sfx] = [ab.labels]
            ex["reg_targets" + sfx] = [ab.bbox_targets]
        ex["transformation"] = self._aug["transformation"]
        return ex


def gtaug_batch(cfg, clouds, gt_boxes, gt_names, rs, db_sampler, device="cuda", frame_hook=None):
    """GT-database sampling of a batch of labelled frames, then the augmentation draws, in the reference's stream order: per frame,
    the sampler's draws (its shuffles when a class stream runs out) come before the frame's noise / global / shuffle draws, and the
    shuffle is sized by the frame's point count after the paste.

    Selection runs on the host (db_sampler.select); the paste runs on the device over the resident database (sessd_gtaug_paste).  The
    host reads the pasted frame offsets back once, before drawing; when db_sampler draws from ``rs`` itself and a class stream has to be
    reshuffled in a later frame, the frames before it are pasted and drawn first (one more read-back per reshuffle), so the stream
    stays the reference's.  Returns (d_points [P', 4], d_frame_off [B+1], frame sizes, boxes per frame (gt then sampled, in their
    dtype), names per frame, Draws, accepted ids per frame).

    frame_hook: None, or f(frame, d_frame_points, size, boxes, names) -> FrameDraws, called for each pasted frame in stream order in
    place of draw_augmentation (the SA-DA path runs the frame's device stages there)."""
    db = db_sampler.device_database(device)
    B = len(clouds)
    ns = [len(c) for c in clouds]
    off = np.zeros(B + 1, np.int64)
    off[1:] = np.cumsum(ns)
    pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, 4) for c in clouds] + [np.zeros((0, 4), np.float32)])
    d_pts = torch.from_numpy(pts).pin_memory().to(device, non_blocking=True)
    ids, boxes, names, frames, groups, pending = [], [], [], [], [], []

    def flush():
        if not pending:
            return
        f0, f1 = pending[0], pending[-1] + 1
        obj_off = np.zeros(f1 - f0 + 1, np.int32)
        obj_off[1:] = np.cumsum([len(ids[f]) for f in range(f0, f1)])
        obj_ids = np.concatenate([ids[f] for f in range(f0, f1)] + [np.zeros(0, np.int64)]).astype(np.int32)
        sub_off = torch.from_numpy((off[f0:f1 + 1] - off[f0]).astype(np.int32)).to(device)
        out, fo = ops.gtaug_paste(d_pts[off[f0]:off[f1]], sub_off, obj_off, obj_ids, db["points"], db["off"], db["count"], db["boxes"],
                                  int(db_sampler.counts[obj_ids].sum()))
        fo = fo.cpu().numpy()                                   # the read-back: each frame's point count after the paste
        sizes = np.diff(fo)
        for f, n in zip(range(f0, f1), sizes):
            frames.append((int(n), len(boxes[f]), True))
            if frame_hook is None:
                draws.frames += draw_augmentation(rs, [frames[-1]], cfg).frames
            else:
                r0 = int(fo[f - f0])
                draws.frames.append(frame_hook(f, out[r0:r0 + int(n)], int(n), boxes[f], names[f]))
        groups.append((out, int(sizes.sum())))
        pending.clear()

    draws = Draws()
    shared = db_sampler._rs is rs
    if shared:
        db_sampler._set_random_state(_FlushOnShuffle(rs, flush))
    try:
        for b in range(B):
            gb = np.asarray(gt_boxes[b]).reshape(-1, 7)
            acc = db_sampler.select(gb, list(gt_names[b]))
            ids.append(acc)
            boxes.append(np.concatenate([gb, db_sampler.boxes[acc]]))
            names.append(np.concatenate([np.asarray(gt_names[b], dtype=object), db_sampler.names[acc].astype(object)]))
            pending.append(b)
        flush()
    finally:
        if shared:
            db_sampler._set_random_state(rs)
    sizes = [f[0] for f in frames]
    new_off = np.zeros(B + 1, np.int32)
    new_off[1:] = np.cumsum(sizes)
    # the frames' rows (the paste's buffer is sized by its capacity); several groups only when a stream was reshuffled mid-batch
    d_points = groups[0][0][:groups[0][1]] if len(groups) == 1 else torch.cat([o[:n] for o, n in groups])
    d_off = torch.from_numpy(new_off).to(device)
    return d_points, d_off, sizes, boxes, names, draws, ids


class _FlushOnShuffle:
    """the RandomState a sampler sees inside gtaug_batch: before it reshuffles a stream, the frames selected so far are pasted and
    their augmentation drawn (those draws precede the reshuffle in the reference's stream)"""

    def __init__(self, rs, flush):
        self._rs, self._flush = rs, flush

    def shuffle(self, x):
        self._flush()
        self._rs.shuffle(x)


class _SadaFrames:
    """The SA-DA path of a batch, one labelled frame at a time in the reference's stream order (Preprocess.__call__:113-161): the
    frame's noise and global draws, its device stages (augment_resident on its rows, perm = identity), its SA-DA (sessd_b200.sada:
    draws, at most one read-back of the swap counts), one read-back of its new size, then its shuffle draw.  ``assemble`` joins the
    frames into augment_batch's layout and shuffles them with one gather."""

    def __init__(self, cfg, sa_da, rs, device, twin=True):
        self.cfg, self.sa_da, self.rs, self.device, self.twin = cfg, sa_da, rs, device, twin
        self.frames = []

    def __call__(self, f, d_points, n, boxes, names):
        from . import sada
        cfg, rs = self.cfg, self.rs
        loc, rot, flip, rotation, scale = _labeled_draws(rs, len(boxes), cfg)
        fd = FrameDraws(loc, rot, flip, rotation, scale, np.arange(n))
        d_off = torch.tensor([0, n], dtype=torch.int32).to(self.device)
        aug = augment_resident(cfg, d_points, d_off, [n], [boxes], [names], Draws([fd]), self.device, student_boxes=True, twin=self.twin)
        k = sum(1 for nm in names if nm in cfg.class_names)
        out, num = sada.sada_frame(aug["points"], aug["sada_boxes"][0], k, rs, self.sa_da)
        size = int(num.item())                                  # the read-back: the shuffle is sized by the frame after SA-DA
        fd.perm = _shuffle(rs, size, cfg)
        self.frames.append((out[:size], aug, fd))
        return fd

    def assemble(self):
        B = len(self.frames)
        dev = self.frames[0][1]["frame_off"].device
        sizes = [len(o) for o, _, _ in self.frames]
        raw_sizes = [len(a["points_raw"]) if self.twin else 0 for _, a, _ in self.frames]
        off = np.zeros(B + 1, np.int32); off[1:] = np.cumsum(sizes)
        raw_off = np.zeros(B + 1, np.int32); raw_off[1:] = np.cumsum(raw_sizes)
        perm = np.concatenate([fd.perm for _, _, fd in self.frames] + [np.zeros(0, np.int64)]).astype(np.int32)
        host = torch.from_numpy(np.concatenate([off, raw_off, perm])).to(dev)
        d_off, d_raw_off, d_perm = host[:B + 1], host[B + 1:2 * B + 2], host[2 * B + 2:]
        pts = torch.cat([o for o, _, _ in self.frames] + [torch.empty((0, 4), dtype=torch.float32, device=dev)])
        points = ops.sada_shuffle(pts, d_off, max(sizes + [0]), d_perm) if len(pts) else pts
        M = max([1] + [a["gt_boxes"].shape[1] for _, a, _ in self.frames])
        res = dict(points=points, points_raw=torch.cat([a["points_raw"] for _, a, _ in self.frames]) if self.twin else None, frame_off=d_off,
                   frame_off_raw=d_raw_off, transformation=Draws([fd for _, _, fd in self.frames]).transformation())
        for key, num_key in (("gt_boxes", "num_gt"), ("gt_boxes_raw", "num_gt_raw")):
            bx = torch.zeros((B, M, 7), dtype=torch.float32, device=dev)
            for b, (_, a, _) in enumerate(self.frames):
                bx[b, :a[key].shape[1]] = a[key][0]
            res[key] = bx
            res[num_key] = torch.cat([a[num_key] for _, a, _ in self.frames])
        sel = torch.full((B, M), -1, dtype=torch.int32, device=dev)
        for b, (_, a, _) in enumerate(self.frames):
            sel[b, :a["selected"].shape[1]] = a["selected"][0]
        res["selected"] = sel
        return res, int(off[-1]), int(raw_off[-1])


def launch_train_batch(cfg, clouds, gt_boxes, gt_names, rs, labeled=None, device="cuda", db_sampler=None, sa_da=None, twin=True):
    """Everything of build_train_batch that runs on the device: the draws (host), augment_batch, the voxeliser on the student's points
    and on the twin, the target assigner on both box sets.  Returns a PendingBatch.

    twin=False builds the student's branch only (a single-model batch, as CIA-SSD pre-training reads): no teacher copy of the points,
    no second voxelisation or assignment, no ``*_raw`` keys.  The draws and the RandomState stream are those of twin=True, so every
    student key is bit-identical to the twin batch of the same stream.

    Without db_sampler nothing waits on the device.  With db_sampler (a det3d.core.sampler DataBaseSamplerV2), GT-database sampling
    runs first (gtaug_batch): it waits once on the pasted frame offsets before drawing the augmentation, because the shuffle is sized
    by each frame's point count after the paste and the next frame's draws follow it in the stream.

    sa_da: None, or a sessd_b200.sada.SadaConfig: shape-aware augmentation runs between the global scaling and the shuffle, as
    Preprocess does.  Its draws depend on each frame's device results, so the frames are then built one at a time (_SadaFrames): per
    frame it waits on the device once for the swap counts, only when a box is swap-selected, and once for the frame's size before the
    shuffle draw.  The voxelisations and assignments then run batched."""
    if labeled is not None and not all(labeled):
        raise ValueError("build_train_batch builds labelled batches (the reference gives unlabelled frames no targets and no twin); "
                         "augment unlabelled frames with augment_batch(..., labeled=...)")
    st = _static(cfg, device)
    B = len(clouds)
    if sa_da is not None:
        frames = _SadaFrames(st["aug"], sa_da, rs, device, twin)
        if db_sampler is None:
            pts = np.concatenate([np.asarray(c, np.float32).reshape(-1, 4) for c in clouds] + [np.zeros((0, 4), np.float32)])
            d_pts = torch.from_numpy(pts).pin_memory().to(device, non_blocking=True)
            r0 = 0
            for b in range(B):
                frames(b, d_pts[r0:r0 + len(clouds[b])], len(clouds[b]), np.asarray(gt_boxes[b]).reshape(-1, 7), list(gt_names[b]))
                r0 += len(clouds[b])
        else:
            gtaug_batch(st["aug"], clouds, gt_boxes, gt_names, rs, db_sampler, device, frame_hook=frames)
        aug, total, total_raw = frames.assemble()
    elif db_sampler is None:
        draws = draw_augmentation(rs, [(len(c), len(b), True) for c, b in zip(clouds, gt_boxes)], st["aug"])
        aug = augment_batch(st["aug"], clouds, gt_boxes, gt_names, draws, device=device, twin=twin)
        total = total_raw = int(sum(len(c) for c in clouds))
    else:
        d_points, d_off, sizes, boxes, names, draws, _ = gtaug_batch(st["aug"], clouds, gt_boxes, gt_names, rs, db_sampler, device)
        aug = augment_resident(st["aug"], d_points, d_off, sizes, boxes, names, draws, device, twin=twin)
        total = total_raw = int(sum(sizes))
    A = st["anchors"].shape[0]
    vox = ops.VoxelBuffers(st["vcfg"], B, max(total, 1), device)
    ops.voxelize(aug["points"], aug["frame_off"], vox)
    asg = ops.AssignBuffers(A, B, aug["gt_boxes"].shape[1], device)
    ops.assign_targets(st["anchors"], aug["gt_boxes"], aug["num_gt"], asg, *st["thr"])
    vox_raw = asg_raw = None
    if twin:
        vox_raw = ops.VoxelBuffers(st["vcfg"], B, max(total_raw, 1), device)
        ops.voxelize(aug["points_raw"], aug.get("frame_off_raw", aug["frame_off"]), vox_raw)
        asg_raw = ops.AssignBuffers(A, B, aug["gt_boxes"].shape[1], device)
        ops.assign_targets(st["anchors"], aug["gt_boxes_raw"], aug["num_gt_raw"], asg_raw, *st["thr"])
    return PendingBatch(st, aug, vox, vox_raw, asg, asg_raw, B, aug["frame_off"], total)


def build_train_batch(cfg, clouds, gt_boxes, gt_names, rs, labeled=None, device="cuda", db_sampler=None, sa_da=None, twin=True):
    """A collated SE-SSD training batch with real augmentation: the ``example`` dict batch_processor_inline takes, with the keys of
    ``synth.train_batch`` (voxels, coordinates with a batch column, num_points, num_voxels, shape, anchors, labels, reg_targets, their
    ``_raw`` twins for the teacher, points with a batch column, metadata, transformation), all tensors on the device.

    cfg: the loaded det3d Config (train_preprocessor, voxel_generator, train_cfg.assigner); clouds: per frame [N, 4] f32; gt_boxes /
    gt_names: per frame [M, 7] and [M] (DontCare / ignore dropped); rs: the numpy RandomState the draws come from (draw_augmentation).
    db_sampler: None, or the GT-database sampler (det3d.builder.build_dbsampler(cfg.db_sampler)): sampled objects are pasted into each
    frame first, as Preprocess does.  The student's frame is noised, flipped, rotated, scaled and shuffled; the teacher's twin is the
    noised frame (Preprocess:131).

    sa_da: None, or a sessd_b200.sada.SadaConfig (its defaults are the car values Preprocess passes): shape-aware augmentation of the
    student's frame between the global scaling and the shuffle.  It leaves the boxes and the teacher's twin as they are.

    Without db_sampler and sa_da the device work is launched without waiting (launch_train_batch); with a db_sampler, GT-AUG reads the
    pasted frame sizes back once before drawing; with sa_da, each frame waits on the device once or twice (see launch_train_batch).
    Forming the dict then reads the two branches' voxel totals back once, because the model consumes exact-count voxel tensors.

    twin=False: the student's branch only, without the ``*_raw`` keys (see launch_train_batch)."""
    return launch_train_batch(cfg, clouds, gt_boxes, gt_names, rs, labeled, device, db_sampler, sa_da, twin).example()
