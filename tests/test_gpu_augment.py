"""GPU training augmentation (csrc/augment.cu through the C ABI, sessd_b200.augment) against the reference's own functions
(tests/golden/augment_cases.npz) and the numpy oracle (oracle/augment_ref.py), one operator at a time, then a batch end to end.

Bars.  Collision matrix, selected tries and the box bookkeeping: bit-exact.  Points and boxes after the per-object and global stages:
bit-exact as well -- every operation is an individually rounded fp32 / fp64 operation or an fma, in the reference's order, and the only
transcendental values computed on the device are the fp64 cos / sin of the draws and box angles (CUDA's double-precision cos / sin are
within 2 ulp, so the fp32 values rounded from them can only differ when the fp64 value lies within 2^-51 relative of an fp32 rounding
boundary: about 1 in 2^22 per value), and the membership test's fp64 frame (points are kept >= 1e-3 from every face, so that cannot flip
a point).  Everything else the global stages need is rounded on the host as the reference rounds it."""
import ctypes as C

import numpy as np
import pytest
import torch

from test_augment_oracle import load_frames, reference_config

pytestmark = pytest.mark.gpu


def _cu(a, dt=None):
    return torch.from_numpy(np.ascontiguousarray(a if dt is None else np.asarray(a, dt))).cuda()


def _batch(frames):
    """pad a list of fixture frames into the device layout"""
    from sessd_b200 import augment
    B = len(frames)
    M = max([1] + [len(d["in_boxes"]) for d in frames])
    boxes = np.zeros((B, M, 7), np.float32); valid = np.zeros((B, M), np.uint8)
    loc = np.zeros((B, M, 100, 3)); rot = np.zeros((B, M, 100)); num = np.zeros(B, np.int32)
    glob = np.zeros((B, 5), np.float32)
    for b, d in enumerate(frames):
        m = len(d["in_boxes"])
        boxes[b, :m] = d["in_boxes"]; valid[b, :m] = d["valid"]; num[b] = m
        loc[b, :m] = d["loc"]; rot[b, :m] = d["rot"]
        glob[b] = augment.global_row(augment.FrameDraws(d["loc"], d["rot"], bool(d["flip"]), float(d["rotation"]), float(d["scale"]),
                                                        d["perm"]))
    return boxes, valid, loc, rot, num, glob


def _groups():
    _, frames = load_frames()
    lab = [d for d in frames if d["labeled"] and float(d["context"]) <= 0]
    ctx = [d for d in frames if d["labeled"] and float(d["context"]) > 0]
    return frames, lab, ctx


def test_collision_matrix_bit_exact():
    from sessd_b200 import ops
    z, _ = load_frames()
    got = ops.box_collision(_cu(z["coll_boxes"]), _cu(z["coll_qboxes"])).cpu().numpy().astype(bool)
    assert np.array_equal(got, z["coll_ref"])


def test_selected_tries_bit_exact():
    from sessd_b200 import ops
    _, lab, ctx = _groups()
    for group in (lab, ctx):
        boxes, valid, loc, rot, num, _ = _batch(group)
        ctxv = float(group[0]["context"])
        sel = ops.noise_per_box(_cu(boxes), _cu(num), _cu(valid), _cu(loc), _cu(rot), ctxv).cpu().numpy()
        for b, d in enumerate(group):
            m = len(d["in_boxes"])
            assert np.array_equal(sel[b, :m], d["selected"]), str(d["name"])
            assert (sel[b, m:] == -1).all()


def test_points_in_boxes_matches_reference_masks():
    """the membership entry point (GT-AUG's points_in_rbbox as well) against points_in_convex_polygon_3d_jit's masks, all boxes"""
    from sessd_b200 import ops
    _, lab, ctx = _groups()
    for d in lab + ctx:
        if not len(d["in_boxes"]) or not len(d["in_points"]):
            continue
        got = ops.points_in_boxes(_cu(d["in_points"]), _cu(d["in_boxes"]), float(d["context"])).cpu().numpy().astype(bool)
        assert np.array_equal(got, d["masks"]), str(d["name"])


def _points_run(group, labeled=None):
    from sessd_b200 import ops
    boxes, valid, loc, rot, num, glob = _batch(group)
    ns = [len(d["in_points"]) for d in group]
    off = np.concatenate([[0], np.cumsum(ns)]).astype(np.int32)
    pts = np.concatenate([d["in_points"] for d in group]).astype(np.float32).reshape(-1, 4)
    perm = np.concatenate([d["perm"] for d in group] + [np.zeros(0, np.int64)]).astype(np.int32)
    ctxv = float(group[0]["context"])
    d_boxes, d_num, d_valid, d_loc, d_rot, d_glob = _cu(boxes), _cu(num), _cu(valid), _cu(loc), _cu(rot), _cu(glob)
    sel = ops.noise_per_box(d_boxes, d_num, d_valid, d_loc, d_rot, ctxv)
    raw, out = ops.augment_points(_cu(pts), _cu(off), max(ns), d_boxes, d_num, d_valid, d_loc, d_rot, sel, d_glob, _cu(perm),
                                  None if labeled is None else _cu(labeled, np.uint8), ctxv)
    return off, raw.cpu().numpy(), out.cpu().numpy(), (d_boxes, d_num, d_valid, d_loc, d_rot, sel, d_glob)


def test_points_membership_transform_twin_and_shuffle():
    frames, lab, ctx = _groups()
    for group in (lab, ctx):
        off, raw, out, _ = _points_run(group)
        for b, d in enumerate(group):
            r, o = raw[off[b]:off[b + 1]], out[off[b]:off[b + 1]]
            assert np.array_equal(r, d["points_raw"]), str(d["name"])          # the teacher's twin: noised, unshuffled
            assert np.array_equal(o, d["points"]), str(d["name"])              # the student's: global stages, then the permutation
            # membership: exactly the points of a valid box moved (bitwise), with the reference's masks
            owner = (d["masks"] & d["valid"][None, :]).any(1) if len(d["in_boxes"]) else np.zeros(len(r), bool)
            moved = (r != d["in_points"]).any(1)
            assert not (moved & ~owner).any()
    unl = [d for d in frames if not d["labeled"]]
    off, raw, out, _ = _points_run(unl, labeled=[0])
    assert np.array_equal(out, unl[0]["points"])
    # the permutation alone: global identity draws leave the shuffled rows bit-equal to the input rows
    d = dict(unl[0]); d.update(flip=False, rotation=0.0, scale=1.0)
    off, raw, out, _ = _points_run([d], labeled=[0])
    assert np.array_equal(out, d["in_points"][d["perm"]])


def test_box_transform_global_and_bookkeeping():
    from det3d.core.bbox import box_np_ops
    from det3d.datasets.pipelines.preprocess import filter_gt_box_outside_range
    from sessd_b200 import ops
    _, lab, _ = _groups()
    rg = (0.0, -40.0, 70.4, 40.0)
    boxes, valid, loc, rot, num, glob = _batch(lab)
    d_boxes, d_num, d_valid, d_loc, d_rot, d_glob = _cu(boxes), _cu(num), _cu(valid), _cu(loc), _cu(rot), _cu(glob)
    sel = ops.noise_per_box(d_boxes, d_num, d_valid, d_loc, d_rot)
    braw, nraw, bout, nout = [t.cpu().numpy() for t in ops.augment_boxes(d_boxes, d_num, d_valid, None, d_loc, d_rot, sel, d_glob, rg)]
    lp = lambda b: np.concatenate([b[:, :6], box_np_ops.limit_period(b[:, 6:7], 0.5, np.pi * 2)], 1).astype(np.float32)  # noqa: E731
    for b, d in enumerate(lab):
        want_raw = lp(d["boxes_raw"])
        keep = filter_gt_box_outside_range(d["boxes"], rg) if len(d["boxes"]) else np.zeros(0, bool)
        want_out = lp(d["boxes"][keep])
        assert nraw[b] == len(want_raw) and np.array_equal(braw[b, :nraw[b]], want_raw), str(d["name"])
        assert nout[b] == len(want_out) and np.array_equal(bout[b, :nout[b]], want_out), str(d["name"])
        assert (braw[b, nraw[b]:] == 0).all() and (bout[b, nout[b]:] == 0).all()


def _train_frames(batch, seed):
    from sessd_data import synth
    clouds = [synth.ring_cloud(seed + b, 20000, 15) for b in range(batch)]
    boxes = [synth.ring_boxes(seed + b, 15) for b in range(batch)]
    names = [np.array(["Car"] * 13 + ["Van", "Pedestrian"]) for _ in range(batch)]
    return clouds, boxes, names


def test_global_boxes_are_the_oracle_global_boxes():
    """augment_boxes' optional output, the boxes SA-DA takes: per frame the class-valid boxes after the noise and the global stages, in
    index order, before the range filter and limit_period, zero padded"""
    from oracle import augment_ref
    from sessd_b200 import augment, ops
    acfg = augment.AugmentConfig.from_config(reference_config())
    clouds, boxes, names = _train_frames(4, 300)
    draws = augment.draw_augmentation(np.random.RandomState(9), [(len(c), len(b), True) for c, b in zip(clouds, boxes)], acfg)
    (_, _), rest, _ = augment._host_inputs(acfg, [len(c) for c in clouds], boxes, names, draws, None)
    d_boxes, d_num, d_valid, _, d_loc, d_rot, d_glob = [_cu(a) for a in rest[:7]]
    sel = ops.noise_per_box(d_boxes, d_num, d_valid, d_loc, d_rot)
    sb, sn = ops.augment_boxes(d_boxes, d_num, d_valid, None, d_loc, d_rot, sel, d_glob, acfg.range_bev, global_boxes=True)[4:]
    sb, sn = sb.cpu().numpy(), sn.cpu().numpy()
    for b in range(4):
        valid = np.array([n in acfg.class_names for n in names[b]])
        f = draws.frames[b]
        o = augment_ref.augment_frame(clouds[b], boxes[b], valid, dict(loc=f.loc, rot=f.rot, flip=f.flip, rotation=f.rotation,
                                                                        scale=f.scale, perm=f.perm))
        assert sn[b] == valid.sum() and np.array_equal(sb[b, :sn[b]], o["boxes"]) and not sb[b, sn[b]:].any()


def test_batch_end_to_end_against_the_oracle():
    """8 ring-20k frames with 15 boxes: both branches' voxels bit-exact against the CPU voxeliser on the oracle-augmented points, targets
    bit-exact against assign_v2 on the oracle-augmented boxes, transformation = the draws, and no host synchronisation while building"""
    from det3d.datasets.pipelines import AssignTarget
    from det3d.datasets.pipelines.preprocess import filter_gt_box_outside_range
    from det3d.core.bbox import box_np_ops
    from det3d.torchie import Config
    from oracle import augment_ref, cpu as ocpu
    from sessd_b200 import augment, ops, synth
    import os
    acfg = augment.AugmentConfig.from_config(reference_config())
    B = 8
    clouds, boxes, names = _train_frames(B, 100)
    draws = augment.draw_augmentation(np.random.RandomState(5), [(len(c), len(b), True) for c, b in zip(clouds, boxes)], acfg)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        res = augment.augment_batch(acfg, clouds, boxes, names, draws)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    assert res["transformation"] == [dict(flipped=f.flip, noise_rotation=f.rotation, noise_scale=f.scale) for f in draws.frames]
    assert {f.flip for f in draws.frames} == {False, True}
    cfg = Config.fromfile(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "examples", "second", "configs",
                                       "config.py"))
    vcfg = ops.make_voxel_cfg(synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
    at = AssignTarget(cfg=cfg.train_cfg.assigner)
    ta, ad = at.target_assigners[0], at.anchor_dicts_by_task[0]
    anchors = _cu(np.ascontiguousarray(list(ad.values())[0]["anchors"].reshape(-1, 7), np.float32))
    off = res["frame_off"].cpu().numpy()
    branches = {}
    for name, pts_key, box_key, num_key in (("student", "points", "gt_boxes", "num_gt"), ("teacher", "points_raw", "gt_boxes_raw",
                                                                                           "num_gt_raw")):
        buf = ops.VoxelBuffers(vcfg, B, int(off[-1]), "cuda")
        ops.voxelize(res[pts_key], res["frame_off"], buf)
        abuf = ops.AssignBuffers(anchors.shape[0], B, res[box_key].shape[1], "cuda")
        ops.assign_targets(anchors, res[box_key], res[num_key], abuf)
        branches[name] = (buf, abuf)
    torch.cuda.synchronize()
    sel = res["selected"].cpu().numpy()
    vbase = {k: np.concatenate([[0], np.cumsum(v[0].num_voxels[:B].cpu().numpy())]) for k, v in branches.items()}   # collate order
    for b in range(B):
        valid = np.array([n in acfg.class_names for n in names[b]])
        f = draws.frames[b]
        o = augment_ref.augment_frame(clouds[b], boxes[b], valid, dict(loc=f.loc, rot=f.rot, flip=f.flip, rotation=f.rotation,
                                                                        scale=f.scale, perm=f.perm))
        assert np.array_equal(sel[b, :15], o["selected"])
        assert np.array_equal(res["points"][off[b]:off[b + 1]].cpu().numpy(), o["points"])
        assert np.array_equal(res["points_raw"][off[b]:off[b + 1]].cpu().numpy(), o["points_raw"])
        keep = filter_gt_box_outside_range(o["boxes"], acfg.range_bev)
        for name, pts, bx in (("student", o["points"], o["boxes"][keep]), ("teacher", o["points_raw"], o["boxes_raw"])):
            buf, abuf = branches[name]
            v, c, n = ocpu.points_to_voxel(pts, synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
            nv = int(buf.num_voxels[b].item())
            base = int(vbase[name][b])
            assert nv == len(c), (name, b)
            assert np.array_equal(buf.coors[base:base + nv, 1:].cpu().numpy(), c), (name, b)
            assert np.array_equal(buf.num_points[base:base + nv].cpu().numpy(), n), (name, b)
            assert np.array_equal(buf.voxels[base:base + nv].cpu().numpy(), v), (name, b)
            bx = bx.copy()
            bx[:, 6] = box_np_ops.limit_period(bx[:, 6], 0.5, np.pi * 2)
            ref = ta.assign_v2(ad, bx, anchors_mask=None, gt_classes=np.ones(len(bx), np.int32), gt_names=np.array(["Car"] * len(bx)),
                               enable_similar_type=True)
            labels = abuf.labels[b].cpu().numpy()
            assert np.array_equal(labels, ref["labels"].astype(np.int32)), (name, b)
            npos = int(abuf.num_pos[b].item())
            assert np.array_equal(abuf.pos_anchor[b, :npos].cpu().numpy(), np.nonzero(ref["labels"] > 0)[0]), (name, b)
            assert np.array_equal(abuf.pos_gt_id[b, :npos].cpu().numpy(), ref["positive_gt_id"][0]), (name, b)
    assert sum(int(branches["student"][1].num_pos[b].item()) for b in range(B)) > 0


def test_build_train_batch_feeds_the_training_step():
    """build_train_batch returns synth.train_batch's keys (same containers and dtypes), launches its device work with no host
    synchronisation (one read-back when the dict is formed), the teacher's voxels are those of the noised frame, and the batch runs
    through batch_processor_inline with a backward pass"""
    import copy
    from det3d.models import build_detector
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
    from oracle import augment_ref, cpu as ocpu
    from sessd_b200 import augment, synth, weights
    cfg = reference_config()
    B = 4
    clouds, boxes, names = _train_frames(B, 200)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        pending = augment.launch_train_batch(cfg, clouds, boxes, names, np.random.RandomState(3))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    ex = pending.example()
    ref = synth.train_batch(cfg, clouds, boxes)
    assert set(ex) == set(ref)
    for k, v in ref.items():
        got = ex[k]
        assert type(got) is type(v), k
        if isinstance(v, torch.Tensor):
            assert got.is_cuda and got.dtype == v.dtype and got.dim() == v.dim() and got.shape[1:] == v.shape[1:], k
        elif isinstance(v, list) and v and isinstance(v[0], torch.Tensor):
            assert got[0].dtype == v[0].dtype and got[0].shape == v[0].shape, k
    assert np.array_equal(ex["shape"], ref["shape"]) and np.array_equal(ex["anchors"][0].cpu().numpy(), ref["anchors"][0].cpu().numpy())
    draws = augment.draw_augmentation(np.random.RandomState(3), [(len(c), len(b), True) for c, b in zip(clouds, boxes)],
                                      augment.AugmentConfig.from_config(cfg))
    assert ex["transformation"] == draws.transformation()
    f = draws.frames[0]
    valid = np.array([n in ("Car", "Van") for n in names[0]])
    o = augment_ref.augment_frame(clouds[0], boxes[0], valid, dict(loc=f.loc, rot=f.rot, flip=f.flip, rotation=f.rotation, scale=f.scale,
                                                                    perm=f.perm))
    v, c, n = ocpu.points_to_voxel(o["points_raw"], synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
    nv = int(ex["num_voxels_raw"][0].item())
    assert nv == len(c) and np.array_equal(ex["coordinates_raw"][:nv].cpu().numpy(), np.concatenate([np.zeros((nv, 1), np.int32), c], 1))
    assert np.array_equal(ex["voxels_raw"][:nv].cpu().numpy(), v) and np.array_equal(ex["num_points_raw"][:nv].cpu().numpy(), n)
    assert np.array_equal(ex["points"][:len(clouds[0]), 1:].cpu().numpy(), o["points"]) and (ex["points"][:len(clouds[0]), 0] == 0).all()
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    model.load_state_dict(weights.random_detector_state(0), strict=True)
    model = model.cuda().train()
    ema = copy.deepcopy(model)
    for p in ema.parameters():
        p.requires_grad_(False)
    out = batch_processor_inline(model, ema, ex, consistency_weight=1.0, train_mode=True)
    assert torch.isfinite(out["loss"]).all() and out["num_samples"] == B
    out["loss"].backward()
    assert any(p.grad is not None and torch.isfinite(p.grad).all() for p in model.parameters())


def test_error_codes_and_the_global_box_pair():
    from sessd_b200._lib import lib
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    x = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(x.data_ptr())
    null = C.c_void_p(0)
    assert lib.sessd_box_collision(null, 1, p, 1, p, st) == -1
    assert lib.sessd_noise_per_box(p, p, p, 1, 4, null, p, 100, -1.0, p, st) == -1
    assert lib.sessd_noise_per_box(p, p, p, 1, 257, p, p, 100, -1.0, p, st) == -2            # SESSD_AUGMENT_MAX_GT
    assert lib.sessd_noise_per_box(p, p, p, 1, 16, p, p, 129, -1.0, p, st) == -2             # SESSD_AUGMENT_MAX_TRY
    assert lib.sessd_noise_per_box(p, p, p, 0, 16, p, p, 100, -1.0, p, st) == -1
    assert lib.sessd_augment_points(p, p, 1, 10, p, p, p, 257, p, p, 100, p, -1.0, p, p, None, None, p, st) == -2
    assert lib.sessd_augment_points(p, null, 1, 10, p, p, p, 4, p, p, 100, p, -1.0, p, p, None, None, p, st) == -1
    assert lib.sessd_augment_points(C.c_void_p(x.data_ptr() + 4), p, 1, 10, p, p, p, 4, p, p, 100, p, -1.0, p, p, None, None, p, st) == -1
    assert lib.sessd_points_in_boxes(null, 1, 4, p, 1, -1.0, p, st) == -1
    assert lib.sessd_points_in_boxes(p, 1, 2, p, 1, -1.0, p, st) == -1
    rg = (C.c_float * 4)(0.0, -40.0, 70.4, 40.0)
    assert lib.sessd_augment_boxes(p, p, p, None, 1, 257, p, p, 100, p, p, rg, p, p, p, p, None, None, st) == -2
    assert lib.sessd_augment_boxes(p, p, p, None, 1, 4, p, p, 100, p, p, None, p, p, p, p, None, None, st) == -1
    assert lib.sessd_augment_boxes(p, p, p, None, 1, 4, p, p, 100, p, p, rg, p, p, p, p, p, None, st) == -1      # the global pair:
    assert lib.sessd_augment_boxes(p, p, p, None, 1, 4, p, p, 100, p, p, rg, p, p, p, p, None, p, st) == -1      # both or neither
    torch.cuda.synchronize()
