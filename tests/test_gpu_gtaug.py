"""GPU GT-database sampling (csrc/gtaug.cu and sessd_gtaug_select_host through the C ABI, sessd_b200.augment with a db_sampler) against
the reference's own DataBaseSamplerV2 run on a crafted database (tests/golden/gtaug_cases.npz) and the numpy oracle
(oracle/gt_aug_ref.py), then a batch end to end.  Bars: bit-exact everywhere (the paste is one fp64 add rounded to fp32 per coordinate;
membership is the fp64 box-frame test with every crafted point at least 1e-3 from every face)."""
import ctypes as C
import os
import pickle

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
from test_augment_oracle import reference_config  # noqa: E402
from test_gtaug_oracle import load, mirror_sampler, write_database  # noqa: E402

pytestmark = pytest.mark.gpu


def _db(z):
    rel = [z["db_rel_points"][o:o + n] for o, n in zip(z["db_off"], z["db_count"])]
    t = lambda a, dt: torch.from_numpy(np.ascontiguousarray(a, dt)).cuda()
    return rel, dict(points=t(z["db_rel_points"], np.float32).reshape(-1, 4), off=t(z["db_off"], np.int32),
                     count=t(z["db_count"], np.int32), boxes=t(z["db_boxes"], np.float64))


def _paste_fixture(z, ids_override=None, repeat=1):
    from sessd_b200 import ops
    F = int(z["num_frames"])
    clouds = [z["f%d_in_points" % f] for f in range(F)] * repeat
    ids = ([z["f%d_ids" % f] for f in range(F)] if ids_override is None else ids_override) * repeat
    off = np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)
    pts = torch.from_numpy(np.concatenate(clouds).astype(np.float32)).cuda()
    obj_off = np.concatenate([[0], np.cumsum([len(i) for i in ids])]).astype(np.int32)
    obj_ids = np.concatenate(ids).astype(np.int32)
    _, db = _db(z)
    max_paste = int(sum(z["db_count"][i] for i in obj_ids if 0 <= i < len(z["db_count"])))
    return ops, pts, torch.from_numpy(off).cuda(), obj_off, obj_ids, db, max_paste


def test_select_host_reproduces_the_fixture_acceptance():
    from oracle import gt_aug_ref
    from sessd_b200 import ops
    z = load()
    from test_gtaug_oracle import db_infos_from
    infos = gt_aug_ref.filter_db(db_infos_from(z), {"Car": int(z["min_points"])}, [-1])
    g = gt_aug_ref.GtAug(infos, [("Car", int(z["max_num"]))], np.random.RandomState(int(z["seed"])), similar=bool(z["similar"]))
    rounds = 0
    for f in range(int(z["num_frames"])):
        pre = "f%d_" % f
        bx, names = z[pre + "in_boxes"], z[pre + "in_names"]
        _, log = g.sample_frame(bx, names)
        all_gt = bx
        for _, cand, acc in log:
            c = np.concatenate([gt_aug_ref.corners(all_gt), gt_aug_ref.corners(g.boxes[cand], True)])
            assert np.array_equal(ops.gtaug_select_host(c, len(all_gt)), acc), f
            all_gt = np.concatenate([all_gt, g.boxes[cand[acc]]])
            rounds += 1
        from test_gtaug_oracle import rest_of_frame
        rest_of_frame(g.streams["Car"][1].rs, z, pre)
    assert rounds >= 10


def test_paste_kernel_reproduces_the_fixture_frames():
    """the fixture's frames as one batch, then four times over (19.5k scene points: the survivor scan spans several tiles, with empty
    frames and frame boundaries inside its tiles)"""
    z = load()
    F = int(z["num_frames"])
    for repeat in (1, 4):
        ops, pts, off, obj_off, obj_ids, db, max_paste = _paste_fixture(z, repeat=repeat)
        out, fo = ops.gtaug_paste(pts, off, obj_off, obj_ids, db["points"], db["off"], db["count"], db["boxes"], max_paste)
        fo = fo.cpu().numpy()
        for f in range(F * repeat):
            assert np.array_equal(out[fo[f]:fo[f + 1]].cpu().numpy(), z["f%d_points_pasted" % (f % F)]), (repeat, f)


def test_builder_draws_ids_and_pasted_frames_follow_the_reference_stream(tmp_path):
    """the fixture's frames as one batch: the tiny database reshuffles in every frame, so gtaug_batch pastes and draws frame by frame
    before each reshuffle -- ids, draws and pasted frames equal the reference's stream on the same seed"""
    from sessd_b200 import augment
    z = load()
    from test_gtaug_oracle import db_infos_from
    write_database(z, str(tmp_path))
    rs = np.random.RandomState(int(z["seed"]))
    s = mirror_sampler(z, db_infos_from(z), rs)
    s.load_database(str(tmp_path))
    fid = np.array([i["image_idx"] for i in s._infos])
    F = int(z["num_frames"])
    clouds = [z["f%d_in_points" % f] for f in range(F)]
    d_pts, d_off, sizes, boxes, names, draws, ids = augment.gtaug_batch(augment.AugmentConfig(), clouds,
                                                                       [z["f%d_in_boxes" % f] for f in range(F)],
                                                                       [z["f%d_in_names" % f] for f in range(F)], rs, s)
    off = d_off.cpu().numpy()
    for f in range(F):
        pre = "f%d_" % f
        assert np.array_equal(fid[ids[f]], z[pre + "ids"]), f
        assert np.array_equal(boxes[f], z[pre + "gt_boxes"]) and list(names[f]) == list(z[pre + "gt_names"])
        assert np.array_equal(d_pts[off[f]:off[f + 1]].cpu().numpy(), z[pre + "points_pasted"]), f
        d = draws.frames[f]
        assert np.array_equal(d.loc, z[pre + "loc"]) and np.array_equal(d.perm, z[pre + "perm"]), f
        assert (d.flip, d.rotation, d.scale) == (bool(z[pre + "flip"]), float(z[pre + "rotation"]), float(z[pre + "scale"]))


# ---------------------------------------------------------------------------------------------------------------- end to end
def synthetic_database(root, n_obj=240, seed=0):
    """a KITTI-like car database: boxes on a ring band, 20..400 points each (fp32 relative to the fp64 centre); returns the pickle path"""
    rs = np.random.RandomState(seed)
    infos = {"Car": [], "Pedestrian": []}
    os.makedirs(os.path.join(root, "gt_database"), exist_ok=True)
    for k in range(n_obj):
        name = "Car" if k % 12 else "Pedestrian"
        r, a = rs.uniform(6, 60), rs.uniform(-0.7, 0.7)
        dims = [1.6, 3.9, 1.56] if name == "Car" else [0.6, 0.8, 1.73]
        b = np.array([r * np.cos(a), r * np.sin(a), -1.0 + rs.uniform(-0.2, 0.2)] + [d + rs.uniform(-0.1, 0.1) for d in dims] +
                     [rs.uniform(-np.pi, np.pi)], np.float64)
        n = int(rs.randint(20, 400))
        loc = rs.uniform(-0.5, 0.5, (n, 3)) * (b[3:6] - 4e-3)
        c, s = np.cos(b[6]), np.sin(b[6])
        p = np.stack([loc[:, 0] * c + loc[:, 1] * s + b[0], -loc[:, 0] * s + loc[:, 1] * c + b[1], loc[:, 2] + b[2],
                      rs.uniform(0, 1, n)], 1).astype(np.float32)
        p[:, :3] -= b[:3]
        path = "gt_database/%06d_%s_0.bin" % (k, name)
        p.tofile(os.path.join(root, path))
        infos[name].append(dict(name=name, path=path, image_idx=k, gt_idx=0, box3d_lidar=b, num_points_in_gt=n, difficulty=0,
                                group_id=k))
    with open(os.path.join(root, "dbinfos_train.pkl"), "wb") as f:
        pickle.dump(infos, f)
    return os.path.join(root, "dbinfos_train.pkl")


def _few_car_frames(batch, seed, cars=3):
    from sessd_data import synth
    clouds = [synth.ring_cloud(seed + b, 20000, 15) for b in range(batch)]
    boxes = [synth.ring_boxes(seed + b, 15)[:cars].astype(np.float64) for b in range(batch)]
    names = [np.array(["Car"] * (cars - 1) + ["Pedestrian"]) for _ in range(batch)]
    return clouds, boxes, names


def _sampler(tmp_path, rs):
    from det3d.builder import build_dbsampler
    cfg = reference_config().db_sampler
    cfg.db_info_path = synthetic_database(str(tmp_path))
    return build_dbsampler(cfg, random_state=rs)


def test_batch_end_to_end_against_the_oracle(tmp_path):
    """8 ring-20k frames with 3 boxes each (most frames paste many objects) through launch_train_batch(db_sampler=...): both branches'
    voxels and the targets bit-exact against the oracle path (gt_aug_ref + augment_ref), the CPU voxeliser and assign_v2"""
    from det3d.core.bbox import box_np_ops
    from det3d.datasets.pipelines import AssignTarget
    from det3d.datasets.pipelines.preprocess import filter_gt_box_outside_range
    from oracle import cpu as ocpu, gt_aug_ref
    from sessd_b200 import augment, synth
    cfg = reference_config()
    B = 8
    clouds, boxes, names = _few_car_frames(B, 300)
    rs = np.random.RandomState(11)
    sampler = _sampler(tmp_path, rs)
    pend = augment.launch_train_batch(cfg, clouds, boxes, names, rs, db_sampler=sampler)
    # the same host selection and draws, replayed: a second sampler on the same seed (the builder's stream order)
    rs2 = np.random.RandomState(11)
    s2 = _sampler(tmp_path, rs2)
    _, _, sizes, _, _, draws, ids = augment.gtaug_batch(augment.AugmentConfig.from_config(cfg), clouds, boxes, names, rs2, s2)
    assert min(len(i) for i in ids) >= 5
    ex = pend.example()
    assert ex["transformation"] == draws.transformation()
    aug = pend._aug
    acfg = pend._st["aug"]
    off = aug["frame_off"].cpu().numpy()
    at = AssignTarget(cfg=cfg.train_cfg.assigner)
    ta, ad = at.target_assigners[0], at.anchor_dicts_by_task[0]
    rel = [sampler._points[o:o + n] for o, n in zip(sampler.offsets, sampler.counts)]
    branches = {"student": (pend._vox, pend._asg), "teacher": (pend._vox_raw, pend._asg_raw)}
    vbase = {k: np.concatenate([[0], np.cumsum(v[0].num_voxels[:B].cpu().numpy())]) for k, v in branches.items()}
    for b in range(B):
        f = draws.frames[b]
        o = gt_aug_ref.preprocess_frame(clouds[b], boxes[b], names[b], ids[b], rel, sampler.boxes, sampler.names, acfg.class_names,
                                        dict(loc=f.loc, rot=f.rot, flip=f.flip, rotation=f.rotation, scale=f.scale, perm=f.perm))
        assert off[b + 1] - off[b] == len(o["points"]) == sizes[b]
        assert np.array_equal(aug["points"][off[b]:off[b + 1]].cpu().numpy(), o["points"])
        assert np.array_equal(aug["points_raw"][off[b]:off[b + 1]].cpu().numpy(), o["points_raw"])
        keep = filter_gt_box_outside_range(o["boxes"], acfg.range_bev)
        tgt = np.array([n in ("Car", "Van") for n in o["names_pasted"]])[np.array([n in acfg.class_names for n in o["names_pasted"]])]
        for name, pts, bx in (("student", o["points"], o["boxes"][keep & tgt]), ("teacher", o["points_raw"], o["boxes_raw"][tgt])):
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
            assert np.array_equal(abuf.labels[b].cpu().numpy(), ref["labels"].astype(np.int32)), (name, b)
            npos = int(abuf.num_pos[b].item())
            assert np.array_equal(abuf.pos_anchor[b, :npos].cpu().numpy(), np.nonzero(ref["labels"] > 0)[0]), (name, b)
    assert sum(int(branches["student"][1].num_pos[b].item()) for b in range(B)) > 0


def test_gtaug_batch_feeds_the_training_step(tmp_path):
    import copy
    from det3d.models import build_detector
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
    from sessd_b200 import augment, weights
    cfg = reference_config()
    B = 4
    clouds, boxes, names = _few_car_frames(B, 400)
    rs = np.random.RandomState(5)
    ex = augment.build_train_batch(cfg, clouds, boxes, names, rs, db_sampler=_sampler(tmp_path, rs))
    assert len(ex["points"]) > sum(len(c) for c in clouds) // 2
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


def test_full_frames_sample_nothing_and_match_the_plain_batch(tmp_path):
    """every frame holds 15 cars: GT-AUG samples nothing, and the batch equals the one built without a sampler, bit for bit"""
    from sessd_b200 import augment, synth as ssynth
    from sessd_data import synth
    cfg = reference_config()
    B = 3
    clouds = [synth.ring_cloud(700 + b, 20000, 15) for b in range(B)]
    boxes = [synth.ring_boxes(700 + b, 15) for b in range(B)]
    names = [np.array(["Car"] * 15) for _ in range(B)]
    rs = np.random.RandomState(9)
    sampler = _sampler(tmp_path, rs)
    state = rs.get_state()
    a = augment.build_train_batch(cfg, clouds, boxes, names, rs, db_sampler=sampler)
    rs.set_state(state)
    b = augment.build_train_batch(cfg, clouds, boxes, names, rs)
    assert set(a) == set(b)
    for k in a:
        x, y = a[k], b[k]
        if isinstance(x, torch.Tensor):
            assert torch.equal(x, y), k
        elif isinstance(x, list) and x and isinstance(x[0], torch.Tensor):
            assert all(torch.equal(p, q) for p, q in zip(x, y)), k
        elif isinstance(x, np.ndarray):
            assert np.array_equal(x, y), k
        else:
            assert x == y, k


def test_error_codes():
    from sessd_b200 import ops
    from sessd_b200._lib import lib
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    x = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(x.data_ptr())
    null = C.c_void_p(0)
    ws = int(lib.sessd_gtaug_paste_workspace_bytes(1, 16, 1))
    assert 0 < ws < (1 << 16)
    args = lambda **k: [k.get("pts", p), p, 1, 16, p, p, 1, 32, p, p, p, p, 4, k.get("ws", p), k.get("wsb", ws), p, k.get("cap", 48), p, st]
    assert lib.sessd_gtaug_paste(*args(pts=null)) == -1
    assert lib.sessd_gtaug_paste(*args(ws=null)) == -1
    assert lib.sessd_gtaug_paste(*args(cap=47)) == -2                        # capacity < num_points + max_paste_points
    assert lib.sessd_gtaug_paste(*args(wsb=ws - 1)) == -3
    assert lib.sessd_gtaug_paste(*args(pts=C.c_void_p(x.data_ptr() + 4))) == -1
    assert lib.sessd_gtaug_select_host(None, 0, 1, None) == -1
    torch.cuda.synchronize()
    # an out-of-range id: rejected by the wrapper; straight to the ABI it pastes nothing and the rest of the batch is intact
    z = load()
    ops_, pts, off, obj_off, obj_ids, db, max_paste = _paste_fixture(z)
    bad = obj_ids.copy()
    bad[3] = len(z["db_count"]) + 5
    with pytest.raises(ValueError):
        ops.gtaug_paste(pts, off, obj_off, bad, db["points"], db["off"], db["count"], db["boxes"], max_paste)
    out, fo = ops.gtaug_paste(pts, off, torch.from_numpy(obj_off).cuda(), torch.from_numpy(bad).cuda(), db["points"], db["off"],
                              db["count"], db["boxes"], max_paste)
    fo = fo.cpu().numpy()
    F = int(z["num_frames"])
    ids = [z["f%d_ids" % f] for f in range(F)]
    frame_of_3 = int(np.searchsorted(obj_off, 3, side="right") - 1)
    ids[frame_of_3] = np.delete(ids[frame_of_3], 3 - obj_off[frame_of_3])
    rel, _ = _db(z)
    from oracle import gt_aug_ref
    for f in range(F):
        exp, _, _, _ = gt_aug_ref.paste(z["f%d_in_points" % f], z["f%d_in_boxes" % f], z["f%d_in_names" % f], ids[f], rel, z["db_boxes"],
                                        z["db_names"])
        assert np.array_equal(out[fo[f]:fo[f + 1]].cpu().numpy(), exp), f
