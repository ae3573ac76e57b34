"""GPU shape-aware augmentation (csrc/sada.cu through the C ABI, sessd_b200.sada and the drop-in pyramid_augment_v0) against the
reference's own pyramid_augment_v0 run on crafted frames (tests/golden/sada_cases.npz) and the numpy oracle (tests/sada_ref.py).  Bars:
bit-exact everywhere (fp32 operations individually rounded in the reference's order; fp64 farthest-point distances)."""
import numpy as np
import pytest
import torch

import sada_ref
from test_sada_oracle import CASES, stage_cfg

pytestmark = pytest.mark.gpu


def _cu(a, dt=None):
    return torch.from_numpy(np.ascontiguousarray(a if dt is None else np.asarray(a, dt))).cuda()


def _mask(bits, a):
    b = bits.cpu().numpy().view(np.uint32)
    return ((b[:, np.arange(a) // 32] >> (np.arange(a) % 32).astype(np.uint32)) & 1).astype(bool)


@pytest.mark.parametrize("case", CASES, ids=[str(c["name"]) for c in CASES])
def test_pyramids_membership_and_counts_match_the_fixture(case):
    from sessd_b200 import ops
    K = len(case["boxes"])
    pyr, planes = ops.sada_pyramids(_cu(case["boxes"], np.float32).reshape(-1, 7))
    assert np.array_equal(pyr.cpu().numpy().reshape(K, 6, 15), case["pyramids"])
    if K == 0 or len(case["points"]) == 0:
        return
    bits, counts, _ = ops.sada_membership(_cu(case["points"], np.float32), planes, np.arange(6 * K))
    assert np.array_equal(_mask(bits, 6 * K), case["mask"])
    assert np.array_equal(counts.cpu().numpy(), case["mask"].sum(0))


@pytest.mark.parametrize("case", CASES, ids=[str(c["name"]) for c in CASES])
def test_stages_and_random_state_match_the_fixture(case):
    from sessd_b200 import sada
    d, sp, sw = stage_cfg(case["cfg"])
    rs = np.random.RandomState(int(case["seed"]))
    stages = {}
    pts = case["points"] if len(case["points"]) else np.zeros((0, 4), np.float32)
    out, num = sada.sada_frame(_cu(pts, np.float32).reshape(-1, 4), _cu(case["boxes"], np.float32).reshape(-1, 7), len(case["boxes"]),
                               rs, sada.SadaConfig(d, sp, sw), stages)
    torch.cuda.synchronize()
    for st in ("dropout", "sparsify", "swap"):
        rows, n = stages[st]
        n = len(pts) if n is None else int(n.item())
        assert np.array_equal(rows[:n].cpu().numpy(), case[st]), st
    assert np.array_equal(out[:int(num.item())].cpu().numpy(), case["swap"])
    _, key, pos = rs.get_state()[:3]
    assert np.array_equal(key, case["state_key"]) and pos == int(case["state_pos"])


@pytest.mark.parametrize("case", CASES, ids=[str(c["name"]) for c in CASES])
def test_drop_in_pyramid_augment_v0_equals_the_reference(case):
    from det3d.datasets.utils.sa_da_v2 import pyramid_augment_v0
    d, sp, sw = stage_cfg(case["cfg"])
    np.random.seed(int(case["seed"]))
    out = pyramid_augment_v0(case["boxes"].astype(np.float32).reshape(-1, 7), case["points"].astype(np.float32).reshape(-1, 4),
                             enable_sa_dropout=d, enable_sa_sparsity=None if sp is None else list(sp),
                             enable_sa_swap=None if sw is None else list(sw))
    assert out.dtype == np.float32 and np.array_equal(out, case["swap"])
    _, key, pos = np.random.get_state()[:3]
    assert np.array_equal(key, case["state_key"]) and pos == int(case["state_pos"])


def _pyramid_cloud(rs, n, dup=0):
    """n points inside pyramid 1 (the +x face) of an axis-aligned box, dup of them repeated, plus 300 points elsewhere"""
    box = np.array([[10.0, 2.0, -1.0, 40.0, 4.0, 3.0, 0.0]], np.float32)
    q = rs.uniform(-1, 1, (8 * n + 1000, 3))
    q = q[(q[:, 0] > np.abs(q[:, 1]) + 0.01) & (q[:, 0] > np.abs(q[:, 2]) + 0.01)][:n]
    p = np.concatenate([q * 0.5 * box[0, 3:6] + box[0, :3], rs.uniform(0, 1, (len(q), 1))], 1).astype(np.float32)
    if dup:
        p[-dup:] = p[rs.randint(0, n - dup, dup)]
    other = np.stack([rs.uniform(-30, -15, 300), rs.uniform(-1, 1, 300) + 2, rs.uniform(-1, 1, 300) - 1, rs.uniform(0, 1, 300)], 1)
    cloud = np.concatenate([other[:150], p, other[150:]]).astype(np.float32)
    return box, cloud


# (pyramid points, duplicated points, device row count or None): the compaction's one-CTA scan (<= 16k rows), its two-launch scan (up to
# 1024 scan tiles) and its three-launch scan (more), with a device row count below the buffer's rows and above them (clamped)
FPS_CASES = [(51, 0, None), (700, 0, None), (4096, 0, None), (4097, 0, None), (20000, 0, None), (300, 120, None), (6000, 3000, None),
             (2100000, 0, None), (6000, 0, 5000), (700, 0, 1 << 30), (20000, 0, 1 << 30)]


@pytest.mark.parametrize("n,dup,rows", FPS_CASES, ids=["%d-%d" % c[:2] + ("" if c[2] is None else "-rows%d" % c[2]) for c in FPS_CASES])
def test_fps_picks_follow_the_contract(n, dup, rows):
    """shared-memory (<= 4096 points) and global-memory pyramids, duplicated points (ties), and stages that read a device row count"""
    from sessd_b200 import ops
    rs = np.random.RandomState(n + dup)
    box, cloud = _pyramid_cloud(rs, n, dup)
    pyr, planes = ops.sada_pyramids(_cu(box))
    pts = _cu(cloud)
    d_n = None if rows is None else _cu(np.array([rows], np.int32))
    N = len(cloud) if rows is None else min(rows, len(cloud))              # the rows the stages read
    bits, counts, _ = ops.sada_membership(pts, planes, [1], n=d_n)
    inside = sada_ref.in_pyramids(cloud, sada_ref.pyramids(box)[0, 1:2])[:, 0]
    assert inside.sum() == n
    inside = inside[:N]
    assert int(counts.item()) == inside.sum()
    out = torch.empty((len(cloud) + 50, 4), dtype=torch.float32, device="cuda")
    _, num = ops.sada_compact(pts, bits, counts, 50, n=d_n, out=out)
    ops.sada_fps(pts, bits, counts, 50, 50, out, num, n=d_n)
    torch.cuda.synchronize()
    mine = cloud[:N][inside]
    want = np.concatenate([cloud[:N][~inside], mine[sada_ref.fps(mine, 50)]])
    assert int(num.item()) == len(want)
    assert np.array_equal(out[:len(want)].cpu().numpy(), want)


def test_shuffle_gathers_each_frame():
    from sessd_b200 import ops
    rs = np.random.RandomState(3)
    sizes = [5, 0, 9, 1]
    pts = rs.uniform(-1, 1, (sum(sizes), 4)).astype(np.float32)
    off = np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
    perm = np.concatenate([rs.permutation(n) for n in sizes]).astype(np.int32)
    out = ops.sada_shuffle(_cu(pts), _cu(off), max(sizes), _cu(perm)).cpu().numpy()
    assert np.array_equal(out, np.concatenate([pts[o:o + n][perm[o:o + n]] for o, n in zip(off, sizes)]))


def test_error_codes():
    import ctypes as C
    from sessd_b200 import ops
    from sessd_b200._lib import lib
    P = C.c_void_p
    pts = torch.zeros((64, 4), dtype=torch.float32, device="cuda")
    bits = torch.zeros((64, 1), dtype=torch.int32, device="cuda")
    counts = torch.full((1,), 60, dtype=torch.int32, device="cuda")
    out = torch.zeros((200, 4), dtype=torch.float32, device="cuda")
    num = torch.zeros((1,), dtype=torch.int32, device="cuda")
    ws = torch.zeros((1 << 16,), dtype=torch.uint8, device="cuda")
    p = lambda t: P(t.data_ptr())
    s = P(torch.cuda.current_stream().cuda_stream)
    # capacity and workspace
    assert lib.sessd_sada_compact(p(pts), 64, None, p(bits), 1, p(counts), -1, p(ws), ws.numel(), p(out), 63, p(num), s) == -2
    assert lib.sessd_sada_compact(p(pts), 64, None, p(bits), 1, p(counts), -1, p(ws), 8, p(out), 64, p(num), s) == -3
    assert lib.sessd_sada_fps(p(pts), 64, None, p(bits), 1, p(counts), 50, 50, p(ws), ws.numel(), p(out), 64 + 49, p(num), s) == -2
    assert lib.sessd_sada_fps(p(pts), 64, None, p(bits), 1, p(counts), 50, 50, p(ws), 16, p(out), 200, p(num), s) == -3
    assert lib.sessd_sada_fps(p(pts), 64, None, p(bits), 1, p(counts), 40, 50, p(ws), ws.numel(), p(out), 200, p(num), s) == -1
    assert lib.sessd_sada_swap(p(pts), 64, None, p(bits), 1, p(counts), p(out), 1, p(num), 10, p(out), 70, p(num), p(num), s) == -2
    assert lib.sessd_sada_membership(p(pts), 64, None, p(out), 1, p(num), 6 * 256 + 1, p(bits), p(counts), s) == -2
    assert lib.sessd_sada_pyramids(p(out), 257, p(out), p(out), s) == -2
    # misaligned rows
    assert lib.sessd_sada_compact(P(pts.data_ptr() + 4), 63, None, p(bits), 1, p(counts), -1, p(ws), ws.numel(), p(out), 64, p(num),
                                  s) == -1
    # the tensor wrappers reject host ids out of range; device ids out of range hold no points and access nothing out of bounds
    box = _cu(np.array([[0, 0, 0, 2, 2, 2, 0]], np.float32))
    _, planes = ops.sada_pyramids(box)
    with pytest.raises(ValueError):
        ops.sada_membership(pts, planes, [6])
    _, c, _ = ops.sada_membership(pts, planes, _cu(np.array([-1, 6, 1 << 30, 0], np.int32)))
    assert c.cpu().tolist()[:3] == [0, 0, 0]
    with pytest.raises(ValueError):
        ops.sada_compact(torch.zeros(64 * 4 + 1, dtype=torch.float32, device="cuda")[1:].view(64, 4), bits, counts)


# ------------------------------------------------------------------------------------------------ the training batch
def _dense_frames(batch, seed):
    """ring-20k frames with 15 cars, each car carrying 400 points on its surface (enough for every pyramid to pass 50)"""
    from sessd_data import synth
    rs = np.random.RandomState(seed)
    clouds, boxes, names = [], [], []
    for b in range(batch):
        bx = synth.ring_boxes(seed + b, 15)
        surf = []
        for x in bx:
            q = rs.uniform(-0.5, 0.5, (400, 3))
            ax = rs.randint(0, 3, 400)
            q[np.arange(400), ax] = np.sign(q[np.arange(400), ax]) * 0.49
            q *= x[3:6]
            c, s = np.cos(x[6]), np.sin(x[6])
            surf.append(np.stack([q[:, 0] * c + q[:, 1] * s + x[0], -q[:, 0] * s + q[:, 1] * c + x[1], q[:, 2] + x[2],
                                  rs.uniform(0, 1, 400)], 1))
        clouds.append(np.concatenate([synth.ring_cloud(seed + b, 20000, 15)] + surf).astype(np.float32))
        boxes.append(bx)
        names.append(np.array(["Car"] * 13 + ["Van", "Pedestrian"]))
    return clouds, boxes, names


def _check_batch(pend, frames, B, cfg):
    """the built batch against oracle frames: student points, twin, both branches' voxels (CPU voxeliser) and targets (assign_v2)"""
    from det3d.core.bbox import box_np_ops
    from det3d.datasets.pipelines import AssignTarget
    from det3d.datasets.pipelines.preprocess import filter_gt_box_outside_range
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    aug, acfg = pend._aug, pend._st["aug"]
    off, roff = aug["frame_off"].cpu().numpy(), aug["frame_off_raw"].cpu().numpy()
    at = AssignTarget(cfg=cfg.train_cfg.assigner)
    ta, ad = at.target_assigners[0], at.anchor_dicts_by_task[0]
    branches = {"student": (pend._vox, pend._asg), "teacher": (pend._vox_raw, pend._asg_raw)}
    vbase = {k: np.concatenate([[0], np.cumsum(v[0].num_voxels[:B].cpu().numpy())]) for k, v in branches.items()}
    for b, (o, names) in enumerate(frames):
        assert np.array_equal(aug["points"][off[b]:off[b + 1]].cpu().numpy(), o["points"]), b
        assert np.array_equal(aug["points_raw"][roff[b]:roff[b + 1]].cpu().numpy(), o["points_raw"]), b
        valid = np.array([n in acfg.class_names for n in names])
        tgt = np.array([n in ("Car", "Van") for n in names])[valid]
        keep = filter_gt_box_outside_range(o["boxes"], acfg.range_bev)
        for name, pts, bx in (("student", o["points"], o["boxes"][keep & tgt]), ("teacher", o["points_raw"], o["boxes_raw"][tgt])):
            buf, abuf = branches[name]
            v, c, n = ocpu.points_to_voxel(pts, synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
            nv, base = int(buf.num_voxels[b].item()), int(vbase[name][b])
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
            assert np.array_equal(abuf.pos_gt_id[b, :npos].cpu().numpy(), ref["positive_gt_id"][0]), (name, b)


RAISED = dict(dropout=0.4, sparsity=(0.5, 50), swap=(0.6, 50))


@pytest.mark.parametrize("probs", ["raised", "car"])
def test_batch_with_sada_against_the_oracle(probs):
    """8 dense ring-20k frames through launch_train_batch(sa_da=...): bit-exact against the chained oracle, the CPU voxeliser and
    assign_v2; the twin and the boxes are SA-DA-free; the RandomState ends where the oracle's does"""
    from sessd_b200 import augment, sada
    from test_augment_oracle import reference_config
    cfg = reference_config()
    B = 8
    clouds, boxes, names = _dense_frames(B, 40)
    sc = sada.SadaConfig(**RAISED) if probs == "raised" else sada.SadaConfig()
    rs, rs_o = np.random.RandomState(21), np.random.RandomState(21)
    pend = augment.launch_train_batch(cfg, clouds, boxes, names, rs, sa_da=sc)
    acfg = pend._st["aug"]
    frames = [(sada_ref.preprocess_frame(clouds[b], boxes[b], names[b], rs_o, acfg, sc), names[b]) for b in range(B)]
    ex = pend.example()
    assert ex["transformation"] == [dict(flipped=o["draws"].flip, noise_rotation=o["draws"].rotation, noise_scale=o["draws"].scale)
                                    for o, _ in frames]
    _check_batch(pend, frames, B, cfg)
    assert np.array_equal(rs.get_state()[1], rs_o.get_state()[1]) and rs.get_state()[2] == rs_o.get_state()[2]
    changed = sum(len(o["points_sada"]) != len(o["points_raw"]) or not np.array_equal(o["points_sada"], o["points_raw"]) for o, _ in frames)
    if probs == "raised":
        assert changed == B


def test_batch_with_sada_and_db_sampler_against_the_oracle(tmp_path):
    """GT-AUG then SA-DA: the pasted frames (read from the device, whose paste is checked in test_gpu_gtaug) replayed through the chained
    oracle in the builder's stream order"""
    from sessd_b200 import augment, sada
    from test_augment_oracle import reference_config
    from test_gpu_gtaug import _few_car_frames, _sampler
    cfg = reference_config()
    B = 8
    clouds, boxes, names = _few_car_frames(B, 300)
    sc = sada.SadaConfig(**RAISED)
    rs = np.random.RandomState(11)
    pend = augment.launch_train_batch(cfg, clouds, boxes, names, rs, db_sampler=_sampler(tmp_path, rs), sa_da=sc)
    acfg = pend._st["aug"]
    rs2 = np.random.RandomState(11)
    frames = []

    def hook(f, d_points, n, bx, nm):
        o = sada_ref.preprocess_frame(d_points.cpu().numpy(), bx, nm, rs2, acfg, sc)
        frames.append((o, nm))
        return o["draws"]

    augment.gtaug_batch(acfg, clouds, boxes, names, rs2, _sampler(tmp_path, rs2), frame_hook=hook)
    pend.example()
    _check_batch(pend, frames, B, cfg)
    assert np.array_equal(rs.get_state()[1], rs2.get_state()[1]) and rs.get_state()[2] == rs2.get_state()[2]


def test_batch_without_sada_is_unchanged():
    """sa_da=None builds exactly the batch the builder built before SA-DA existed: the draws and kernels of draw_augmentation +
    augment_batch, every tensor compared"""
    from sessd_b200 import augment
    from test_augment_oracle import reference_config
    from test_gpu_augment import _train_frames
    cfg = reference_config()
    clouds, boxes, names = _train_frames(4, 500)
    a = augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(2), sa_da=None)
    acfg = augment.AugmentConfig.from_config(cfg)
    draws = augment.draw_augmentation(np.random.RandomState(2), [(len(c), len(b), True) for c, b in zip(clouds, boxes)], acfg)
    aug = augment.augment_batch(acfg, clouds, boxes, names, draws)
    assert torch.equal(a["points"][:, 1:], aug["points"])
    b = augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(2))
    for k, v in a.items():
        w = b[k]
        if isinstance(v, torch.Tensor):
            assert torch.equal(v, w), k
        elif isinstance(v, list) and v and isinstance(v[0], torch.Tensor):
            assert all(torch.equal(x, y) for x, y in zip(v, w)), k
        else:
            assert np.array_equal(np.asarray(v), np.asarray(w)) if not isinstance(v, list) else v == w, k


def test_sada_batch_feeds_the_training_step():
    import copy
    from det3d.models import build_detector
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
    from sessd_b200 import augment, sada, weights
    from test_augment_oracle import reference_config
    cfg = reference_config()
    B = 2
    clouds, boxes, names = _dense_frames(B, 70)
    ex = augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(4), sa_da=sada.SadaConfig(**RAISED))
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
