"""Shared seeded test inputs (the same generators tests/golden/make_golden.py used)."""
import hashlib

import numpy as np

from sessd_data import synth


def sha(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), np.uint8)


def voxel_cases():
    rng = np.random.default_rng(123)
    cases = []
    cases.append(("uniform2k", synth.uniform_cloud(1, 2000), 5, 20000))
    cases.append(("uniform20k", synth.uniform_cloud(0, 20000), 5, 20000))
    cases.append(("ring20k", synth.ring_cloud(0, 20000), 5, 20000))
    cases.append(("cut300", synth.uniform_cloud(2, 5000), 5, 300))
    ctr = rng.uniform([5, -10, -2], [40, 10, 0], (40, 3))
    p = ctr[rng.integers(0, 40, 6000)] + rng.normal(0, 0.04, (6000, 3))
    cases.append(("clustered", np.concatenate([p, rng.uniform(0, 1, (6000, 1))], 1).astype(np.float32), 5, 20000))
    q = synth.uniform_cloud(3, 3000)
    q[::7, 0] = -0.01
    q[1::11, 1] = 40.0
    q[2::13, 2] = 1.0
    q[3::17, 0] = 70.4
    q[4::19] = np.float32([0.0, -40.0, -3.0, 0.5])
    q[5::23, 0] = np.nextafter(np.float32(70.4), np.float32(0))
    cases.append(("edges", q, 5, 20000))
    cases.append(("clustered_mp3_cut", cases[4][1][:4000].copy(), 3, 500))
    cases.append(("empty", np.zeros((0, 4), np.float32), 5, 20000))
    return cases


def iou_inputs():
    b1, _ = synth.random_boxes(11, 160, spread=0.25)
    b2, _ = synth.random_boxes(12, 120, spread=0.25)
    b2[:10] = b1[:10]
    b2[10:15, :2] = b1[10:15, :2] + np.float32([1.6, 0.0]); b2[10:15, 3:7] = b1[10:15, 3:7]
    b1[20, 3] = 0.0
    b1[21:25, 6] = np.float32([0.0, np.pi / 2, -np.pi / 2, np.pi])
    return b1, b2


def assign_cases():
    """(name, gt_boxes [M,7]) inputs of the IoU target assigner (anchors: the 70 400 KITTI car anchors)."""
    out = []
    g12, _ = synth.random_boxes(21, 12)
    g12[:, 2] = -1.0
    out.append(("m12", g12))
    out.append(("m0", np.zeros((0, 7), np.float32)))
    out.append(("m1", synth.random_boxes(22, 1)[0]))
    out.append(("m40", synth.random_boxes(23, 40)[0]))
    e, _ = synth.random_boxes(24, 10)
    e[0, 0] = -20.0                       # no overlap with any anchor => its column max is 0 => never forces a positive
    e[1, 0] = 95.0
    e[2, 3:5] = np.float32([0.5, 0.6])    # pedestrian-sized: max IoU < 0.45, positives only through the forced rule
    e[3, 3:5] = np.float32([0.6, 1.7])
    e[4] = e[5]                           # duplicate GT: argmax ties resolve to the first
    e[6, :2] = np.float32([10.2, 0.2]); e[6, 3:7] = np.float32([1.6, 3.9, 1.56, 0.0])      # exactly an anchor (IoU 1)
    e[7, :2] = np.float32([10.4, 4.4]); e[7, 3:7] = np.float32([1.6, 3.9, 1.56, 0.0])      # half-way between 2 anchors: tie
    e[8, 6] = np.float32(np.pi / 4)       # on the near-bbox swap boundary
    e[9, 6] = np.float32(-3 * np.pi / 4)
    out.append(("edge", e))
    return out


def kitti_wire_case():
    """A KITTI-style calibration (typical values of the training split), image shape and a 5-object annotation dict (1 DontCare)."""
    P2 = np.array([[7.215377e+02, 0.0, 6.095593e+02, 4.485728e+01], [0.0, 7.215377e+02, 1.728540e+02, 2.163791e-01],
                   [0.0, 0.0, 1.0, 2.745884e-03], [0.0, 0.0, 0.0, 1.0]], np.float32)
    R0 = np.eye(4, dtype=np.float32)
    R0[:3, :3] = np.array([[0.9999239, 0.00983776, -0.00744505], [-0.0098698, 0.9999421, -0.00427846],
                           [0.00740253, 0.00435161, 0.9999631]], np.float32)
    Tr = np.eye(4, dtype=np.float32)
    Tr[:3, :4] = np.array([[7.533745e-03, -9.999714e-01, -6.166020e-04, -4.069766e-03], [1.480249e-02, 7.280733e-04, -9.998902e-01, -7.631618e-02],
                           [9.998621e-01, 7.523790e-03, 1.480755e-02, -2.717806e-01]], np.float32)
    rng = np.random.default_rng(77)
    n = 5
    annos = dict(name=np.array(["Car", "DontCare", "Pedestrian", "Car", "Cyclist"]),
                 location=np.stack([rng.uniform(-10, 10, n), rng.uniform(1.2, 1.9, n), rng.uniform(5, 60, n)], 1),
                 dimensions=np.stack([rng.normal(3.9, 0.3, n), rng.normal(1.56, 0.1, n), rng.normal(1.6, 0.1, n)], 1),
                 rotation_y=rng.uniform(-np.pi, np.pi, n), bbox=rng.uniform(0, 300, (n, 4)), difficulty=np.arange(n, dtype=np.int32))
    info = dict(calib={"P2": P2, "R0_rect": R0, "Tr_velo_to_cam": Tr}, image={"image_shape": np.array([375, 1242], np.int32)}, annos=annos,
                point_cloud={"velodyne_path": "training/velodyne/000007.bin"})
    return info


def head_loss_case():
    """Inputs of the supervised head loss: fused head tensor [2, 35200, 24] (seeded), labels / regression targets of two assigner cases."""
    import torch
    from oracle import anchors as oa
    anc = oa.create_anchors_3d_range().reshape(-1, 7)
    cases = dict(assign_cases())
    labels, targets = [], []
    for name in ("m12", "m40"):
        r = oa.assign_targets(anc, cases[name])
        labels.append(r["labels"])
        targets.append(r["bbox_targets"])
    g = torch.Generator().manual_seed(41)
    head = torch.randn(2, 35200, 24, generator=g) * 0.5
    head[..., 14:16] -= 2.0                       # mostly-negative classification logits, like an early training step
    return head.numpy(), anc, np.stack(labels, 0).astype(np.int32), np.stack(targets, 0).astype(np.float32)


def odiou_pairs():
    """(gboxes, qboxes) [n,7] for the ODIoU loss: predictions = targets + noise at three scales, plus disjoint / contained / identical /
    perpendicular / zero-height-overlap pairs."""
    rng = np.random.default_rng(91)
    g, _ = synth.random_boxes(92, 48)
    q = g.copy()
    for k, s in enumerate((0.02, 0.1, 0.4)):
        sl = slice(16 * k, 16 * (k + 1))
        q[sl] += rng.normal(0, 1, (16, 7)).astype(np.float32) * np.float32([s, s, 0.3 * s, 0.3 * s, 0.5 * s, 0.3 * s, s])
    extra_g = np.float32([[10, 0, -1, 1.6, 3.9, 1.5, 0.3]] * 6)
    extra_q = extra_g.copy()
    extra_q[0, :2] += np.float32([8.0, 6.0])                      # disjoint
    extra_q[1, 3:6] *= np.float32(0.5)                            # contained
    extra_q[2] = extra_g[2]                                       # identical
    extra_q[3, 6] += np.float32(np.pi / 2)                        # perpendicular
    extra_q[4, 2] += np.float32(3.0)                              # no height overlap
    extra_q[5, :2] += np.float32([0.4, -1.1]); extra_q[5, 6] -= np.float32(2.5)
    return np.concatenate([g, extra_g], 0), np.concatenate([q, extra_q], 0)


def checkpoint_model(seed):
    """Small module with the parameter kinds of an SE-SSD checkpoint: a spconv-layout weight [kz,ky,kx,Cin,Cout], BatchNorm1d
    (incl. num_batches_tracked), a Conv2d with bias.  Seeded."""
    import torch
    from torch import nn

    class M(nn.Module):
        def __init__(self):
            super().__init__()
            self.middle_conv = nn.Module()
            self.middle_conv.weight = nn.Parameter(torch.zeros(3, 3, 3, 4, 16))
            self.bn = nn.BatchNorm1d(16, eps=1e-3, momentum=0.01)
            self.conv_box = nn.Conv2d(8, 14, 1)

    g = torch.Generator().manual_seed(seed)
    m = M()
    with torch.no_grad():
        for p in m.parameters():
            p.copy_(torch.randn(p.shape, generator=g))
        m.bn.running_mean.copy_(torch.randn(16, generator=g))
        m.bn.running_var.copy_(torch.rand(16, generator=g) + 0.5)
        m.bn.num_batches_tracked.fill_(seed)
    return m


def consistency_case():
    """Student / teacher head outputs of two frames for the SE-SSD consistency loss: ~60 objects per frame predicted by both models at
    different anchors (teacher in its own augmentation frame: flip / global rotation / scale undone by the loss), plus unmatched and
    out-of-range predictions.  Returns (preds_stu, preds_tea) as dicts of [2, A, k] float32 arrays, anchors [A, 7], the two transformation
    dicts and the number of planted objects."""
    import torch
    from oracle import anchors as oa
    anc = oa.create_anchors_3d_range().reshape(-1, 7).astype(np.float32)
    A = anc.shape[0]
    rng = np.random.default_rng(2024)
    trans = [dict(flipped=False, noise_rotation=0.031, noise_scale=1.02), dict(flipped=True, noise_rotation=-0.044, noise_scale=0.97)]

    def encode(b, a):                                              # second_box_encode (box_np_ops.py), per pair
        diag = np.sqrt(a[:, 3] ** 2 + a[:, 4] ** 2)
        return np.stack([(b[:, 0] - a[:, 0]) / diag, (b[:, 1] - a[:, 1]) / diag, (b[:, 2] - a[:, 2]) / a[:, 5], np.log(b[:, 3] / a[:, 3]),
                         np.log(b[:, 4] / a[:, 4]), np.log(b[:, 5] / a[:, 5]), b[:, 6] - a[:, 6]], 1).astype(np.float32)

    out = []
    for f in range(2):
        n = 60
        boxes = np.stack([rng.uniform(5, 65, n), rng.uniform(-35, 35, n), rng.uniform(-1.6, -0.6, n), rng.uniform(1.5, 1.8, n),
                          rng.uniform(3.6, 4.4, n), rng.uniform(1.4, 1.7, n), rng.uniform(-3.1, 3.1, n)], 1).astype(np.float32)
        t = trans[f]
        # the same objects in the teacher's frame: undo scale, rotation and flip (inverse of mg_head_sessd.py:668-673)
        tb = boxes.copy()
        tb[:, :6] /= np.float32(t["noise_scale"])
        tb[:, 6] -= np.float32(t["noise_rotation"])
        c, s = np.cos(-t["noise_rotation"]), np.sin(-t["noise_rotation"])
        x, y = tb[:, 0].copy(), tb[:, 1].copy()
        tb[:, 0], tb[:, 1] = x * c + y * s, -x * s + y * c
        if t["flipped"]:
            tb[:, 1] = -tb[:, 1]
            tb[:, 6] = np.float32(np.pi) - tb[:, 6]
        preds = []
        for who, bx in (("stu", boxes), ("tea", tb)):
            g = np.random.default_rng(100 * f + (1 if who == "stu" else 2))
            box = (g.normal(0, 0.05, (A, 7))).astype(np.float32)
            cls = np.full((A, 1), -5.0, np.float32) + g.normal(0, 0.2, (A, 1)).astype(np.float32)
            dr = g.normal(0, 1, (A, 2)).astype(np.float32)
            iou = g.uniform(-1, 1, (A, 1)).astype(np.float32)
            idx = g.choice(A, n + 25, replace=False)
            noisy = bx + g.normal(0, 1, bx.shape).astype(np.float32) * np.float32([0.08, 0.08, 0.03, 0.03, 0.06, 0.03, 0.03])
            noisy[:6] += np.float32([1.5, 1.2, 0, 0, 0, 0, 0.6])       # six objects whose two predictions overlap too little to match
            box[idx[:n]] = encode(noisy, anc[idx[:n]])
            cls[idx[:n], 0] = g.uniform(0.0, 3.0, n).astype(np.float32)
            cls[idx[n:n + 15], 0] = g.uniform(-0.7, 2.0, 15).astype(np.float32)   # confident predictions without a partner
            far = idx[n + 15:]
            box[far, 2] = np.float32(9.0)                                # decoded z above the post-processing range
            cls[far, 0] = np.float32(2.0)
            preds.append(dict(box_preds=box, cls_preds=cls, dir_cls_preds=dr, iou_preds=iou))
        out.append(preds)
    stu = {k: np.stack([out[0][0][k], out[1][0][k]], 0) for k in out[0][0]}
    tea = {k: np.stack([out[0][1][k], out[1][1][k]], 0) for k in out[0][1]}
    return stu, tea, anc, trans


def assert_tile_lists_match(rec, nbr, n):
    """sessd_rulebook_tile_lists records (uint32 [tiles, 160 + 128 kvol]) vs a numpy regrouping of the neighbour table nbr [>= n, kvol]
    for its first n rows: per tile of 128 rows the pair count of every offset (zero for offsets >= kvol), the 128-bit row mask of every
    offset and the (input row << 7 | tile row) entries offset by offset in ascending tile row -- bit-exact."""
    kvol = nbr.shape[1]
    assert rec.dtype == np.uint32 and rec.shape[1] == 160 + 128 * kvol
    for t in range(-(-n // 128)):
        rows = nbr[t * 128:min(n, (t + 1) * 128)]
        pos = 160
        for k in range(kvol):
            valid = np.nonzero(rows[:, k] >= 0)[0]
            assert rec[t, k] == len(valid), (t, k)
            mask = np.zeros(4, np.uint64)
            np.add.at(mask, valid >> 5, np.uint64(1) << (valid & 31).astype(np.uint64))      # distinct bits: sum == or
            assert np.array_equal(rec[t, 32 + 4 * k:36 + 4 * k], mask), (t, k)
            want = (rows[valid, k].astype(np.uint32) << np.uint32(7)) | valid.astype(np.uint32)
            assert np.array_equal(rec[t, pos:pos + len(valid)], want), (t, k)
            pos += len(valid)
        assert not rec[t, kvol:32].any()


# ------------------------------------------------------------------------------------------------ assigner edge cases
F32_PI4 = np.float32(np.pi / 4)
# GT yaws and anchor yaws where the near-bbox w / l swap (|limit_period(r, 0.5, pi)| > pi / 4) or limit_period's floor changes
EDGE_YAWS = np.float32([F32_PI4, np.nextafter(F32_PI4, np.float32(1)), np.nextafter(F32_PI4, np.float32(0)), -F32_PI4,
                        np.float32(3 * np.pi / 4), np.float32(-3 * np.pi / 4),
                        np.float32(np.pi / 2), np.nextafter(np.float32(np.pi / 2), np.float32(2)),
                        np.nextafter(np.float32(np.pi / 2), np.float32(0)), np.float32(-np.pi / 2),
                        np.nextafter(np.float32(-np.pi / 2), np.float32(-2)), np.nextafter(np.float32(-np.pi / 2), np.float32(0))])
# one GT per frame on the KITTI grid: (anchor, IoU with that anchor under the reference's rounding, GT).  The GT is centred on another
# anchor (its best), so the forced rule cannot label the listed anchor; found by a search over the GT's x and l with the numpy oracle.
ASSIGN_THRESHOLD_GTS = (
    (17600, np.float32(0.6), [0.5999999642372131, -19.799999237060547, -1.0, 1.600000023841858, 3.9000000953674316, 1.559999942779541, 0.0]),
    (17600, np.nextafter(np.float32(0.6), np.float32(0)),
     [0.6000000238418579, -19.799999237060547, -1.0, 1.600000023841858, 3.9000000953674316, 1.559999942779541, 0.0]),
    (17600, np.nextafter(np.float32(0.6), np.float32(1)),
     [0.5999999046325684, -19.799999237060547, -1.0, 1.600000023841858, 3.9000000953674316, 1.559999942779541, 0.0]),
    (21120, np.float32(0.45), [0.8068957328796387, -15.800000190734863, -1.0, 1.600000023841858, 3.900005340576172, 1.559999942779541, 0.0]),
    (21120, np.nextafter(np.float32(0.45), np.float32(0)),
     [0.8068965673446655, -15.800000190734863, -1.0, 1.600000023841858, 3.9000000953674316, 1.559999942779541, 0.0]),
    (21120, np.nextafter(np.float32(0.45), np.float32(1)),
     [0.8068965077400208, -15.800000190734863, -1.0, 1.600000023841858, 3.9000000953674316, 1.559999942779541, 0.0]),
)
# (anchor i, anchor j, GT index) pairs with bit-identical IoUs across a CTA boundary (line anchors), and (best, one ulp lower) pairs
LINE_TIES = ((255, 256, 0), (511, 512, 1))
LINE_NEAR_TIES = ((255, 256, 0),)


def line_anchors(A, near=False):
    """A custom anchors on a line: x = 0.5 i - 128, y = 0, w 1.5, l 4, h 1.5, yaw 0 -- dyadic, so the IoUs of a GT centred between two
    anchors are bit-identical; the first len(EDGE_YAWS) anchors take the boundary yaws.  near: anchor 256 one ulp wider, so the GT
    between 255|256 has its best anchor in CTA 0 and the next best, one ulp lower, in CTA 1."""
    anc = np.zeros((513, 7), np.float32)
    anc[:, 0] = np.float32(0.5) * np.arange(513, dtype=np.float32) - np.float32(128)
    anc[:, 2] = -1.0
    anc[:, 3:6] = np.float32([1.5, 4.0, 1.5])
    anc[:len(EDGE_YAWS), 6] = EDGE_YAWS
    if near:
        anc[256, 3] = np.nextafter(np.float32(1.5), np.float32(2))
    return np.ascontiguousarray(anc[:A])


def assign_edge_cases():
    """(name, anchors [A, 7], per-frame GT lists [[M_f, 7]], matched, unmatched) of the assigner's edge cases (tests/golden/
    assign_edge_cases.npz; the generator asserts every crafted condition in the reference's own overlap matrix)."""
    from oracle import anchors as oa
    kitti = oa.create_anchors_3d_range().reshape(-1, 7)
    f32 = np.float32
    out = []
    thr = [np.float32([g]) for _, _, g in ASSIGN_THRESHOLD_GTS]
    out.append(("thresholds", kitti, thr, 0.6, 0.45))
    out.append(("thresholds_05_05", kitti, thr, 0.5, 0.5))
    out.append(("thresholds_07_03", kitti, thr, 0.7, 0.3))
    # yaw boundaries on GTs over the KITTI grid, in three rows of four
    yg = np.zeros((len(EDGE_YAWS), 7), f32)
    for i, r in enumerate(EDGE_YAWS):
        yg[i] = [10.0 + 6.0 * (i % 4), -20.0 + 12.0 * (i // 4), -1.0, 1.6, 3.9, 1.56, r]
    out.append(("yaw_boundaries", kitti, [yg], 0.6, 0.45))
    # line anchors: exact ties across CTAs 0|1 and 1|2, GTs over the boundary-yaw anchors, every anchor count
    tie = f32([[-0.25, 0, -1, 1.5, 4.0, 1.5, 0], [127.75, 0, -1, 1.5, 4.0, 1.5, 0]])
    over_yaws = f32([[-128.0 + 0.5 * i + 0.1, 0.3, -1, 1.6, 3.9, 1.5, EDGE_YAWS[(i + 3) % len(EDGE_YAWS)]] for i in range(0, 12, 3)])
    line = line_anchors(513)
    # tie IoUs are 0.714: with matched 0.8 / unmatched 0.75 only the forced rule labels the tied anchors positive
    out.append(("line513", line, [np.concatenate([tie, over_yaws]), f32([[-0.25, 0, -1, 1.5, 4.0, 1.5, 0]])], 0.8, 0.75))
    out.append(("line513_near_ties", line_anchors(513, near=True), [tie[:1]], 0.8, 0.75))
    for A in (1, 255, 256, 257):
        g = f32([[-128.0, 0, -1, 1.5, 4.0, 1.5, 0], [0.5 * (A - 1) - 128.25, 0.2, -1, 1.5, 4.0, 1.5, 0.1],
                 [0.5 * (A // 2) - 128, 0, -1, 1.5, 4.0, 1.5, EDGE_YAWS[4]]])
        out.append(("line%d" % A, line_anchors(A), [g], 0.6, 0.45))
    # KITTI grid, positives only at anchors >= 65 536 (CTAs 256-274): GTs in the rows y >= 35.2
    hi = f32([[5.0 + 9.0 * i, 36.0 + 1.2 * (i % 3), -1.0, 1.6, 3.9, 1.56, 0.4 * i] for i in range(7)])
    out.append(("kitti_high", kitti, [hi], 0.6, 0.45))
    # GT sets: 1024 GTs in one frame (the shared-memory stage's limit), duplicates, a GT without any overlap, a GT equal to an anchor
    rng = np.random.default_rng(41)
    many = np.zeros((1024, 7), f32)
    many[:, 0], many[:, 1] = rng.uniform(0.5, 70, 1024), rng.uniform(-39.5, 39.5, 1024)
    many[:, 2], many[:, 3:6] = -1.0, rng.uniform([0.5, 0.6, 1.4], [2.0, 4.8, 1.8], (1024, 3))
    many[:, 6] = rng.uniform(-np.pi, np.pi, 1024)
    many[1000:1010] = many[500:510]                                       # duplicates: argmax ties resolve to the first
    many[1010] = [-30.0, 0, -1, 1.6, 3.9, 1.56, 0]                       # no overlap with any anchor
    many[1011] = kitti[12345]
    misc = f32([[-30.0, 0, -1, 1.6, 3.9, 1.56, 0], kitti[777], kitti[777], kitti[40001], [30.0, 10.0, -1, 1.6, 3.9, 1.56, 1.0],
                [30.0, 10.0, -1, 1.6, 3.9, 1.56, 1.0]])
    out.append(("gt_sets", kitti, [many, misc], 0.6, 0.45))
    return out
