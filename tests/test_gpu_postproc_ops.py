"""Detection post-processing (csrc/postproc.cu) and the rotated-box kernels (csrc/iou3d.cu, csrc/rotbox.cuh) one operator at a
time, called through sessd_b200.ops on crafted inputs and compared with tests/post_model.py.

Bounds (derived in post_model's docstring): x, y, z, r of every returned box are bit-exact, including the + float32(pi) flip;
w, l, h lie within 5.01 * 2^-24 relative of exp(t) * anchor and scores within 7.01 * 2^-24 relative of sigmoid(c) * q^4
(CUDA expf is within 2 ulp; every other operation rounds once).  Keep sets, counts, anchor indices, labels and padding are
exact: every crafted pair's IoU is at least 1e-3 (relative) away from the threshold, or exactly representable.

Rotated overlaps: at angle 0 no sinf / cosf is involved and the kernels equal the fp32 oracle bit for bit.  Otherwise they are
within the oracle tolerance (2e-5), and against the exact fp64 clip within
    |dev - exact| <= 2^-20 * ((C + R) * (Pa + Pb) + Sa + Sb)
for pairs with no vertex within 1e-3 of the other box's boundary, where C is the largest centre coordinate, R the larger
half-diagonal, P the perimeters and S the areas: each rotated corner carries an error below 2^-21 (C + R) (a few roundings of
coordinates of size C + R, and cosf / sinf within 2 ulp), which moves the clipped area by at most that times the perimeters,
and the shoelace fan adds a few roundings of terms no larger than the areas.
"""
import math

import numpy as np
import pytest
import torch

import post_model as pm

pytestmark = pytest.mark.gpu

def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


@pytest.fixture(scope="module")
def anchors():
    a = pm.kitti_anchors()
    return a, _dev(a)


def _cfg(batch, kw, use_frustum=False):
    from sessd_b200 import ops
    c = dict(pm.POST_DEFAULTS)
    c.update(kw)
    return ops.make_post_cfg(batch=batch, head_stride=24, score_thresh=c["score_thresh"], nms_pre_max=c["nms_pre_max"],
                             nms_post_max=c["nms_post_max"], nms_iou_thresh=c["nms_iou_thresh"], nms_ge=c["nms_ge"],
                             post_range=c["post_range"], direction_offset=c["direction_offset"], use_frustum=use_frustum)


def _poison(buf, packed, meta):
    buf.boxes.fill_(float("nan"))
    buf.scores.fill_(float("nan"))
    for t in (buf.labels, buf.count, buf.aux, buf.sel_anchor, meta):
        t.fill_(-7)
    packed.fill_(float("nan"))


def _alloc(cfg):
    from sessd_b200 import ops
    buf = ops.PostBuffers(cfg, "cuda")
    packed = torch.empty((cfg.batch, cfg.nms_post_max, 8), dtype=torch.float32, device="cuda")
    meta = torch.empty((cfg.batch, 8 + cfg.nms_post_max), dtype=torch.int32, device="cuda")
    return buf, packed, meta


def _run(heads, cfg, dan, planes=None, bufs=None, ws_fill=None, nv=None, status=None, poison=True):
    from sessd_b200 import ops
    buf, packed, meta = bufs or _alloc(cfg)
    if ws_fill is not None:
        buf.ws.fill_(ws_fill)
    if poison:
        _poison(buf, packed, meta)
    head = _dev(np.stack(heads))
    ops.postprocess_packed(head, dan, None if planes is None else _dev(np.stack(planes)), buf, packed, meta,
                           None if nv is None else _dev(np.asarray(nv, np.int32)), None if status is None else _dev(np.asarray([status], np.int32)))
    torch.cuda.synchronize()
    out = dict(boxes=buf.boxes.cpu().numpy(), scores=buf.scores.cpu().numpy(), labels=buf.labels.cpu().numpy(),
               count=buf.count.cpu().numpy(), aux=buf.aux.cpu().numpy(), sel=buf.sel_anchor.cpu().numpy(),
               packed=packed.cpu().numpy(), meta=meta.cpu().numpy())
    return out, (buf, packed, meta)


def _frame_out(o, b):
    return {k: v[b] for k, v in o.items()}


def _check(f, mdl, nv=0, status=0):
    """every output slot of one frame against the model"""
    P = mdl["boxes"].shape[0]
    assert int(f["count"]) == mdl["count"]
    assert np.array_equal(f["aux"], mdl["aux"])
    assert np.array_equal(f["sel"], mdl["sel_anchor"])
    assert np.array_equal(f["labels"], mdl["labels"])
    xb = f["boxes"]
    assert np.array_equal(xb[:, [0, 1, 2, 6]].view(np.uint32), mdl["boxes"][:, [0, 1, 2, 6]].view(np.uint32)), "x, y, z, r not bit-exact"
    c = mdl["count"]
    assert np.array_equal(xb[c:].view(np.uint32), np.zeros((P - c, 7), np.uint32)) and np.all(f["scores"][c:].view(np.uint32) == 0)
    if c:
        rw = np.abs(xb[:c, 3:6] - mdl["whl"][:c]) / (pm.W_BOUND * mdl["whl"][:c])
        rs = np.abs(f["scores"][:c] - mdl["scores"][:c]) / (pm.S_BOUND * mdl["scores"][:c])
        assert rw.max() <= 1 and rs.max() <= 1
    pk = f["packed"]
    assert np.array_equal(pk[:, :7].view(np.uint32), xb.view(np.uint32)) and np.array_equal(pk[:, 7].view(np.uint32), f["scores"].view(np.uint32))
    mt = f["meta"]
    assert mt[:8].tolist() == [c, mdl["aux"][0], mdl["aux"][1], mdl["aux"][2], nv, status, 0, 0]
    assert np.array_equal(mt[8:], mdl["anchor"])


GPU_SWEEP = [dict(kw) for kw in (
    [dict(n=n, K=1000, P=100) for n in (999, 1000, 1001, 1023, 1024, 1025, 2049)] +
    [dict(n=m, K=1000, P=100, pattern=("chain", "cluster")[i % 2]) for i, m in
     enumerate([1, 31, 32, 33, 63, 64, 65, 95, 96, 97, 127, 128, 129])] +
    [dict(n=50, K=1, P=1), dict(n=100, K=33, P=100, pattern="cluster"), dict(n=1500, K=1000, P=100, tie_levels=1),
     dict(n=600, K=500, P=100, tie_levels=40, pattern="cluster"), dict(n=2, K=1000, P=1, pattern="far"),
     dict(n=99, K=1000, P=100, pattern="far"), dict(n=100, K=1000, P=100, pattern="far"), dict(n=101, K=1000, P=100, pattern="far"),
     dict(n=4095, K=5000, P=4096, pattern="far"), dict(n=4096, K=5000, P=4096, pattern="far"),
     dict(n=4097, K=5000, P=4096, pattern="far"), dict(n=3000, K=2048, P=4096, pattern="chain"),
     dict(n=70400, K=16384, P=4096, all_anchors=True), dict(n=70400, K=1000, P=100, all_anchors=True, pattern="cluster")])]


@pytest.mark.parametrize("kw", GPU_SWEEP, ids=lambda kw: "-".join("%s%s" % (k, v) for k, v in kw.items()))
def test_postprocess_matches_model(kw, anchors):
    an, dan = anchors
    h, cfg = pm.frame(**kw)
    mdl = pm.post_frame(h, an, cfg)
    assert pm.robust(mdl["ious"], 0.01) and mdl["clear"]
    o, _ = _run([h], _cfg(1, cfg), dan, nv=[1234], status=5)
    _check(_frame_out(o, 0), mdl, 1234, 5)


def test_exact_ties_across_the_k_cut(anchors):
    """1500 bit-identical scores, K = 1000: the 1000 lowest anchor indices are selected"""
    an, dan = anchors
    h, cfg = pm.frame(n=1500, K=1000, P=1000, pattern="far", tie_levels=1)
    mdl = pm.post_frame(h, an, cfg)
    cand = np.sort(np.nonzero(h[:, 14:16].reshape(-1) > 0)[0])
    assert mdl["aux"][2] == 1000 and np.array_equal(np.sort(mdl["sel_anchor"]), cand[:1000])
    o, _ = _run([h], _cfg(1, cfg), dan)
    _check(_frame_out(o, 0), mdl)


def test_boundaries(anchors):
    """centres on every range bound, a frustum plane sign of exactly 0, r == direction_offset (non-zero) with equal and with
    unequal dir logits, and the P cap filled by out-of-range boxes"""
    an, dan = anchors
    h, cfg, planes, _idx = pm.boundary_frame()
    mdl = pm.post_frame(h, an, cfg, planes)
    o, _ = _run([h], _cfg(1, cfg, use_frustum=True), dan, planes=[planes])
    _check(_frame_out(o, 0), mdl)
    # without the frustum the sign-0 box is returned
    mdl2 = pm.post_frame(h, an, cfg)
    assert mdl2["count"] == mdl["count"] + 1
    o2, _ = _run([h], _cfg(1, cfg), dan)
    _check(_frame_out(o2, 0), mdl2)


def test_batch_frames_are_independent(anchors):
    an, dan = anchors
    kws = [dict(n=0), dict(n=70400, all_anchors=True, pattern="cluster"), dict(n=129, pattern="chain")]
    heads = [pm.frame(K=1000, P=100, seed=s, **kw)[0] for s, kw in enumerate(kws)]
    cfg = dict(nms_pre_max=1000, nms_post_max=100)
    mdls = [pm.post_frame(h, an, cfg) for h in heads]
    o3, _ = _run(heads, _cfg(3, cfg), dan, nv=[7, 8, 9], status=2)
    r3, _ = _run(heads[::-1], _cfg(3, cfg), dan, nv=[9, 8, 7], status=2)
    for b in range(3):
        _check(_frame_out(o3, b), mdls[b], 7 + b, 2)
        o1, _ = _run([heads[b]], _cfg(1, cfg), dan, nv=[7 + b], status=2)
        for k in o1:
            assert _frame_out(o3, b)[k].tobytes() == _frame_out(o1, 0)[k].tobytes(), k
            if k != "meta":
                assert _frame_out(r3, 2 - b)[k].tobytes() == _frame_out(o1, 0)[k].tobytes(), k


def test_stale_or_poisoned_state_does_not_leak(anchors):
    an, dan = anchors
    big, cfgd = pm.frame(n=1000, K=1000, P=100, pattern="chain", seed=3)
    small, _ = pm.frame(n=65, K=1000, P=100, pattern="cluster", seed=4)
    cfg = _cfg(1, cfgd)
    ref_small, _ = _run([small], cfg, dan)
    _check(_frame_out(ref_small, 0), pm.post_frame(small, an, cfgd))
    for fill in (0xFF, 0x00):
        o, _ = _run([small], cfg, dan, ws_fill=fill)
        for k in o:
            assert o[k].tobytes() == ref_small[k].tobytes(), (fill, k)
    bufs = _alloc(cfg)
    _run([big], cfg, dan, bufs=bufs, ws_fill=0xFF)
    o, _ = _run([small], cfg, dan, bufs=bufs)           # stale mask words, keys and boxes of the large frame
    for k in o:
        assert o[k].tobytes() == ref_small[k].tobytes(), k


# ------------------------------------------------------------------------------------------------------------ stand-alone NMS
def _rotate_nms(det, scores, n_dev, max_boxes, pre, post, thr, ge=True):
    from sessd_b200 import ops
    keep, num = ops.rotate_nms(_dev(det), _dev(scores), torch.tensor([n_dev], dtype=torch.int32, device="cuda"), max_boxes, pre, post,
                               thr, ge)
    torch.cuda.synchronize()
    k = int(num.item())
    kk = keep.cpu().numpy()
    assert np.all(kk[k:] == -1)
    return kk[:k]


@pytest.mark.parametrize("pat,m,n_dev,pre,post", [("chain", 1000, 700, 500, 100), ("cluster", 700, 700, 129, 4096),
                                                  ("chain", 129, 129, 1000, 60), ("standup", 200, 150, 150, 150),
                                                  ("cluster", 3000, 2900, 2048, 4096)])
def test_rotate_nms_crafted(pat, m, n_dev, pre, post):
    det, perm = pm.gen_boxes(pat, m, 11)
    scores = ((m - perm) / m).astype(np.float32)
    ref = pm.rotate_nms_model(det[:n_dev], scores[:n_dev], 0.01, True, pre, post)
    assert np.array_equal(_rotate_nms(det, scores, n_dev, m, pre, post, 0.01), ref)


def test_rotate_nms_exact_threshold():
    det, thr = pm.exact_threshold_set()
    sc = np.array([0.9, 0.8, 0.7, 0.6], np.float32)
    assert _rotate_nms(det, sc, 4, 4, 4, 4, float(thr), True).tolist() == [0, 2, 3]
    assert _rotate_nms(det, sc, 4, 4, 4, 4, float(thr), False).tolist() == [0, 1, 3]


def test_rotate_nms_negative_and_signed_zero_scores():
    det = np.array([[10, 0, 1.6, 3.9, 0], [10.5, 0, 1.6, 3.9, 0]], np.float32)      # IoU ~0.52
    assert _rotate_nms(det, np.array([-0.9, -0.1], np.float32), 2, 2, 2, 2, 0.01).tolist() == [1]
    assert _rotate_nms(det, np.array([-0.1, -0.9], np.float32), 2, 2, 2, 2, 0.01).tolist() == [0]
    assert _rotate_nms(det, np.array([-1e-30, 1e-30], np.float32), 2, 2, 2, 2, 0.01).tolist() == [1]
    for s in ([0.0, -0.0], [-0.0, 0.0]):                 # +0 and -0 tie: the lower index wins
        assert _rotate_nms(det, np.array(s, np.float32), 2, 2, 2, 2, 0.01).tolist() == [0]
    for pat, m in (("chain", 1000), ("cluster", 129)):
        dets, perm = pm.gen_boxes(pat, m, 5)
        mixed = ((m // 2 - perm) / m).astype(np.float32)
        mixed[perm == m // 2] = -0.0                        # the one zero score, negative
        for scores in (mixed, (-(perm + 1) / m).astype(np.float32) * np.float32(1e3)):
            ref = pm.rotate_nms_model(dets, scores, 0.01, True, 700, 100)
            assert np.array_equal(_rotate_nms(dets, scores, m, m, 700, 100, 0.01), ref)


def test_public_rotate_nms_mirrors_with_negative_scores():
    from det3d.core.bbox import box_torch_ops
    from det3d.ops.nms import nms_cpu
    det, perm = pm.gen_boxes("chain", 400, 9)
    scores = (-(perm + 1) / 400.0 + 0.3).astype(np.float32)         # distinct, both signs
    ref = pm.rotate_nms_model(det, scores, 0.01, True, 300, 50)
    got = box_torch_ops.rotate_nms(_dev(det), _dev(scores), 300, 50, 0.01)
    assert np.array_equal(got.cpu().numpy(), ref)
    dets = np.concatenate([det, scores[:, None]], 1)
    assert nms_cpu.rotate_nms_cc(dets, 0.01) == pm.rotate_nms_model(det, scores, 0.01).tolist()


# ------------------------------------------------------------------------------------------------------------ nms_sorted
def _axis_ious(bev):
    out = {}
    for i, j in pm.overlapping_pairs(np.asarray(bev, np.float64)[:, :4]):
        a, b = bev[i].astype(np.float64), bev[j].astype(np.float64)
        w = max(min(a[2], b[2]) - max(a[0], b[0]), 0.0)
        h = max(min(a[3], b[3]) - max(a[1], b[1]), 0.0)
        inter = w * h
        out[(i, j)] = inter / max((a[2] - a[0]) * (a[3] - a[1]) + (b[2] - b[0]) * (b[3] - b[1]) - inter, 1e-8)
    return out


@pytest.mark.parametrize("mode", [0, 1, 2])
@pytest.mark.parametrize("n", [1, 63, 64, 65, 127, 128, 129, 700])
def test_nms_sorted_crafted(mode, n):
    from sessd_b200 import ops
    for pat in ("chain", "cluster"):
        det, perm = pm.gen_boxes(pat, n, 21 + n)
        det = det[np.argsort(perm)]
        bev = pm.bev_of(det)
        if mode == 1:
            bx = np.stack([bev[:, 0], bev[:, 1], np.full(n, -1.78, np.float32), bev[:, 2], bev[:, 3], np.full(n, -0.22, np.float32),
                           bev[:, 4]], 1).astype(np.float32)
            ious = {p: pm.iou3d64(bx[p[0]], bx[p[1]]) for p in pm.pair_ious(det)}
        elif mode == 2:
            bx = bev
            ious = _axis_ious(bev)
        else:
            bx = bev
            ious = pm.pair_ious(det)
        thr = 0.25
        assert pm.robust(ious, thr)
        keep, num = ops.nms_sorted(_dev(bx), thr, mode)
        got = keep[: int(num.item())].cpu().numpy()
        assert got.tolist() == pm.greedy(n, ious, thr, ge=False), (pat, mode, n)
    if n == 1:
        det, thr = pm.exact_threshold_set()
        keep, num = ops.nms_sorted(_dev(pm.bev_of(det)), float(thr), 0)
        assert keep[: int(num.item())].cpu().tolist() == [0, 1, 3]          # IoU == thr is not '>'


# ------------------------------------------------------------------------------------------------------------ matrix kernels
def _b5(x, y, w, l, r):
    return [x - w / 2, y - l / 2, x + w / 2, y + l / 2, r]


def _crafted_pairs():
    """(name, a5, b5) in [x1, y1, x2, y2, ang]"""
    P = [("identical", _b5(10, 0, 1.6, 3.9, 0.3), _b5(10, 0, 1.6, 3.9, 0.3)),
         ("square_pi2", _b5(5, 5, 2, 2, 0), _b5(5, 5, 2, 2, np.pi / 2)),
         ("shared_edge", _b5(0, 0, 2, 4, 0), _b5(2, 0, 2, 4, 0)),
         ("corner_touch", _b5(0, 0, 2, 2, 0), _b5(2, 2, 2, 2, 0)),
         ("contain_a_in_b", _b5(3, 3, 1, 1, 0), _b5(3, 3, 4, 4, 0)),
         ("contain_b_in_a", _b5(3, 3, 6, 6, 0.2), _b5(3.5, 2.5, 1, 2, 0.7)),
         ("cross_8", _b5(0, 0, 1, 6, 0), _b5(0, 0, 6, 1, 0)),
         ("cross_8_rot", _b5(20, 3, 1, 6, 0.4), _b5(20, 3, 1, 6, 0.4 + np.pi / 2)),
         ("near_parallel", _b5(10, 10, 1.6, 3.9, 0.1), _b5(10.3, 10.1, 1.6, 3.9, 0.1 + 1e-6)),
         ("thin", _b5(0, 0, 1e-3, 4, 0.3), _b5(0, 0, 2, 2, 0)),
         ("zero_width", _b5(0, 0, 0, 4, 0.3), _b5(0, 0, 2, 2, 0)),
         ("far_x", _b5(70.4, 39.9, 1.6, 3.9, 0.5), _b5(70.0, 39.5, 1.6, 3.9, 1.0)),
         ("far_neg", _b5(0.2, -39.9, 1.6, 3.9, -np.pi), _b5(0.5, -39.0, 1.6, 3.9, np.pi)),
         ("angle_2pi", _b5(30, 0, 1.6, 3.9, 2 * np.pi), _b5(30.4, 0.3, 1.6, 3.9, 0.0)),
         ("angle_100", _b5(30, 10, 1.6, 3.9, 100.0), _b5(30.4, 10.3, 1.6, 3.9, 0.25)),
         ("disjoint", _b5(0, 0, 1, 1, 0), _b5(5, 5, 1, 1, 0.3)),
         ("axis_dyadic", _b5(0, 0, 4, 2, 0), _b5(3, 0.5, 4, 2, 0))]
    rng = np.random.default_rng(5)
    for k in range(40):
        x, y = rng.uniform(0, 70), rng.uniform(-40, 40)
        P.append(("rand%d" % k, _b5(x, y, 1.6, 3.9, rng.uniform(-np.pi, np.pi)),
                  _b5(x + rng.uniform(-2, 2), y + rng.uniform(-2, 2), rng.uniform(1, 2), rng.uniform(3, 5), rng.uniform(-np.pi, np.pi))))
    return [(nm, np.array(a, np.float32), np.array(b, np.float32)) for nm, a, b in P]


def _geom_bound(a5, b5):
    C = max(abs(float(v)) for v in (a5[0], a5[1], a5[2], a5[3], b5[0], b5[1], b5[2], b5[3]))
    dims = [(float(q[2] - q[0]), float(q[3] - q[1])) for q in (a5, b5)]
    R = max(math.hypot(w, l) / 2 for w, l in dims)
    return 2.0 ** -20 * ((C + R) * sum(2 * (w + l) for w, l in dims) + sum(w * l for w, l in dims))


def test_matrix_kernels_crafted_pairs():
    from oracle import cpu as ocpu
    from sessd_b200 import ops
    pairs = _crafted_pairs()
    A = np.stack([a for _n, a, _b in pairs])
    B = np.stack([b for _n, _a, b in pairs])
    n = len(pairs)
    ov = ops.boxes_overlap_bev(_dev(A), _dev(B), torch.zeros((n, n), device="cuda")).cpu().numpy()
    iou = ops.boxes_iou_bev(_dev(A), _dev(B), torch.zeros((n, n), device="cuda")).cpu().numpy()
    al = ops.boxes_aligned_overlap_bev(_dev(A), _dev(B), torch.zeros((n,), device="cuda")).cpu().numpy()
    o_ov, o_iou = ocpu.boxes_overlap_bev(A, B), ocpu.boxes_iou_bev(A, B)
    np.testing.assert_allclose(ov, o_ov, rtol=2e-5, atol=2e-5)
    np.testing.assert_allclose(iou, o_iou, rtol=2e-5, atol=2e-5)
    assert np.array_equal(al.view(np.uint32), np.diag(ov).copy().view(np.uint32))
    ang0 = (A[:, 4] == 0)[:, None] & (B[:, 4] == 0)[None, :]
    assert np.array_equal(ov[ang0].view(np.uint32), o_ov[ang0].view(np.uint32))
    assert np.array_equal(iou[ang0].view(np.uint32), o_iou[ang0].view(np.uint32))
    checked = 0
    for i, (nm, a, b) in enumerate(pairs):
        ex = pm.overlap64(a, b)
        if nm in ("identical", "square_pi2", "contain_a_in_b", "disjoint", "cross_8", "axis_dyadic") or pm.clear_of_boundaries(a, b):
            r = abs(float(ov[i, i]) - ex) / _geom_bound(a, b)
            assert r <= 1, (nm, ov[i, i], ex)
            checked += 1
    assert checked >= 30
    # 3-D: z touching, barely overlapping, contained
    A7 = np.array([[9.2, -1.95, -1.0, 10.8, 1.95, 0.5, 0.3]] * 4, np.float32)
    B7 = np.array([[9.4, -1.8, 0.5, 11.0, 2.1, 2.0, 0.35], [9.4, -1.8, 0.499, 11.0, 2.1, 2.0, 0.35],
                   [9.4, -1.8, -0.5, 11.0, 2.1, 0.2, 0.35], [9.2, -1.95, -1.0, 10.8, 1.95, 0.5, 0.3]], np.float32)
    i3 = ops.boxes_iou3d(_dev(A7), _dev(B7), torch.zeros((4, 4), device="cuda")).cpu().numpy()
    np.testing.assert_allclose(i3, ocpu.boxes_iou_3d(A7, B7), rtol=2e-5, atol=2e-5)
    assert i3[0, 0] == 0.0 and i3[1, 1] > 0
    for k in range(4):
        assert abs(i3[k, k] - pm.iou3d64(A7[k], B7[k])) <= 1e-5


@pytest.mark.parametrize("n,m", [(0, 5), (5, 0), (1, 300), (300, 1), (600, 600)])
def test_matrix_kernel_shapes(n, m):
    from oracle import cpu as ocpu
    from sessd_b200 import ops
    rng = np.random.default_rng(n * 1000 + m)

    def boxes(k):
        xy = rng.uniform([0, -40], [70.4, 40], (k, 2))
        return np.array([_b5(x, y, 1.6, 3.9, r) for (x, y), r in zip(xy, rng.uniform(-np.pi, np.pi, k))], np.float32).reshape(k, 5)
    # dense enough to overlap: half the boxes of b sit near boxes of a
    A, B = boxes(n), boxes(m)
    if n and m:
        k = min(n, m) // 2
        B[:k, :4] = A[:k, :4] + np.float32(0.5)
    for fn, ref in ((ops.boxes_overlap_bev, ocpu.boxes_overlap_bev), (ops.boxes_iou_bev, ocpu.boxes_iou_bev)):
        out = torch.full((max(n, 1), max(m, 1)), -3.0, device="cuda")
        fn(_dev(A), _dev(B), out[:n, :m] if n and m else out)
        got = out.cpu().numpy()
        if n == 0 or m == 0:
            assert np.all(got == -3.0)
        else:
            np.testing.assert_allclose(got, ref(A, B), rtol=2e-5, atol=2e-5)
    if n == 0:
        out = torch.full((3,), -3.0, device="cuda")
        ops.boxes_aligned_overlap_bev(_dev(A), _dev(A), out)
        assert torch.all(out == -3.0)


# ------------------------------------------------------------------------------------------------------------ refused calls
def test_refused_calls_leave_outputs_untouched(anchors):
    from sessd_b200 import ops
    from sessd_b200._lib import SessdError
    an, dan = anchors
    h, _ = pm.frame(n=10)
    head = _dev(h[None])
    for kw, shrink in ((dict(nms_pre_max=16385), False), (dict(nms_post_max=4097), False), (dict(), True), (dict(apl=1), False)):
        cfg = _cfg(1, {k: v for k, v in kw.items() if k != "apl"})
        if "apl" in kw:
            cfg.anchors_per_loc = 1
        buf, packed, meta = _alloc(cfg)
        if shrink:
            buf.ws = buf.ws[:-256]
        _poison(buf, packed, meta)
        with pytest.raises(SessdError):
            ops.postprocess_packed(head, dan, None, buf, packed, meta)
        torch.cuda.synchronize()
        assert torch.all(buf.count == -7) and torch.all(buf.aux == -7) and torch.all(meta == -7) and torch.all(buf.sel_anchor == -7)
        assert torch.all(torch.isnan(buf.boxes)) and torch.all(torch.isnan(packed))
    det = _dev(np.zeros((4, 5), np.float32))
    sc = _dev(np.ones(4, np.float32))
    cnt = torch.tensor([4], dtype=torch.int32, device="cuda")
    for pre, post in ((16385, 10), (10, 4097), (0, 10), (10, 0)):
        with pytest.raises(SessdError):
            ops.rotate_nms(det, sc, cnt, 4, pre, post, 0.01)

