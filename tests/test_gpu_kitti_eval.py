"""GPU: KITTI evaluation on the device (csrc/kitti_eval.cu) against the reference's golden results and the numpy oracle."""
import json
import os
import pickle

import numpy as np
import pytest
import torch

from kitti_eval_cases import CLASSES, dt_annos_of, load_golden, make_set
from oracle import kitti_eval_ref as ref

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_eval_cases.npz")
AOS_TOL = 1e-6        # alpha comes from atan2 of fp32 operands in fp32, which may differ in its last bit between libraries


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


def _close_detail(a, b, tol, aos_tol=None):
    assert a.keys() == b.keys()
    for cls in a:
        assert a[cls].keys() == b[cls].keys(), cls
        for k in a[cls]:
            t = aos_tol if (aos_tol is not None and k == "aos") else tol
            np.testing.assert_allclose(a[cls][k], b[cls][k], rtol=0, atol=t, err_msg="%s %s" % (cls, k))


def test_device_overlaps_match_reference_and_oracle(golden):
    from sessd_b200 import kitti_eval as ke
    g, infos, _, dt_annos = golden
    gt_annos = [i["annos"] for i in infos]
    frames = ke.Frames(ke.DeviceGT(gt_annos), ke.DeviceDT.from_annos(dt_annos))
    for m, tol in ((0, 1e-12), (1, 2e-5), (2, 2e-5)):
        dev = frames.overlaps(m)
        for f in range(len(infos)):
            want = g["ov%d_%d" % (m, f)]
            assert dev[f].shape == want.shape
            np.testing.assert_allclose(dev[f], want, rtol=tol, atol=tol, err_msg="metric %d frame %d" % (m, f))
            orc = ref.overlaps_frame(m, ref.records(dt_annos[f], "score"), ref.records(gt_annos[f], "truncated"))
            np.testing.assert_allclose(dev[f], orc, rtol=tol, atol=tol)


def test_result_functions_reproduce_reference(golden):
    from det3d.datasets.kitti import get_coco_eval_result, get_official_eval_result, get_official_eval_result_v2
    g, infos, _, dt_annos = golden
    gt_annos = [i["annos"] for i in infos]
    for name, fn in (("official", get_official_eval_result), ("official_v2", get_official_eval_result_v2),
                     ("coco", get_coco_eval_result)):
        r = fn(gt_annos, dt_annos, CLASSES, z_axis=1, z_center=1.0)
        assert r["result"] == str(g[name + "_result"]), name
        _close_detail(r["detail"], json.loads(str(g[name + "_detail"])), 1e-9)


def test_dataset_evaluation_from_device_tensors(golden, tmp_path):
    from det3d.datasets.kitti import KittiDataset
    g, infos, dets, _ = golden
    p = tmp_path / "infos.pkl"
    p.write_bytes(pickle.dumps(infos))
    ds = KittiDataset(str(tmp_path), str(p), class_names=CLASSES)
    det_dev = {k: {"box3d_lidar": torch.from_numpy(v["box3d_lidar"]).cuda(), "scores": torch.from_numpy(v["scores"]).cuda(),
                   "label_preds": torch.from_numpy(v["label_preds"]).cuda(), "metadata": v["metadata"]} for k, v in dets.items()}
    before = {k: v["box3d_lidar"].clone() for k, v in det_dev.items()}
    results, dt_annos = ds.evaluation(det_dev)
    want = json.loads(str(g["dataset_results"]))
    assert results["results"] == want["results"]
    assert results["results_2"] == want["results_2"]
    for part in ("official", "coco"):
        _close_detail(results["detail"]["eval.kitti"][part], want["detail"]["eval.kitti"][part], 1e-9, AOS_TOL)
    for f, a in enumerate(dt_annos):
        assert list(a["name"]) == list(g["dt%d_name" % f])
        assert a["metadata"] == dets[str(infos[f]["image"]["image_idx"])]["metadata"]
        for k in ("bbox", "location", "dimensions", "rotation_y", "score"):
            np.testing.assert_allclose(a[k].reshape(g["dt%d_%s" % (f, k)].shape), g["dt%d_%s" % (f, k)], rtol=1e-12, atol=1e-9)
        np.testing.assert_allclose(a["alpha"], g["dt%d_alpha" % f], rtol=0, atol=AOS_TOL)
    assert all(torch.equal(before[k], v["box3d_lidar"]) for k, v in det_dev.items())      # the caller's tensors are not modified


@pytest.fixture(scope="module")
def random_set():
    infos, dets = make_set(11, 200, max_dets=100, special=False)
    return infos, dets


def _device_eval(infos, dets, classes, mo):
    from sessd_b200 import kitti_eval as ke
    calib = ke.DeviceCalib(infos)
    keys = [str(i["image"]["image_idx"]) for i in infos]
    per = [tuple(torch.from_numpy(dets[k][f]).cuda() for f in ("box3d_lidar", "scores", "label_preds")) for k in keys]
    dt, _ = ke.convert_detections(per, calib, CLASSES)
    frames = ke.Frames(ke.DeviceGT([i["annos"] for i in infos]), dt)
    return ke.evaluate(frames, classes, [0, 1, 2], mo, (0,))


def test_random_sets_match_oracle_and_repeat_bitwise(random_set):
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, _coco_overlaps
    infos, dets = random_set
    assert max(len(d["box3d_lidar"]) for d in dets.values()) > 60
    assert {"Car", "Pedestrian", "Cyclist"} <= {n for i in infos for n in i["annos"]["name"]}
    classes = [0, 1, 10]
    mo = np.concatenate([OFFICIAL_OVERLAPS[:, :, classes], _coco_overlaps(classes)], axis=0)   # what KittiDataset.evaluation runs
    dev = _device_eval(infos, dets, classes, mo)
    orc = ref.evaluate([i["annos"] for i in infos], dt_annos_of(infos, dets), classes, [0, 1, 2], mo)
    for m in range(3):
        np.testing.assert_array_equal(dev[m]["thresholds"], orc[m]["thresholds"], err_msg="metric %d" % m)
        np.testing.assert_array_equal(dev[m]["precision"], orc[m]["precision"], err_msg="metric %d" % m)
        np.testing.assert_allclose(dev[m]["orientation"], orc[m]["orientation"], rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(dev[m]["map"], orc[m]["map"], rtol=1e-12, atol=1e-12)
    again = _device_eval(infos, dets, classes, mo)
    for m in range(3):
        for k in ("thresholds", "precision", "orientation", "map"):
            assert np.array_equal(dev[m][k], again[m][k], equal_nan=True), (m, k)


def test_frames_without_detections_or_ground_truth(golden):
    from det3d.datasets.kitti import get_official_eval_result
    from sessd_b200.kitti_eval import empty_anno
    _, infos, _, dt_annos = golden
    gt_annos = [i["annos"] for i in infos]
    r = get_official_eval_result(gt_annos, [empty_anno() for _ in gt_annos], CLASSES)
    assert all(v == [0.0, 0.0, 0.0] for c in r["detail"].values() for v in c.values())
    no_gt = [{k: (v[:0] if hasattr(v, "__len__") else v) for k, v in a.items()} for a in gt_annos]
    r = get_official_eval_result(no_gt, dt_annos, CLASSES)
    assert all(v == [0.0, 0.0, 0.0] for c in r["detail"].values() for v in c.values())


# ------------------------------------------------------------------------------------------------ crafted decision edges
# kitti_eval_edges.npz: the reference's results on frames that each sit on one decision edge (tests/kitti_eval_edges.py).  Their
# overlaps are exact by construction, so every overlap, threshold and precision must match bit for bit (NaN where the reference
# has NaN); AOS within kitti_eval_edges.aos_bound.
EDGES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_eval_edges.npz")


@pytest.fixture(scope="module")
def edges():
    from kitti_eval_edges import load_edges
    return load_edges(EDGES)


def _same(a, b):
    return np.array_equal(np.asarray(a), np.asarray(b), equal_nan=True)


def test_edge_overlaps_bit_for_bit(edges):
    from sessd_b200 import kitti_eval as ke
    g, names, gts, dts = edges
    frames = ke.Frames(ke.DeviceGT(gts), ke.DeviceDT.from_annos(dts))
    for m in range(3):
        dev = frames.overlaps(m)
        for f, name in enumerate(names):
            assert dev[f].tobytes() == g["ov%d_%d" % (m, f)].tobytes(), (name, m, dev[f], g["ov%d_%d" % (m, f)])


def _edge_set_run(gts, dts, mo):
    from kitti_eval_edges import CODES
    from sessd_b200 import kitti_eval as ke
    frames = ke.Frames(ke.DeviceGT(gts), ke.DeviceDT.from_annos(dts))
    return ke.evaluate(frames, CODES, [0, 1, 2], mo, (0,))


def test_edge_set_evaluation_bit_for_bit_and_repeatable(edges):
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, _coco_overlaps
    from kitti_eval_edges import CODES, aos_bound, map_aos_bound
    g, names, gts, dts = edges
    mo = np.concatenate([OFFICIAL_OVERLAPS[:, :, CODES], _coco_overlaps(CODES)], axis=0)
    dev = _edge_set_run(gts, dts, mo)
    n_tp = sum(len(a["name"]) for a in dts)
    for m in range(3):
        np.testing.assert_array_equal(dev[m]["thresholds"], g["set%d_thresholds" % m], err_msg="metric %d" % m)
        np.testing.assert_array_equal(dev[m]["precision"], g["set%d_precision" % m], err_msg="metric %d" % m)
        np.testing.assert_allclose(dev[m]["orientation"], g["set%d_orientation" % m], rtol=0, atol=aos_bound(n_tp))
        p = g["set%d_precision" % m]
        assert _same(dev[m]["map"][..., 0], ref.map_r11(p)) and _same(dev[m]["map"][..., 1], ref.map_r40(p)), m
        o = g["set%d_orientation" % m]
        np.testing.assert_allclose(dev[m]["map"][..., 2], ref.map_r11(o), rtol=0, atol=map_aos_bound(n_tp))
        np.testing.assert_allclose(dev[m]["map"][..., 3], ref.map_r40(o), rtol=0, atol=map_aos_bound(n_tp))
    again = _edge_set_run(gts, dts, mo)
    for m in range(3):
        for k in ("thresholds", "precision", "orientation", "map"):
            assert _same(dev[m][k], again[m][k]), (m, k)


def test_edge_set_result_functions_reproduce_reference(edges):
    from det3d.datasets.kitti import get_coco_eval_result, get_official_eval_result, get_official_eval_result_v2
    from kitti_eval_edges import CLASSES, map_aos_bound
    g, _, gts, dts = edges
    n_tp = sum(len(a["name"]) for a in dts)
    for name, fn in (("official", get_official_eval_result), ("official_v2", get_official_eval_result_v2),
                     ("coco", get_coco_eval_result)):
        r = fn(gts, dts, CLASSES, z_axis=1, z_center=1.0)
        assert r["result"] == str(g[name + "_result"]), name
        _close_detail(r["detail"], json.loads(str(g[name + "_detail"])), 0, map_aos_bound(n_tp))


def test_each_edge_frame_alone_bit_for_bit(edges):
    from kitti_eval_edges import aos_bound, golden_checks, map_aos_bound
    from sessd_b200 import kitti_eval as ke
    g, names, gts, dts = edges
    nan_seen = False
    for f, name, key in golden_checks(g, names):
        metric, cls, diff = (int(x) for x in g[key + "_config"])
        frames = ke.Frames(ke.DeviceGT([gts[f]]), ke.DeviceDT.from_annos([dts[f]]))
        out = {k: v.cpu().numpy() for k, v in frames.eval_metric(metric, [(cls, diff)], [float(g[key + "_min_overlap"])],
                                                                  metric == 0).items()}
        thr, p, o = g[key + "_thresholds"], g[key + "_precision"], g[key + "_orientation"]
        n_thr = len(g[key + "_stats"])
        assert int(out["num_thresholds"][0]) == n_thr, name
        assert _same(out["thresholds"][0], thr), (name, out["thresholds"][0], thr)
        assert _same(out["precision"][0], p), (name, out["precision"][0], p)
        assert _same(out["map"][0, :2], [ref.map_r11(p), ref.map_r40(p)]), name
        n = len(dts[f]["name"])
        np.testing.assert_allclose(out["aos"][0], o, rtol=0, atol=aos_bound(n), err_msg=name)
        np.testing.assert_allclose(out["map"][0, 2:], [ref.map_r11(o), ref.map_r40(o)], rtol=0, atol=map_aos_bound(n), err_msg=name)
        # a NaN at curve point 0 reaches R11 (points 0, 4, ..., 40) but not R40 (points 1 ... 40)
        nan_seen |= bool(np.isnan(out["precision"][0, 0]) and np.isnan(out["map"][0, [0, 2]]).all())
    assert nan_seen


# ------------------------------------------------------------------------------------------------ capacity
@pytest.fixture(scope="module")
def capacity():
    from kitti_eval_edges import capacity_set
    return capacity_set()


def test_capacity_frames_match_oracle_bit_for_bit(capacity):
    """Frames that keep exactly 0 ... 1024 records (the matching detection last), a 1024-record frame without GT, a 300-GT frame
    and two frames whose conversion drops detections: through the conversion and through exact-count annotations, the whole set
    and each frame alone, bit for bit against the oracle."""
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS
    from kitti_eval_edges import CAPACITY_COUNTS, CODES
    from sessd_b200 import kitti_eval as ke
    infos, dets, kind = capacity
    classes = CODES[:2]
    mo = OFFICIAL_OVERLAPS[:, :, classes]
    calib = ke.DeviceCalib(infos)
    keys = [str(i["image"]["image_idx"]) for i in infos]
    per = [tuple(torch.from_numpy(dets[k][f]).cuda() for f in ("box3d_lidar", "scores", "label_preds")) for k in keys]
    dt, labels = ke.convert_detections(per, calib, CLASSES)
    assert dt.capacity.tolist() == list(CAPACITY_COUNTS) + [1024, 64, 40, 1024]
    orc_dt = dt_annos_of(infos, dets)
    cnt = dt.cnt.cpu().numpy()
    assert cnt.tolist() == [len(a["name"]) for a in orc_dt]
    counted = [f for f, k in enumerate(kind) if k == "count"]
    assert [int(cnt[f]) for f in counted] == list(CAPACITY_COUNTS) + [1024, 64]           # every listed count is evaluated
    assert all(cnt[f] < dt.capacity[f] for f, k in enumerate(kind) if k == "drop")
    for f, a in enumerate(ke.dt_annos_from_device(dt, labels, CLASSES)):
        assert list(a["name"]) == list(orc_dt[f]["name"]), f
        for k in ("bbox", "location", "dimensions", "rotation_y", "score"):
            np.testing.assert_allclose(a[k].reshape(orc_dt[f][k].shape), orc_dt[f][k], rtol=1e-12, atol=1e-9, err_msg="%d %s" % (f, k))
        np.testing.assert_allclose(a["alpha"], orc_dt[f]["alpha"], rtol=0, atol=AOS_TOL)
    gt_annos = [i["annos"] for i in infos]

    def compare(route, dev, orc):
        for m in range(3):
            np.testing.assert_array_equal(dev[m]["thresholds"], orc[m]["thresholds"], err_msg="%s metric %d" % (route, m))
            np.testing.assert_array_equal(dev[m]["precision"], orc[m]["precision"], err_msg="%s metric %d" % (route, m))
            np.testing.assert_allclose(dev[m]["orientation"], orc[m]["orientation"], rtol=1e-12, atol=1e-12)
            np.testing.assert_array_equal(dev[m]["map"][..., :2], orc[m]["map"][..., :2], err_msg="%s metric %d" % (route, m))

    orc = ref.evaluate(gt_annos, orc_dt, classes, [0, 1, 2], mo)
    for route, dev_dt in (("convert", dt), ("annos", ke.DeviceDT.from_annos(orc_dt))):
        compare(route, ke.evaluate(ke.Frames(ke.DeviceGT(gt_annos), dev_dt), classes, [0, 1, 2], mo, (0,)), orc)
    # each frame with one GT alone, Car only: its one TP is the last detection (score 0.99), so the threshold is 0.99 and the
    # precision at it counts the frame's Car fillers as FPs
    car = OFFICIAL_OVERLAPS[:, :, :1]
    for f in range(len(infos)):
        if len(gt_annos[f]["name"]) != 1 or cnt[f] == 0:
            continue
        o = ref.evaluate([gt_annos[f]], [orc_dt[f]], [0], [0, 1, 2], car)
        assert all(o[m]["thresholds"][0, 0, 0, 0] == np.float32(0.99) for m in range(3)), f
        compare("frame %d alone" % f, ke.evaluate(ke.Frames(ke.DeviceGT([gt_annos[f]]), ke.DeviceDT.from_annos([orc_dt[f]])), [0],
                                                 [0, 1, 2], car, (0,)), o)


def test_frames_refuse_1025_detections():
    import ctypes as C
    from sessd_b200 import _lib, kitti_eval as ke
    from sessd_b200.kitti_eval import empty_anno
    gt = ke.DeviceGT([empty_anno()])
    full = ke.DeviceDT.from_annos([{"name": np.array(["Car"] * 1024), "alpha": np.zeros(1024), "bbox": np.tile([0, 0, 50.0, 50], (1024, 1)),
                                    "dimensions": np.ones((1024, 3)), "location": np.ones((1024, 3)), "rotation_y": np.zeros(1024),
                                    "score": np.full(1024, 0.5, np.float32)}])
    frames = ke.Frames(gt, full)                                     # 1024 is the limit: accepted
    assert frames.max_frame_dt == 1024
    # Frames checks the input capacity, not the count left after conversion
    over = ke.DeviceDT(full.off, full.cnt, full.rec, full.code, np.array([1025]))
    with pytest.raises(ValueError):
        ke.Frames(gt, over)
    out = frames.eval_metric(0, [(0, 0)], [0.7], False)
    ws_bytes = _lib.lib.sessd_kitti_eval_workspace_bytes(1, 0, 0, 1, 0)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device="cuda")
    cfg = torch.zeros(1, 2, dtype=torch.int32, device="cuda")
    mo = torch.full((1,), 0.7, dtype=torch.float64, device="cuda")
    p = ke._ptr
    rc = _lib.lib.sessd_kitti_eval(C.byref(frames.struct), 1025, 0, 1, 1.0, 1, p(cfg), p(mo), 0, 0, 0, p(out["thresholds"]),
                                   p(out["num_thresholds"]), p(out["precision"]), p(out["aos"]), p(out["map"]), p(ws),
                                   C.c_size_t(ws_bytes), ke._stream(torch.device("cuda")))
    assert rc == -2                                                  # SESSD_ECAPACITY


def test_conversion_edges_match_reference(edges):
    """The device conversion of the conversion-edge frame (kitti_eval_edges.conversion_set) against the reference's."""
    from kitti_eval_edges import conversion_golden
    from sessd_b200 import kitti_eval as ke
    info, det, want = conversion_golden(edges[0])
    per = [tuple(torch.from_numpy(det[k]).cuda() for k in ("box3d_lidar", "scores", "label_preds"))]
    dt, labels = ke.convert_detections(per, ke.DeviceCalib([info]), CLASSES)
    assert int(dt.cnt[0]) == len(want["name"]) < len(det["box3d_lidar"])
    a = ke.dt_annos_from_device(dt, labels, CLASSES)[0]
    assert list(a["name"]) == list(want["name"])
    for k in ("bbox", "location", "dimensions", "rotation_y", "score"):
        np.testing.assert_allclose(a[k], want[k], rtol=1e-12, atol=1e-9, err_msg=k)          # NaN where the reference has NaN
    np.testing.assert_allclose(a["alpha"], want["alpha"], rtol=0, atol=AOS_TOL)
