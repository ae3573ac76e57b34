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
