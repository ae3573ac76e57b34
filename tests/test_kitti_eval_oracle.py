"""CPU: the numpy KITTI evaluation (oracle/kitti_eval_ref.py) against the reference's own results on the golden cases, and the
host packing / class-code mapping of sessd_b200.kitti_eval."""
import json
import os

import numpy as np
import pytest

from kitti_eval_cases import CLASSES, load_golden, make_set
from oracle import kitti_eval_ref as ref

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_eval_cases.npz")


@pytest.fixture(scope="module")
def golden():
    return load_golden(GOLDEN)


@pytest.fixture(scope="module")
def oracle_results(golden):
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, _coco_overlaps
    g, infos, _dets, dt_annos = golden
    classes = [0, 1, 10]
    mo = np.concatenate([OFFICIAL_OVERLAPS[:, :, classes], _coco_overlaps(classes)], axis=0)
    return ref.evaluate([i["annos"] for i in infos], dt_annos, classes, [0, 1, 2], mo), classes


def _close_detail(a, b, tol):
    assert a.keys() == b.keys()
    for cls in a:
        assert a[cls].keys() == b[cls].keys(), cls
        for k in a[cls]:
            np.testing.assert_allclose(a[cls][k], b[cls][k], rtol=0, atol=tol, err_msg="%s %s" % (cls, k))


def test_oracle_conversion_matches_reference(golden):
    g, infos, dets, _ = golden
    for f, info in enumerate(infos):
        d = dets[str(info["image"]["image_idx"])]
        a = ref.convert_frame(d["box3d_lidar"], d["scores"], d["label_preds"], info, CLASSES)
        assert list(a["name"]) == list(g["dt%d_name" % f]), f
        for k in ("bbox", "location", "dimensions", "rotation_y", "score"):
            np.testing.assert_allclose(a[k].reshape(g["dt%d_%s" % (f, k)].shape), g["dt%d_%s" % (f, k)], rtol=1e-12, atol=1e-9)
        np.testing.assert_allclose(a["alpha"], g["dt%d_alpha" % f], rtol=0, atol=1e-6)          # atan2 of fp32 operands, in fp32


def test_oracle_overlaps_match_reference(golden):
    g, infos, _, dt_annos = golden
    for f, info in enumerate(infos):
        d, gt = ref.records(dt_annos[f], "score"), ref.records(info["annos"], "truncated")
        for m, tol in ((0, 1e-12), (1, 2e-5), (2, 2e-5)):
            want = g["ov%d_%d" % (m, f)]
            got = ref.overlaps_frame(m, d, gt)
            assert got.shape == want.shape
            np.testing.assert_allclose(got, want, rtol=tol, atol=tol, err_msg="metric %d frame %d" % (m, f))


def test_oracle_reproduces_reference_results(golden, oracle_results):
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, format_coco, format_official
    g = golden[0]
    ret, classes = oracle_results
    off = OFFICIAL_OVERLAPS[:, :, classes]
    for name, r in (("official", format_official(ret, classes, off, True, 0)), ("official_v2", format_official(ret, classes, off, True, 1)),
                    ("coco", format_coco(ret, classes, True, k0=2))):
        assert r["result"] == str(g[name + "_result"]), name
        _close_detail(r["detail"], json.loads(str(g[name + "_detail"])), 1e-9)


def test_golden_cases_cover_the_edge_cases(golden, oracle_results):
    g, infos, dets, dt_annos = golden
    names = [n for i in infos for n in i["annos"]["name"]]
    assert {"DontCare", "Van", "Person_sitting"} <= set(names)
    assert any(len(i["annos"]["name"]) == 0 for i in infos)
    assert any(len(a["name"]) == 0 for a in dt_annos)
    assert any(set(i["annos"]["name"]) == {"DontCare"} for i in infos)
    assert "Cyclist" not in names                                                  # a class with zero valid ground truth
    ret, _ = oracle_results
    assert (ret[0]["thresholds"][2] == 0).all()
    ov2 = [g["ov1_%d" % f] for f in range(len(infos))]
    assert max(o.max() for o in ov2 if o.size) > 0.999                             # identical boxes
    n_in = sum(len(d["box3d_lidar"]) for d in dets.values())
    assert n_in > sum(len(a["name"]) for a in dt_annos)                            # some detections fall outside the image
    assert _edge_sharing_pairs(g, infos, dt_annos)


def _edge_sharing_pairs(g, infos, dt_annos):
    """(frame, detection, GT) of axis-aligned camera-BEV pairs that share an edge: the gap along x is below 1e-5, the z ranges
    overlap, the clip keeps vertices, and the reference's BEV overlap is 0."""
    out = []
    for f, info in enumerate(infos):
        d, gt = ref.records(dt_annos[f], "score"), ref.records(info["annos"], "truncated")
        for j in range(len(d)):
            for i in range(len(gt)):
                bd, bg = ref._bev(d[j:j + 1], 1), ref._bev(gt[i:i + 1], 1)
                if bd[0, 4] != 0 or bg[0, 4] != 0:
                    continue
                gap = abs(abs(bd[0, 0] - bg[0, 0]) - (bd[0, 2] + bg[0, 2]) / 2)
                zo = min(bd[0, 1] + bd[0, 3] / 2, bg[0, 1] + bg[0, 3] / 2) - max(bd[0, 1] - bd[0, 3] / 2, bg[0, 1] - bg[0, 3] / 2)
                if gap < 1e-5 and zo > 0:
                    _, n = ref.rbox_inter(bg, bd, with_count=True)
                    if n[0] > 0 and g["ov1_%d" % f][j, i] == 0:
                        out.append((f, j, i))
    return out


def test_class_codes_and_host_packing(golden):
    from sessd_b200 import kitti_eval as ke
    assert [ke.class_code(n) for n in ("Car", "PEDESTRIAN", "Cyclist", "Van", "Person_sitting", "DontCare", "Tram")] == \
        [0, 1, 10, ke.VAN, ke.PERSON_SITTING, -1, -1]
    _, infos, _, dt_annos = golden
    gt = [i["annos"] for i in infos]
    h = ke.pack_gt(gt)
    assert h["gt_off"][-1] == sum(len(a["name"]) for a in gt) == len(h["gt"]) == len(h["gt_code"])
    assert h["dc_off"][-1] == sum(int((a["name"] == "DontCare").sum()) for a in gt)
    f = int(np.argmax(np.diff(h["gt_off"])))
    r = h["gt"][h["gt_off"][f]:h["gt_off"][f + 1]]
    np.testing.assert_array_equal(r[:, 0:4], gt[f]["bbox"])
    np.testing.assert_array_equal(r[:, 8:11], gt[f]["dimensions"])
    np.testing.assert_array_equal(r[:, 12], gt[f]["truncated"])
    d = ke.pack_dt(dt_annos)
    assert d["dt_off"][-1] == len(d["dt"]) == sum(len(a["name"]) for a in dt_annos)
    np.testing.assert_array_equal(d["dt"][:, 12], np.concatenate([a["score"] for a in dt_annos]))


def test_eval_entry_points_reject_bad_arguments():
    import ctypes as C
    from sessd_b200 import _lib
    fr = _lib.KittiFrames()
    assert _lib.lib.sessd_kitti_overlaps(C.byref(fr), 0, 1, 1.0, None, None) == -1
    assert _lib.lib.sessd_kitti_eval_workspace_bytes(0, 0, 0, 1, 0) == 0
    assert _lib.lib.sessd_kitti_convert_workspace_bytes(0) == 0


def test_dataset_mirror_surface(tmp_path):
    import pickle
    from det3d.datasets import DATASETS
    from det3d.datasets.kitti.kitti_common import empty_result_anno, get_start_result_anno
    infos, _ = make_set(1, 2)
    p = tmp_path / "infos.pkl"
    p.write_bytes(pickle.dumps(infos))
    ds = DATASETS.get("KittiDataset")(str(tmp_path), str(p), class_names=CLASSES)
    assert len(ds) == 2 and list(ds.ground_truth_annotations[1]["name"]) == list(infos[1]["annos"]["name"])
    with pytest.raises(NotImplementedError):
        ds[0]
    assert get_start_result_anno()["bbox"] == [] and empty_result_anno()["bbox"].shape == (0, 4)
