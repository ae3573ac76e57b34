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


# ------------------------------------------------------------------------------------------------ crafted decision edges
# kitti_eval_edges.npz holds the reference's results on frames that each sit on one decision edge (tests/kitti_eval_edges.py).
# Thresholds and precision must match bit for bit (NaN where the reference has NaN); AOS within kitti_eval_edges.aos_bound, the
# difference between numpy's and the device's fp64 cos.
EDGES = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_eval_edges.npz")


@pytest.fixture(scope="module")
def edges():
    from kitti_eval_edges import load_edges
    return load_edges(EDGES)


def test_edge_min_overlaps_reach_the_evaluation_bit_for_bit(edges):
    """The mirror's OFFICIAL_OVERLAPS and _coco_overlaps give the reference's min overlaps exactly (0.8999999999999999 etc.)."""
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, _coco_overlaps
    from kitti_eval_edges import CODES
    mo = np.concatenate([OFFICIAL_OVERLAPS[:, :, CODES], _coco_overlaps(CODES)], axis=0)
    assert mo.tobytes() == edges[0]["min_overlaps"].tobytes()


def test_oracle_reproduces_edge_golden(edges):
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, format_coco, format_official
    from kitti_eval_edges import CODES, aos_bound, map_aos_bound
    g, names, gts, dts = edges
    mo = g["min_overlaps"]
    res = ref.evaluate(gts, dts, CODES, [0, 1, 2], mo)
    n_tp = sum(len(a["name"]) for a in dts)
    for m in range(3):
        for f in range(len(names)):
            assert res[m]["overlaps"][f].tobytes() == g["ov%d_%d" % (m, f)].tobytes(), (names[f], m)
        np.testing.assert_array_equal(res[m]["thresholds"], g["set%d_thresholds" % m], err_msg="metric %d" % m)
        np.testing.assert_array_equal(res[m]["precision"], g["set%d_precision" % m], err_msg="metric %d" % m)
        np.testing.assert_allclose(res[m]["orientation"], g["set%d_orientation" % m], rtol=0, atol=aos_bound(n_tp))
    off = OFFICIAL_OVERLAPS[:, :, CODES]
    for name, r in (("official", format_official(res, CODES, off, True, 0)), ("official_v2", format_official(res, CODES, off, True, 1)),
                    ("coco", format_coco(res, CODES, True, k0=2))):
        assert r["result"] == str(g[name + "_result"]), name
        _close_detail(r["detail"], json.loads(str(g[name + "_detail"])), map_aos_bound(n_tp))


def _check_frame(mod, g, gts, dts, f, key, min_ov=None):
    """(thresholds, precision, orientation, [(tp, fp, similarity)]) of one golden check, frame f alone, with oracle module mod."""
    metric, cls, diff = (int(x) for x in g[key + "_config"])
    mo = float(g[key + "_min_overlap"]) if min_ov is None else min_ov
    d, gt = mod.records(dts[f], "score"), mod.records(gts[f], "truncated")
    ov = mod.overlaps_frame(metric, d, gt)
    dc = mod.dontcare_boxes(gts[f])
    th, p, o = mod.eval_config([ov], [gt], [d], [gts[f]], [dts[f]], [dc], metric, cls, diff, mo, metric == 0)
    ig, idt = mod.gt_flags(gts[f], cls, diff), mod.dt_flags(dts[f], cls, diff)
    st = [mod.match(ov, gt, d, ig, idt, dc, metric, mo, t, True, True)[:3] for t in th[:int((th != 0).sum())]]
    return th, p, o, st


def _frame_differs(mod, g, gts, dts, f, key, min_ov=None):
    th, p, o, st = _check_frame(mod, g, gts, dts, f, key, min_ov)
    want = [tuple(int(x) for x in s[:2]) for s in g[key + "_stats"]]
    return (not np.array_equal(th, g[key + "_thresholds"], equal_nan=True)
            or not np.array_equal(p, g[key + "_precision"], equal_nan=True)
            or [tuple(int(x) for x in s[:2]) for s in st] != want
            or not np.allclose(o, g[key + "_orientation"], rtol=0, atol=1e-9, equal_nan=True))


def test_oracle_decides_each_edge_frame_as_the_reference(edges):
    from kitti_eval_edges import aos_bound, golden_checks
    g, names, gts, dts = edges
    checks = golden_checks(g, names)
    assert len(checks) >= len(names)
    for f, name, key in checks:
        th, p, o, st = _check_frame(ref, g, gts, dts, f, key)
        np.testing.assert_array_equal(th, g[key + "_thresholds"], err_msg=name)
        np.testing.assert_array_equal(p, g[key + "_precision"], err_msg=name)
        n = len(dts[f]["name"])
        np.testing.assert_allclose(o, g[key + "_orientation"], rtol=0, atol=aos_bound(n), err_msg=name)
        want = g[key + "_stats"]
        assert [(tp, fp) for tp, fp, _ in st] == [(int(a), int(b)) for a, b, _ in want], name
        sims = [s if s != -1 else -1.0 for _, _, s in st]
        np.testing.assert_allclose(sims, want[:, 2], rtol=0, atol=len(gts[f]["name"]) * 2.0 ** -50, err_msg=name)
    assert any(np.isnan(g[k + "_precision"]).any() for _, _, k in checks)            # the NaN case is present


# Planted mistakes: each is applied to a fresh copy of the oracle's source and must change the result of at least one edge
# frame.  Equivalent mutant, not listed: dropping `taken_ignored` from the displacement test.  A short detection is only taken
# while nothing is held, and it leaves the best overlap at 0, so any normal detection above the min overlap displaces it anyway.
MUTANTS = {
    "ge_at_min_overlap": [("(ov[:, i] > min_ov)", "(ov[:, i] >= min_ov)")],
    "ge_at_dontcare_min_overlap": [("odc[j, c] > min_ov", "odc[j, c] >= min_ov")],
    "no_fp32_storage": [(".astype(f4).astype(f8).reshape(nd, ng)", ".reshape(nd, ng)"), ("out = rinc.copy()", "out = rinc.astype(f8)")],
    "lt_on_gt_height": [("h <= MIN_HEIGHT[diff]", "h < MIN_HEIGHT[diff]")],
    "ge_on_truncation": [('anno["truncated"][i] > MAX_TRUNCATION[diff]', 'anno["truncated"][i] >= MAX_TRUNCATION[diff]')],
    "le_on_det_height": [("]) < MIN_HEIGHT[diff]:", "]) <= MIN_HEIGHT[diff]:")],
    "last_index_wins_ties": [("dt[j, 12] > best_key", "dt[j, 12] >= best_key"), ("ov[j, i] > best_key)", "ov[j, i] >= best_key)")],
    "short_not_displaced": [("(best < 0 or taken_ignored or ov[j, i] > best_key)",
                             "(best < 0 or (not taken_ignored and ov[j, i] > best_key))")],
    "dontcare_absorbs_twice": [("if free[j] and not assigned[j] and odc[j, c] > min_ov:", "if free[j] and odc[j, c] > min_ov:")],
    "dontcare_absorbs_assigned": [("odc = box2d_overlap(dt[:, :4], dc, 0)", "odc, hit = box2d_overlap(dt[:, :4], dc, 0), set()"),
                                  ("if free[j] and not assigned[j] and odc[j, c] > min_ov:\n                    assigned[j] = True",
                                   "if idt[j] == 0 and not below[j] and j not in hit and odc[j, c] > min_ov:\n"
                                   "                    hit.add(j)")],
    "nan_dropped_from_suffix_max": [("prec[t] = np.max(prec[t:])", "prec[t] = np.fmax.reduce(prec[t:])")],
}


def _mutant(patches):
    import inspect
    import types
    src = inspect.getsource(ref)
    for old, new in patches:
        assert src.count(old) == 1, old
        src = src.replace(old, new)
    mod = types.ModuleType("kitti_eval_ref_mutant")
    exec(compile(src, "kitti_eval_ref_mutant", "exec"), mod.__dict__)
    return mod


def test_unmutated_oracle_differs_on_no_edge_frame(edges):
    """The control of the planted mistakes below: with no patch, no frame may count as changed."""
    from kitti_eval_edges import golden_checks
    g, names, gts, dts = edges
    mod = _mutant([])
    with np.errstate(divide="ignore", invalid="ignore"):
        assert [nm for f, nm, key in golden_checks(g, names) if _frame_differs(mod, g, gts, dts, f, key)] == []
        assert [nm for f, nm, key in golden_checks(g, names) if _frame_differs(ref, g, gts, dts, f, key)] == []


@pytest.mark.parametrize("name", sorted(MUTANTS))
def test_planted_mistake_fails_an_edge_frame(edges, name):
    from kitti_eval_edges import golden_checks
    g, names, gts, dts = edges
    mod = _mutant(MUTANTS[name])
    with np.errstate(divide="ignore", invalid="ignore"):
        hit = [nm for f, nm, key in golden_checks(g, names) if _frame_differs(mod, g, gts, dts, f, key)]
    assert hit, name


def test_planted_coco_grid_as_decimal_steps_fails_an_edge_frame(edges):
    """COCO min overlaps computed as first + 0.05 k instead of np.linspace: 0.9, 0.45 and 0.65 land on their decimals."""
    from kitti_eval_edges import COCO_CAR, COCO_PED, golden_checks
    g, names, gts, dts = edges
    hit = []
    for f, nm, key in golden_checks(g, names):
        mo, cls = float(g[key + "_min_overlap"]), int(g[key + "_config"][1])
        grid, first = (COCO_CAR, 0.5) if cls == 0 else (COCO_PED, 0.25)
        if mo in grid.tolist():
            if _frame_differs(ref, g, gts, dts, f, key, first + 0.05 * grid.tolist().index(mo)):
                hit.append(nm)
    assert {"2d_iou_0.9_car_coco_match", "2d_iou_0.45_ped_coco_match"} <= set(hit), hit


def test_oracle_conversion_edges_match_reference(edges):
    """u0 == W and u1 == 0 kept, a corner on the camera plane (NaN bbox, inf clipped), boxes behind the camera, ry at fp32 +-pi
    and +-3 pi: the oracle's conversion against the reference's."""
    from kitti_eval_edges import conversion_golden
    info, det, want = conversion_golden(edges[0])
    with np.errstate(divide="ignore", invalid="ignore"):
        a = ref.convert_frame(det["box3d_lidar"], det["scores"], det["label_preds"], info, CLASSES)
    assert list(a["name"]) == list(want["name"]) and len(want["name"]) < len(det["box3d_lidar"])
    assert np.isnan(want["bbox"]).any()
    for k in ("bbox", "location", "dimensions", "rotation_y", "score"):
        np.testing.assert_allclose(a[k], want[k], rtol=1e-12, atol=1e-9, err_msg=k)
    np.testing.assert_allclose(a["alpha"], want["alpha"], rtol=0, atol=1e-6)
