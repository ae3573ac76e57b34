"""KITTI data preparation on the GPU: the kernels with the reference's planes, a KITTI-size batch against the oracle, edge cases, error
codes and kitti_data_prep end to end against the reference's files (tests/golden/kitti_prep_cases.npz)."""
import ctypes as C
import io
import os
import pickle

import numpy as np
import pytest
import torch

import kitti_prep_cases as cases
from oracle import kitti_prep_ref as ref

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "kitti_prep_cases.npz")


@pytest.fixture(scope="module")
def golden():
    return dict(np.load(GOLDEN))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    root = tmp_path_factory.mktemp("kitti")
    cases.write_tree(str(root))
    return root


def _pkl(g, name):
    return pickle.load(io.BytesIO(g["file:" + name].tobytes()))


def _csr(sizes):
    return torch.tensor(np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32), device="cuda")


def _run(frames):
    from sessd_b200 import kitti_prep
    return kitti_prep.run_frames(frames, batch_frames=4)


def test_kernels_with_the_reference_planes(golden, tree):
    from sessd_b200 import kitti_prep
    infos = _pkl(golden, "kitti_infos_train.pkl") + _pkl(golden, "kitti_infos_val.pkl")
    frames = []
    for info in infos:
        idx = info["image"]["image_idx"]
        db = golden["planes_db:%d" % idx] if ("planes_db:%d" % idx) in golden else None
        cen = kitti_prep.db_boxes(info)[0][:, :3] if db is not None else None
        frames.append(kitti_prep.Frame(str(tree / info["point_cloud"]["velodyne_path"]), golden["planes_frustum:training/%d" % idx],
                                       golden["planes_count:%d" % idx], db, cen, tag=info))
    for r in _run(frames):
        info = r.frame.tag
        idx = info["image"]["image_idx"]
        assert r.reduced.tobytes() == golden["file:training/velodyne_reduced/%06d.bin" % idx].tobytes()
        n = len(r.counts)
        assert np.array_equal(r.counts, info["annos"]["num_points_in_gt"][:n])
        names = kitti_prep.db_boxes(info)[1]["name"] if r.frame.db_planes.shape[0] else []
        for i, rows in enumerate(r.db_rows):
            assert rows.tobytes() == golden["file:gt_database/%d_%s_%d.bin" % (idx, names[i], i)].tobytes()


def test_point_on_a_plane_is_outside():
    from sessd_b200 import ops
    x0 = np.float32(1.25)
    pl = np.tile(np.array([0.0, 0.0, 0.0, -1.0]), (1, 6, 1))
    pl[0, 0] = (1.0, 0.0, 0.0, -float(x0))               # x - x0 < 0 inside: x == x0 gives sign 0
    pts = np.array([[x0, 0, 0, 1], [np.nextafter(x0, np.float32(0)), 0, 0, 2], [np.nextafter(x0, np.float32(2)), 0, 0, 3]], np.float32)
    out, off = ops.prep_frustum_compact(torch.from_numpy(pts).cuda(), _csr([3]), torch.from_numpy(pl).cuda())
    assert int(off[1]) == 1 and out[0, 3].item() == 2.0
    c = ops.prep_box_count(torch.from_numpy(pts).cuda(), _csr([3]), torch.from_numpy(pl).cuda(), _csr([1]))
    assert c.tolist() == [1]


def _ring(seed, n):
    rs = np.random.RandomState(seed)
    az, r = rs.uniform(-np.pi, np.pi, n), rs.uniform(1, 80, n)
    return np.stack([r * np.cos(az), r * np.sin(az), rs.uniform(-2.5, 1.0, n), rs.uniform(0, 1, n)], 1).astype(np.float32)


def _boxes(seed, k):
    rs = np.random.RandomState(seed + 1000)
    return np.stack([rs.uniform(-40, 40, k), rs.uniform(-30, 30, k), rs.uniform(-1.5, -0.5, k), rs.uniform(1.5, 2.5, k),
                     rs.uniform(3.5, 6, k), rs.uniform(1.4, 2.0, k), rs.uniform(-3, 3, k)], 1)


def _frustum(k):
    c = np.eye(4)
    p2 = np.array([[721.5, 0, 609.6, 44.9], [0, 721.5, 172.9, 0.2], [0, 0, 1, 0.003], [0, 0, 0, 1]])
    tr = np.array([[0, -1, 0, 0], [0, 0, -1, -0.08], [1, 0, 0, -0.27], [0, 0, 0, 1.0]])
    return ref.frustum_planes(c, tr, p2, cases.SIZES[k % 4])


def test_kitti_size_batch_against_the_oracle():
    """16 ring frames of ~120k points with ~15 boxes each (one empty frame, one without boxes): multi-CTA tiles and the scan paths"""
    from sessd_b200 import kitti_prep
    frames, want = [], []
    for f in range(16):
        pts = np.zeros((0, 4), np.float32) if f == 3 else _ring(f, 120000 + 37 * f)
        boxes = np.zeros((0, 7)) if f == 5 else _boxes(f, 15)
        if f == 7:
            boxes[0, :3] = (500.0, 500.0, 0.0)                 # an object with zero points
        fr = _frustum(f) if f % 2 else kitti_prep.ALL_PASS
        frames.append(kitti_prep.Frame(pts, fr, ref.box_planes(boxes), ref.box_planes(boxes), boxes[:, :3]))
        red = pts[ref.inside(pts, fr[None])[:, 0]] if len(pts) else pts
        m = ref.inside(red, ref.box_planes(boxes))
        rows = []
        for i in range(len(boxes)):
            r = red[m[:, i]].copy()
            r[:, :3] -= boxes[i, :3]
            rows.append(r)
        want.append((red, m.sum(0).astype(np.int32), rows))
    got = kitti_prep.run_frames(frames, batch_frames=16)
    for f, (r, (red, cnt, rows)) in enumerate(zip(got, want)):
        assert r.reduced.tobytes() == red.tobytes(), f
        assert np.array_equal(r.counts, cnt) and np.array_equal(r.db_counts, cnt), f
        for a, b in zip(r.db_rows, rows):
            assert a.tobytes() == b.tobytes(), f
    assert want[7][1][0] == 0 and len(got[3].reduced) == 0 and len(got[5].counts) == 0


def test_error_codes():
    from sessd_b200._lib import lib
    p = lambda t: C.c_void_p(t.data_ptr())
    null, st = C.c_void_p(0), C.c_void_p(torch.cuda.current_stream().cuda_stream)
    pts = torch.zeros((8, 4), dtype=torch.float32, device="cuda")
    off, pl = _csr([8]), torch.zeros((1, 6, 4), dtype=torch.float64, device="cuda")
    out, fo = torch.zeros((8, 4), dtype=torch.float32, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    wsb = int(lib.sessd_prep_frustum_compact_workspace_bytes(8))
    ws = torch.zeros(wsb, dtype=torch.uint8, device="cuda")
    f = lib.sessd_prep_frustum_compact
    assert f(p(pts), p(off), 1, 8, p(pl), p(ws), wsb, p(out), 8, p(fo), st) == 0
    assert f(null, p(off), 1, 8, p(pl), p(ws), wsb, p(out), 8, p(fo), st) == -1
    assert f(p(pts), p(off), 1, -1, p(pl), p(ws), wsb, p(out), 8, p(fo), st) == -1
    assert f(p(pts), p(off), 1, 8, p(pl), p(ws), wsb, p(out), 7, p(fo), st) == -2
    assert f(p(pts), p(off), 1, 8, p(pl), p(ws), wsb - 1, p(out), 8, p(fo), st) == -3
    mis = C.c_void_p(pts.data_ptr() + 4)
    assert f(mis, p(off), 1, 7, p(pl), p(ws), wsb, p(out), 8, p(fo), st) == -1
    cnt, boff = torch.zeros(1, dtype=torch.int32, device="cuda"), _csr([1])
    assert lib.sessd_prep_box_count(p(pts), p(off), 1, 8, p(pl), p(boff), 1, p(cnt), st) == 0
    assert lib.sessd_prep_box_count(p(pts), p(off), 1, 8, null, p(boff), 1, p(cnt), st) == -1
    assert lib.sessd_prep_box_count(p(pts), p(off), 1, 8, p(pl), p(boff), -1, p(cnt), st) == -1
    assert lib.sessd_prep_box_count(mis, p(off), 1, 7, p(pl), p(boff), 1, p(cnt), st) == -1
    gb = int(lib.sessd_prep_box_gather_workspace_bytes(1))
    gws, oo = torch.zeros(gb, dtype=torch.uint8, device="cuda"), torch.zeros(2, dtype=torch.int32, device="cuda")
    cen = torch.zeros((1, 3), dtype=torch.float64, device="cuda")
    g = lib.sessd_prep_box_gather
    assert g(p(pts), p(off), 1, 8, p(pl), p(cen), p(boff), 1, p(cnt), 4, p(gws), gb, p(out), 8, p(oo), st) == 0
    assert g(p(pts), p(off), 1, 8, p(pl), p(cen), p(boff), 1, p(cnt), 9, p(gws), gb, p(out), 8, p(oo), st) == -2
    assert g(p(pts), p(off), 1, 8, p(pl), p(cen), p(boff), 1, p(cnt), 4, p(gws), gb - 1, p(out), 8, p(oo), st) == -3
    assert g(p(pts), p(off), 1, 8, p(pl), null, p(boff), 1, p(cnt), 4, p(gws), gb, p(out), 8, p(oo), st) == -1
    assert g(p(pts), p(off), 1, 8, p(pl), p(cen), p(boff), 1, p(cnt), 4, p(gws), gb, C.c_void_p(out.data_ptr() + 8), 7, p(oo), st) == -1
    torch.cuda.synchronize()


def _same(a, b, path="x"):
    assert type(a) is type(b), path
    if isinstance(a, dict):
        assert list(a) == list(b), path
        for k in a:
            _same(a[k], b[k], path + "." + str(k))
    elif isinstance(a, list):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same(x, y, "%s[%d]" % (path, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and np.array_equal(a, b), path
    else:
        assert a == b, path


def test_kitti_data_prep_end_to_end(golden, tree):
    from sessd_b200.kitti_prep import kitti_data_prep
    kitti_data_prep(str(tree), used_classes=cases.USED_CLASSES, batch_frames=3)
    for k, v in golden.items():
        if not k.startswith("file:"):
            continue
        rel = k[5:]
        data = (tree / rel).read_bytes()
        if rel.endswith(".bin"):
            assert data == v.tobytes(), rel
        else:
            _same(pickle.loads(data), pickle.loads(v.tobytes()), rel)
    # the outputs work with the mirror: the loader takes the reduced file, the sampler loads the database, evaluation runs
    from det3d.datasets.pipelines.loading import LoadPointCloudFromFile
    info = pickle.loads((tree / "kitti_infos_train.pkl").read_bytes())[0]
    res = {"metadata": {"image_prefix": str(tree), "num_point_features": 4}, "lidar": {}}
    res, _ = LoadPointCloudFromFile()(res, info)
    assert res["lidar"]["points"].tobytes() == golden["file:training/velodyne_reduced/000000.bin"].tobytes()
    from det3d.builder import build_dbsampler
    from test_augment_oracle import reference_config
    cfg = reference_config().db_sampler
    cfg.db_info_path = str(tree / "dbinfos_train.pkl")
    sampler = build_dbsampler(cfg, random_state=np.random.RandomState(0))
    assert sampler is not None
    from det3d.datasets.kitti import KittiDataset
    from sessd_b200 import kitti_prep
    ds = KittiDataset(str(tree), str(tree / "kitti_infos_val.pkl"), class_names=["Car"])
    dets = {}
    for info in ds._kitti_infos:
        b = kitti_prep.db_boxes(info)[0]
        dets[str(info["image"]["image_idx"])] = {"box3d_lidar": torch.from_numpy(b.astype(np.float32)).cuda(),
                                                 "scores": torch.ones(len(b), device="cuda"),
                                                 "label_preds": torch.zeros(len(b), dtype=torch.int64, device="cuda"),
                                                 "metadata": {"image_idx": info["image"]["image_idx"]}}
    results, _ = ds.evaluation(dets)
    assert "official_AP_11" in results["results"]
