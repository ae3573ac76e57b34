"""Training and validation from a prepared KITTI tree on the device: loader batches against direct build_train_batch calls and the host
test pipeline, a two-epoch train_detector run with checkpoints and the final validation, and resume against the uninterrupted run.

The tree is written here: 8 train and 4 val frames of a few thousand points with 3-6 cars each, every car carrying 60 points, so the GT
database passes the config's Car=5 minimum and SA-DA selects boxes; kitti_data_prep then writes the infos, reduced clouds and database."""
import os
import re
import shutil

import numpy as np
import pytest
import torch

import kitti_prep_cases as cases
from oracle import kitti_prep_ref as ref
from test_kitti_train import reference_config

pytestmark = pytest.mark.gpu
SEED = 5


def _write_tree(root, n_train=8, n_val=4, points=3000, seed=11):
    rs = np.random.RandomState(seed)
    os.makedirs(os.path.join(root, "ImageSets"), exist_ok=True)
    ids = {"train": list(range(n_train)), "val": list(range(n_train, n_train + n_val)), "test": []}
    for s, v in ids.items():
        with open(os.path.join(root, "ImageSets", s + ".txt"), "w") as f:
            f.write("".join("%06d\n" % i for i in v))
    for d in ("calib", "label_2", "velodyne", "image_2"):
        os.makedirs(os.path.join(root, "training", d), exist_ok=True)
    os.makedirs(os.path.join(root, "testing"), exist_ok=True)
    for k in range(n_train + n_val):
        h, w = cases.SIZES[k % 4]
        with open(os.path.join(root, "training", "image_2", "%06d.png" % k), "wb") as f:
            f.write(cases.png(h, w))
        text, cal = cases.calib(rs, k)
        with open(os.path.join(root, "training", "calib", "%06d.txt" % k), "w") as f:
            f.write(text)
        slots = rs.permutation(8)[:rs.randint(3, 7)]            # cars on a grid inside the camera's view, never overlapping
        objs = [("Car", 0.0, 0, -1.2, (500.0, 150.0, 600.0, 190.0), (1.52, 1.63, 3.9),
                 (-6.0 + 4.0 * (s % 4) + rs.uniform(-0.3, 0.3), 1.7, 14.0 + 9.0 * (s // 4) + rs.uniform(-0.5, 0.5)),
                 float(rs.uniform(-1.0, 1.0))) for s in slots]
        objs.insert(1, ("DontCare", -1, -1, -10, (700.0, 160.0, 720.0, 180.0), (-1, -1, -1), (-1000, -1000, -1000), -10))
        text = cases.label_text(objs)
        with open(os.path.join(root, "training", "label_2", "%06d.txt" % k), "w") as f:
            f.write(text)
        boxes = ref.db_boxes({"annos": cases._anno(text), "calib": cal})[0]
        cases.cloud(rs, points, boxes).tofile(os.path.join(root, "training", "velodyne", "%06d.bin" % k))


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    from sessd_b200.kitti_prep import kitti_data_prep
    root = str(tmp_path_factory.mktemp("kitti_train"))
    _write_tree(root)
    kitti_data_prep(root)
    return root


def _cfg(tree, work_dir, epochs=2):
    cfg = reference_config(tree)
    cfg.data.samples_per_gpu = 2
    cfg.total_epochs = epochs
    cfg.workflow = [("train", epochs), ("val", 1)]
    cfg.work_dir = str(work_dir)
    cfg.load_from = None
    cfg.seed = SEED
    cfg.log_config.interval = 1
    cfg.test_cfg.score_threshold = 0.001          # a briefly trained detector scores low: keep its boxes so the evaluation sees some
    return cfg


def _same(a, b):
    if isinstance(a, torch.Tensor):
        return isinstance(b, torch.Tensor) and a.dtype == b.dtype and a.shape == b.shape and torch.equal(a, b)
    if isinstance(a, np.ndarray):
        return np.array_equal(a, b)
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(_same(a[k], b[k]) for k in a)
    if isinstance(a, (list, tuple)):
        return len(a) == len(b) and all(_same(x, y) for x, y in zip(a, b))
    return a == b


def test_loader_train_batch_equals_direct_build(tree, monkeypatch):
    from det3d.builder import build_dbsampler
    from det3d.datasets import build_dataloader, build_dataset
    from sessd_b200 import augment, sada
    from sessd_b200.kitti_loader import epoch_streams, restart_sampler
    cfg = _cfg(tree, tree)
    ds = build_dataset(cfg.data.train)
    loader = build_dataloader(ds, 2, 2, cfg=cfg, seed=SEED)
    assert len(loader) == 4
    loader.set_epoch(1)
    ex = next(iter(loader))
    order, rs = epoch_streams(SEED, 1, len(ds))
    frames = [ds[int(i)] for i in order[:2]]
    db = build_dbsampler(cfg.db_sampler)
    restart_sampler(db, rs)
    select, pick = db.select, sada.draw_pick
    counted = {"paste": 0, "pick": 0}

    def select_count(*a):
        out = select(*a)
        counted["paste"] += len(out)
        return out

    def pick_count(*a):
        out = pick(*a)
        counted["pick"] += int(np.sum(out[1]))
        return out
    db.select = select_count
    monkeypatch.setattr(sada, "draw_pick", pick_count)
    lidar = [f["lidar"] for f in frames]
    direct = augment.build_train_batch(cfg, [l["points"] for l in lidar], [l["gt_boxes"] for l in lidar],
                                       [l["gt_names"] for l in lidar], rs, db_sampler=db, sa_da=sada.SadaConfig())
    assert counted["paste"] > 0 and counted["pick"] > 0
    assert _same(ex["metadata"], [f["metadata"] for f in frames])
    assert sorted(ex) == sorted(direct)
    for k in direct:
        if k != "metadata":
            assert _same(ex[k], direct[k]), k


def test_loader_val_batch_equals_host_pipeline(tree):
    from det3d.datasets import build_dataloader, build_dataset
    from det3d.datasets.pipelines import AssignTarget, Reformat, Voxelization
    from det3d.models import build_detector
    from det3d.torchie.parallel import collate_kitti
    from det3d.torchie.trainer.trainer_sessd import example_to_device
    from sessd_b200 import weights
    cfg = _cfg(tree, tree)
    ds = build_dataset(cfg.data.val)
    loader = build_dataloader(ds, 2, 2, cfg=cfg, seed=SEED)
    ex = next(iter(loader))
    tf = [Voxelization(cfg=cfg.voxel_generator), AssignTarget(cfg=cfg.train_cfg.assigner), Reformat()]
    frames = []
    for i in range(2):
        res = ds[i]
        for t in tf:
            res, _ = t(res, None)
        frames.append(res)
    host = example_to_device(collate_kitti(frames), "cuda")
    assert ex["coordinates"].shape[0] > 1000 and loader.train is False and ds[0]["mode"] == "val"
    for k in ("voxels", "coordinates", "num_points", "num_voxels"):
        assert torch.equal(ex[k].cpu(), host[k].cpu().to(ex[k].dtype)), k
    assert np.array_equal(ex["shape"], host["shape"])
    assert torch.equal(ex["anchors"][0].cpu(), host["anchors"][0].cpu().float())
    for k in host["calib"]:
        assert torch.equal(ex["calib"][k].cpu(), host["calib"][k].cpu()), k
    assert _same(ex["metadata"], host["metadata"])
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    model.load_state_dict(weights.random_detector_state(0), strict=True)
    model = model.cuda().eval()
    with torch.no_grad():
        a, b = model(ex, return_loss=False), model(host, return_loss=False)
    assert len(a) == 2 and _same(a, b)


def _train(tree, work_dir, resume_from=None):
    from det3d.torchie.apis import train_detector
    from sessd_b200.kitti_train import build_datasets
    from det3d.models import build_detector
    cfg = _cfg(tree, work_dir)
    cfg.resume_from = resume_from
    torch.manual_seed(0)
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    init = {k: v.clone() for k, v in model.state_dict().items()}
    return cfg, init, train_detector(model, build_datasets(cfg), cfg)


def _ckpt(path):
    return torch.load(path, map_location="cpu", weights_only=True)


def test_train_detector_two_epochs_validate_and_resume(tree, tmp_path):
    from det3d.datasets import build_dataloader, build_dataset
    from det3d.models import build_detector
    from det3d.torchie.trainer import load_checkpoint
    from det3d.torchie.trainer.trainer_sessd import compute_on_dataset
    cfg, init, results = _train(tree, tmp_path / "a")
    wd = tmp_path / "a"
    for n in (1, 2):
        for name in ("epoch_%d.pth" % n, "epoch_%d_ema.pth" % n):
            ck = _ckpt(str(wd / name))
            assert set(ck) == {"meta", "state_dict", "optimizer"} and ck["meta"]["epoch"] == n and ck["meta"]["iter"] == 4 * n
            assert set(ck["state_dict"]) == set(init)
    assert os.readlink(str(wd / "latest.pth")) == "epoch_2.pth" and os.readlink(str(wd / "latest_ema.pth")) == "epoch_2_ema.pth"
    final = _ckpt(str(wd / "epoch_2.pth"))
    for k, v in init.items():
        if v.is_floating_point() and not k.endswith(("running_mean", "running_var")):
            assert not torch.equal(final["state_dict"][k], v), k             # every student parameter moved
    log = open(str(next(wd.glob("*.log")))).read()
    lines = [l for l in log.splitlines() if "Epoch [" in l]
    assert len(lines) == 8
    for l in lines:
        vals = [float(x) for x in re.findall(r"[-+]?\d+\.\d+(?:e[-+]?\d+)?|nan|inf", l.split("data_time")[1])]
        assert vals and np.isfinite(vals).all(), l
    assert "Evaluation official_AP_11" in log and "Evaluation official_AP_40" in log
    # the returned results are the evaluation of the final student's predictions
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    load_checkpoint(model, str(wd / "epoch_2.pth"), map_location="cpu")
    val = build_dataset(cfg.data.val)
    preds = compute_on_dataset(model.cuda(), build_dataloader(val, 2, 2, cfg=cfg))
    assert len(preds) == 4 and sum(len(p["scores"]) for p in preds.values()) > 0
    want, _ = val.evaluation(preds)
    assert results["results"] == want["results"] and results["results_2"] == want["results_2"]
    # two identical runs, then a run resumed from the first one's epoch 1: the same student, teacher and optimiser state
    _train(tree, tmp_path / "b")
    os.makedirs(str(tmp_path / "c"))
    for name in ("epoch_1.pth", "epoch_1_ema.pth"):
        shutil.copy(str(wd / name), str(tmp_path / "c" / name))
    _train(tree, tmp_path / "c", resume_from=str(tmp_path / "c" / "epoch_1.pth"))
    for name in ("epoch_2.pth", "epoch_2_ema.pth"):
        a = _ckpt(str(wd / name))
        assert _same(a, _ckpt(str(tmp_path / "b" / name))), "two identical runs differ: " + name
        assert _same(a, _ckpt(str(tmp_path / "c" / name))), "the resumed run differs: " + name
