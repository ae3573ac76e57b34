"""Frame loading, dataset building and the training loop on the CPU: KittiDataset on the crafted KITTI tree with the reference-written
info files (tests/golden/kitti_prep_cases.npz), build_dataset from the reference config, and the Trainer's schedule, EMA steps,
workflow, checkpoints and resume with a stand-in model, optimiser and loader."""
import json
import os
import pickle
from collections import OrderedDict

import numpy as np
import pytest
import torch

import kitti_prep_cases as cases

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "kitti_prep_cases.npz")
REF_CFG = os.path.join(ROOT, "tests", "golden", "reference_config.json")


def reference_config(data_root):
    """the reference config (its values as Config.fromfile reads them) with the data root overridden"""
    from det3d.torchie import Config
    from sessd_b200.kitti_train import override_data_root
    d = json.load(open(REF_CFG))
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    d["model"]["neck"]["logger"] = ours.model.neck.logger
    d["model"]["bbox_head"]["box_coder"] = ours.model.bbox_head.box_coder
    return override_data_root(Config(d), data_root)


@pytest.fixture(scope="module")
def tree(tmp_path_factory):
    """the crafted tree plus the reference's info files and reduced clouds"""
    root = tmp_path_factory.mktemp("kitti")
    cases.write_tree(str(root))
    g = np.load(GOLDEN)
    for key in g.files:
        if key.startswith("file:") and not key.startswith("file:gt_database"):
            path = os.path.join(str(root), key[5:])
            os.makedirs(os.path.dirname(path), exist_ok=True)
            g[key].tofile(path)
    return str(root)


def _dataset(tree, split="train", **kw):
    from det3d.datasets import KittiDataset
    cfg = reference_config(tree)
    return KittiDataset(cfg.data[split].root_path, cfg.data[split].info_path, pipeline=cfg.data[split].pipeline,
                        class_names=cfg.class_names, **kw)


def test_getitem_runs_the_two_loaders_and_drops_dontcare(tree):
    from det3d.core.bbox import box_np_ops
    from det3d.datasets.pipelines import LoadPointCloudAnnotations, LoadPointCloudFromFile
    ds = _dataset(tree)
    infos = pickle.load(open(os.path.join(tree, "kitti_infos_train.pkl"), "rb"))
    assert len(ds) == len(infos) == 5
    saw_dontcare = False
    for i, info in enumerate(infos):
        res = ds[i]
        assert list(res.keys()) == ["type", "lidar", "metadata", "calib", "cam", "mode", "labeled"]
        assert res["mode"] == "train" and res["labeled"] is True and res["type"] == "KittiDataset"
        idx = info["image"]["image_idx"]
        meta = res["metadata"]
        assert list(meta) == ["image_prefix", "num_point_features", "image_idx", "image_shape", "token"]
        assert (meta["image_prefix"], meta["num_point_features"], meta["image_idx"], meta["token"]) == (tree, 4, idx, str(idx))
        assert np.array_equal(meta["image_shape"], info["image"]["image_shape"])
        red = np.fromfile(os.path.join(tree, "training", "velodyne_reduced", "%06d.bin" % idx), np.float32).reshape(-1, 4)
        assert np.array_equal(res["lidar"]["points"], red)                       # the reduced cloud, as the loader prefers it
        want = {"type": "KittiDataset", "lidar": {}, "metadata": dict(res["metadata"])}
        want, _ = LoadPointCloudFromFile()(want, info)
        want, _ = LoadPointCloudAnnotations(with_bbox=True)(want, info)
        for k in ("rect", "Trv2c", "P2", "frustum"):
            assert np.array_equal(res["calib"][k], want["calib"][k]), k
        c = info["calib"]
        assert np.array_equal(res["calib"]["frustum"], box_np_ops.get_valid_frustum(c["R0_rect"], c["Tr_velo_to_cam"], c["P2"],
                                                                                   info["image"]["image_shape"]))
        names = np.asarray(info["annos"]["name"])
        keep = names != "DontCare"
        saw_dontcare |= not keep.all()
        assert list(res["lidar"]["gt_names"]) == list(names[keep])
        assert np.array_equal(res["lidar"]["gt_boxes"], want["lidar"]["annotations"]["boxes"])
        assert res["lidar"]["gt_boxes"].shape == (int(keep.sum()), 7)
    assert saw_dontcare


def test_test_mode_and_by_index(tree):
    assert _dataset(tree, "val")[0]["mode"] == "val"                       # the val pipeline's Preprocess sets the mode
    ds = _dataset(tree, "val", test_mode=True)
    res = ds.get_sensor_data(5, by_index=True)
    assert res["mode"] == "val" and res["metadata"]["token"] == "5" and "gt_boxes" not in res["lidar"]
    assert res["lidar"]["annotations"] is not None                        # evaluation-side annotations are still loaded
    with pytest.raises(NotImplementedError):
        ds.get_sensor_data(0, with_gp=True)


def test_unknown_pipeline_stage_raises(tree):
    from det3d.datasets import KittiDataset
    cfg = reference_config(tree)
    pipeline = list(cfg.data.train.pipeline) + [dict(type="ObjectSample")]
    with pytest.raises(ValueError, match="ObjectSample"):
        KittiDataset(cfg.data.train.root_path, cfg.data.train.info_path, pipeline=pipeline, class_names=["Car"])


def test_build_dataset_from_the_reference_config(tree):
    from det3d.datasets import KittiDataset, build_dataset
    cfg = reference_config(tree)
    assert cfg.db_sampler.db_info_path == os.path.join(tree, "dbinfos_train.pkl")
    assert cfg.train_preprocessor.db_sampler.db_info_path == os.path.join(tree, "dbinfos_train.pkl")
    train, val = build_dataset(cfg.data.train), build_dataset(cfg.data.val)
    assert isinstance(train, KittiDataset) and len(train) == 5 and len(val) == 2
    assert train.test_mode is False and set(train.device_stages) == {"Preprocess", "Voxelization", "AssignTarget", "Reformat"}
    unl = build_dataset(cfg.data.train_unlabel_val)
    assert unl.labeled is False and unl[0]["labeled"] is False and "gt_boxes" not in unl[0]["lidar"]


# ------------------------------------------------------------------------------------------------ the loop with stand-ins
class StandIn(torch.nn.Module):
    def __init__(self, seed):
        super().__init__()
        torch.manual_seed(seed)
        self.lin = torch.nn.Linear(3, 2)

    def forward(self, example, return_loss=True, **kw):
        if not return_loss:
            return [{"box3d_lidar": torch.zeros(0, 7), "scores": torch.zeros(0), "label_preds": torch.zeros(0, dtype=torch.long),
                     "metadata": m} for m in example["metadata"]]
        return self.lin(example["x"]).square().sum()


class StandInOpt:
    """the optimiser surface the loop and OneCycle use: lr / mom attributes, zero_grad, step, state_dict"""

    def __init__(self, params):
        self.inner = torch.optim.SGD(params, lr=0.01)
        self.lr = self.mom = None
        self.steps = []
        self.loaded = None

    def zero_grad(self):
        self.inner.zero_grad()

    def step(self):
        self.steps.append((self.lr, self.mom))
        self.inner.step()

    def state_dict(self):
        return {"steps": len(self.steps)}

    def load_state_dict(self, sd):
        self.loaded = sd


class Loader:
    def __init__(self, n_batches, dataset, log, name):
        self.n, self.dataset, self.log, self.name = n_batches, dataset, log, name

    def __len__(self):
        return self.n

    def set_epoch(self, e):
        self.log.append((self.name, "set_epoch", e))

    def __iter__(self):
        self.log.append((self.name, "iter"))
        for i in range(self.n):
            yield {"x": torch.full((2, 3), float(i + 1)), "metadata": [{"token": "%d" % (2 * i + j)} for j in range(2)]}


class EvalSet:
    def __init__(self, log):
        self.log = log

    def evaluation(self, detections, output_dir=None):
        self.log.append(("val", "evaluation", sorted(detections)))
        return {"results": {"official_AP_11": "r11"}, "results_2": {"official_AP_40": "r40"}}, None


def _setup(tmp_path, monkeypatch, n_batches=3, epochs=2, seed=0):
    from det3d.solver.learning_schedules_fastai import OneCycle
    from det3d.torchie.trainer import trainer_sessd as T
    log, weights, emas = [], [], []

    def processor(model, model_ema, data, consistency_weight, train_mode):
        weights.append(consistency_weight)
        return dict(loss=model(data), log_vars=OrderedDict(loss=[1.0 + len(weights)], loc_loss_elem=[[0.5, 0.25]]), num_samples=2)

    def ema(model, model_ema, global_step):
        emas.append(global_step)
        with torch.no_grad():
            for p, q in zip(model.parameters(), model_ema.parameters()):
                q.mul_(0.5).add_(0.5 * p)
    monkeypatch.setattr(T, "update_ema_variables", ema)
    model, teacher = StandIn(seed), StandIn(seed + 100)
    for p in teacher.parameters():
        p.requires_grad_(False)
    opt = StandInOpt(model.parameters())
    sched = OneCycle(opt, epochs * n_batches, 0.003, [0.95, 0.85], 10.0, 0.4)
    tr = T.Trainer(model, teacher, processor, opt, sched, str(tmp_path))
    tr.register_training_hooks(None, dict(grad_clip=dict(max_norm=35, norm_type=2)), dict(interval=1, meta=dict(config="c")),
                               dict(interval=2))
    loaders = [Loader(n_batches, None, log, "train"), Loader(2, EvalSet(log), log, "val")]
    return tr, loaders, log, weights, emas, opt


def test_trainer_schedule_ema_workflow_and_checkpoints(tmp_path, monkeypatch):
    from det3d.solver.learning_schedules_fastai import OneCycle
    from det3d.torchie.trainer import sigmoid_rampup
    tr, loaders, log, weights, emas, opt = _setup(tmp_path, monkeypatch)
    res = tr.run(loaders, [("train", 60), ("val", 1)], 2)
    assert res["results"]["official_AP_11"] == "r11"
    # the schedule at every global step, and the consistency weight of each epoch
    ref = StandInOpt([torch.zeros(1, requires_grad=True)])
    sched = OneCycle(ref, 6, 0.003, [0.95, 0.85], 10.0, 0.4)
    want = []
    for s in range(6):
        sched.step(s)
        want.append((ref.lr, ref.mom))
    assert opt.steps == want
    assert weights == [sigmoid_rampup(0, 2)] * 3 + [sigmoid_rampup(1, 2)] * 3
    assert emas == list(range(6))
    # train epochs first, then one val pass on the last loader
    assert log == [("train", "set_epoch", 0), ("train", "iter"), ("train", "set_epoch", 1), ("train", "iter"), ("val", "iter"),
                   ("val", "evaluation", ["0", "1", "2", "3"])]
    assert tr.epoch == 2 and tr.iter == 6
    for n in (1, 2):
        for name in ("epoch_%d.pth" % n, "epoch_%d_ema.pth" % n):
            ck = torch.load(str(tmp_path / name), weights_only=True)
            assert ck["meta"] == {"config": "c", "epoch": n, "iter": 3 * n} and ck["optimizer"] == {"steps": 3 * n}
    assert os.readlink(str(tmp_path / "latest.pth")) == "epoch_2.pth"
    assert os.readlink(str(tmp_path / "latest_ema.pth")) == "epoch_2_ema.pth"
    ck = torch.load(str(tmp_path / "epoch_2_ema.pth"), weights_only=True)
    assert torch.equal(ck["state_dict"]["lin.weight"], tr.model_ema.lin.weight)
    logs = [f for f in os.listdir(str(tmp_path)) if f.endswith(".log")]
    text = open(str(tmp_path / logs[0])).read()
    assert "Epoch [1/2][2/3]" in text and "Evaluation official_AP_40: r40" in text and "loc_loss_elem: [[0.5, 0.25]]" in text


def test_resume_and_load_from(tmp_path, monkeypatch):
    tr, loaders, _, _, _, _ = _setup(tmp_path, monkeypatch)
    tr.run(loaders, [("train", 1)], 1)
    student = {k: v.clone() for k, v in tr.model.state_dict().items()}
    teacher = {k: v.clone() for k, v in tr.model_ema.state_dict().items()}
    assert not torch.equal(student["lin.weight"], teacher["lin.weight"])
    tr2, loaders2, log2, weights2, emas2, opt2 = _setup(tmp_path, monkeypatch, seed=7)
    tr2.resume(str(tmp_path / "epoch_1.pth"), map_location="cpu")
    assert tr2.epoch == 1 and tr2.iter == 3 and opt2.loaded == {"steps": 3}
    assert all(torch.equal(v, student[k]) for k, v in tr2.model.state_dict().items())
    assert all(torch.equal(v, teacher[k]) for k, v in tr2.model_ema.state_dict().items())      # from the _ema file
    tr2.run(loaders2, [("train", 60), ("val", 1)], 2)
    assert emas2 == [3, 4, 5] and log2[0] == ("train", "set_epoch", 1) and log2[-1][1] == "evaluation"
    tr3, _, _, _, _, opt3 = _setup(tmp_path, monkeypatch, seed=9)
    tr3.load_checkpoint_from_scratch(str(tmp_path / "epoch_1.pth"))
    assert all(torch.equal(v, student[k]) for k, v in tr3.model.state_dict().items())
    assert all(torch.equal(v, student[k]) for k, v in tr3.model_ema.state_dict().items())
    assert opt3.loaded == {"steps": 3} and tr3.epoch == 0
