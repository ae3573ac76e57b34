"""CIA-SSD pre-training on the CPU: the ``--pretrain`` / ``--load-from`` command line, the datasets and the ignored ``load_from`` of the
first stage, DI-NMS as its validation default, and the single-model Trainer's step order (schedule, batch processor hooks, one fused
clip + AdamW step without EMA), epochs and checkpoint files with stand-in models."""
import logging
import os
from collections import OrderedDict

import pytest
import torch

from test_kitti_train import EvalSet, Loader, StandIn, reference_config, tree  # noqa: F401  (tree: the crafted KITTI tree fixture)

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUR_CFG = os.path.join(ROOT, "examples", "second", "configs", "config.py")


def test_cli_pretrain_and_load_from(tmp_path, monkeypatch):
    from sessd_b200 import kitti_train
    seen = []
    monkeypatch.setattr(kitti_train, "train", lambda cfg, pretrain=False: seen.append((cfg, pretrain)))
    monkeypatch.chdir(tmp_path)
    kitti_train.main([OUR_CFG, "--pretrain", "--work-dir", "w1", "--total-epochs", "2"])
    kitti_train.main([OUR_CFG, "--work-dir", "w2", "--load-from", "w1/latest.pth", "--resume-from", "epoch_1.pth"])
    (c1, p1), (c2, p2) = seen
    assert p1 is True and c1.work_dir == "w1" and c1.total_epochs == 2
    assert p2 is False and c2.load_from == str(tmp_path / "w1" / "latest.pth") and c2.resume_from == os.path.join("w2", "epoch_1.pth")


def test_pretrain_builds_no_unlabelled_dataset(tree):  # noqa: F811
    from sessd_b200.kitti_train import build_datasets
    cfg = reference_config(tree)
    assert cfg.my_paras.enable_ssl and cfg.workflow[-1][0] == "val"
    stage2, stage1 = build_datasets(cfg), build_datasets(cfg, pretrain=True)
    assert len(stage2) == 3 and not stage2[1].labeled
    assert len(stage1) == 2 and all(ds.labeled for ds in stage1) and stage1[1].mode == "val"


def test_train_detector_ignores_load_from_and_defaults_to_dinms(tree, monkeypatch):  # noqa: F811
    from det3d.torchie.apis import train as T
    from det3d.torchie.trainer.trainer import Trainer
    cfg = reference_config(tree)
    cfg.work_dir = None
    cfg.load_from = "/no/such/epoch_60.pth"
    assert "nms_type" not in cfg.test_cfg.nms
    built, ran = [], []
    monkeypatch.setattr(T, "build_loaders", lambda ds, cfg, twin=True: built.append(twin) or [Loader(3, None, [], "train")])
    monkeypatch.setattr(Trainer, "run", lambda self, loaders, workflow, max_epochs: ran.append((self, workflow, max_epochs)) or "ran")
    model = StandIn(0)
    model.cuda = lambda: model
    model.test_cfg = cfg.test_cfg
    logged = []

    class Capture(logging.Handler):
        def emit(self, record):
            logged.append(record.getMessage())
    logger = logging.getLogger("ciassd-test")
    logger.addHandler(Capture())
    logger.setLevel(logging.INFO)
    assert T.train_detector(model, ["train", "val"], cfg, logger=logger) == "ran"
    assert built == [False] and ran[0][1] == cfg.workflow and ran[0][2] == cfg.total_epochs
    assert any("load_from /no/such/epoch_60.pth is ignored" in m for m in logged)
    assert model.test_cfg.nms.nms_type == "rotate_weighted_nms" and "nms_type" not in cfg.test_cfg.nms
    model.test_cfg.nms.nms_type = "rotate_nms"
    assert T.with_default_nms(model.test_cfg).nms.nms_type == "rotate_nms"               # a named NMS is kept


class CiassdStandIn(StandIn):
    """a detector whose CIA-SSD loss is a reference-shaped dict, recording how it was called"""

    def __init__(self, seed, log):
        super().__init__(seed)
        self.log = log

    def forward(self, example, return_loss=True, stage="sessd", **kw):
        self.log.append(("forward", stage, return_loss))
        if not return_loss:
            return super().forward(example, return_loss=False)
        loss = self.lin(example["x"]).square().sum()
        return dict(loss=[loss], cls_loss_reduced=[torch.tensor(0.5)], loc_loss_elem=[[torch.tensor(0.1 * i) for i in range(7)]],
                    num_pos=[torch.tensor(11)])


def _setup(tmp_path, monkeypatch, log, seed=0, n_batches=3, epochs=2):
    from det3d.solver.learning_schedules_fastai import OneCycle
    from det3d.torchie.apis.train import batch_processor
    from det3d.torchie.trainer.trainer import Trainer
    from sessd_b200.train import ArenaAdamW, ParamArena

    def step(self, max_grad_norm=None, ema=None, global_step=None):
        log.append(("step", max_grad_norm, ema, global_step, round(self.lr, 8)))
        with torch.no_grad():
            self.arena.flat.add_(self.arena.grad_flat, alpha=-0.01)
    monkeypatch.setattr(ArenaAdamW, "step", step)
    monkeypatch.setattr(ArenaAdamW, "zero_grad", lambda self: log.append("zero_grad") or self.arena.zero_grad())
    model = CiassdStandIn(seed, log)
    opt = ArenaAdamW(ParamArena(model), lr=3e-3, betas=(0.9, 0.99), weight_decay=0.01)
    sched = OneCycle(opt, epochs * n_batches, 0.003, [0.95, 0.85], 10.0, 0.4)

    def processor(model, data, train_mode):             # the stand-in loader's batches of two frames, with anchors
        return batch_processor(model, dict(data, anchors=[torch.zeros(2, 4, 7)]), train_mode, device="cpu", hooks=log.append)
    tr = Trainer(model, processor, opt, sched, str(tmp_path))
    tr.register_training_hooks(None, dict(grad_clip=dict(max_norm=35, norm_type=2)), dict(interval=1, meta=dict(config="c")),
                               dict(interval=2))
    return tr, [Loader(n_batches, None, log, "train"), Loader(2, EvalSet(log), log, "val")], opt


def test_single_model_trainer_step_order_checkpoints_and_resume(tmp_path, monkeypatch):
    log = []
    tr, loaders, opt = _setup(tmp_path, monkeypatch, log)
    res = tr.run(loaders, [("train", 60), ("val", 1)], 2)
    assert res["results"]["official_AP_11"] == "r11" and tr.epoch == 2 and tr.iter == 6
    per_step = ["after_data_to_device", ("forward", "ciassd", True), "after_forward", "after_parse_loss", "zero_grad"]
    steps = [e for e in log if isinstance(e, tuple) and e[0] == "step"]
    assert [s[1:4] for s in steps] == [(35, None, None)] * 6                                # clip at 35, no EMA
    first = log.index(("train", "iter")) + 1
    assert log[first:first + 6] == per_step + [steps[0]]
    assert log[-4:] == [("val", "iter"), ("forward", "sessd", False), ("forward", "sessd", False), ("val", "evaluation", ["0", "1", "2", "3"])]
    files = sorted(f for f in os.listdir(str(tmp_path)) if f.endswith(".pth"))
    assert files == ["epoch_1.pth", "epoch_2.pth", "latest.pth"] and os.readlink(str(tmp_path / "latest.pth")) == "epoch_2.pth"
    ck = torch.load(str(tmp_path / "epoch_1.pth"), weights_only=True)
    assert ck["meta"] == {"config": "c", "epoch": 1, "iter": 3} and set(ck["optimizer"]) == set(opt.state_dict())
    text = open(str(next(tmp_path.glob("*.log")))).read()
    assert "Epoch [1/2][2/3]" in text and "loc_loss_elem: [[0.0, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6]]" in text
    # resume from epoch 1: the model, the optimiser, the epoch and the iteration, then the same second epoch as the uninterrupted run
    final = {k: v.clone() for k, v in tr.model.state_dict().items()}
    log2 = []
    tr2, loaders2, opt2 = _setup(tmp_path / "r", monkeypatch, log2, seed=7)
    tr2.resume(str(tmp_path / "epoch_1.pth"), map_location="cpu")
    assert tr2.epoch == 1 and tr2.iter == 3
    assert all(torch.equal(v, ck["state_dict"][k]) for k, v in tr2.model.state_dict().items())
    tr2.run(loaders2, [("train", 60), ("val", 1)], 2)
    assert [e[3:] for e in log2 if isinstance(e, tuple) and e[0] == "step"] == [s[3:] for s in steps[3:]]
    assert all(torch.equal(v, final[k]) for k, v in tr2.model.state_dict().items())
    with pytest.raises(NotImplementedError):
        tr2.load_checkpoint_from_scratch(str(tmp_path / "epoch_1.pth"))


def test_batch_processor_eval_mode_returns_detections():
    from det3d.torchie.apis.train import batch_processor
    log = []
    model = CiassdStandIn(0, log)
    out = batch_processor(model, {"x": torch.ones(2, 3), "metadata": [{"token": "a"}]}, train_mode=False, device="cpu")
    assert log == [("forward", "sessd", False)] and out[0]["metadata"] == {"token": "a"}
    res = batch_processor(model, {"x": torch.ones(2, 3), "anchors": [torch.zeros(2, 4, 7)]}, train_mode=True, device="cpu")
    assert res["num_samples"] == 2 and res["log_vars"]["num_pos"] == [11.0] and res["loss"].requires_grad
    assert isinstance(res["log_vars"], OrderedDict)
