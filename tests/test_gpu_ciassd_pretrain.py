"""CIA-SSD pre-training on the device: ``MultiGroupHead.loss_ciassd`` against the reference's own CIA-SSD loss and its gradient
(tests/golden/ciassd_loss_case.npz, make_ciassd_golden.py), the student-only training batch against the twin batch of the same stream,
and the first stage end to end on a small prepared tree -- two identical runs and a resumed run, checkpoints without ``_ema`` files, a
checkpoint the SE-SSD model loads strictly, and the SE-SSD stage started from it."""
import os
import shutil

import numpy as np
import pytest
import torch

from test_gpu_kitti_train import SEED, _cfg, _ckpt, _same, tree  # noqa: F401  (tree: the prepared synthetic KITTI tree fixture)

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _head():
    from det3d.models import build_detector
    from det3d.torchie import Config
    cfg = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    return build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg).bbox_head


def test_loss_ciassd_matches_reference_golden(golden_dir):
    g = np.load(os.path.join(golden_dir, "ciassd_loss_case.npz"))
    B, A = g["labels"].shape
    H, W = 16, A // 32
    packed = torch.zeros(B, H, W, 24)
    packed[..., 0:14] = torch.from_numpy(g["box_preds"]).reshape(B, H, W, 14)
    packed[..., 14:16] = torch.from_numpy(g["cls_preds"]).reshape(B, H, W, 2)
    packed[..., 16:20] = torch.from_numpy(g["dir_cls_preds"]).reshape(B, H, W, 4)
    packed[..., 20:22] = torch.from_numpy(g["iou_preds"]).reshape(B, H, W, 2)
    packed[..., 22:] = 7.0                                               # padding channels: read by nothing, no gradient
    packed = packed.cuda().requires_grad_(True)
    anchors = torch.from_numpy(g["anchors"]).cuda()[None].expand(B, -1, -1).contiguous()
    example = dict(anchors=[anchors], labels=[torch.from_numpy(g["labels"].astype(np.int32)).cuda()],
                   reg_targets=[torch.from_numpy(g["reg_targets"]).cuda()])
    preds = dict(box_preds=packed[..., 0:14], cls_preds=packed[..., 14:16], dir_cls_preds=packed[..., 16:20], iou_preds=packed[..., 20:22],
                 _packed=packed)
    out = _head().loss_ciassd(example, [preds])
    keys = {"loss", "cls_loss_reduced", "loc_loss_reduced", "dir_loss_reduced", "iou_pred_loss", "loc_loss_elem", "cls_pos_loss",
            "cls_neg_loss", "num_pos", "num_neg"}
    assert set(out) == keys and all(isinstance(v, list) and len(v) == 1 for v in out.values())
    for k in ("loss", "cls_loss_reduced", "loc_loss_reduced", "dir_loss_reduced", "iou_pred_loss", "cls_pos_loss", "cls_neg_loss"):
        assert float(out[k][0].detach()) == pytest.approx(float(g[k]), rel=2e-5, abs=1e-7), k
    np.testing.assert_allclose([float(e) for e in out["loc_loss_elem"][0]], g["loc_loss_elem"], rtol=2e-5, atol=1e-7)
    assert int(out["num_pos"][0]) == int(g["num_pos"]) and int(out["num_neg"][0]) == int(g["num_neg"])
    # the reference's quirk: dir_loss_reduced is reported without its 0.2, the total sums 0.2 * dir
    total = float(g["cls_loss_reduced"] + g["loc_loss_reduced"] + 0.2 * g["dir_loss_reduced"] + g["iou_pred_loss"])
    assert float(g["loss"]) == pytest.approx(total, rel=1e-6)
    out["loss"][0].backward()
    grad = packed.grad.cpu().reshape(B, H, W, 24)
    for name, sl in (("box_preds", slice(0, 14)), ("cls_preds", slice(14, 16)), ("dir_cls_preds", slice(16, 20)),
                     ("iou_preds", slice(20, 22))):
        want = g["grad_" + name]
        # the IoU-prediction target comes from the device's aligned IoU here and the reference's CPU overlap there (about 1e-6 apart)
        atol = (1e-4 if name == "iou_preds" else 2e-6) * np.abs(want).max()
        np.testing.assert_allclose(grad[..., sl].numpy(), want, rtol=2e-4, atol=atol, err_msg=name)
    assert float(grad[..., 22:].abs().sum()) == 0.0
    assert float(np.abs(g["grad_box_preds"]).sum()) > 1.0 and (grad[1, ..., 0:14] == 0).all()       # frame 1 has no positives


def test_student_only_batch_equals_twin_batch(tree):  # noqa: F811
    """build_train_batch(twin=False) with GT-AUG and SA-DA: no ``*_raw`` keys, every student key bit-equal to the twin batch of the same
    seed, and the RandomState left where the twin batch leaves it"""
    from det3d.builder import build_dbsampler
    from det3d.datasets import build_dataset
    from sessd_b200 import augment, sada
    from sessd_b200.kitti_loader import epoch_streams, restart_sampler
    cfg = _cfg(tree, tree)
    ds = build_dataset(cfg.data.train)
    out = {}
    for twin in (True, False):
        order, rs = epoch_streams(SEED, 1, len(ds))
        frames = [ds[int(i)]["lidar"] for i in order[:4]]
        db = build_dbsampler(cfg.db_sampler)
        restart_sampler(db, rs)
        ex = augment.build_train_batch(cfg, [f["points"] for f in frames], [f["gt_boxes"] for f in frames], [f["gt_names"] for f in frames],
                                       rs, db_sampler=db, sa_da=sada.SadaConfig(), twin=twin)
        out[twin] = (ex, rs.get_state()[1].copy(), rs.get_state()[2])
    full, single = out[True][0], out[False][0]
    assert not any(k.endswith("_raw") for k in single) and any(k.endswith("_raw") for k in full)
    assert sorted(single) == sorted(k for k in full if not k.endswith("_raw"))
    for k in single:
        assert _same(single[k], full[k]), k
    assert np.array_equal(out[True][1], out[False][1]) and out[True][2] == out[False][2]
    assert int((single["labels"][0] > 0).sum()) > 0 and single["voxels"].shape[0] > 1000


def _pretrain(tree, work_dir, resume_from=None, load_from=None):
    from det3d.models import build_detector
    from det3d.torchie.apis.train import train_detector
    from sessd_b200.kitti_train import build_datasets
    cfg = _cfg(tree, work_dir)
    cfg.resume_from, cfg.load_from = resume_from, load_from
    torch.manual_seed(0)
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    return cfg, train_detector(model, build_datasets(cfg, pretrain=True), cfg)


def test_pretrain_runs_resumes_and_hands_off_to_sessd(tree, tmp_path, monkeypatch):  # noqa: F811
    from det3d.models import build_detector
    from det3d.torchie.trainer import load_checkpoint
    from det3d.torchie.trainer import trainer_sessd
    wd = tmp_path / "a"
    cfg, results = _pretrain(tree, wd, load_from=str(tmp_path / "no_such_checkpoint.pth"))
    assert sorted(f for f in os.listdir(str(wd)) if f.endswith(".pth")) == ["epoch_1.pth", "epoch_2.pth", "latest.pth"]
    for n in (1, 2):
        ck = _ckpt(str(wd / ("epoch_%d.pth" % n)))
        assert set(ck) == {"meta", "state_dict", "optimizer"} and ck["meta"]["epoch"] == n and ck["meta"]["iter"] == 4 * n
    log = open(str(next(wd.glob("*.log")))).read()
    assert "is ignored" in log and "Evaluation official_AP_11" in log and "official_AP_11" in results["results"]
    assert len([l for l in log.splitlines() if "Epoch [" in l and "loc_loss_reduced" in l and "ious_loss" not in l]) == 8
    # the checkpoint is the SE-SSD model's, key for key
    sessd = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    load_checkpoint(sessd, str(wd / "latest.pth"), map_location="cpu", strict=True)
    stage1 = _ckpt(str(wd / "latest.pth"))["state_dict"]
    # two identical runs, and a run resumed after epoch 1: bitwise the same model and optimiser state
    _pretrain(tree, tmp_path / "b")
    os.makedirs(str(tmp_path / "c"))
    shutil.copy(str(wd / "epoch_1.pth"), str(tmp_path / "c" / "epoch_1.pth"))
    _pretrain(tree, tmp_path / "c", resume_from=str(tmp_path / "c" / "epoch_1.pth"))
    a = _ckpt(str(wd / "epoch_2.pth"))
    assert _same(a, _ckpt(str(tmp_path / "b" / "epoch_2.pth"))), "two identical runs differ"
    assert _same(a, _ckpt(str(tmp_path / "c" / "epoch_2.pth"))), "the resumed run differs"
    # the SE-SSD stage from the stage-1 checkpoint: student == teacher == stage 1 when its loop starts, and it trains
    from det3d.torchie.apis import train_detector
    from sessd_b200.kitti_train import build_datasets
    start = {}
    run = trainer_sessd.Trainer.run

    def record_then_run(self, *args, **kwargs):
        start["student"] = {k: v.detach().cpu().clone() for k, v in self.model.state_dict().items()}
        start["teacher"] = {k: v.detach().cpu().clone() for k, v in self.model_ema.state_dict().items()}
        return run(self, *args, **kwargs)
    monkeypatch.setattr(trainer_sessd.Trainer, "run", record_then_run)
    cfg2 = _cfg(tree, tmp_path / "s2")
    cfg2.load_from = str(wd / "latest.pth")
    assert cfg2.my_paras.enable_ssl
    torch.manual_seed(1)
    model = build_detector(cfg2.model, train_cfg=cfg2.train_cfg, test_cfg=cfg2.test_cfg)
    res2 = train_detector(model, build_datasets(cfg2), cfg2)
    assert _same(start["student"], stage1) and _same(start["teacher"], stage1)
    assert "official_AP_11" in res2["results"] and os.path.exists(str(tmp_path / "s2" / "epoch_2_ema.pth"))
