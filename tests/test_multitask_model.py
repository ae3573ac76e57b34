"""Multi-class inference on the CPU: the per-task anchors against the reference's (tests/golden/anchors_multitask.npz), the head
weight packing of several tasks, a three-class config's head, the engine's label recovery against the reference's concatenation of
per-task detections, the post-processing config's new fields and the training entry points that stay single-task."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import multitask_cases as mc
from cases import sha

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "anchors_multitask.npz")


def test_task_anchors_equal_the_reference_bit_for_bit():
    from sessd_b200.weights import task_anchors
    g = np.load(GOLDEN)
    got = task_anchors(dict(anchor_generators=mc.GENERATORS, tasks=mc.TASKS))
    assert len(got) == 3
    for name, a in zip(mc.NAMES, got):
        assert a.dtype == np.float32 and a.shape == tuple(g[name + "_shape"])
        assert np.array_equal(sha(a), g[name + "_sha"]), name
        assert np.array_equal(a[:704].view(np.uint32), g[name + "_head"].view(np.uint32))
        assert np.array_equal(a[-704:].view(np.uint32), g[name + "_tail"].view(np.uint32))
    with pytest.raises(NotImplementedError):
        task_anchors(dict(anchor_generators=mc.GENERATORS, tasks=[dict(num_class=3, class_names=mc.NAMES)]))


def test_head_packing_stacks_tasks_at_24_channel_blocks():
    from sessd_b200.runners import head_launch, head_weight, pack_head
    g = torch.Generator().manual_seed(3)
    sd = {}
    for t in range(3):
        for nm, co in (("conv_box", 14), ("conv_cls", 2), ("conv_dir", 4), ("conv_iou", 2)):
            sd["tasks.%d.%s.weight" % (t, nm)] = torch.randn((co, 128, 1, 1), generator=g)
            sd["tasks.%d.%s.bias" % (t, nm)] = torch.randn(co, generator=g)
    w, b = pack_head(sd, ["tasks.0.", "tasks.1.", "tasks.2."], "cpu")
    assert tuple(w.shape) == (72, 128, 1, 1) and tuple(b.shape) == (72,)
    for t in range(3):
        o = 24 * t
        one_w, one_b = pack_head(sd, "tasks.%d." % t, "cpu")
        assert torch.equal(w[o:o + 24], one_w) and torch.equal(b[o:o + 24], one_b)
        cat_w = torch.cat([sd["tasks.%d.%s.weight" % (t, n)] for n in ("conv_box", "conv_cls", "conv_dir", "conv_iou")])
        assert torch.equal(w[o:o + 22], cat_w) and torch.all(w[o + 22:o + 24] == 0) and torch.all(b[o + 22:o + 24] == 0)
    # one task: the layout of the single-task head, module parameters keep their graph
    w1, _ = head_weight(lambda n: sd["tasks.0." + n])
    assert torch.equal(w1, w[:24])
    assert head_launch(3).cout == 72 and head_launch(1).cout == 24 and head_launch(3).name == "head"


def test_three_class_config_builds_a_three_task_head():
    from det3d.models import build_detector
    from det3d.torchie import Config
    import json
    cfg = Config(mc.three_class(json.load(open(mc.REF_CFG))))
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    cfg.model.neck.logger = ours.model.neck.logger
    cfg.model.bbox_head.box_coder = ours.model.bbox_head.box_coder
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    head = model.bbox_head
    assert len(head.tasks) == 3 and head.num_classes == [1, 1, 1] and head.class_names == [["Car"], ["Pedestrian"], ["Cyclist"]]
    keys = {k for k in model.state_dict() if k.startswith("bbox_head.tasks.")}
    assert {k.split(".")[2] for k in keys} == {"0", "1", "2"}
    assert cfg.class_names == mc.NAMES


def _reference_merge(per_task, num_classes):
    """MultiGroupHead.predict's concatenation of the reference (mg_head_sessd.py:923-943): boxes and scores concatenated in task
    order, labels offset by the classes of the earlier tasks"""
    flag, labels = 0, []
    for r, n in zip(per_task, num_classes):
        labels.append(r["label_preds"] + flag)
        flag += n
    return dict(box3d_lidar=np.concatenate([r["box3d_lidar"] for r in per_task]), scores=np.concatenate([r["scores"] for r in per_task]),
                label_preds=np.concatenate(labels))


def test_packed_results_unpack_to_the_reference_concatenation():
    from sessd_b200.engine import unpack_results
    rs = np.random.RandomState(0)
    A, T, P = 70400, 3, 100
    for counts in ((5, 0, 3), (0, 0, 0), (100, 100, 100), (0, 7, 0)):
        per_task = [dict(box3d_lidar=rs.randn(c, 7).astype(np.float32), scores=rs.rand(c).astype(np.float32),
                         label_preds=np.zeros(c, np.int64), anchor=rs.randint(0, A, c)) for c in counts]
        result = np.zeros((1, T * P, 8), np.float32)
        meta = np.full((1, 8 + T * P), -1, np.int32)
        meta[0, :8] = [sum(counts), 11, 10, 9, 4, 0, 0, 0]
        o = 0
        for t, r in enumerate(per_task):
            c = counts[t]
            result[0, o:o + c, :7], result[0, o:o + c, 7] = r["box3d_lidar"], r["scores"]
            meta[0, 8 + o:8 + o + c] = t * A + r["anchor"]
            o += c
        (got,) = unpack_results(result, meta, A)
        ref = _reference_merge(per_task, [1, 1, 1])
        for k in ref:
            assert np.array_equal(got[k], ref[k]), (counts, k)
        assert got["label_preds"].dtype == np.int64
        assert np.array_equal(got["anchor_index"] % A, np.concatenate([r["anchor"] for r in per_task]).astype(np.int64))


def test_post_cfg_new_fields_zero_mean_one_task():
    from sessd_b200 import ops
    from sessd_b200._lib import PostCfg
    names = [f[0] for f in PostCfg._fields_]
    assert names[-2:] == ["num_tasks", "task_stride"]
    assert PostCfg.num_tasks.offset >= PostCfg.dinms.offset + C.sizeof(PostCfg._fields_[names.index("dinms")][1])
    c1 = ops.make_post_cfg(batch=2)
    assert c1.num_tasks == 0 and c1.task_stride == 0 and ops.post_tasks(c1) == 1 and ops.post_capacity(c1) == 100
    z = PostCfg()
    assert z.num_tasks == 0 and z.task_stride == 0 and ops.post_tasks(z) == 1
    # the old fields keep their values and offsets: a one-task config is byte for byte the old struct plus two zero ints
    raw = bytes(c1)
    assert raw[PostCfg.num_tasks.offset:] == bytes(C.sizeof(PostCfg) - PostCfg.num_tasks.offset)
    c3 = ops.make_post_cfg(batch=2, head_stride=72, num_tasks=3, nms_type="rotate_weighted_nms")
    assert (c3.num_tasks, c3.task_stride) == (3, 24) and ops.post_capacity(c3) == 3000
    assert bytes(c3)[:PostCfg.num_tasks.offset] == bytes(ops.make_post_cfg(batch=2, head_stride=72,
                                                                           nms_type="rotate_weighted_nms"))[:PostCfg.num_tasks.offset]
    with pytest.raises(ValueError):
        ops.make_post_cfg(batch=1, num_tasks=0)


def test_training_entry_points_raise_for_several_tasks():
    from det3d.models.bbox_heads.mg_head_sessd import MultiGroupHead
    from det3d.models import build_detector
    from det3d.torchie import Config
    from sessd_b200 import augment
    import json
    cfg = Config(mc.three_class(json.load(open(mc.REF_CFG))))
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    cfg.model.neck.logger = ours.model.neck.logger
    cfg.model.bbox_head.box_coder = ours.model.bbox_head.box_coder
    head = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg).bbox_head
    assert isinstance(head, MultiGroupHead)
    preds = [dict(_packed=torch.zeros(1, 4, 4, 24))] * 3
    for fn in (head.loss, head.loss_ciassd):
        with pytest.raises(NotImplementedError, match="training is single-task"):
            fn({}, preds)
    head.train()
    with pytest.raises(NotImplementedError, match="training is single-task"):
        head(torch.zeros(1, 128, 8, 8))
    with pytest.raises(NotImplementedError, match="single-task"):
        augment._static(cfg, "cpu")
