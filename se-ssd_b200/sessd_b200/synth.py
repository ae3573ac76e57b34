"""Seeded synthetic inputs: the generators of sessd_data.synth (re-exported; they live in the library-free package) and
``train_batch``, a collated SE-SSD training batch built from them with the det3d pipelines and the device target assigner."""
from sessd_data.synth import *  # noqa: F401,F403
from sessd_data.synth import PC_RANGE, VOXEL_SIZE, random_boxes, ring_cloud, uniform_cloud  # noqa: F401


def train_batch(cfg, clouds, gt_boxes):
    """a collated SE-SSD training batch (the format batch_processor_inline takes) from point clouds and GT boxes: the config's test
    pipeline (voxels, anchors), targets from TargetAssigner.assign_batch_gpu, the teacher's ``_raw`` twins equal to the student's inputs
    and an identity augmentation (``transformation``)"""
    from det3d.datasets.pipelines import AssignTarget, Reformat, Voxelization
    from det3d.torchie.parallel import collate_kitti
    tf = [Voxelization(cfg=cfg.voxel_generator), AssignTarget(cfg=cfg.train_cfg.assigner), Reformat()]
    frames = []
    for i, c in enumerate(clouds):
        res = dict(mode="val", metadata=dict(token=i), lidar=dict(points=c))
        for t in tf:
            res, _ = t(res, None)
        frames.append(res)
    ex = collate_kitti(frames)
    at = tf[1]
    tg = at.target_assigners[0].assign_batch_gpu(at.anchor_dicts_by_task[0], gt_boxes)
    ex["labels"], ex["reg_targets"] = [tg["labels"]], [tg["bbox_targets"]]
    for k in ("voxels", "num_points", "coordinates", "num_voxels", "shape", "anchors", "labels", "reg_targets"):
        ex[k + "_raw"] = ex[k]
    ex["transformation"] = [dict(flipped=False, noise_rotation=0.0, noise_scale=1.0) for _ in clouds]
    return ex
