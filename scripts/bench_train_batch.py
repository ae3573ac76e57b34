"""Time the device-built SE-SSD training batch at batch 8 on ring-20k clouds with 15 GT boxes per frame.  Prints one JSON object with
the card's name, power limit and SM clock (read in the same run) and, from CUDA events after warm-up (median, min, max):
  * build_train_batch_ms: sessd_b200.augment.build_train_batch, the whole call -- host draws and packing, the one host-to-device copy,
    augmentation, both voxelisations, both target assignments and the one read-back of the voxel totals that forms the dict;
  * launch_train_batch_ms: the same without forming the dict (no read-back);
  * augment_batch_ms / kernels_only_ms: the augmentation alone, and its three kernels on inputs already on the device;
  * train_step_ms (--step): batch_processor_inline forward (teacher + student + losses) and backward on the built batch;
a torch.profiler kernel table of build_train_batch from a separate run, and, for comparison, CPU times per frame on the same machine:
  * reference_numba_ms: the reference's own numba functions (noise_per_object_v4_, random_flip_v2, global_rotation_v3,
    global_scaling_v3 and the shuffle) when --reference points at a checkout of it, else "not measured";
  * host_voxelize_assign_ms: the CPU voxeliser (oracle/cpu.py points_to_voxel) of both branches plus TargetAssigner.assign_v2 of both
    box sets.

    python scripts/bench_train_batch.py [--batch 8] [--steps 30] [--warmup 5] [--step] [--reference DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "se-ssd_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_encoder_train import card  # noqa: E402
from bench_train_step import sm_clock_mhz, timed  # noqa: E402


def frames(batch, seed=100):
    from sessd_data import synth
    clouds = [synth.ring_cloud(seed + b, 20000, 15) for b in range(batch)]
    boxes = [synth.ring_boxes(seed + b, 15) for b in range(batch)]
    names = [np.array(["Car"] * 13 + ["Van", "Pedestrian"]) for _ in range(batch)]
    return clouds, boxes, names


def cpu_ms(fn, reps=3):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return round(float(np.median(ts)), 2)


def reference_numba(ref_dir, cloud, boxes, valid, seed):
    """the reference's functions on one frame, timed after a JIT warm-up (imported where they lie, as tests/golden/make_augment_golden.py
    does)"""
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import make_augment_golden as g
    g.REF = ref_dir
    prep, _ = g.load_reference()

    def run():
        rs = np.random.RandomState(seed)
        pts, bx = cloud.copy(), boxes.copy()
        with g.draws_from(rs, []):
            prep.noise_per_object_v4_(bx, pts, valid, rotation_perturb=[-0.785, 0.785], center_noise_std=[1.0, 1.0, 0.5],
                                      global_random_rot_range=[0.0, 0.0], group_ids=None, num_try=100, data_aug_with_context=-1.0,
                                      data_aug_random_drop=-1.0)
            bx = bx[valid]
            bx, pts, _ = prep.random_flip_v2(bx, pts)
            bx, pts, _ = prep.global_rotation_v3(bx, pts, [-0.785, 0.785])
            bx, pts, _ = prep.global_scaling_v3(bx, pts, 0.95, 1.05)
            pts = pts[np.random.choice(np.arange(pts.shape[0]), pts.shape[0], replace=False)]
    run()
    return cpu_ms(run)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--reference", default=None)
    ap.add_argument("--step", action="store_true")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_train_batch.py measures the GPU; there is no CPU fallback"
    from det3d.datasets.pipelines import AssignTarget
    from det3d.datasets.pipelines.preprocess import filter_gt_box_outside_range
    from det3d.torchie import Config
    from oracle import augment_ref, cpu as ocpu
    from sessd_b200 import augment, ops, synth

    d = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_config.json")))     # the upstream config's values, plus its two
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))   # constructed objects from the repo's config
    d["model"]["neck"]["logger"] = ours.model.neck.logger
    d["model"]["bbox_head"]["box_coder"] = ours.model.bbox_head.box_coder
    cfg = Config(d)
    acfg = augment.AugmentConfig.from_config(cfg)
    clouds, boxes, names = frames(a.batch)
    sizes = [(len(c), len(b), True) for c, b in zip(clouds, boxes)]
    draws = augment.draw_augmentation(np.random.RandomState(0), sizes, acfg)

    def build():
        return augment.augment_batch(acfg, clouds, boxes, names, draws)

    full = timed(build, a.steps, a.warmup)
    built = timed(lambda: augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(0)), a.steps, a.warmup)
    launched = timed(lambda: augment.launch_train_batch(cfg, clouds, boxes, names, np.random.RandomState(0)), a.steps, a.warmup)
    step = "not measured"
    if a.step:
        import copy
        from det3d.models import build_detector
        from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
        from sessd_b200 import weights
        model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
        model.load_state_dict(weights.random_detector_state(0), strict=True)
        model = model.cuda().train()
        ema = copy.deepcopy(model)
        for p in ema.parameters():
            p.requires_grad_(False)
        ex = augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(0))

        def fwd_bwd():
            model.zero_grad(set_to_none=True)
            batch_processor_inline(model, ema, ex, consistency_weight=1.0, train_mode=True)["loss"].backward()
        step = timed(fwd_bwd, max(3, a.steps // 3), 2)
    # the three kernels on inputs already on the device
    res = build()
    B, M = res["selected"].shape
    d_boxes = torch.zeros((B, M, 7), dtype=torch.float32, device="cuda")
    for b in range(B):
        d_boxes[b, :len(boxes[b])] = torch.from_numpy(boxes[b])
    d_num = torch.tensor([len(x) for x in boxes], dtype=torch.int32, device="cuda")
    d_valid = torch.tensor([[n in acfg.class_names for n in nm] for nm in names], dtype=torch.uint8, device="cuda")
    d_loc = torch.from_numpy(np.stack([f.loc for f in draws.frames])).cuda()
    d_rot = torch.from_numpy(np.stack([f.rot for f in draws.frames])).cuda()
    d_glob = torch.from_numpy(np.stack([augment.global_row(f) for f in draws.frames])).cuda()
    d_pts = torch.from_numpy(np.concatenate(clouds)).cuda()
    d_perm = torch.from_numpy(np.concatenate([f.perm for f in draws.frames]).astype(np.int32)).cuda()
    d_off = res["frame_off"]
    raw, out = torch.empty_like(d_pts), torch.empty_like(d_pts)

    def kernels():
        sel = ops.noise_per_box(d_boxes, d_num, d_valid, d_loc, d_rot)
        ops.augment_points(d_pts, d_off, 20000, d_boxes, d_num, d_valid, d_loc, d_rot, sel, d_glob, d_perm, None, -1.0, raw, out)
        ops.augment_boxes(d_boxes, d_num, d_valid, d_valid, d_loc, d_rot, sel, d_glob, acfg.range_bev)

    kern = timed(kernels, a.steps, a.warmup)
    name, pl = card()
    sm_clock = sm_clock_mhz()

    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
        augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(0))
        torch.cuda.synchronize()
    table = [dict(name=e.key[:60], calls=e.count, device_us=round(e.device_time_total, 1))
             for e in sorted(prof.key_averages(), key=lambda e: -e.device_time_total) if e.device_time_total > 0][:14]

    # CPU comparison, per frame, on this machine
    f0 = draws.frames[0]
    valid0 = np.array([n in acfg.class_names for n in names[0]])
    dr0 = dict(loc=f0.loc, rot=f0.rot, flip=f0.flip, rotation=f0.rotation, scale=f0.scale, perm=f0.perm)
    o = augment_ref.augment_frame(clouds[0], boxes[0], valid0, dr0)       # the augmented frame the host voxeliser / assigner get
    at = AssignTarget(cfg=cfg.train_cfg.assigner)
    ta, ad = at.target_assigners[0], at.anchor_dicts_by_task[0]
    keep = filter_gt_box_outside_range(o["boxes"], acfg.range_bev)

    def host_vox_assign():
        for pts, bx in ((o["points"], o["boxes"][keep]), (o["points_raw"], o["boxes_raw"])):
            ocpu.points_to_voxel(pts, synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
            ta.assign_v2(ad, bx, anchors_mask=None, gt_classes=np.ones(len(bx), np.int32), gt_names=np.array(["Car"] * len(bx)),
                         enable_similar_type=True)
    host_ms = cpu_ms(host_vox_assign)
    ref_ms = "not measured"
    if a.reference and os.path.isdir(a.reference):
        ref_ms = reference_numba(a.reference, clouds[0], boxes[0], valid0, 0)

    print(json.dumps(dict(gpu=name, power_limit=pl, sm_clock_mhz_now_max=sm_clock, batch=a.batch, points_per_frame=20000, gt_per_frame=15,
                          build_train_batch_ms=built, launch_train_batch_ms=launched, augment_batch_ms=full, kernels_only_ms=kern,
                          train_step_ms=step, profile=table,
                          cpu_per_frame=dict(reference_numba_ms=ref_ms,
                                             host_voxelize_assign_ms=host_ms, where="CPU of the machine that ran this script"))))


if __name__ == "__main__":
    main()
