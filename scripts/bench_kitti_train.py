"""Measure the SE-SSD training loop on a prepared synthetic KITTI tree, split into its parts.

    python scripts/bench_kitti_train.py [--frames 64] [--batch 4] [--steps 20] [--warmup 3]

Writes, under a temporary directory, FRAMES train and FRAMES val frames of ring-20k clouds with 15 cars each (60 points per car) and
runs kitti_data_prep on it.  Then, with the reference config's recipe (GT-AUG, SA-DA, one-cycle AdamW with clip 35 and the fused
teacher EMA), it times each loop step after warm-up with a device synchronise between the parts: the batch (waiting on the reader
thread, the host draws and the device build), the train step (both forwards, backward, optimiser), the whole loop step; then the
validation pass in frames/s (second pass over the val split).  In the same call it runs scripts/bench_train_step.py --recipe, the
identity-augmentation step on synthetic batches, at the same batch size.  Prints one JSON line with the card's name, power limit and
SM clock.
"""
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "se-ssd_b200"), os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)


def write_tree(root, n_train, n_val, points=20000, cars=15, seed=0):
    import kitti_prep_cases as cases
    from oracle import kitti_prep_ref as ref
    from sessd_b200 import synth
    rs = np.random.RandomState(seed)
    ids = {"train": list(range(n_train)), "val": list(range(n_train, n_train + n_val)), "test": []}
    os.makedirs(os.path.join(root, "ImageSets"))
    for s, v in ids.items():
        with open(os.path.join(root, "ImageSets", s + ".txt"), "w") as f:
            f.write("".join("%06d\n" % i for i in v))
    for d in ("calib", "label_2", "velodyne", "image_2"):
        os.makedirs(os.path.join(root, "training", d))
    os.makedirs(os.path.join(root, "testing"))
    for k in range(n_train + n_val):
        with open(os.path.join(root, "training", "image_2", "%06d.png" % k), "wb") as f:
            f.write(cases.png(*cases.SIZES[k % 4]))
        text, cal = cases.calib(rs, k % 7)
        with open(os.path.join(root, "training", "calib", "%06d.txt" % k), "w") as f:
            f.write(text)
        slots = rs.permutation(30)[:cars]                       # a 6 x 5 grid in front of the car: no two boxes overlap
        objs = [("Car", 0.0, 0, -1.2, (500.0, 150.0, 600.0, 190.0), (1.52, 1.63, 3.9),
                 (-12.5 + 5.0 * (s % 6) + rs.uniform(-0.3, 0.3), 1.7, 10.0 + 9.0 * (s // 6) + rs.uniform(-0.5, 0.5)),
                 float(rs.uniform(-1.0, 1.0))) for s in slots]
        text = cases.label_text(objs)
        with open(os.path.join(root, "training", "label_2", "%06d.txt" % k), "w") as f:
            f.write(text)
        boxes = ref.db_boxes({"annos": cases._anno(text), "calib": cal})[0]
        inside = cases.cloud(rs, 0, boxes)
        np.concatenate([synth.ring_cloud(k, points), inside]).astype(np.float32).tofile(
            os.path.join(root, "training", "velodyne", "%06d.bin" % k))


def main():
    import argparse
    import torch

    from bench_encoder_train import card
    from bench_train_step import sm_clock_mhz
    from test_kitti_train import reference_config
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    import copy

    from det3d.datasets import build_dataloader, build_dataset
    from det3d.models import build_detector
    from det3d.torchie.apis import _create_learning_rate_scheduler, build_one_cycle_optimizer
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline, compute_on_dataset
    from sessd_b200.kitti_prep import kitti_data_prep
    from sessd_b200.train import ParamArena
    from sessd_b200 import weights

    # the identity-augmentation step first, in its own process, while this one holds no device memory
    step = subprocess.run([sys.executable, os.path.join(HERE, "bench_train_step.py"), "--batch", str(a.batch), "--recipe", "--steps",
                           str(a.steps), "--warmup", "5", "--layer-reps", "1"], capture_output=True, text=True)
    lines = [l for l in step.stdout.splitlines() if l.startswith("{")]
    identity = json.loads(lines[-1])["step_ms"] if lines else "failed: " + step.stderr[-500:]
    with tempfile.TemporaryDirectory() as root:
        t0 = time.time()
        write_tree(root, a.frames, a.frames)
        kitti_data_prep(root)
        prep_s = time.time() - t0
        cfg = reference_config(root)
        cfg.data.samples_per_gpu = a.batch
        train_loader = build_dataloader(build_dataset(cfg.data.train), a.batch, 2, cfg=cfg, seed=0)
        val_loader = build_dataloader(build_dataset(cfg.data.val), a.batch, 2, cfg=cfg)
        model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
        model.load_state_dict(weights.random_detector_state(0), strict=True)
        model = model.cuda()
        ema = copy.deepcopy(model)
        for p in ema.parameters():
            p.requires_grad_(False)
        arena_ema = ParamArena(ema, with_grad=False)
        _, opt = build_one_cycle_optimizer(model, cfg.optimizer)
        need = a.steps + a.warmup
        sched = _create_learning_rate_scheduler(opt, cfg.lr_config, need + len(train_loader))
        model.train()
        ema.train()
        parts = {"batch_ms": [], "train_step_ms": [], "loop_step_ms": []}
        gs, it = 0, iter(train_loader)
        torch.cuda.synchronize()
        while gs < need:
            t0 = time.perf_counter()
            try:
                batch = next(it)
            except StopIteration:
                it = iter(train_loader)
                continue
            torch.cuda.synchronize()
            t1 = time.perf_counter()
            sched.step(gs)
            out = batch_processor_inline(model, ema, batch, 1.0, train_mode=True)
            opt.zero_grad()
            out["loss"].backward()
            opt.step(max_grad_norm=35.0, ema=arena_ema, global_step=gs)
            torch.cuda.synchronize()
            t2 = time.perf_counter()
            if gs >= a.warmup:
                for k, v in (("batch_ms", t1 - t0), ("train_step_ms", t2 - t1), ("loop_step_ms", t2 - t0)):
                    parts[k].append(1e3 * v)
            gs += 1
        sm_clock = sm_clock_mhz()
        stats = {k: dict(median=round(float(np.median(v)), 2), min=round(float(np.min(v)), 2), max=round(float(np.max(v)), 2),
                         n=len(v)) for k, v in parts.items()}
        compute_on_dataset(model, val_loader)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        compute_on_dataset(model, val_loader)
        torch.cuda.synchronize()
        val_fps = a.frames / (time.perf_counter() - t0)
    name, pl = card()
    print(json.dumps(dict(gpu=name, power_limit=pl, sm_clock_mhz_now_max=sm_clock, batch=a.batch, frames=a.frames, prep_s=round(prep_s, 1),
                          **stats, val_frames_per_s=round(val_fps, 1), identity_aug_train_step_ms=identity)))


if __name__ == "__main__":
    main()
