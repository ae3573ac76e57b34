"""Measure the CIA-SSD pre-training step (the first stage of SE-SSD training) next to the SE-SSD step, on a prepared synthetic KITTI tree.

    python scripts/bench_pretrain_step.py [--frames 64] [--batch 4] [--steps 20] [--warmup 3]

Writes the tree of scripts/bench_kitti_train.py (FRAMES train frames of ring-20k clouds with 15 cars each) under a temporary directory
and runs kitti_data_prep on it.  Then, with the reference config's recipe (GT-AUG, SA-DA, one-cycle AdamW with clip 35), it times after
warm-up, with CUDA events and one synchronise per step:
  * pretrain: the student-only batch (twin=False: one voxelisation, one assignment) and the single-model step (one forward, the CIA-SSD
    loss, backward, the fused clip + AdamW pass);
  * sessd: the twin batch and the teacher / student step (two forwards, the SE-SSD loss with the consistency term, backward, the fused
    clip + AdamW + EMA pass).
Both loops start from the same weights and alternate in blocks of ``--block`` steps, so drift of the card's clock affects both alike.
Prints one JSON line with the card's name, power limit and SM clock.
"""
import json
import os
import sys
import tempfile

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
for p in (ROOT, os.path.join(ROOT, "se-ssd_b200"), os.path.join(ROOT, "tests"), HERE):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    import argparse
    import copy

    import torch

    from bench_encoder_train import card
    from bench_kitti_train import write_tree
    from bench_train_step import sm_clock_mhz
    from test_kitti_train import reference_config
    from det3d.datasets import build_dataloader, build_dataset
    from det3d.models import build_detector
    from det3d.torchie.apis import _create_learning_rate_scheduler, build_one_cycle_optimizer
    from det3d.torchie.apis.train import batch_processor
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
    from sessd_b200 import weights
    from sessd_b200.kitti_prep import kitti_data_prep
    from sessd_b200.train import ParamArena
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=64)
    ap.add_argument("--batch", type=int, default=4)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--block", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_pretrain_step.py measures on the GPU and found none")
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.frames, 4)
        kitti_data_prep(root)
        cfg = reference_config(root)
        cfg.data.samples_per_gpu = a.batch
        need = a.steps + a.warmup
        runs = {}
        for name, twin in (("pretrain", False), ("sessd", True)):
            loader = build_dataloader(build_dataset(cfg.data.train), a.batch, 2, cfg=cfg, seed=0, twin=twin)
            model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
            model.load_state_dict(weights.random_detector_state(0), strict=True)
            model = model.cuda().train()
            ema = None
            if twin:
                ema = copy.deepcopy(model)
                for p in ema.parameters():
                    p.requires_grad_(False)
                ema._arena = ParamArena(ema, with_grad=False)
            _, opt = build_one_cycle_optimizer(model, cfg.optimizer)
            sched = _create_learning_rate_scheduler(opt, cfg.lr_config, 2 * need + len(loader))
            runs[name] = dict(loader=loader, it=iter(loader), model=model, ema=ema, opt=opt, sched=sched, gs=0,
                              batch_ms=[], step_ms=[], loop_ms=[])

        def one_step(r):
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
            ev[0].record()
            while True:
                try:
                    batch = next(r["it"])
                    break
                except StopIteration:
                    r["it"] = iter(r["loader"])
            ev[1].record()
            r["sched"].step(r["gs"])
            if r["ema"] is None:
                out = batch_processor(r["model"], batch, train_mode=True)
                r["opt"].zero_grad()
                out["loss"].backward()
                r["opt"].step(max_grad_norm=35.0)
            else:
                out = batch_processor_inline(r["model"], r["ema"], batch, 1.0, train_mode=True)
                r["opt"].zero_grad()
                out["loss"].backward()
                r["opt"].step(max_grad_norm=35.0, ema=r["ema"]._arena, global_step=r["gs"])
            ev[2].record()
            ev[2].synchronize()
            if r["gs"] >= a.warmup:
                r["batch_ms"].append(ev[0].elapsed_time(ev[1]))
                r["step_ms"].append(ev[1].elapsed_time(ev[2]))
                r["loop_ms"].append(ev[0].elapsed_time(ev[2]))
            r["gs"] += 1

        torch.cuda.synchronize()
        while any(r["gs"] < need for r in runs.values()):
            for r in runs.values():
                for _ in range(a.block):
                    if r["gs"] < need:
                        one_step(r)
        sm_clock = sm_clock_mhz()
    stats = {name: {k: dict(median=round(float(np.median(r[k])), 2), min=round(float(np.min(r[k])), 2), max=round(float(np.max(r[k])), 2),
                            n=len(r[k])) for k in ("batch_ms", "step_ms", "loop_ms")} for name, r in runs.items()}
    name, pl = card()
    print(json.dumps(dict(gpu=name, power_limit=pl, sm_clock_mhz_now_max=sm_clock, batch=a.batch, frames=a.frames, **stats)))


if __name__ == "__main__":
    main()
