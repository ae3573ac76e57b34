"""Time the optimiser tail of one SE-SSD training step on the student arena (~3.8 M parameters): the fused path (sessd_grad_sqnorm +
sessd_adamw_clip_ema_step: clip, AdamW and teacher EMA in two launches) against the unfused one (torch clip_grad_norm_ over the
parameter views + sessd_adamw_step + sessd_axpby).  CUDA-event medians over --reps calls after --warmup, alternating the two paths in
rounds.  Prints one JSON object with the card's name, power limit and SM clock, and the bytes each path moves per parameter.

    python scripts/bench_optim_tail.py [--reps 200] [--warmup 20] [--rounds 5]
"""
import argparse
import copy
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "se-ssd_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_encoder_train import card  # noqa: E402
from bench_train_step import sm_clock_mhz  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_optim_tail.py needs a GPU")
    from det3d.models import build_detector
    from det3d.torchie import Config
    from sessd_b200.train import ArenaAdamW, ParamArena, update_ema_variables

    cfg = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg).cuda()
    ema = copy.deepcopy(model)
    arena, arena_ema = ParamArena(model), ParamArena(ema, with_grad=False)
    views = [p for p in model.parameters()]
    opt = ArenaAdamW(arena, lr=1e-3, weight_decay=0.01)
    g = torch.Generator(device="cuda").manual_seed(0)
    grads = torch.randn(arena.numel, device="cuda", generator=g) * 0.05      # norm ~100: every step clips
    n_params = sum(p.numel() for p in views)

    def fused():
        arena.grad_flat.copy_(grads)
        opt.step(max_grad_norm=35.0, ema=arena_ema, global_step=100)

    def unfused():
        arena.grad_flat.copy_(grads)
        torch.nn.utils.clip_grad_norm_(views, max_norm=35.0)
        opt.step()
        update_ema_variables(arena, arena_ema, 100)

    def refill():
        arena.grad_flat.copy_(grads)

    def time_of(fn):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.reps):
            fn()
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) * 1e3 / a.reps                             # us per call

    for fn in (fused, unfused, refill):
        for _ in range(a.warmup):
            fn()
    torch.cuda.synchronize()
    t = {"fused": [], "unfused": [], "refill": []}
    for _ in range(a.rounds):
        for name, fn in (("fused", fused), ("unfused", unfused), ("refill", refill)):
            t[name].append(time_of(fn))
    sm_clock = sm_clock_mhz()
    med = {k: float(np.median(v)) for k, v in t.items()}
    name, pl = card()
    print(json.dumps(dict(
        gpu=name, power_limit=pl, sm_clock_mhz_now_max=sm_clock, params=n_params, arena_floats=int(arena.numel),
        tail_us=dict(fused=round(med["fused"] - med["refill"], 1), unfused=round(med["unfused"] - med["refill"], 1)),
        with_grad_refill_us={k: [round(x, 1) for x in v] for k, v in t.items()},
        bytes_per_param=dict(fused=44, unfused=52),
        note="tail_us = median per call minus the median of the gradient refill (a 2 x 4 B/param copy) both paths start with")))


if __name__ == "__main__":
    main()
