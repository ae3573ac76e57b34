"""One SE-SSD training step at the training shape (BASELINE config #3: student + teacher forward, loss, backward, AdamW, EMA; batch 8,
ring-20k clouds, seeded GT boxes, targets from TargetAssigner.assign_batch_gpu, identity augmentation).  Prints one JSON object with the
card's name, power limit and SM clock, the step time from CUDA events after warm-up (median, min, max), per-launch neck / head forward, data-gradient
and weight-gradient times of the BevConvFunction on that launch's shapes (CUDA events; the gradient times include the split of the output
gradient into planes) with TFLOP/s from FLOPs computed from the shapes (each of the three products counted as the launch's forward FLOPs),
and a torch.profiler kernel table of one step from a separate run.

    python scripts/bench_train_step.py [--batch 8] [--steps 20] [--warmup 5] [--layer-reps 10] [--recipe]

--recipe runs the reference's optimiser recipe: the one-cycle lr / momentum schedule before each step, and clip (max-norm 35), AdamW
and the teacher EMA as one fused device pass (ArenaAdamW.step(max_grad_norm=35, ema=..., global_step=...)).
"""
import argparse
import copy
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "se-ssd_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)

from bench_encoder_train import card  # noqa: E402


def timed(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        fn()
        e1.record()
        torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return dict(median=round(float(np.median(ts)), 3), min=round(float(np.min(ts)), 3), max=round(float(np.max(ts)), 3), n=len(ts),
                all=[round(t, 2) for t in ts])


def sm_clock_mhz():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=clocks.sm,clocks.max.sm", "--format=csv,noheader", "-i",
                               str(torch.cuda.current_device())], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        return "unknown"


def launch_flop(L, in_hw, out_hw, batch):
    """forward FLOPs of one neck / head launch: 2 Cin Cout per tap and output pixel (conv), per tap and input pixel (deconv)"""
    if L.kind == "deconv":
        return 2.0 * batch * in_hw[0] * in_hw[1] * L.cin * L.cout * 9
    return 2.0 * batch * out_hw[0] * out_hw[1] * L.cin * L.cout * L.k * L.k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--layer-reps", type=int, default=10)
    ap.add_argument("--recipe", action="store_true")
    a = ap.parse_args()
    from det3d.models import build_detector
    from det3d.torchie import Config
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
    from sessd_b200 import bev_grad, synth, weights
    from sessd_b200.train import ArenaAdamW, ParamArena, update_ema_variables
    from sessd_data.layers import SSFA_LAUNCHES, ssfa_extents

    cfg = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    model.load_state_dict(weights.random_detector_state(0), strict=True)       # the benchmark's weights (bench.py)
    model = model.cuda().train()
    ema = copy.deepcopy(model)
    for p in ema.parameters():
        p.requires_grad_(False)
    arena, arena_ema = ParamArena(model), ParamArena(ema, with_grad=False)
    opt = ArenaAdamW(arena, lr=1e-3)
    clouds = [synth.ring_cloud(b, 20000) for b in range(a.batch)]
    gts = []
    for b in range(a.batch):
        gt = synth.random_boxes(100 + b, 15, spread=0.4)[0]
        gt[:, 2] = -1.0
        gts.append(gt)
    ex = synth.train_batch(cfg, clouds, gts)
    state = dict(n=0)
    if a.recipe:
        from det3d.solver import OneCycle
        sched = OneCycle(opt, a.steps + a.warmup + 3, 0.003, [0.95, 0.85], 10.0, 0.4)

    def step():
        arena.zero_grad()
        if a.recipe:
            sched.step(state["n"])
        out = batch_processor_inline(model, ema, ex, consistency_weight=1.0, train_mode=True)
        out["loss"].backward()
        if a.recipe:
            opt.step(max_grad_norm=35.0, ema=arena_ema, global_step=state["n"])
            state["n"] += 1
            return
        opt.step()
        state["n"] += 1
        update_ema_variables(arena, arena_ema, state["n"])

    step_ms = timed(step, a.steps, a.warmup)
    sm_clock = sm_clock_mhz()                                   # right after the timed steps: the clock the card ran them at

    h, w = 200, 176
    layers, g = [], torch.Generator(device="cuda").manual_seed(1)
    Fn = bev_grad.BevConvFunction
    for L in SSFA_LAUNCHES:
        in_hw, out_hw = ssfa_extents(L, h, w)
        wshape = (L.cin, L.cout, 3, 3) if L.kind == "deconv" else (L.cout, L.cin, L.k, L.k)
        W = (torch.randn(wshape, device="cuda", generator=g) * 0.05).requires_grad_(True)
        bias = torch.zeros(L.cout, device="cuda", requires_grad=True) if L.name == "head" else None
        x = torch.relu(torch.randn((a.batch,) + in_hw + (L.cin,), device="cuda", generator=g)).requires_grad_(True)
        with torch.no_grad():
            t_fwd = timed(lambda: Fn.apply(x, W, bias, L, in_hw, out_hw), a.layer_reps, 2)
        # one graph per gradient: the Function computes every gradient its inputs require
        y_x = Fn.apply(x, W.detach(), None, L, in_hw, out_hw)
        y_w = Fn.apply(x.detach(), W, None, L, in_hw, out_hw)
        gy = torch.randn(y_x.shape, device="cuda", generator=g)
        t_dx = timed(lambda: torch.autograd.grad(y_x, x, gy, retain_graph=True), a.layer_reps, 2)
        t_dw = timed(lambda: torch.autograd.grad(y_w, W, gy, retain_graph=True), a.layer_reps, 2)
        flop = launch_flop(L, in_hw, out_hw, a.batch)
        tf = lambda t: round(flop / t["median"] * 1e-9, 2)       # noqa: E731
        layers.append(dict(name=L.name, kind=L.kind, cin=L.cin, cout=L.cout, k=L.k, stride=L.stride, gflop=round(flop * 1e-9, 2),
                           fwd_ms=t_fwd["median"], dgrad_ms=t_dx["median"], wgrad_ms=t_dw["median"], fwd_tflops=tf(t_fwd),
                           dgrad_tflops=tf(t_dx), wgrad_tflops=tf(t_dw)))
        del y_x, y_w
    neck_gflop = sum(l["gflop"] for l in layers)

    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "cuda" in str(ev.device_type).lower() and ev.device_time_total > 0:
            kernels[ev.key] = dict(calls=int(ev.count), us=round(float(ev.device_time_total), 1))
    tops = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["us"])[:30])
    name, pl = card()
    print(json.dumps(dict(gpu=name, power_limit=pl, sm_clock_mhz_now_max=sm_clock, batch=a.batch, recipe=a.recipe, step_ms=step_ms,
                          neck_head_fwd_gflop=round(neck_gflop, 2), neck_head_bwd_gflop=round(2 * neck_gflop, 2),
                          neck_fwd_ms=round(sum(l["fwd_ms"] for l in layers), 3),
                          neck_dgrad_ms=round(sum(l["dgrad_ms"] for l in layers), 3),
                          neck_wgrad_ms=round(sum(l["wgrad_ms"] for l in layers), 3), layers=layers, kernels=tops)))


if __name__ == "__main__":
    main()
