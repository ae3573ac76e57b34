"""Time detection post-processing with DI-NMS (nms_type "rotate_weighted_nms") against the default rotated NMS on the H100.  Prints
one JSON object with the card's name and power limit (read in the same run) and, from CUDA events after warm-up (median, min, max):
  * post_ms[mode][workload][batch]: ops.postprocess of both modes, alternated call by call, at batch 1 and 8, on
    - "bench": head maps of the bench's ring-20k clouds and weights (FrameEngine), ~400 candidates per frame;
    - "saturated": synthetic heads with >= 1000 candidates per frame, so k = nms_pre_max = 1000;
  * kernel_us[workload]: the DI-NMS overlap stage (dinms_iou_kernel) and cluster loop (dinms_cluster_kernel) per call at batch 8, from
    torch.profiler in a run of its own;
  * picks / clusters / candidates per frame;
  * engine_fps[mode]: FrameEngine graph replays at batch 8 on the ring-20k clouds (input copies included).

    python scripts/bench_dinms.py [--steps 50] [--warmup 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path[:0] = [os.path.join(ROOT, "se-ssd_b200"), ROOT]

MODES = ("rotate_nms", "rotate_weighted_nms")


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def stats(v):
    v = np.asarray(v, np.float64)
    return dict(median=float(np.median(v)), min=float(v.min()), max=float(v.max()))


def saturated_heads(batch, seed=0, n_pos=3000):
    rng = np.random.default_rng(seed)
    h = np.zeros((batch, 200, 176, 24), np.float32)
    h[..., 0:14] = rng.normal(0, 0.25, h[..., 0:14].shape)
    h[..., 14:16] = -4.0
    h[..., 16:20] = rng.normal(0, 1, h[..., 16:20].shape)
    h[..., 20:22] = rng.uniform(-0.5, 1.0, h[..., 20:22].shape)
    for b in range(batch):
        ys, xs, rs = rng.integers(0, 200, n_pos), rng.integers(0, 176, n_pos), rng.integers(0, 2, n_pos)
        h[b, ys, xs, 14 + rs] = rng.uniform(-0.8, 4.0, n_pos)
    return torch.from_numpy(h.reshape(batch, -1, 24)).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dinms.py measures on the GPU; there is no CPU mode"
    from sessd_b200 import ops, synth, weights
    from sessd_b200.engine import FrameEngine

    anchors_np = weights.kitti_car_anchors()
    anchors = torch.from_numpy(anchors_np).cuda()
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    clouds = [synth.ring_cloud(100 + i, 20000) for i in range(8)]
    out = dict(card=card(), steps=args.steps, warmup=args.warmup, post_ms={}, kernel_us={}, per_frame={}, engine_fps={})

    # head maps of the bench frames
    eng = FrameEngine(batch=8, max_points_per_frame=20000)
    eng.load_weights(layers, ssfa, head, anchors_np)
    eng.infer(clouds)
    bench_heads = eng.neck.buf["head"].reshape(8, -1, eng.neck.buf["head"].shape[-1]).clone()
    heads = {"bench": bench_heads, "saturated": saturated_heads(8)}
    stride = {k: int(v.shape[-1]) for k, v in heads.items()}

    for wl, hd8 in heads.items():
        for batch in (1, 8):
            hd = hd8[:batch].contiguous()
            bufs = {m: ops.PostBuffers(ops.make_post_cfg(batch=batch, head_stride=stride[wl], nms_type=m), "cuda") for m in MODES}
            times = {m: [] for m in MODES}
            for it in range(args.warmup + args.steps):
                for m in MODES:                      # alternated, call by call
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    ops.postprocess(hd, anchors, None, bufs[m])
                    e1.record()
                    torch.cuda.synchronize()
                    if it >= args.warmup:
                        times[m].append(e0.elapsed_time(e1))
            for m in MODES:
                out["post_ms"].setdefault(m, {}).setdefault(wl, {})[str(batch)] = stats(times[m])
            if batch == 8:
                aux = bufs["rotate_weighted_nms"].aux.cpu().numpy()
                out["per_frame"][wl] = dict(candidates=stats(aux[:, 1]), picks=stats(aux[:, 3]), clusters=stats(aux[:, 2]),
                                            rotate_nms_kept=stats(bufs["rotate_nms"].aux.cpu().numpy()[:, 2]))
                # kernel times of the two DI-NMS stages (profiler run of its own)
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    for _ in range(20):
                        ops.postprocess(hd, anchors, None, bufs["rotate_weighted_nms"])
                    torch.cuda.synchronize()
                ks = {}
                for ev in prof.key_averages():
                    for name in ("dinms_iou_kernel", "dinms_cluster_kernel", "post_finalize_kernel", "post_select_kernel", "post_score_kernel"):
                        if name in ev.key:
                            ks[name] = ks.get(name, 0.0) + ev.device_time_total / 20.0
                out["kernel_us"][wl] = ks

    for m in MODES:
        e = FrameEngine(batch=8, max_points_per_frame=20000, post_kwargs={"nms_type": m})
        e.load_weights(layers, ssfa, head, anchors_np)
        e.stage(clouds)
        e.capture()
        for _ in range(args.warmup):
            e.launch()
        e.stream.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        with torch.cuda.stream(e.stream):
            e0.record()
        for _ in range(args.steps):
            e.launch()
        with torch.cuda.stream(e.stream):
            e1.record()
        e.stream.synchronize()
        out["engine_fps"][m] = 8 * args.steps / (e0.elapsed_time(e1) / 1e3)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
