"""Multi-class inference cost: FrameEngine frames/s with one task (Car) and three (Car, Pedestrian, Cyclist) on seeded ring-20k clouds
and seeded random weights, the two engines alternated in one run, plus the post-processing alone at T = 1 and T = 3 on the head maps
those engines produce.  Prints one JSON line with the card's name and power limit, read in the same run.

    python scripts/bench_multiclass.py [--frames 200] [--rounds 5] [--out results/bench_multiclass.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "se-ssd_b200"))

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else torch.cuda.get_device_name(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=200, help="frames per timed window")
    ap.add_argument("--rounds", type=int, default=5, help="alternated windows per engine")
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_multiclass needs a GPU"
    from sessd_b200 import ops, weights
    from sessd_b200.engine import FrameEngine
    from sessd_data import synth
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    head3 = dict(head)
    for t in (1, 2):                                    # two more tasks at the car head's scale
        for k, v in head.items():
            if k.startswith("tasks.0."):
                head3[k.replace("tasks.0.", "tasks.%d." % t)] = v * (1.0 - 0.05 * t) if k.endswith("weight") else v + 0.2 * t
    gens = [dict(type="anchor_generator_range", sizes=s, anchor_ranges=[0, -40.0, z, 70.4, 40.0, z], rotations=[0, 1.57])
            for s, z in (([1.6, 3.9, 1.56], -1.0), ([0.6, 0.8, 1.73], -0.6), ([0.6, 1.76, 1.73], -0.6))]
    anchors = weights.task_anchors(dict(anchor_generators=gens))
    clouds = [synth.ring_cloud(j, 20000) for j in range(16)]
    eng = {1: FrameEngine(batch=1, max_points_per_frame=20000), 3: FrameEngine(batch=1, max_points_per_frame=20000, num_tasks=3)}
    eng[1].load_weights(layers, ssfa, head, anchors[0])
    eng[3].load_weights(layers, ssfa, head3, anchors)
    for e in eng.values():
        e.stage([clouds[0]])
        e.capture()
        e.launch()
        e.results()
    dets = {T: [] for T in eng}
    fps = {T: [] for T in eng}
    for _ in range(a.rounds):
        for T, e in eng.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for f in range(a.frames):
                e.stage([clouds[f % len(clouds)]])
                e.launch()
                r = e.results()[0]
                if f < len(clouds):
                    dets[T].append(len(r["scores"]))
            fps[T].append(a.frames / (time.perf_counter() - t0))
    # post-processing alone on the head map of the last frame, CUDA events around many calls
    post = {}
    for T, e in eng.items():
        head_map = e.neck.buf["head"]
        for _ in range(10):
            ops.postprocess(head_map, e.anchors, None, e.post)
        torch.cuda.synchronize()
        st, en = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        times = []
        for _ in range(a.rounds):
            st.record()
            for _ in range(100):
                ops.postprocess(head_map, e.anchors, None, e.post)
            en.record()
            en.synchronize()
            times.append(st.elapsed_time(en) / 100 * 1000.0)
        post[T] = times
    line = dict(card=card(), frames_per_window=a.frames, rounds=a.rounds,
                frames_per_s={"T1": fps[1], "T3": fps[3]},
                frames_per_s_median={"T1": float(np.median(fps[1])), "T3": float(np.median(fps[3]))},
                postprocess_us_median={"T1": float(np.median(post[1])), "T3": float(np.median(post[3]))},
                postprocess_us={"T1": post[1], "T3": post[3]},
                detections_per_frame_mean={"T1": float(np.mean(dets[1])), "T3": float(np.mean(dets[3]))})
    print(json.dumps(line))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
