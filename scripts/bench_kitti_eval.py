"""Time the full KITTI evaluation (official R11 + R40 + COCO, with AOS) on the device, on a KITTI-val-shaped synthetic set: 3769
frames, up to 100 detections and about 8 ground-truth + DontCare boxes per frame, detections as lidar-frame device tensors.  The timed
region is the detection conversion, the three metrics' kernels (cars, pedestrians, cyclists; 2 official + 10 COCO min-overlap sets)
and the one copy of their results back to the host.  CUDA events, median over --reps runs after --warmup.  The
numpy oracle (oracle/kitti_eval_ref.py) is timed on the CPU on the first --oracle-frames frames, and labelled as such.  Prints one
JSON object with the card's name and power limit.

    python scripts/bench_kitti_eval.py [--frames 3769] [--reps 5] [--warmup 2] [--oracle-frames 100]
"""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "se-ssd_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
sys.path.insert(0, HERE)

from bench_encoder_train import card  # noqa: E402
from kitti_eval_cases import CLASSES, calib  # noqa: E402
from oracle import kitti_eval_ref as ref  # noqa: E402

_SIZE = {0: (1.6, 3.9, 1.56), 1: (0.6, 0.8, 1.73), 2: (0.6, 1.76, 1.73)}


def synth(frames, seed=0, max_dets=100):
    """Infos with ground truth (cars, vans, pedestrians, cyclists, one DontCare) and lidar detections around them plus clutter."""
    rng = np.random.default_rng(seed)
    names_pool = ["Car", "Car", "Car", "Car", "Van", "Pedestrian", "Cyclist"]
    infos, dets = [], []
    for f in range(frames):
        info = {"image": {"image_idx": f, "image_shape": np.array([375, 1242])}, "calib": calib(rng)}
        ng = int(rng.integers(4, 12))
        names = [names_pool[i] for i in rng.integers(0, len(names_pool), ng)]
        lab = np.array([{"Pedestrian": 1, "Cyclist": 2}.get(n, 0) for n in names])
        x = rng.uniform(5, 45, ng)
        box = np.stack([x, rng.uniform(-0.4, 0.4, ng) * x, np.full(ng, -1.0)] +
                       [np.array([_SIZE[l][i] for l in lab]) * rng.uniform(0.9, 1.1, ng) for i in range(3)] +
                       [rng.uniform(-np.pi, np.pi, ng)], 1).astype(np.float32)
        a = ref.convert_frame(box, np.ones(ng, np.float32), np.arange(ng), info, names)
        n = len(a["name"])
        a["occluded"] = rng.integers(0, 3, n)
        a["truncated"] = rng.choice([0.0, 0.1, 0.3], n)
        a.pop("score")
        a["name"] = np.concatenate([a["name"], ["DontCare"]])
        a["bbox"] = np.concatenate([a["bbox"].reshape(-1, 4), [[500.0, 150.0, 560.0, 200.0]]])
        for k, v in (("alpha", -10.0), ("rotation_y", -10.0), ("truncated", -1.0), ("occluded", -1)):
            a[k] = np.concatenate([a[k], [v]])
        a["location"] = np.concatenate([a["location"].reshape(-1, 3), [[-1000.0] * 3]])
        a["dimensions"] = np.concatenate([a["dimensions"].reshape(-1, 3), [[-1.0] * 3]])
        info["annos"] = a
        nd = int(rng.integers(0, max_dets + 1))
        hit = box[rng.integers(0, ng, min(nd, 2 * ng))].copy()
        hit[:, :2] += rng.normal(0, 0.3, (len(hit), 2)).astype(np.float32)
        hit[:, 6] += rng.normal(0, 0.1, len(hit)).astype(np.float32)
        nc = nd - len(hit)
        xc = rng.uniform(3, 60, nc)
        clutter = np.stack([xc, rng.uniform(-0.6, 0.6, nc) * xc, np.full(nc, -1.0), np.full(nc, 1.6), np.full(nc, 3.9), np.full(nc, 1.5),
                            rng.uniform(-np.pi, np.pi, nc)], 1).astype(np.float32)
        b = np.concatenate([hit, clutter]).astype(np.float32)
        dets.append((b, rng.uniform(0.05, 1, len(b)).astype(np.float32), rng.integers(0, 3, len(b))))
        infos.append(info)
    return infos, dets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=3769)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--oracle-frames", type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_kitti_eval.py needs a GPU")
    from det3d.datasets.kitti.eval import evaluate_all
    from sessd_b200 import kitti_eval as ke

    infos, dets = synth(a.frames)
    gt = ke.DeviceGT([i["annos"] for i in infos])
    cal = ke.DeviceCalib(infos)
    dev = [tuple(torch.from_numpy(x).cuda() for x in d) for d in dets]

    def run():
        dt, _ = ke.convert_detections(dev, cal, CLASSES)
        return evaluate_all(ke.Frames(gt, dt), CLASSES, True)

    for _ in range(a.warmup):
        run()
    times = []
    for _ in range(a.reps):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record()
        official, _, _ = run()
        e.record()
        torch.cuda.synchronize()
        times.append(s.elapsed_time(e))
    n = a.oracle_frames
    dt_annos = [ref.convert_frame(b, sc, lb, info, CLASSES) for (b, sc, lb), info in zip(dets[:n], infos[:n])]
    classes = [0, 1, 10]
    from det3d.datasets.kitti.eval import OFFICIAL_OVERLAPS, _coco_overlaps
    mo = np.concatenate([OFFICIAL_OVERLAPS[:, :, classes], _coco_overlaps(classes)], axis=0)
    t0 = time.perf_counter()
    ref.evaluate([i["annos"] for i in infos[:n]], dt_annos, classes, [0, 1, 2], mo)
    t_oracle = time.perf_counter() - t0
    name, pl = card()
    print(json.dumps({"card": name, "power_limit": pl, "frames": a.frames, "detections": int(sum(len(d[0]) for d in dets)),
                      "gt_boxes": int(gt.total), "device_eval_ms_median": float(np.median(times)), "device_eval_ms_all": times,
                      "oracle_cpu_frames": n, "oracle_cpu_s": t_oracle, "car_r11_moderate": official["detail"]["car"]["3d@0.70"][1]}))


if __name__ == "__main__":
    main()
