"""Device time of each of the 13 BEV neck conv / deconv launches of the frame-ring workload (ring-20k cloud, batch 1), each launch timed
alone with CUDA events on the engine stream and the L2 flushed before every launch (as bench.py's roofline leg times one layer).  Two
settings per launch: `dense` runs every work item; `skip` runs the work items of the frame's skip plan plus the fill of the skipped tiles,
as the frame graph does.  Writes JSON to --out and prints a table.

    python scripts/neck_layers.py --out FILE [--reps 20]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "se-ssd_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)


def launches(neck):
    """(name, closure(skip)) of the 13 launches of SSFAPlanesRunner.forward"""
    from sessd_data.layers import SSFA_LAUNCHES
    return [(L.name, lambda skip, L=L: neck._launch(L, skip)) for L in SSFA_LAUNCHES]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    a = ap.parse_args()

    import numpy as np
    import torch

    from sessd_b200.engine import FrameEngine
    from sessd_data import synth, weights

    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    eng = FrameEngine(batch=1)
    eng.load_weights(layers, ssfa, head, weights.kitti_car_anchors())
    for s in range(4):                   # module loads; the neck's buffers, info slots and skip plan then hold a real frame's state
        eng.infer([synth.ring_cloud(s, 20000)])
    torch.cuda.synchronize()
    neck = eng.neck
    flush = torch.empty((64 * 1024 * 1024,), dtype=torch.float32, device=eng.device)     # 256 MB > L2
    res = dict(gpu=torch.cuda.get_device_name(), reps=a.reps, layers={})
    with torch.cuda.stream(eng.stream):
        for name, launch in launches(neck):
            rec = {}
            for mode in ("dense", "skip"):
                skip = mode == "skip"
                for _ in range(3):
                    launch(skip)
                ms = []
                for _ in range(a.reps):
                    flush.zero_()
                    t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    t0.record(eng.stream)
                    launch(skip)
                    t1.record(eng.stream)
                    eng.stream.synchronize()
                    ms.append(t0.elapsed_time(t1))
                rec[mode + "_us"] = float(np.mean(ms)) * 1000.0
                rec[mode + "_us_min"] = float(np.min(ms)) * 1000.0
            res["layers"][name] = rec
    res["total_dense_us"] = sum(r["dense_us"] for r in res["layers"].values())
    res["total_skip_us"] = sum(r["skip_us"] for r in res["layers"].values())
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print("neck launches alone (us, mean of %d, L2 flushed), %s" % (a.reps, res["gpu"]))
    for name, r in res["layers"].items():
        print("  %-20s dense %8.1f   skip %8.1f" % (name, r["dense_us"], r["skip_us"]))
    print("  %-20s dense %8.1f   skip %8.1f" % ("total", res["total_dense_us"], res["total_skip_us"]))


if __name__ == "__main__":
    main()
