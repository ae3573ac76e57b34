"""Measure the KITTI data preparation (sessd_b200.kitti_prep.kitti_data_prep) on a synthetic KITTI-shaped tree.

    python scripts/bench_kitti_prep.py [--frames 256] [--points 120000] [--oracle-frames 8]

Writes, under a temporary directory, FRAMES training frames (half train, half val) and a few test frames of 64-beam-like 360-degree ring
clouds with 12 labelled cars each, then reports: the full preparation in frames per second (files included; the tree was just written,
so the page cache is warm), the device stages alone (CUDA events, summed over batches), and the numpy oracle's reduce + count + database
per frame on this host's CPU over a subset.  Prints one JSON line.
"""
import json
import os
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "se-ssd_b200"), os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def main():
    import argparse
    import torch

    import kitti_prep_cases as cases
    from oracle import kitti_prep_ref as ref
    from sessd_b200 import kitti_prep
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=256)
    ap.add_argument("--points", type=int, default=120000)
    ap.add_argument("--oracle-frames", type=int, default=8)
    a = ap.parse_args()
    rs = np.random.RandomState(0)
    with tempfile.TemporaryDirectory() as root:
        n = a.frames
        ids = {"train": list(range(0, n, 2)), "val": list(range(1, n, 2)), "test": [0, 1]}
        os.makedirs(os.path.join(root, "ImageSets"))
        for s, v in ids.items():
            with open(os.path.join(root, "ImageSets", s + ".txt"), "w") as f:
                f.write("".join("%06d\n" % i for i in v))
        for part, cnt in (("training", n), ("testing", 2)):
            for d in ("calib", "label_2", "velodyne", "image_2"):
                os.makedirs(os.path.join(root, part, d))
            for k in range(cnt):
                with open(os.path.join(root, part, "image_2", "%06d.png" % k), "wb") as f:
                    f.write(cases.png(*cases.SIZES[k % 4]))
                text, _ = cases.calib(rs, k % 7)
                with open(os.path.join(root, part, "calib", "%06d.txt" % k), "w") as f:
                    f.write(text)
                objs = [cases.objects(3)[0][:6] + ((rs.uniform(-15, 15), 1.7, rs.uniform(5, 60)), rs.uniform(-3, 3)) for _ in range(12)]
                with open(os.path.join(root, part, "label_2", "%06d.txt" % k), "w") as f:
                    f.write(cases.label_text(objs))
                beam = rs.randint(0, 64, a.points)
                az = rs.uniform(-np.pi, np.pi, a.points)
                el = np.deg2rad(-24.9 + beam * (26.9 / 63))
                r = rs.uniform(3, 80, a.points)
                pts = np.stack([r * np.cos(el) * np.cos(az), r * np.cos(el) * np.sin(az), 1.73 + r * np.sin(el), rs.uniform(0, 1, a.points)], 1)
                pts.astype(np.float32).tofile(os.path.join(root, part, "velodyne", "%06d.bin" % k))
        kitti_prep.kitti_data_prep(root, batch_frames=16)          # warm-up (CUDA context, page cache)
        torch.cuda.synchronize()
        ev = []
        orig = kitti_prep.Runner.run

        def run(self, frames, cb):
            orig(self, frames, cb)
            ev.append(self.event_ms)
        kitti_prep.Runner.run = run
        t0 = time.perf_counter()
        kitti_prep.kitti_data_prep(root, batch_frames=16)
        wall = time.perf_counter() - t0
        kitti_prep.Runner.run = orig
        total = n + 2
        infos = kitti_prep.image_info(root, 0, True, True, True, True)
        t1 = time.perf_counter()
        for k in range(a.oracle_frames):
            info = kitti_prep.image_info(root, 2 * k, True, True, True, True)
            raw = np.fromfile(os.path.join(root, info["point_cloud"]["velodyne_path"]), np.float32).reshape(-1, 4)
            c = info["calib"]
            red = ref.reduce_frame(raw, c["R0_rect"], c["Tr_velo_to_cam"], c["P2"], info["image"]["image_shape"])
            ref.num_points_in_gt(red, info)
            ref.db_objects(red, info)
        cpu = (time.perf_counter() - t1) / a.oracle_frames
        del infos
        print(json.dumps({"frames": total, "points_per_frame": a.points, "objects_per_frame": 12, "page_cache": "warm",
                          "full_prep_fps": round(total / wall, 1), "full_prep_s": round(wall, 3),
                          "device_stages_ms": round(sum(ev), 2), "oracle_cpu_ms_per_frame": round(1000 * cpu, 1),
                          "gpu": torch.cuda.get_device_name(0)}))


if __name__ == "__main__":
    main()
