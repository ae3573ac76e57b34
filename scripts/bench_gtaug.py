"""Time GT-database sampling (GT-AUG) in the device-built SE-SSD training batch: batch 8 of ring-20k clouds with 3 GT boxes per frame
(2 cars and a pedestrian, so every frame asks the sampler for 13 cars), on a synthetic car database.  Prints one JSON object with the
card's name and power limit (read in the same run), the database size, and, from CUDA events after warm-up (median, min, max):
  * build_train_batch_ms / build_train_batch_gtaug_ms: sessd_b200.augment.build_train_batch without and with db_sampler;
  * paste_ms: ops.gtaug_paste on resident inputs (the kernels of csrc/gtaug.cu and its survivor scan, plus the wrapper);
  * select_host_ms: DataBaseSamplerV2.select for the 8 frames (host, perf_counter);
  * oracle_paste_host_ms: the ORACLE's numpy paste (oracle/gt_aug_ref.py paste: gather + point removal) of the same 8 frames on this
    machine's CPU -- a stand-in for the reference's host path, which is not measured here.

    python scripts/bench_gtaug.py [--batch 8] [--steps 20] [--warmup 3] [--objects 3000] [--tiny]

--tiny is a CPU rehearsal: a small database and batch, host timings only.
"""
import argparse
import json
import os
import pickle
import sys
import tempfile
import time

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "se-ssd_b200"))
sys.path.insert(0, ROOT)
sys.path.insert(0, HERE)


def database(root, n_obj, seed=0):
    """cars (and 1 in 12 pedestrians) on a ring band in front of the sensor, 20..400 points each; returns (pickle path, mean points)"""
    rs = np.random.RandomState(seed)
    infos = {"Car": [], "Pedestrian": []}
    os.makedirs(os.path.join(root, "gt_database"), exist_ok=True)
    total = 0
    for k in range(n_obj):
        name = "Car" if k % 12 else "Pedestrian"
        r, a = rs.uniform(6, 60), rs.uniform(-0.7, 0.7)
        dims = [1.6, 3.9, 1.56] if name == "Car" else [0.6, 0.8, 1.73]
        b = np.array([r * np.cos(a), r * np.sin(a), -1.0] + dims + [rs.uniform(-np.pi, np.pi)], np.float64)
        n = int(rs.randint(20, 400))
        p = np.concatenate([(rs.uniform(-0.5, 0.5, (n, 3)) * b[3:6]), rs.uniform(0, 1, (n, 1))], 1).astype(np.float32)
        path = "gt_database/%06d_%s_0.bin" % (k, name)
        p.tofile(os.path.join(root, path))
        total += n
        infos[name].append(dict(name=name, path=path, image_idx=k, gt_idx=0, box3d_lidar=b, num_points_in_gt=n, difficulty=0, group_id=k))
    with open(os.path.join(root, "dbinfos_train.pkl"), "wb") as f:
        pickle.dump(infos, f)
    return os.path.join(root, "dbinfos_train.pkl"), total / max(n_obj, 1)


def frames(batch, n_points, seed=300):
    from sessd_data import synth
    clouds = [synth.ring_cloud(seed + b, n_points, 15) for b in range(batch)]
    boxes = [synth.ring_boxes(seed + b, 15)[:3].astype(np.float64) for b in range(batch)]
    names = [np.array(["Car", "Car", "Pedestrian"]) for _ in range(batch)]
    return clouds, boxes, names


def host_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median=round(float(np.median(ts)), 3), min=round(float(np.min(ts)), 3), max=round(float(np.max(ts)), 3), n=len(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--objects", type=int, default=3000)
    ap.add_argument("--tiny", action="store_true")
    a = ap.parse_args()
    from det3d.builder import build_dbsampler
    from det3d.torchie import Config
    from oracle import gt_aug_ref
    batch, n_points, n_obj = (2, 2000, 200) if a.tiny else (a.batch, 20000, a.objects)
    d = json.load(open(os.path.join(ROOT, "tests", "golden", "reference_config.json")))     # the upstream config's values, plus its two
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))   # constructed objects from the repo's config
    d["model"]["neck"]["logger"] = ours.model.neck.logger
    d["model"]["bbox_head"]["box_coder"] = ours.model.bbox_head.box_coder
    cfg = Config(d)
    sampler_cfg = dict(cfg.db_sampler)                                                        # the reference's db_sampler, a local database
    out = dict(batch=batch, points_per_frame=n_points, gt_per_frame=3, cars_asked_per_frame=13)
    with tempfile.TemporaryDirectory() as tmp:
        sampler_cfg["db_info_path"], mean_pts = database(tmp, n_obj)
        rs = np.random.RandomState(0)
        sampler = build_dbsampler(sampler_cfg, random_state=rs)
        sampler.load_database()
        out["database"] = dict(objects=n_obj, mean_points_per_object=round(mean_pts, 1), points_per_object="uniform 20..399")
        clouds, boxes, names = frames(batch, n_points)
        ids = []
        out["select_host_ms"] = host_ms(lambda: ids.append([sampler.select(b, list(n)) for b, n in zip(boxes, names)]), a.steps)
        last = ids[-1]
        out["accepted_per_frame"] = [len(i) for i in last]
        rel = [sampler._points[o:o + n] for o, n in zip(sampler.offsets, sampler.counts)]
        out["oracle_paste_host_ms"] = host_ms(lambda: [gt_aug_ref.paste(c, b, n, i, rel, sampler.boxes, sampler.names)
                                                       for c, b, n, i in zip(clouds, boxes, names, last)], 3)
        if not a.tiny and torch.cuda.is_available():
            from bench_encoder_train import card
            from bench_train_step import timed
            from sessd_b200 import augment, ops
            out["gpu"], out["power_limit"] = card()
            rs2 = np.random.RandomState(1)
            out["build_train_batch_ms"] = timed(lambda: augment.build_train_batch(cfg, clouds, boxes, names, rs2), a.steps, a.warmup)
            sampler._set_random_state(rs2)
            out["build_train_batch_gtaug_ms"] = timed(lambda: augment.build_train_batch(cfg, clouds, boxes, names, rs2, db_sampler=sampler),
                                                      a.steps, a.warmup)
            db = sampler.device_database("cuda")
            pts = torch.from_numpy(np.concatenate(clouds).astype(np.float32)).cuda()
            off = torch.from_numpy(np.concatenate([[0], np.cumsum([len(c) for c in clouds])]).astype(np.int32)).cuda()
            oo = torch.from_numpy(np.concatenate([[0], np.cumsum([len(i) for i in last])]).astype(np.int32)).cuda()
            oi = torch.from_numpy(np.concatenate(last).astype(np.int32)).cuda()
            mp = int(sampler.counts[np.concatenate(last)].sum())
            out["pasted_points_per_batch"] = mp
            out["paste_ms"] = timed(lambda: ops.gtaug_paste(pts, off, oo, oi, db["points"], db["off"], db["count"], db["boxes"], mp),
                                    a.steps, a.warmup)
            for k in ("build_train_batch_ms", "build_train_batch_gtaug_ms", "paste_ms"):
                out[k].pop("all", None)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
