"""Time shape-aware augmentation (SA-DA) in the device-built SE-SSD training batch: batch 8 of ring-20k clouds with 15 cars, each car
carrying 400 surface points, with the car values of Preprocess (dropout 0.25, sparsity (0.05, 50), swap (0.1, 50)) and with raised
probabilities (0.4, (0.5, 50), (0.6, 50)) so that every stage fires.  Prints one JSON object with the card's name and power limit (read in
the same run) and, from CUDA events after warm-up (median, min, max):
  * kernels_ms: each SA-DA entry on frame 0's globally augmented points (pyramids, membership over all pyramids, compact, fps of the
    sparsified pyramids, swap of 8 pairs, the batch shuffle);
  * build_train_batch_ms / build_train_batch_sada_ms / build_train_batch_sada_raised_ms: sessd_b200.augment.build_train_batch without
    and with SA-DA, alternated step by step in one run;
  * readbacks_per_batch: the device-to-host waits of one batch with SA-DA (swap counts, frame sizes, the voxel totals);
  * oracle_sada_host_ms: tests/sada_ref.py's numpy SA-DA of the same 8 frames on this machine's CPU.  The reference's own path (numba
    plus cKDTree, with the external ifp package) is not measured.

    python scripts/bench_sada.py [--steps 20] [--warmup 3] [--tiny]

--tiny is a CPU rehearsal: two small frames, host timings only.
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
for p in (os.path.join(ROOT, "se-ssd_b200"), ROOT, HERE, os.path.join(ROOT, "tests")):
    sys.path.insert(0, p)

RAISED = dict(dropout=0.4, sparsity=(0.5, 50), swap=(0.6, 50))


def frames(batch, n_points, seed=40):
    from sessd_data import synth
    rs = np.random.RandomState(seed)
    clouds, boxes, names = [], [], []
    for b in range(batch):
        bx = synth.ring_boxes(seed + b, 15)
        surf = []
        for x in bx:
            q = rs.uniform(-0.5, 0.5, (400, 3))
            ax = rs.randint(0, 3, 400)
            q[np.arange(400), ax] = np.sign(q[np.arange(400), ax]) * 0.49
            q *= x[3:6]
            c, s = np.cos(x[6]), np.sin(x[6])
            surf.append(np.stack([q[:, 0] * c + q[:, 1] * s + x[0], -q[:, 0] * s + q[:, 1] * c + x[1], q[:, 2] + x[2],
                                  rs.uniform(0, 1, 400)], 1))
        clouds.append(np.concatenate([synth.ring_cloud(seed + b, n_points, 15)] + surf).astype(np.float32))
        boxes.append(bx)
        names.append(np.array(["Car"] * 13 + ["Van", "Pedestrian"]))
    return clouds, boxes, names


def host_ms(fn, reps):
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return dict(median=round(float(np.median(ts)), 3), min=round(float(np.min(ts)), 3), max=round(float(np.max(ts)), 3), n=len(ts))


def stats(ts):
    return dict(median=round(float(np.median(ts)), 3), min=round(float(np.min(ts)), 3), max=round(float(np.max(ts)), 3), n=len(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--tiny", action="store_true")
    a = ap.parse_args()
    import sada_ref
    from oracle import augment_ref
    from sessd_b200 import augment, sada
    from test_augment_oracle import reference_config
    cfg = reference_config()
    acfg = augment.AugmentConfig.from_config(cfg)
    batch, n_points = (2, 2000) if a.tiny else (8, 20000)
    clouds, boxes, names = frames(batch, n_points)
    out = dict(batch=batch, points_per_frame=len(clouds[0]), cars_per_frame=15, surface_points_per_car=400)
    # the frames as SA-DA receives them (after the noise and global stages), for the oracle and the kernel timings
    draws = augment.draw_augmentation(np.random.RandomState(0), [(len(c), len(b), True) for c, b in zip(clouds, boxes)], acfg)
    glob = []
    for b in range(batch):
        f = draws.frames[b]
        valid = np.array([n in acfg.class_names for n in names[b]])
        o = augment_ref.augment_frame(clouds[b], boxes[b], valid, dict(loc=f.loc, rot=f.rot, flip=f.flip, rotation=f.rotation,
                                                                        scale=f.scale, perm=np.arange(len(clouds[b]))))
        glob.append((o["points"], o["boxes"]))
    rs_o = np.random.RandomState(1)
    out["oracle_sada_host_ms"] = host_ms(lambda: [sada_ref.sada(p, bx, rs_o) for p, bx in glob], 3)
    if not a.tiny and torch.cuda.is_available():
        from bench_encoder_train import card
        from bench_train_step import timed
        from sessd_b200 import ops
        out["gpu"], out["power_limit"] = card()
        p0, b0 = (torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in glob[0])
        K = b0.shape[0]
        pyr, planes = ops.sada_pyramids(b0)
        ids_all = np.arange(6 * K)
        _, counts_all, _ = ops.sada_membership(p0, planes, ids_all, with_bits=False)
        cnt = counts_all.cpu().numpy().reshape(K, 6)
        big = [6 * i + int(np.argmax(cnt[i])) for i in range(K)]
        pairs = big[:8] + big[8:16][::-1] if K >= 16 else big[:K // 2] + big[K // 2:2 * (K // 2)]
        bits_s, counts_s, _ = ops.sada_membership(p0, planes, big)
        bits_w, counts_w, d_pairs = ops.sada_membership(p0, planes, pairs)
        extra = int(counts_w.sum().item())
        n0 = p0.shape[0]
        buf = torch.empty((n0 + 50 * len(big) + extra, 4), dtype=torch.float32, device="cuda")
        kept = torch.zeros((1,), dtype=torch.int32, device="cuda")
        allp = torch.cat([torch.from_numpy(np.ascontiguousarray(p)).cuda() for p, _ in glob])
        off = torch.from_numpy(np.concatenate([[0], np.cumsum([len(p) for p, _ in glob])]).astype(np.int32)).cuda()
        perm = torch.from_numpy(np.concatenate([np.random.RandomState(2).permutation(len(p)) for p, _ in glob]).astype(np.int32)).cuda()
        kern = dict(
            pyramids=lambda: ops.sada_pyramids(b0),
            membership_all_pyramids=lambda: ops.sada_membership(p0, planes, ids_all, with_bits=False),
            membership_bits=lambda: ops.sada_membership(p0, planes, big),
            compact=lambda: ops.sada_compact(p0, bits_s, counts_s, 50, out=buf),
            fps=lambda: ops.sada_fps(p0, bits_s, counts_s, 50, 50, buf, kept.zero_()),
            swap=lambda: ops.sada_swap(p0, bits_w, counts_w, pyr, d_pairs, extra, buf, kept.zero_()),
            shuffle=lambda: ops.sada_shuffle(allp, off, max(len(p) for p, _ in glob), perm))
        out["kernels_ms"] = {k: {kk: v for kk, v in timed(fn, a.steps, a.warmup).items() if kk != "all"} for k, fn in kern.items()}
        out["kernel_inputs"] = dict(points=n0, boxes=K, fps_pyramids=len(big), fps_points=counts_s.cpu().tolist(), swap_pairs=len(pairs) // 2,
                                    swap_points=extra)
        # the builder, with and without SA-DA, alternated
        variants = dict(build_train_batch_ms=None, build_train_batch_sada_ms=sada.SadaConfig(),
                        build_train_batch_sada_raised_ms=sada.SadaConfig(**RAISED))
        rss = {k: np.random.RandomState(3) for k in variants}
        ts = {k: [] for k in variants}
        for step in range(a.warmup + a.steps):
            for k, sc in variants.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                augment.build_train_batch(cfg, clouds, boxes, names, rss[k], sa_da=sc)
                torch.cuda.synchronize()
                if step >= a.warmup:
                    ts[k].append((time.perf_counter() - t0) * 1e3)
        out.update({k: stats(v) for k, v in ts.items()})
        # read-backs of one batch: count the host waits the builder makes (swap counts, frame sizes, voxel totals)
        calls = dict(n=0)
        orig_cpu, orig_item = torch.Tensor.cpu, torch.Tensor.item

        def cpu(t, *x, **k):
            if t.is_cuda:
                calls["n"] += 1
            return orig_cpu(t, *x, **k)

        def item(t):
            if t.is_cuda:
                calls["n"] += 1
            return orig_item(t)
        for name, sc in (("car", sada.SadaConfig()), ("raised", sada.SadaConfig(**RAISED)), ("off", None)):
            calls["n"] = 0
            torch.Tensor.cpu, torch.Tensor.item = cpu, item
            try:
                augment.build_train_batch(cfg, clouds, boxes, names, np.random.RandomState(5), sa_da=sc)
            finally:
                torch.Tensor.cpu, torch.Tensor.item = orig_cpu, orig_item
            out.setdefault("readbacks_per_batch", {})[name] = calls["n"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
