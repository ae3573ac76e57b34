"""Per-kernel achieved rates against the GPU roofline, on BASELINE config #5's shape (dense-scene stress: uniform 200k-point
clouds, batch 8 per launch, one GPU) and on config #2's shape (ring-20k, batch 1).  SURVEY.md 8(d): batch-1 frames are
launch/latency-bound, so the roofline fractions of the bandwidth-bound kernels are quoted from the stress shape.

Every launch group of the frame is bracketed by CUDA events on the engine stream (eager launches, median of --iters passes);
ALGORITHMIC bytes / flops per group follow SURVEY.md 8(d) / DESIGN.md section 4:
  voxelise+VFE   16 N + 112 M                       (read points; write voxels 80, coors 12(+4 batch), num 4, mean 16)
  rulebook       16 N_in + 4 kvol N_out + 16 N_out  (read coords; write the output-major nbr table + output coords)
  sparse conv    flops 2 P Cin Cout ; bytes 4 N_in Cin + 4 N_out Cout + 4 kvol N_out + 4 kvol Cin Cout
  dense()        4 B H W C written + 4 N_out C read
  neck conv      flops 2 H W Cin Cout taps
  post           3.1 MB / frame read
Prints one JSON object; `python scripts/kernel_rooflines.py --shape stress|frame`.
"""
import argparse, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "se-ssd_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)
import numpy as np, torch


def load_peaks():
    peaks = {}
    try:
        peaks = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))
    except Exception:
        pass
    return (float(peaks.get("hbm_gbs", 3350.0)), float(peaks.get("bf16_tflops_sustained", peaks.get("bf16_tflops", 989.0))),
            "MEASURED_PEAKS.json (of measured)" if peaks else "H100 SXM datasheet (HBM3 3.35 TB/s, dense bf16 989 TFLOP/s)")


def group_rooflines(eng, clouds, iters=5):
    """Per-launch-group times (CUDA events on the engine stream, eager launches, median of `iters` passes after one warm-up pass)
    and achieved rates of one batch of `clouds` through `eng` (a FrameEngine with weights loaded).  Returns the JSON-able record."""
    from sessd_b200 import ops
    HBM, TF, src = load_peaks()
    B = eng.batch
    npts = eng.stage(clouds)
    st = eng.stream
    flush = torch.empty((64 * 1024 * 1024,), dtype=torch.float32, device=eng.device)
    runs = []
    for it in range(iters + 1):
        marks = []

        def mark(label):
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(st)
            marks.append((label, ev))

        with torch.cuda.stream(st):
            eng.d_points.copy_(eng.h_points, non_blocking=True); eng.d_off.copy_(eng.h_off, non_blocking=True)
            flush.zero_()
            mark("start")
            ops.voxelize(eng.d_points, eng.d_off, eng.vox)
            mark("voxelize")
            hd = eng.sparse_and_neck(mark=mark)
            ops.postprocess(hd, eng.anchors, None, eng.post)
            mark("post")
            st.synchronize()
        if it:
            runs.append([marks[i][1].elapsed_time(marks[i + 1][1]) for i in range(len(marks) - 1)])
    labels = [m[0] for m in marks[1:]]
    ms = np.median(np.array(runs), 0)

    # ---- algorithmic work per group --------------------------------------------------------------------------------
    M = int(eng.vox.num_voxels[B].item())
    mid = eng.middle
    n_lvl = [M] + [int(l["n"].item()) for l in mid.levels[1:]]
    work = {}
    work["voxelize"] = ("hbm", 16.0 * npts + 112.0 * M)
    work["hash_build"] = ("hbm", 16.0 * M + 8.0 * M)
    work["sort0"] = ("hbm", 16.0 * M * 2 + 16.0 * M * 2)
    seen = set()
    for li, p in enumerate(mid.plan):
        n_in, n_out = n_lvl[p["lin"]], n_lvl[p["lout"]]
        kvol = p["ks"][0] * p["ks"][1] * p["ks"][2]
        pairs = int((p["nbr"][:n_out] >= 0).sum().item())
        key = "rulebook:%s" % p["key"] if p["kind"] == "subm" else "rulebook:sp%d" % p["lout"]
        if key not in seen:
            seen.add(key)
            work[key] = ("hbm", 16.0 * n_in + 4.0 * kvol * n_out + 16.0 * n_out)
        work["conv:%d" % li] = ("tensor", 2.0 * pairs * p["cin"] * p["cout"],
                                4.0 * n_in * p["cin"] + 4.0 * n_out * p["cout"] + 4.0 * kvol * n_out + 4.0 * kvol * p["cin"] * p["cout"],
                                dict(kind=p["kind"], impl=p.get("impl"), cin=p["cin"], cout=p["cout"], n_out=n_out, pairs=pairs))
    for li, p in enumerate(mid.plan):
        if mid.planes[li] is not None:
            work["split:%d" % li] = ("hbm", 8.0 * n_lvl[p["lout"]] * p["cout"])
    work["dense"] = ("hbm", 4.0 * mid.dense.numel() + 4.0 * n_lvl[-1] * 64)
    h, w = eng.neck.h, eng.neck.w
    NECK = {"bottom_up_block_0.1": (h, w, 128, 128, 9), "bottom_up_block_0.4": (h, w, 128, 128, 9), "bottom_up_block_0.7": (h, w, 128, 128, 9),
            "bottom_up_block_1.0": (h // 2, w // 2, 128, 256, 9), "bottom_up_block_1.3": (h // 2, w // 2, 256, 256, 9),
            "bottom_up_block_1.6": (h // 2, w // 2, 256, 256, 9), "trans_0.0": (h, w, 128, 128, 1), "trans_1.0": (h // 2, w // 2, 256, 256, 1),
            "deconv_block_0.0": (h // 2, w // 2, 256, 128, 9), "deconv_block_1.0": (h // 2, w // 2, 256, 128, 9),
            "conv_0.0": (h, w, 128, 128, 9), "conv_1.0": (h, w, 128, 128, 9)}
    for k, (hh, ww, ci, co, t) in NECK.items():
        in_px = 4 * hh * ww if k == "bottom_up_block_1.0" else hh * ww          # stride-2 conv reads the 200x176 map
        out_px = 4 * hh * ww if "deconv" in k else hh * ww                      # deconvs write the 200x176 map
        work["neck:" + k] = ("tensor", 2.0 * B * hh * ww * ci * co * t, 4.0 * B * (in_px * ci + out_px * co) + 4.0 * t * ci * co, None)
    work["neck:fuse+head"] = ("hbm", 4.0 * B * h * w * (3 * 128 + 128 + 24))
    work["post"] = ("hbm", 4.0 * B * 70400 * 11)
    rows = []
    for lab, t in zip(labels, ms):
        wk = work.get(lab)
        row = {"group": lab, "ms": round(float(t), 4)}
        if wk is not None:
            if wk[0] == "hbm":
                row.update(bound="hbm", alg_bytes=wk[1], GBps=round(wk[1] / (t / 1e3) / 1e9, 1), frac=round(wk[1] / (t / 1e3) / 1e9 / HBM, 4))
            else:
                row.update(bound="tensor", alg_flops=wk[1], TFLOPs=round(wk[1] / (t / 1e3) / 1e12, 2), frac_bf16=round(wk[1] / (t / 1e3) / 1e12 / TF, 4),
                           alg_bytes=wk[2], GBps=round(wk[2] / (t / 1e3) / 1e9, 1))
                if wk[3]:
                    row.update(wk[3])
        rows.append(row)
    return {"batch": B, "points": int(npts), "voxels": M, "active_sites": n_lvl, "capacity_status": int(mid.status.item()),
            "peaks": {"hbm_GBps": HBM, "bf16_TFLOPs_sustained": TF, "source": src},
            "total_ms": round(float(ms.sum()), 3), "frames_per_sec_eager": round(B / (ms.sum() / 1e3), 1),
            "mem_GB": round(torch.cuda.memory_allocated() / 2 ** 30, 1), "groups": rows,
            "note": "eager launches, CUDA events between launch groups on the engine stream, median of %d passes, L2 flushed once per pass" % iters}


def main():
    from sessd_data import synth, weights
    from sessd_b200.engine import FrameEngine
    ap = argparse.ArgumentParser()
    ap.add_argument("--shape", default="stress", choices=["stress", "frame", "frame-uniform"])
    ap.add_argument("--batch", type=int, default=None)
    ap.add_argument("--points", type=int, default=None)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--cg-deep", type=int, default=0, help="1: deep pipeline, one CTA per SM")
    a = ap.parse_args()
    from sessd_b200._lib import lib
    lib.sessd_set_sp_cg_deep(int(a.cg_deep))
    if a.shape == "stress":
        B, N = a.batch or 8, a.points or 200000
        clouds = [synth.uniform_cloud(1000 + f, N) for f in range(B)]
        eng = FrameEngine(batch=B, max_points_per_frame=N, max_voxels=200000, growth=(1.0, 8.0, 8.0, 8.0, 8.0))
        kind = "uniform"
    else:
        B, N = a.batch or 1, a.points or 20000
        kind = "ring" if a.shape == "frame" else "uniform"
        clouds = [(synth.ring_cloud if kind == "ring" else synth.uniform_cloud)(f, N) for f in range(B)]
        eng = FrameEngine(batch=B, max_points_per_frame=max(c.shape[0] for c in clouds))
    layers, ssfa, head = weights.bench_detector_state(kind, 0)
    eng.load_weights(layers, ssfa, head, weights.kitti_car_anchors())
    out = group_rooflines(eng, clouds, a.iters)
    out["shape"] = a.shape
    out["cg_deep"] = int(a.cg_deep)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
