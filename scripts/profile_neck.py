"""Per-kernel device time per frame of the frame-ring workload (ring-20k clouds, batch 1), split into neck / sparse / other, with the
neck's constant-region skipping (csrc/bevskip.cu) on and off.  Each setting is profiled with torch.profiler in a process of its own;
the summaries (JSON) and the Chrome traces go under --out.

    python scripts/profile_neck.py --out DIR [--frames 32]
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "se-ssd_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

NECK = ("bev_conv_p2", "bev_skip", "ssfa_fuse", "bev_split", "absmax_kernel")
SPARSE = ("spconv", "rulebook", "nbr_kernel", "hash_", "tile_lists", "dense_gather", "enumerate", "scan", "mark_", "pair_", "cg_")


def group(name):
    if any(k in name for k in NECK):
        return "neck"
    if any(k in name for k in SPARSE):
        return "sparse"
    return "other"


def child(skip, frames, out):
    import torch
    from torch.profiler import ProfilerActivity, profile

    from sessd_b200.engine import FrameEngine
    from sessd_data import synth, weights

    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    eng = FrameEngine(batch=1, skip_constant=skip)
    eng.load_weights(layers, ssfa, head, weights.kitti_car_anchors())
    clouds = [synth.ring_cloud(s, 20000) for s in range(16)]
    for c in clouds:                      # warm-up: every shape and module load
        eng.infer([c])
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(frames):
            eng.infer([clouds[i % len(clouds)]])
        torch.cuda.synchronize()
    tag = "skip_on" if skip else "skip_off"
    prof.export_chrome_trace(os.path.join(out, tag + ".pt.trace.json"))
    kernels = {}
    for ev in prof.key_averages():
        t = getattr(ev, "self_device_time_total", None)
        if t is None:
            t = ev.self_cuda_time_total
        if t <= 0 or ev.key.startswith("Memcpy") or ev.key.startswith("Memset"):
            continue
        kernels[ev.key] = dict(us_per_frame=t / frames, calls_per_frame=ev.count / frames, group=group(ev.key))
    groups = {}
    for k in kernels.values():
        groups[k["group"]] = groups.get(k["group"], 0.0) + k["us_per_frame"]
    res = dict(skip_constant=skip, frames=frames, gpu=torch.cuda.get_device_name(), groups_us_per_frame=groups, kernels=kernels)
    with open(os.path.join(out, tag + ".json"), "w") as f:
        json.dump(res, f, indent=1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--frames", type=int, default=32)
    ap.add_argument("--child", choices=["on", "off"], default=None)
    a = ap.parse_args()
    os.makedirs(a.out, exist_ok=True)
    if a.child:
        child(a.child == "on", a.frames, a.out)
        return
    res = {}
    for mode in ("off", "on"):
        subprocess.check_call([sys.executable, os.path.abspath(__file__), "--out", a.out, "--frames", str(a.frames), "--child", mode])
        with open(os.path.join(a.out, "skip_%s.json" % mode)) as f:
            res[mode] = json.load(f)
    print("device time per frame (us), %s, %d frames" % (res["on"]["gpu"], a.frames))
    for g in ("neck", "sparse", "other"):
        print("  %-7s off %9.1f   on %9.1f" % (g, res["off"]["groups_us_per_frame"].get(g, 0.0), res["on"]["groups_us_per_frame"].get(g, 0.0)))
    names = sorted(set(res["off"]["kernels"]) | set(res["on"]["kernels"]), key=lambda n: -res["off"]["kernels"].get(n, {}).get("us_per_frame", 0))
    print("  neck kernels:")
    for n in names:
        ko, kn = res["off"]["kernels"].get(n), res["on"]["kernels"].get(n)
        if (ko or kn)["group"] != "neck":
            continue
        print("    %9.1f %9.1f  %s" % (ko["us_per_frame"] if ko else 0.0, kn["us_per_frame"] if kn else 0.0, n[:110]))


if __name__ == "__main__":
    main()
