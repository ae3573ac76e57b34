"""Stall profile of bev_conv_p2_kernel per warp role, for the 13 BEV neck launches of one ring-20k frame (batch 1).

Runs the launches through the PROFILE instantiation of the lab library (sessd_bev_conv_p2_profile / sessd_bev_deconv_p2_profile,
include/sessd_b200_lab.h), which writes the clock64() counters of every CTA (P2Prof in csrc/bevconv_p2.cuh), in two settings:
  * alone: each launch on its own (dense: every work item; skip: the items of the frame's skip plan), timed with CUDA events;
  * concurrent: --engines frame engines replaying their frame graphs at once, as bench.py's frame-ring workload does (the counters of
    every engine's last frame, summed per launch).
Per launch it reports items, rounds (most items of one CTA), µs (alone), the share of the consumer's item clocks spent waiting on
b_full / patch_full / wgmma_wait and in the epilogue, the producers' shares waiting on their *_empty barriers, and the main-loop clocks
per tap step against the tensor-core floor (6 * n_tile clocks: 128 px x 32 cin x 3 n_tile fp16 FMA at 2048 FMA/clk/SM).  The card's
name, power limit and SM clocks are read in the same run.  The counters cost clocks of their own: the µs here are not bench numbers.

--loads adds the L2 -> SM ceiling of the 3x3 128 -> 128 launch: the launch alone through the loader-only probe
(sessd_bev_conv_p2_loads: the TMA producers run unchanged, the consumers only wait on the full barriers and release them), dense once
with the three patch copies shared-memory A descriptors would need and once with the single copy the register-fed A reads, then on the
frame's segment record (sessd_bev_conv_p2_seg_loads: one 3 x 10-row window per segment).  Bytes are counted from the shapes (per item
and 32-channel chunk: the patch boxes plus nine 16 KB weight stages; segments: the windows of the item's segments); reported per clock
and SM and as TB/s.

    python scripts/p2_stall_profile.py --out FILE [--reps 20] [--engines 12] [--frames 8] [--loads]
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for _p in (ROOT, os.path.join(ROOT, "se-ssd_b200")):
    if _p not in sys.path:
        sys.path.insert(0, _p)

WORDS = 16          # kP2ProfWords
# P2Prof word order (csrc/bevconv_p2.cuh)
CTA, ITEMS, STEPS, ITEM_CLK, B_FULL, PATCH_FULL, MMA_WAIT, EPILOGUE, PATCH_EMPTY, PATCH_TOTAL, B_EMPTY, B_TOTAL = range(12)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout
        return dict(zip(q.split(","), [s.strip() for s in out.strip().splitlines()[0].split(",")]))
    except (OSError, IndexError, subprocess.SubprocessError):
        return {}


class Profiler:
    """Routes ops.bev_conv_p2 / ops.bev_deconv_p2 to the PROFILE entry points, one counter buffer per (engine, launch, setting)"""

    def __init__(self, device, num_sms):
        import torch

        from sessd_b200 import ops
        self.torch, self.ops, self.device, self.num_sms = torch, ops, device, num_sms
        self.bufs, self.key = {}, None
        # 0 / 1: route conv() to the loader-only probe with that patch plan ("segs": on the launch's segment record), counters filed
        # under self.key
        self.loads_smem_a = None
        ops.bev_conv_p2, ops.bev_deconv_p2 = self.conv, self.deconv

    def buf(self):
        if self.key not in self.bufs:
            self.bufs[self.key] = self.torch.zeros((self.num_sms, WORDS), dtype=self.torch.int64, device=self.device)
        return self.bufs[self.key]

    def conv(self, in_planes, in_info, weight_h2, scale, shift, residual, resid_info, gain, shift_max, out_f32, out_planes, out_info, desc,
             items=None, segs=None):
        o = self.ops
        if self.loads_smem_a == "segs":
            o.check(o.lib.sessd_bev_conv_p2_seg_loads(o._p(in_planes), o._p(in_info), o._p(weight_h2), int(weight_h2.shape[2]), o._p(scale),
                                                      o._p(shift), o._p(residual), o._p(resid_info), float(gain), float(shift_max),
                                                      o._p(out_f32), o._p(out_planes), o._p(out_info), C.byref(desc), o._p(segs),
                                                      o._p(self.buf()), o._st()), "sessd_bev_conv_p2_seg_loads")
            return
        if self.loads_smem_a is not None:
            o.check(o.lib.sessd_bev_conv_p2_loads(o._p(in_planes), o._p(in_info), o._p(weight_h2), int(weight_h2.shape[2]), o._p(scale),
                                                  o._p(shift), o._p(residual), o._p(resid_info), float(gain), float(shift_max), o._p(out_f32),
                                                  o._p(out_planes), o._p(out_info), C.byref(desc), o._p(items), int(self.loads_smem_a),
                                                  o._p(self.buf()), o._st()), "sessd_bev_conv_p2_loads")
            return
        o.check(o.lib.sessd_bev_conv_p2_profile(o._p(in_planes), o._p(in_info), o._p(weight_h2), int(weight_h2.shape[2]), o._p(scale),
                                                o._p(shift), o._p(residual), o._p(resid_info), float(gain), float(shift_max), o._p(out_f32),
                                                o._p(out_planes), o._p(out_info), C.byref(desc), o._p(items), o._p(segs), o._p(self.buf()),
                                                o._st()),
                "sessd_bev_conv_p2_profile")

    def deconv(self, in_planes, in_info, weight_h2, scale, shift, residual, resid_info, gain, shift_max, out_f32, out_planes, out_info,
               relu=True, items=None, segs=None):
        o = self.ops
        _two, b, h, w, cin = in_planes.shape
        cout = (out_f32 if out_f32 is not None else out_planes).shape[-1]
        o.check(o.lib.sessd_bev_deconv_p2_profile(o._p(in_planes), o._p(in_info), o._p(weight_h2), int(weight_h2.shape[2]), o._p(scale),
                                                  o._p(shift), o._p(residual), o._p(resid_info), float(gain), float(shift_max),
                                                  o._p(out_f32), o._p(out_planes), o._p(out_info), int(b), int(h), int(w), int(cin), int(cout),
                                                  int(bool(relu)), o._p(items), o._p(segs), o._p(self.buf()), o._st()),
                "sessd_bev_deconv_p2_profile")

    def tag(self, eng_id, neck):
        """every launch of this engine's neck files its counters under (eng_id, launch name, dense | skip)"""
        orig = neck._launch

        def launch(L, skip=False):
            if self.loads_smem_a is None:
                self.key = (eng_id, L.name, "skip" if skip else "dense")
            orig(L, skip)

        neck._launch = launch


def summarize(recs, n_tile):
    """recs: int64 [grid, WORDS] of one or more launches (summed) -> per-role shares and per-step clocks"""
    import numpy as np
    r = np.asarray(recs, dtype=np.float64)
    tot = r.sum(axis=0)
    steps, item_clk = max(tot[STEPS], 1.0), max(tot[ITEM_CLK], 1.0)
    floor = 6 * n_tile
    main = tot[ITEM_CLK] - tot[EPILOGUE]
    busy = r[:, CTA]
    return dict(
        items=int(tot[ITEMS]), steps=int(tot[STEPS]), rounds=int(r[:, ITEMS].max()), ctas=int((r[:, ITEMS] > 0).sum()),
        consumer_share=dict(b_full=tot[B_FULL] / item_clk, patch_full=tot[PATCH_FULL] / item_clk, wgmma_wait=tot[MMA_WAIT] / item_clk,
                            epilogue=tot[EPILOGUE] / item_clk,
                            other=1.0 - (tot[B_FULL] + tot[PATCH_FULL] + tot[MMA_WAIT] + tot[EPILOGUE]) / item_clk),
        producer_share=dict(patch_empty=tot[PATCH_EMPTY] / max(tot[PATCH_TOTAL], 1.0), b_empty=tot[B_EMPTY] / max(tot[B_TOTAL], 1.0)),
        clk_per_step_main=main / steps, clk_per_step_with_epilogue=item_clk / steps, floor_clk_per_step=floor,
        floor_share_main=floor / (main / steps) if main > 0 else None,
        epilogue_clk_per_item=tot[EPILOGUE] / max(tot[ITEMS], 1.0),
        cta_clk_max=float(busy.max()), cta_clk_mean_active=float(busy[r[:, ITEMS] > 0].mean()) if (r[:, ITEMS] > 0).any() else 0.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--engines", type=int, default=12)
    ap.add_argument("--frames", type=int, default=8, help="frames per engine in the concurrent leg")
    ap.add_argument("--loads", action="store_true", help="also measure the loader-only ceiling of the 3x3 128->128 launch")
    a = ap.parse_args()

    import numpy as np
    import torch

    from sessd_b200.engine import FrameEngine
    from sessd_data import synth, weights
    from sessd_data.layers import SSFA_LAUNCHES

    if not torch.cuda.is_available():
        raise SystemExit("p2_stall_profile: no CUDA device (the profile is a GPU measurement)")
    dev = torch.device("cuda")
    num_sms = torch.cuda.get_device_properties(dev).multi_processor_count
    prof = Profiler(dev, num_sms)
    n_tile = {L.name: (32 if L.cout <= 32 else 128) for L in SSFA_LAUNCHES}
    layers, ssfa, head = weights.bench_detector_state("ring", 0)
    res = dict(gpu=gpu_info(), torch_device=torch.cuda.get_device_name(), num_sms=num_sms, reps=a.reps, alone={}, concurrent={})

    # ---- alone: one engine, eager, each launch timed on its own after a frame left its buffers and skip plan
    eng = FrameEngine(batch=1)
    eng.load_weights(layers, ssfa, head, weights.kitti_car_anchors())
    prof.tag(0, eng.neck)
    for s in range(4):
        eng.infer([synth.ring_cloud(s, 20000)])
    torch.cuda.synchronize()
    with torch.cuda.stream(eng.stream):
        for L in SSFA_LAUNCHES:
            rec = {}
            for mode in ("dense", "skip"):
                for _ in range(3):
                    eng.neck._launch(L, mode == "skip")
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(eng.stream)
                for _ in range(a.reps):
                    eng.neck._launch(L, mode == "skip")
                t1.record(eng.stream)
                eng.stream.synchronize()
                us = t0.elapsed_time(t1) * 1000.0 / a.reps
                s = summarize(prof.bufs[(0, L.name, mode)].cpu().numpy(), n_tile[L.name])
                s["us"] = us
                s["sm_mhz_from_clock64"] = s["cta_clk_max"] / us if us > 0 else None
                rec[mode] = s
            res["alone"][L.name] = rec
        if a.loads:
            # the 3x3 128 -> 128 launch: per (item, chunk) 2 planes x 18 x (8 + 2) rows (one copy) or 3 copies x 2 x 18 x 8 rows of
            # 64 B, plus 9 weight stages of 2 x 128 rows of 64 B
            L = next(L for L in SSFA_LAUNCHES if L.kind == "conv" and L.cin == 128 and L.cout == 128 and L.k == 3 and L.stride == 1)
            res["loads"] = dict(launch=L.name)
            # segments: 2 planes x 3 x 10 rows of 64 B per segment of the item
            seg_rec = eng.neck.skip.seg_record(eng.neck.SKIP_LAUNCHES.index(L.name)).cpu().numpy()
            groups = seg_rec[32:32 + 16 * int(seg_rec[2])]
            seg_patch = 2 * 3 * 10 * 64 * float((groups >= 0).sum()) / max(len(groups) // 16, 1)
            for smem_a, patch, name in ((1, 3 * 2 * 18 * 8 * 64, "smem_a"), (0, 2 * 18 * 10 * 64, "reg_a"), ("segs", seg_patch, "segs")):
                prof.loads_smem_a = smem_a
                prof.key = (0, L.name, "loads_%s" % name)
                skip = smem_a == "segs"
                for _ in range(3):
                    eng.neck._launch(L, skip)
                t0, t1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0.record(eng.stream)
                for _ in range(a.reps):
                    eng.neck._launch(L, skip)
                t1.record(eng.stream)
                eng.stream.synchronize()
                us = t0.elapsed_time(t1) * 1000.0 / a.reps
                r = prof.bufs[prof.key].cpu().numpy().astype(np.float64)
                item_bytes = (L.cin // 32) * (patch + 9 * 2 * 128 * 64)
                act = r[:, ITEMS] > 0
                res["loads"][name] = dict(
                    us=us, items=int(r[:, ITEMS].sum()), bytes_per_item=item_bytes, patch_bytes_per_chunk=patch,
                    bytes_per_step=item_bytes / (9 * (L.cin // 32)),
                    bytes_per_clk_per_sm=float((r[act, ITEMS] * item_bytes / r[act, CTA]).mean()),
                    tb_per_s=float(r[:, ITEMS].sum() * item_bytes / (us * 1e-6) / 1e12))
            prof.loads_smem_a = None
    clock_probe = gpu_info()
    del eng
    torch.cuda.synchronize()

    # ---- concurrent: the frame-ring shape, every engine replaying its frame graph on its own stream
    clouds = [synth.ring_cloud(s, 20000) for s in range(16)]
    engines = []
    for k in range(a.engines):
        e = FrameEngine(batch=1)
        e.load_weights(layers, ssfa, head, weights.kitti_car_anchors())
        prof.tag(1 + k, e.neck)
        e.stage([clouds[k % len(clouds)]])
        e.capture()
        engines.append(e)
    torch.cuda.synchronize()
    t0 = torch.cuda.Event(enable_timing=True)
    t1 = torch.cuda.Event(enable_timing=True)
    t0.record()
    for _ in range(a.frames):
        for e in engines:
            e.launch()
    for e in engines:
        e.stream.synchronize()
    t1.record()
    t1.synchronize()
    res["concurrent_frames_per_s_profiled"] = a.engines * a.frames / (t0.elapsed_time(t1) / 1000.0)
    for L in SSFA_LAUNCHES:
        recs = [prof.bufs[(1 + k, L.name, "skip")].cpu().numpy() for k in range(a.engines) if (1 + k, L.name, "skip") in prof.bufs]
        if recs:
            res["concurrent"][L.name] = summarize(np.concatenate(recs), n_tile[L.name])
    res["gpu_after_alone_leg"] = clock_probe

    # ---- totals over the 3x3 / deconv launches (n_tile 128)
    for leg, key in (("alone", "dense"), ("alone", "skip"), ("concurrent", None)):
        allr = []
        for L in SSFA_LAUNCHES:
            if n_tile[L.name] != 128:
                continue
            allr.append(prof.bufs[(0, L.name, key)].cpu().numpy() if leg == "alone" else
                        np.concatenate([prof.bufs[(1 + k, L.name, "skip")].cpu().numpy() for k in range(a.engines)]))
        res["total_%s%s" % (leg, "_" + key if key else "")] = summarize(np.concatenate(allr), 128)
    res["alone_total_us"] = {m: sum(r[m]["us"] for r in res["alone"].values()) for m in ("dense", "skip")}

    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(res, f, indent=1)
    print("bev_conv_p2 stall profile, %s, %s" % (res["torch_device"], res["gpu"]))
    print("  %-20s %5s %6s %8s %8s | %6s %6s %6s %6s | %6s %6s | %7s %5s" % (
        "launch (alone)", "items", "rounds", "dense_us", "skip_us", "b_full", "patch", "wgmma", "epi", "p_emp", "b_emp", "clk/st", "floor"))
    for name, r in res["alone"].items():
        d = r["dense"]
        c, pr = d["consumer_share"], d["producer_share"]
        print("  %-20s %5d %6d %8.1f %8.1f | %6.3f %6.3f %6.3f %6.3f | %6.3f %6.3f | %7.0f %5d" % (
            name, d["items"], d["rounds"], d["us"], r["skip"]["us"], c["b_full"], c["patch_full"], c["wgmma_wait"], c["epilogue"],
            pr["patch_empty"], pr["b_empty"], d["clk_per_step_main"], d["floor_clk_per_step"]))
    for k in ("total_alone_dense", "total_alone_skip", "total_concurrent"):
        t = res[k]
        print("  %-20s clk/step main %.0f (floor %d), with epilogue %.0f; consumer %s; producers %s" % (
            k, t["clk_per_step_main"], t["floor_clk_per_step"], t["clk_per_step_with_epilogue"],
            {x: round(v, 3) for x, v in t["consumer_share"].items()}, {x: round(v, 3) for x, v in t["producer_share"].items()}))
    if a.loads:
        for k in ("smem_a", "reg_a", "segs"):
            r = res["loads"][k]
            print("  loader-only %-6s %s: %.1f us, %d items, %d B per item, %d B per step, %.1f B/clk/SM, %.2f TB/s" % (
                k, res["loads"]["launch"], r["us"], r["items"], r["bytes_per_item"], r["bytes_per_step"], r["bytes_per_clk_per_sm"],
                r["tb_per_s"]))
    print("  alone totals (us): %s; concurrent frames/s while profiled: %.0f" % (res["alone_total_us"], res["concurrent_frames_per_s_profiled"]))


if __name__ == "__main__":
    main()
