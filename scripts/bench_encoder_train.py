"""SpMiddleFHD in train mode at the training shape (ring-20k clouds, batch 8): forward and forward + backward time from CUDA events after
warm-up (median, min, max over the steps: the strided rulebooks sync the host once per level, so single steps vary), per-layer forward /
data-gradient / weight-gradient times from CUDA events around each layer's own Function on its own rulebook (the gradient times include the
split of the output gradient into planes on the tensor-core layers), FLOP/s from the rulebook pair counts (2 P Cin Cout per product), and
per-kernel device time of one forward + backward from torch.profiler (a separate run).  Prints one JSON object (with the card's name and
power limit).

    python scripts/bench_encoder_train.py [--batch 8] [--steps 30] [--warmup 3] [--layer-reps 10]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(os.path.dirname(HERE), "se-ssd_b200"))
sys.path.insert(0, os.path.dirname(HERE))


def card():
    name = torch.cuda.get_device_name()
    try:
        pl = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", str(torch.cuda.current_device())],
                            capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError):
        pl = "unknown"
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=8)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--layer-reps", type=int, default=10)
    a = ap.parse_args()
    from det3d.models.backbones.scn import SpMiddleFHD
    from oracle import cpu as ocpu
    from sessd_b200 import sparse_grad, synth
    import spconv
    feats, coors = [], []
    for b in range(a.batch):
        v, c, n = ocpu.points_to_voxel(synth.ring_cloud(b, 20000), synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
        coors.append(np.concatenate([np.full((len(c), 1), b, np.int32), c], 1))
        feats.append((v.sum(1) / n[:, None]).astype(np.float32))
    feats = torch.from_numpy(np.concatenate(feats)).cuda()
    coors = torch.from_numpy(np.concatenate(coors)).cuda()
    torch.manual_seed(0)
    m = SpMiddleFHD(num_input_features=4).cuda().train()
    shape = [1408, 1600, 40]
    R = torch.randn((a.batch, 128, 200, 176), device="cuda")

    def fwd():
        return m(feats, coors, a.batch, shape)

    def step():
        m.zero_grad(set_to_none=True)
        (fwd() * R).sum().backward()

    def timed(fn, steps, warmup):
        for _ in range(warmup):
            fn()
        torch.cuda.synchronize()
        ts = []
        for _ in range(steps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            torch.cuda.synchronize()
            ts.append(e0.elapsed_time(e1))
        return dict(median=round(float(np.median(ts)), 3), min=round(float(np.min(ts)), 3), max=round(float(np.max(ts)), 3), n=len(ts))

    fwd_ms = timed(fwd, a.steps, a.warmup)
    step_ms = timed(step, a.steps, a.warmup)
    # every conv's rulebook and input, captured in one train-mode pass (the layer list of encoder_forward)
    captured, rulebooks = [], {}
    x = spconv.SparseConvTensor(feats, coors, [41, 1600, 1408], a.batch)
    with torch.no_grad():
        for mod in m.middle_conv._modules.values():
            if isinstance(mod, spconv.SparseModule):
                feat_in = x.features
                x, rb = sparse_grad.sparse_conv(mod, x, rulebooks)
                captured.append((mod, rb, feat_in))
            else:
                x.features = mod(x.features)
    layers = []
    Fn = sparse_grad.SparseConvFunction
    for i, (conv, rb, feat_in) in enumerate(captured):
        p = int((rb.nbr[:rb.n_out] >= 0).sum())
        flop = 2.0 * p * conv.in_channels * conv.out_channels      # per product: forward, data gradient, weight gradient alike
        w = conv.weight.detach()
        with torch.no_grad():
            t_fwd = timed(lambda: Fn.apply(feat_in, w, rb), a.layer_reps, 2)
        xr = feat_in.detach().requires_grad_(True)
        out_x = Fn.apply(xr, w, rb)
        g = torch.randn_like(out_x)
        wr = w.clone().requires_grad_(True)
        out_w = Fn.apply(feat_in.detach(), wr, rb)
        t_wgrad = timed(lambda: torch.autograd.grad(out_w, wr, g, retain_graph=True), a.layer_reps, 2)
        row = dict(layer=i, cin=conv.in_channels, cout=conv.out_channels, kvol=rb.kvol, subm=rb.subm, pairs=p, n_out=rb.n_out,
                   impl=sparse_grad.conv_impl(conv.in_channels), gflop_per_product=round(flop * 1e-9, 4), fwd_ms=t_fwd["median"],
                   wgrad_ms=t_wgrad["median"], wgrad_tflops=round(flop / t_wgrad["median"] * 1e-9, 2),
                   fwd_tflops=round(flop / t_fwd["median"] * 1e-9, 2))
        if i > 0:                                                  # layer 0's input (the VFE mean) takes no gradient
            t_dgrad = timed(lambda: torch.autograd.grad(out_x, xr, g, retain_graph=True), a.layer_reps, 2)
            row.update(dgrad_ms=t_dgrad["median"], dgrad_tflops=round(flop / t_dgrad["median"] * 1e-9, 2))
        row["wgrad_over_fwd"] = round(t_wgrad["median"] / t_fwd["median"], 2)
        layers.append(row)
        del out_x, out_w
    from torch.profiler import ProfilerActivity, profile
    step()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        step()
        torch.cuda.synchronize()
    kernels = {}
    for ev in prof.key_averages():
        if ev.device_type is not None and "cuda" in str(ev.device_type).lower() and ev.device_time_total > 0:
            kernels[ev.key] = dict(calls=int(ev.count), us=round(float(ev.device_time_total), 1))
    tops = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["us"])[:30])
    wgrad_us = sum(v["us"] for k, v in kernels.items() if "wgrad_" in k and "reduce" not in k)
    total_gflop = sum(l["gflop_per_product"] for l in layers)
    name, pl = card()
    print(json.dumps(dict(gpu=name, power_limit=pl, batch=a.batch, voxels=int(feats.shape[0]), fwd_ms=fwd_ms,
                          fwd_bwd_ms=step_ms, wgrad_kernels_us=round(wgrad_us, 1),
                          wgrad_tflops_all_layers=round(total_gflop / wgrad_us * 1e3, 3) if wgrad_us else None,
                          layers=layers, kernels=tops)))


if __name__ == "__main__":
    main()
