"""CPU checks of the constant-region skip model (tests/skip_model.py): on small maps, every pixel it calls constant equals its
output-parity class constant in an fp64 restatement of the neck (oracle/bev_ref.py), and the plan it derives covers every tile."""
import numpy as np
import pytest
import torch

import skip_model as sm

H, W = 48, 64


def _occ(points, h=H, w=W):
    occ = np.zeros((h, w), bool)
    for y, x in points:
        occ[y, x] = True
    return occ


CASES = {
    "empty": [],
    "corners": [(0, 0), (H - 1, W - 1)],
    "seams": [(7, 15), (8, 16), (23, 31), (24, 32)],
    "centre": [(H // 2, W // 2)],
    "cluster": [(y, x) for y in range(10, 14) for x in range(40, 45)] + [(30, 5)],
}


@pytest.mark.parametrize("case", sorted(CASES))
def test_constant_pixels_equal_their_class_constant_fp64(case):
    from oracle import bev_ref
    occ = _occ(CASES[case])
    sd = bev_ref.ssfa_random_state(3, torch.float64)
    hsd = bev_ref.head_random_state(4, torch.float64)
    g = torch.Generator().manual_seed(5)
    x = torch.zeros((1, 128, H, W), dtype=torch.float64)
    ys, xs = np.nonzero(occ)
    x[0, :, ys, xs] = torch.rand((128, len(ys)), generator=g, dtype=torch.float64) + 0.5
    trace = {}
    out = bev_ref.ssfa_forward(x, sd, trace)
    head = bev_ref.head_forward(out, hsd)
    trace["out"] = out
    trace["head"] = torch.cat([head[k].permute(0, 3, 1, 2) for k in ("box_preds", "cls_preds", "dir_cls_preds", "iou_preds")], 1)
    masks = sm.masks(occ)
    checked = 0
    for name, t in trace.items():
        a = t[0].numpy()
        const = ~masks[name]
        scale = np.abs(a).max() + 1e-30
        for py in (0, 1):
            for px in (0, 1):
                sel = const[py::2, px::2]
                vals = a[:, py::2, px::2][:, sel]
                if vals.shape[1]:
                    assert np.abs(vals - vals[:, :1]).max() <= 1e-12 * scale, (name, py, px)
                    checked += vals.shape[1]
        # the masks are not vacuous: a map this sparse keeps constant pixels, and non-constant ones do differ somewhere
        assert const.any(), name
    assert checked > 0
    if case != "empty":
        x0 = trace["x0"][0].numpy()
        nc = masks["x0"] & ~sm._dilate3(np.zeros_like(occ))        # non-constant because of a site, not of the border
        assert nc.any()
        c = x0[:, ~masks["x0"]][:, :1]
        assert np.abs(x0[:, nc] - c).max() > 0


@pytest.mark.parametrize("case", sorted(CASES))
@pytest.mark.parametrize("batch", [1, 2])
def test_plan_runs_every_non_constant_tile(case, batch):
    occ = np.stack([_occ(CASES[case])] + [_occ([])] * (batch - 1))
    for rec in sm.plan(occ):
        g = rec["geometry"]
        per_cls = g["nblocks"] * g["tiles"]
        run = {(g["order"][i // per_cls], i % g["tiles"]) for i in rec["items"]}
        for c in range(g["nclass"]):
            for t in range(g["tiles"]):
                if rec["flags"][c, t]:
                    assert (c, t) in run
                listed = (c * g["tiles"] + t) in set(rec["skipped"].tolist())
                assert listed != ((c, t) in run), (rec["name"], c, t)       # every tile either runs or is filled
            if rec["rep"][c] >= 0:
                assert not rec["flags"][c, rec["rep"][c]]
        # every n-block of a tile that runs, in the launcher's order
        assert len(rec["items"]) == g["nblocks"] * len(run)
        assert np.all(np.diff(rec["items"]) > 0)


def test_plan_geometry_matches_the_launcher_on_the_neck_maps():
    occ = np.zeros((1, 200, 176), bool)
    recs = {r["name"]: r["geometry"] for r in sm.plan(occ)}
    assert not recs["b0a"]["u_is_x"] and recs["b0a"]["tiles"] == 25 * 11
    assert recs["b1a"]["u_is_x"] and recs["b1a"]["tiles"] == 11 * 7 and recs["b1a"]["nblocks"] == 2
    assert recs["m0"]["order"] == [3, 1, 2, 0] and recs["m0"]["nclass"] == 4
    assert recs["head"]["nblocks"] == 1
