"""The numpy restatement of the neck's segment records (tests/seg_model.py) against the pixel maps it is derived from: every
non-constant pixel lies in a segment that runs, every skipped segment and every representative is all-constant, a skipped segment's
representative has its class and v parity, and the segments cut the tile plan's work on sparse maps."""
import numpy as np
import pytest

import seg_model
import skip_model as sm


def _occ(kind, batch, h, w, seed):
    rng = np.random.default_rng(seed)
    occ = np.zeros((batch, h, w), bool)
    if kind == "points":
        for b in range(batch):
            occ[b, rng.integers(0, h, 40), rng.integers(0, w, 40)] = True
    elif kind == "full":
        occ[:] = True
    return occ


def _segment_pixels(g, nseg, c, s, deconv):
    """output (b, y, x) of the 8 pixels of segment s of class c (inside the map)"""
    su, rest = s % g["tiles_u"], s // g["tiles_u"]
    v, b = rest % g["grid_v"], rest // g["grid_v"]
    py, px = (c >> 1, c & 1) if deconv else (0, 0)
    out = []
    for u in range(su * sm.TU, min(su * sm.TU + sm.TU, g["grid_u"])):
        gy, gx = (v, u) if g["u_is_x"] else (u, v)
        out.append((b, gy * g["stride"] + py, gx * g["stride"] + px))
    return out


@pytest.mark.parametrize("kind,batch,hw", [("points", 1, (48, 64)), ("points", 2, (40, 72)), ("empty", 1, (48, 64)), ("full", 1, (32, 48))])
def test_segment_model_covers_the_non_constant_pixels(kind, batch, hw):
    h, w = hw
    occ = _occ(kind, batch, h, w, 3)
    masks = [sm.masks(occ[b]) for b in range(batch)]
    for name, deconv, _ in sm.LAUNCHES:
        if name in seg_model.TILE_ONLY:
            continue
        e = seg_model.plan(occ)[name]
        g, nseg = e["geometry"], e["nseg"]
        running = {int(v) for v in e["groups"].reshape(-1) if v >= 0}
        for c in range(g["nclass"]):
            for s in range(nseg):
                pix = _segment_pixels(g, nseg, c, s, deconv)
                nonconst = len(pix) < sm.TU or any(masks[b][name][y, x] for b, y, x in pix)
                assert e["flags"][c, s] == nonconst, (name, c, s)
                assert (((c << 24) | s) in running) == (nonconst or s in e["rep"][c]), (name, c, s)
        for ent in e["skipped"]:
            c, s = divmod(int(ent), nseg)
            par = (s // g["tiles_u"]) % g["grid_v"] & 1
            r = e["rep"][c][par]
            assert r >= 0 and not e["flags"][c, r] and (r // g["tiles_u"]) % g["grid_v"] & 1 == par
        # every group holds one class, padded only at the end of the class's last group
        for grp in e["groups"]:
            live = grp[grp >= 0]
            assert len(live) and len({int(v) >> 24 for v in live}) == 1 and (grp[:len(live)] >= 0).all()
        assert e["count"] == len(e["groups"]) * g["nblocks"]


def test_segments_cut_the_tile_work_on_sparse_maps():
    occ = _occ("points", 1, 200, 176, 7)
    tiles = {p["name"]: p for p in sm.plan(occ)}
    segs = seg_model.plan(occ)
    for name in ("b0a", "b0b", "x0"):
        assert len(segs[name]["groups"]) * seg_model.SLOTS < len(tiles[name]["items"]) * sm.TV, name
