"""numpy restatement of the segment records of the SSFA neck's skip plan (csrc/bevskip.cu, bev_skip_seg_kernel).

Every stride-1 launch runs segments rather than tiles: 8 pixels along the launcher's u in one v row.  A segment is live when it holds a
non-constant pixel (skip_model.masks) or leaves the map.  Per class and v parity, the first all-constant segment is a representative and
runs too.  The live segments and the representatives are packed 16 to a group, per class in the launcher's heavy-first order, by
ascending segment index (b * grid_v + v) * tiles_u + u / 8; a class's last group is padded with -1.  Every other segment is filled from
the representative of its class and v parity.
"""
import numpy as np

import skip_model as sm

SLOTS = 16
HEADER = 32
TILE_ONLY = ("b1a",)      # the stride-2 conv: tiles only


def plan(occ):
    """occ [B, h, w] bool -> {launch name: dict(groups [n, 16], skipped, rep [nclass][2], count, flags)} for every segment launch"""
    B, h, w = occ.shape
    fm = [sm.masks(occ[b]) for b in range(B)]
    out = {}
    for name, deconv, cout in sm.LAUNCHES:
        if name in TILE_ONLY:
            continue
        half = name in ("b1b", "x1", "t1") or deconv
        g = sm.geometry(B, h // 2 if half else h, w // 2 if half else w, cout, deconv)
        nseg = B * g["grid_v"] * g["tiles_u"]
        flags = np.zeros((g["nclass"], nseg), bool)
        for c in range(g["nclass"]):
            py, px = (c >> 1, c & 1) if deconv else (0, 0)
            for b in range(B):
                mm = fm[b][name][py::g["stride"], px::g["stride"]] if deconv else fm[b][name]
                if not g["u_is_x"]:
                    mm = mm.T                                   # [u, v] -> [v, u]
                mm = mm[: g["grid_v"], : g["grid_u"]]
                pad = np.ones((g["grid_v"], g["tiles_u"] * sm.TU), bool)      # a segment past the map's u edge always runs
                pad[:, : g["grid_u"]] = mm
                live = pad.reshape(g["grid_v"], g["tiles_u"], sm.TU).any(axis=2)
                flags[c, b * g["grid_v"] * g["tiles_u"]:(b + 1) * g["grid_v"] * g["tiles_u"]] = live.reshape(-1)
        parity = (np.arange(nseg) // g["tiles_u"]) % g["grid_v"] & 1
        rep = []
        for c in range(g["nclass"]):
            r = []
            for p in (0, 1):
                cand = np.flatnonzero(~flags[c] & (parity == p))
                r.append(int(cand[0]) if len(cand) else -1)
            rep.append(r)
        groups = []
        for c in g["order"]:
            run = np.flatnonzero(flags[c] | np.isin(np.arange(nseg), rep[c]))
            ents = (c << 24) | run
            n = -(-len(ents) // SLOTS) * SLOTS
            groups.append(np.concatenate([ents, -np.ones(n - len(ents), np.int64)]).reshape(-1, SLOTS))
        groups = np.concatenate(groups) if groups else np.zeros((0, SLOTS), np.int64)
        skipped = [c * nseg + s for c in range(g["nclass"]) for s in range(nseg) if not flags[c, s] and s != rep[c][parity[s]]]
        out[name] = dict(geometry=g, nseg=nseg, flags=flags, rep=rep, groups=groups.astype(np.int64),
                         skipped=np.array(skipped, np.int64), count=len(groups) * g["nblocks"])
    return out


def read_seg_record(rec):
    """one segment record of the device plan (numpy int32) -> (count, groups [n, 16], skipped, rep [nclass][2])"""
    count, nskip, ngroups, nclass = (int(v) for v in rec[0:4])
    groups = rec[HEADER:HEADER + SLOTS * ngroups].astype(np.int64).reshape(-1, SLOTS)
    skip_off = int(rec[28])
    rep = [[int(rec[20 + 2 * c]), int(rec[21 + 2 * c])] for c in range(nclass)]
    return count, groups, rec[skip_off:skip_off + nskip].astype(np.int64), rep
