"""numpy restatement of the SSFA neck's constant-region skip plan (csrc/bevskip.cu, runners.SSFAPlanesRunner.SKIP_LAUNCHES).

A pixel of a neck tensor is "non-constant" when its value may differ from the empty-space constant of its output-parity class: the
input pixel holds a site of the last sparse level, a tap of the conv that makes it falls outside the map, or a tap / the residual it
reads is non-constant.  Each launch runs the 8 (u) x 16 (v) tiles that hold a non-constant pixel or leave the map, plus the first
all-constant tile of every class (its representative); the other tiles are filled with the representative's values.
"""
import numpy as np

TU, TV = 8, 16
HEADER = 32


def _dilate3(m):
    """non-constant pixels of a 3x3 / pad 1 conv of a map with non-constant pixels m (out-of-map taps are non-constant)"""
    h, w = m.shape
    p = np.ones((h + 2, w + 2), bool)
    p[1:-1, 1:-1] = m
    out = np.zeros_like(m)
    for dy in range(3):
        for dx in range(3):
            out |= p[dy:dy + h, dx:dx + w]
    return out


def _deconv(t):
    """ConvTranspose2d(k3, s2, p1, op1): out[2g + p] reads in[g] and, for p = 1, in[g + 1] (per axis)"""
    h2, w2 = t.shape
    p = np.ones((h2 + 1, w2 + 1), bool)
    p[:h2, :w2] = t
    out = np.zeros((2 * h2, 2 * w2), bool)
    for py in (0, 1):
        for px in (0, 1):
            o = p[:h2, :w2].copy()
            if py:
                o |= p[1:, :w2]
            if px:
                o |= p[:h2, 1:]
            if py and px:
                o |= p[1:, 1:]
            out[py::2, px::2] = o
    return out


def masks(occ):
    """occ [h, w] bool (one frame) -> dict of the non-constant maps of every neck tensor (t0 = x0, t1 = x1 pixel for pixel)"""
    m = {"x": occ.astype(bool)}
    m["b0a"] = _dilate3(m["x"])
    m["b0b"] = _dilate3(m["b0a"])
    m["x0"] = _dilate3(m["b0b"])
    m["b1a"] = _dilate3(m["x0"])[0::2, 0::2][: occ.shape[0] // 2, : occ.shape[1] // 2]
    m["b1b"] = _dilate3(m["b1a"])
    m["x1"] = _dilate3(m["b1b"])
    m["t0"], m["t1"] = m["x0"], m["x1"]
    m["m1"] = _deconv(m["t1"])
    m["m0"] = m["m1"] | m["t0"]
    m["o0"] = _dilate3(m["m0"])
    m["o1"] = _dilate3(m["m1"])
    m["out"] = m["o0"] | m["o1"]
    m["head"] = m["out"]
    return m


# launch -> (output map, deconv, cout) in the order of SSFAPlanesRunner.SKIP_LAUNCHES
LAUNCHES = (("b0a", False, 128), ("b0b", False, 128), ("x0", False, 128), ("b1a", False, 256), ("b1b", False, 256), ("x1", False, 256),
            ("t0", False, 128), ("t1", False, 256), ("m0", True, 128), ("m1", True, 128), ("o0", False, 128), ("o1", False, 128),
            ("head", False, 24))


def geometry(batch, grid_h, grid_w, cout, deconv):
    """the bev_conv_p2 launcher's geometry: orientation, tiles, n-blocks, heavy-first class order"""
    cdiv = lambda a, b: -(-a // b)  # noqa: E731
    u_is_x = cdiv(grid_w, TU) * cdiv(grid_h, TV) <= cdiv(grid_h, TU) * cdiv(grid_w, TV)
    gu, gv = (grid_w, grid_h) if u_is_x else (grid_h, grid_w)
    tu, tv = cdiv(gu, TU), cdiv(gv, TV)
    ntaps = [(1 + (c >> 1)) * (1 + (c & 1)) for c in range(4)] if deconv else [9]
    order = sorted(range(len(ntaps)), key=lambda c: -ntaps[c])       # stable: the launcher's insertion sort
    return dict(u_is_x=u_is_x, grid_u=gu, grid_v=gv, tiles_u=tu, tiles_v=tv, tiles=tu * tv * batch,
                nblocks=cdiv(cout, 32 if cout <= 32 else 128), order=order, nclass=len(ntaps), stride=2 if deconv else 1)


def plan(occ):
    """occ [B, h, w] bool -> per launch dict(items, skipped, rep, flags) as the device writes them"""
    B, h, w = occ.shape
    fm = [masks(occ[b]) for b in range(B)]
    out = []
    for name, deconv, cout in LAUNCHES:
        half = name in ("b1a", "b1b", "x1", "t1") or deconv
        g = geometry(B, h // 2 if half else h, w // 2 if half else w, cout, deconv)
        flags = np.zeros((g["nclass"], g["tiles"]), bool)
        for c in range(g["nclass"]):
            py, px = (c >> 1, c & 1) if deconv else (0, 0)
            for t in range(g["tiles"]):
                tu, rest = t % g["tiles_u"], t // g["tiles_u"]
                tv, b = rest % g["tiles_v"], rest // g["tiles_v"]
                u0, v0 = tu * TU, tv * TV
                if u0 + TU > g["grid_u"] or v0 + TV > g["grid_v"]:
                    flags[c, t] = True
                    continue
                ys, xs = (slice(v0, v0 + TV), slice(u0, u0 + TU)) if g["u_is_x"] else (slice(u0, u0 + TU), slice(v0, v0 + TV))
                mm = fm[b][name][py::g["stride"], px::g["stride"]] if deconv else fm[b][name]
                flags[c, t] = bool(mm[ys, xs].any())
        rep = [int(np.flatnonzero(~flags[c])[0]) if (~flags[c]).any() else -1 for c in range(g["nclass"])]
        items = []
        for rank, c in enumerate(g["order"]):
            for nb in range(g["nblocks"]):
                for t in range(g["tiles"]):
                    if flags[c, t] or t == rep[c]:
                        items.append((rank * g["nblocks"] + nb) * g["tiles"] + t)
        skipped = [c * g["tiles"] + t for c in range(g["nclass"]) for t in range(g["tiles"]) if not flags[c, t] and t != rep[c]]
        out.append(dict(name=name, geometry=g, flags=flags, rep=rep, items=np.array(items, np.int64), skipped=np.array(skipped, np.int64)))
    return out


def occupancy_from_bitmap(words, batch, depth, h, w):
    """the last sparse level's bitmap index (int32 [words, 2], bit lin & 31 of word lin >> 5 in column 0) -> [B, h, w] bool"""
    bits = np.unpackbits(words[:, 0].astype("<u4").view(np.uint8), bitorder="little").astype(bool)
    n = batch * depth * h * w
    return bits[:n].reshape(batch, depth, h, w).any(axis=1)


def read_record(rec):
    """one launch record of the device plan (numpy int32) -> (items, skipped, rep)"""
    n, ns = int(rec[0]), int(rec[1])
    items = rec[HEADER:HEADER + n].astype(np.int64)
    skip_off = int(rec[23])
    return items, rec[skip_off:skip_off + ns].astype(np.int64), [int(v) for v in rec[19:23]]
