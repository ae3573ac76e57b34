"""A numpy model of how spconv_cg.cu stages its A operand across the tiles of a persistent launch, and crafted rulebooks built against
the grid the kernel launches.

The kernel (spconv_cg_kernel<CP, COUT, DEEP>) runs grid = min(ceil(max_out / 128), blocks_per_sm x SMs) persistent CTAs; CTA b runs the
tiles b, b + grid, ... in turn.  Each CTA carries a ring of kStages shared-memory stages from tile to tile: a tile with nact active
offsets fills the ring positions P .. P + nact - 1 (P = the fills of the CTA's earlier tiles), so its first fill lands in stage
st0 = P mod kStages with phase bit ph0 = (P / kStages) & 1.  Position p is filled by producer group p mod kGroups; each of the group's
warps keeps, in registers, which of its own rows of each of its stages hold data (the dirty masks) and clears a row of the stage when it
held data for the stage's previous offset and gets none for the new one.  A row that is not cleared keeps the input row of that
previous offset, which the wgmma then multiplies by the new offset's weights: a stale product.

replay() follows that bookkeeping fill by fill, for the kernel as written or with one of three staging faults, and reports what a
launch reaches (ring positions, clear slots) and which stale products a faulty kernel would add.
"""
import numpy as np

BM = 128                        # kCgBM: output rows per tile
MAX_K = 27                      # kCgMaxK
PROD_WARPS = 4                  # kCgProdWarps
THREADS = 12 * 32               # kCgThreads
CG_SHAPES = ((32, 32), (32, 64), (64, 32), (64, 64))      # (cp, cout): layers 3-4, 5, the 32 -> 64 data gradient, layers 6-12
NACTS = (1, 2, 3, 4, 5, 7, 8, 9, 27)                      # kStages - 1, kStages, kStages + 1 for kStages 2, 4, 8; 1 and 27
LONGEST_RING = 2 * 8                                      # (st0, ph0) of the 8-stage ring is P mod 16, which fixes it for 2 and 4
FAULTS = ("reset_at_tile", "half_never_clears", "no_rotation")


class CgLayout:
    """CgCfg<cp, cout, deep> restated: the ring, its producer groups and the dynamic shared memory of one CTA"""

    def __init__(self, cp, cout, deep):
        self.cp, self.cout, self.deep = cp, cout, int(bool(deep))
        wide = cp == 64
        self.stages = (2 if wide else 4) * (2 if deep else 1)
        self.groups = min(self.stages, PROD_WARPS)               # group g owns stages g, g + groups, ...
        self.group_warps = PROD_WARPS // self.groups             # 2 or 1
        self.group_stages = self.stages // self.groups           # 1 or 2
        self.own_rows = BM // self.group_warps                   # rows of a stage whose zero state one warp keeps: 128 or 64
        a_tile = (2 if wide else 1) * BM * 128
        b_tile = (2 if wide else 1) * cout * 128
        stage = a_tile + -(-b_tile // 1024) * 1024
        meta = (BM * MAX_K * 4 + MAX_K * 16 + 2 * cout * 4 + 32 * 4 + 33 * 4 + 32 * 4 + 3 * self.stages * 8 + 24)
        self.smem = self.stages * stage + meta + 1024

    def faults(self):
        """the staging faults this layout can have: every layout can lose its masks; only two-warp groups have a second warp's rows,
        only two-stage warps rotate"""
        return ("reset_at_tile",) + (("half_never_clears",) if self.group_warps == 2 else ()) + \
            (("no_rotation",) if self.group_stages == 2 else ())

    def __repr__(self):
        return "CgLayout(cp=%d, cout=%d, deep=%d: %d stages, %d groups x %d warps, %d stages per group)" % (
            self.cp, self.cout, self.deep, self.stages, self.groups, self.group_warps, self.group_stages)


def predicted_blocks_per_sm(layout, smem_per_sm, smem_reserved_per_block=1024, max_blocks=2):
    """CTAs per SM that the shared memory of layout.smem allows, capped by the kernel's __launch_bounds__ (2: 80 registers each)"""
    return min(max_blocks, smem_per_sm // (layout.smem + smem_reserved_per_block))


def cg_grid(cp, cout, deep, max_out):
    """the grid launch_spconv_cg launches: min(ceil(max_out / 128), blocks_per_sm x SMs) of the current device"""
    import torch
    from sessd_b200 import ops
    sms = torch.cuda.get_device_properties(torch.cuda.current_device()).multi_processor_count
    return min(-(-int(max_out) // BM), ops.spconv_cg_blocks_per_sm(cp, cout, deep) * sms)


def tile_ring(nbr, n, grid):
    """(cta, round, P, nact) of every tile of a launch at `grid` over the first n rows: P = fills of the CTA's earlier tiles"""
    ntiles = -(-n // BM)
    valid = nbr[:n] >= 0
    nact = np.array([int(valid[t * BM:(t + 1) * BM].any(0).sum()) for t in range(ntiles)], np.int64)
    p = np.zeros(ntiles, np.int64)
    for b in range(min(grid, ntiles)):
        ts = np.arange(b, ntiles, grid)
        p[ts] = np.concatenate([[0], np.cumsum(nact[ts])[:-1]])
    t = np.arange(ntiles)
    return t % grid, t // grid, p, nact


class Replay:
    """What one launch reaches.
    positions: {(nact, st0, ph0)} of every tile;
    clears: {(kind, stage, word)} of every dirty-row clear, kind "within" (the stale row is from the same tile), "across" (from the
      CTA's previous tile) or "older" (from an earlier one), word = tile row // 32 (its owner: warp word // (4 / group_warps) of the
      stage's group);
    gap_clears: {(stage, word)} of the clears whose stale row is from a tile the CTA ran before an empty tile;
    stale: (out_row, in_row, k) int64 [m, 3] of the products the replayed kernel adds that the rulebook does not have (none for the
      kernel as written)."""

    def __init__(self, positions, clears, gap_clears, stale):
        self.positions, self.clears, self.gap_clears, self.stale = positions, clears, gap_clears, stale

    def missing_positions(self, stages, nacts=NACTS):
        return sorted({(a, s, p) for a in nacts for s in range(stages) for p in (0, 1)} - self.positions)

    def missing_clears(self, stages, kinds=("within", "across")):
        return sorted({(kd, s, w) for kd in kinds for s in range(stages) for w in range(4)} - self.clears)

    def missing_gap_clears(self, stages):
        return sorted({(s, w) for s in range(stages) for w in range(4)} - self.gap_clears)


def replay(nbr, n, max_out, grid, layout, fault=None):
    """Replay the producers' staging of a launch of spconv_cg at `grid` CTAs over the table nbr [>= max_out, kvol] with n rows on the
    device.  fault: None (the kernel as written) or one of FAULTS --
      reset_at_tile: the dirty masks are zeroed at the head of every tile (a stage's rows from the CTA's previous tile are never cleared);
      half_never_clears: the second warp of a two-warp group never clears its 64 rows (its masks still follow the fills);
      no_rotation: a warp that owns two stages keeps one mask for both (it clears against its other stage's previous fill)."""
    assert fault is None or fault in FAULTS, fault
    n = min(int(n), int(max_out))
    assert 1 <= grid <= -(-int(max_out) // BM)
    S, G, GW, GS, OWN = layout.stages, layout.groups, layout.group_warps, layout.group_stages, layout.own_rows
    ntiles = -(-n // BM)
    positions, clears, gap_clears, stale = set(), set(), set(), []
    for b in range(min(grid, ntiles)):
        P = 0
        mem = np.full((S, BM), -1, np.int64)                 # input row held by each row of each stage (-1: zeros)
        mem_tile = np.full((S, BM), -1, np.int64)            # the tile whose fill wrote it
        dirty = np.zeros((PROD_WARPS, GS, OWN), bool)        # per warp: its rows of its stages, [0] = the stage of its next fill
        last_empty = -1                                      # the CTA's latest tile without any pair
        for t in range(b, ntiles, grid):
            rows = np.full((BM, nbr.shape[1]), -1, np.int64)
            live = nbr[t * BM:min(n, (t + 1) * BM)]
            rows[:len(live)] = live
            v = rows >= 0
            klist = np.nonzero(v.any(0))[0]
            positions.add((len(klist), P % S, (P // S) & 1))
            if fault == "reset_at_tile":
                dirty[:] = False
            for j, k in enumerate(klist):
                pos = P + j
                s, grp = pos % S, pos % G
                vs = v[:, k]
                for gw in range(GW):
                    warp = grp * GW + gw
                    own = vs[gw * OWN:(gw + 1) * OWN]
                    z = dirty[warp, 0] & ~own
                    dirty[warp, 0] = own
                    if z.any() and not (fault == "half_never_clears" and gw == 1):
                        rr = np.nonzero(z)[0] + gw * OWN
                        src = mem_tile[s, rr]
                        kinds = np.where(src == t, "within", np.where(src == t - grid, "across", "older"))
                        for kind, word, gap in zip(kinds, rr // 32, src < last_empty):
                            clears.add((str(kind), s, int(word)))
                            if gap:
                                gap_clears.add((s, int(word)))
                        mem[s, rr] = -1
                    if GS > 1 and fault != "no_rotation":
                        dirty[warp] = np.roll(dirty[warp], -1, axis=0)
                mem[s, v[:, k]] = rows[v[:, k], k]
                mem_tile[s, v[:, k]] = t
                extra = np.nonzero((mem[s] >= 0) & ~v[:, k] & (t * BM + np.arange(BM) < n))[0]
                if len(extra):
                    stale.append(np.stack([t * BM + extra, mem[s, extra], np.full(len(extra), k)], 1))
            if len(klist) == 0:
                last_empty = t
            P += len(klist)
    stale = np.concatenate(stale) if stale else np.zeros((0, 3), np.int64)
    return Replay(positions, clears, gap_clears, stale)


# ------------------------------------------------------------------------------------------------------------------ crafted tables
def sparse_tile(rng, rows, nact, n_in, kvol=MAX_K):
    """one tile [rows, kvol]: nact active offsets, every row 1 - 4 pairs among them, every active offset keeps >= 1 pair"""
    tile = np.full((rows, kvol), -1, np.int64)
    if nact == 0:
        return tile
    ks = np.sort(rng.choice(kvol, nact, replace=False))
    key = rng.random((rows, nact))
    j = np.arange(nact)
    key[j % rows, j] = -1.0                                  # row j % rows takes offset j first
    rank = np.argsort(np.argsort(key, 1), 1)
    ok = rank < np.minimum(rng.integers(1, 5, rows), nact)[:, None]
    sub = np.where(ok, rng.integers(0, n_in, (rows, nact)), -1)
    tile[:, ks] = sub
    return tile


def grid_table(grid, ntiles, last_rows, n_in, seed, empty=lambda t: False):
    """nbr [(ntiles - 1) * 128 + last_rows, 27] of sparse tiles (1 - 4 pairs per row) whose active-offset counts steer the CTAs of a
    launch at `grid` over every (nact in NACTS, P mod 16): every ring position of every ring length; tiles with empty(t) have no pair."""
    rng = np.random.default_rng(seed)
    n = (ntiles - 1) * BM + last_rows
    todo = {(a, p) for a in NACTS for p in range(LONGEST_RING)}
    P = np.zeros(grid, np.int64)
    tiles = []
    for t in range(ntiles):
        b = t % grid
        rows = min(BM, n - t * BM)
        if empty(t):
            nact = 0
        else:
            here = [a for a in NACTS if (a, P[b] % LONGEST_RING) in todo]
            if here:
                nact = here[rng.integers(len(here))]
            else:                                            # steer to the position with the most counts still to meet
                score = [sum((a, (P[b] + m) % LONGEST_RING) in todo for a in NACTS) + rng.random() for m in range(1, MAX_K + 1)]
                nact = 1 + int(np.argmax(score))
        tile = sparse_tile(rng, rows, nact, n_in)
        nact = int((tile >= 0).any(0).sum())
        todo.discard((nact, P[b] % LONGEST_RING))
        P[b] += nact
        tiles.append(tile)
    return np.concatenate(tiles)


def carry_table(grid, n_in, seed):
    """every CTA runs >= 3 busy tiles (3 grid + 1, the last one partial): a stage's rows of one tile are cleared by the CTA's next"""
    return grid_table(grid, 3 * grid + 1, 77, n_in, seed)


def gap_table(grid, n_in, seed):
    """busy, empty, busy on the even CTAs (round 1 of the launch has no pair there), busy throughout on the odd ones"""
    return grid_table(grid, 3 * grid + 1, 45, n_in, seed, empty=lambda t: (t // grid) == 1 and (t % grid) % 2 == 0)


def edge_specs(grid):
    """(name, ntiles, last_rows, max_out) around a device grid: tiles = grid - 1, grid, grid + 1, 2 grid + 1 with a partial last tile,
    and a table whose max_out sizes more tiles than the grid while the device count covers less than half of it (most CTAs leave at
    once).  The launch grid is min(ceil(max_out / 128), grid)."""
    def rows(ntiles, last):
        return (ntiles - 1) * BM + last
    return [("grid-1", grid - 1, 127, rows(grid - 1, 127)),               # grid - 1 CTAs, one tile each
            ("grid", grid, 1, rows(grid, 1) + 40),                        # one tile on every CTA, max_out inside the last tile
            ("grid+1", grid + 1, 64, rows(grid + 1, 64) + 3 * BM),        # CTA 0 runs a second, partial tile
            ("2grid+1", 2 * grid + 1, 100, rows(2 * grid + 1, 100)),      # CTA 0 runs three tiles, the others two
            ("exit", grid // 2, 33, (2 * grid + 3) * BM)]


def tile_permutation(kind, full, grid):
    """a permutation of the `full` whole tiles of a table (new position -> old tile): reverse, rotate (by one tile), or shuffle, which
    moves every tile to another CTA and another round of its launch at `grid`"""
    t = np.arange(full)
    if kind == "reverse":
        return t[::-1].copy()
    if kind == "rotate":
        return np.roll(t, 1)
    assert kind == "shuffle" and full % grid == 0 and full >= 2 * grid, (full, grid)
    rounds = full // grid
    r, b = t // grid, t % grid
    new = ((r + 1) % rounds) * grid + (b + 1 + 2 * r) % grid           # tile (round r, CTA b) -> (round r + 1, CTA b + 1 + 2r)
    perm = np.empty(full, np.int64)
    perm[new] = t
    return perm


def permute_tiles(nbr, n, perm):
    """the table with its whole tiles reordered by perm (new position -> old tile); rows past the permuted tiles (the partial last tile
    and anything past n) stay in place"""
    full = len(perm)
    out = nbr.copy()
    out[:full * BM] = nbr[:full * BM].reshape(full, BM, -1)[perm].reshape(full * BM, -1)
    return out
