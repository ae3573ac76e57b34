"""CPU restatement of the frame's front end -- the voxeliser (csrc/voxelize.cu), the rulebook builders (csrc/rulebook.cu) and the
device scan both use (csrc/common.cuh) -- with generators of crafted inputs that reach every code path.  Used by
tests/test_frontend_model.py (CPU) and tests/test_gpu_frontend_ops.py.

Everything here is integer work (the voxel cell is IEEE fp32 subtract / divide / floor, which numpy float32 rounds the same way),
so every device output is expected bit for bit.  The models take a set of mutation flags; each flag is one plausible wrong
kernel, and the CPU tests check that each changes at least one crafted expectation:

  "no_x_bound" / "no_yz_bound"   neighbour lookups skip the x (resp. y and z) range check, so a face site's neighbour index wraps
                                 into the next row (frame)
  "no_parity"                    a strided conv marks outputs whose tap is not divisible by the stride (floor division instead)
  "inclusive"                    the bitmap prefix is inclusive instead of exclusive
  "lost_carry"                   a scan tile of kScanTile words loses the sum of the tiles before it
  "untruncated"                  an overflowed level keeps answering lookups with ranks >= its capacity
  "cut_off_by_one"               the max_voxels cut lets one voxel too many through
  "keep_last"                    a voxel keeps its last max_points points instead of its first
  "no_frame_key"                 the voxel key misses the frame index (frames share cells)
"""
import numpy as np

F32 = np.float32
U64 = np.uint64
SCAN_TILE = 256 * 8                 # kScanTile: items per tile of the multi-CTA scan
SCAN_SMALL_MAX = 16 * 1024          # kScanSmallMax: capacity up to which one CTA scans
SCAN_SELF_PREFIX_TILES = 1024       # kScanSelfPrefixTiles: tiles up to which every apply CTA sums the tiles before it
WORD_THRESHOLDS = (SCAN_SMALL_MAX, SCAN_SMALL_MAX + 1, SCAN_TILE * SCAN_SELF_PREFIX_TILES, SCAN_TILE * SCAN_SELF_PREFIX_TILES + 1)


# ------------------------------------------------------------------------------------------------------------ hash
def hash_mix(keys):
    """fmix64 of common.cuh's hash_mix, low 32 bits (uint64 arrays wrap like the device's 64-bit multiplies)"""
    k = np.array(keys, dtype=U64, ndmin=1)
    k ^= k >> U64(33)
    k *= U64(0xff51afd7ed558ccd)
    k ^= k >> U64(33)
    k *= U64(0xc4ceb9fe1a85ec53)
    k ^= k >> U64(33)
    return (k & U64(0xFFFFFFFF)).astype(np.int64)


def hash_capacity(rows):
    """slots of the open-addressing table for `rows` keys: the smallest power of two >= max(1024, 2 rows)"""
    cap = 1024
    while cap < 2 * rows:
        cap <<= 1
    return cap


def home_slot(keys, cap):
    return hash_mix(keys) & (cap - 1)


def vox_key(f, cells_xyz, grid_xyz):
    """voxeliser key ((f gz + z) gy + y) gx + x"""
    c = np.asarray(cells_xyz, np.int64).reshape(-1, 3)
    gx, gy, gz = (int(v) for v in grid_xyz)
    return ((np.asarray(f, np.int64) * gz + c[:, 2]) * gy + c[:, 1]) * gx + c[:, 0]


def rb_key(coors, shape):
    """rulebook key ((b D + z) H + y) W + x of (b, z, y, x) rows"""
    c = np.asarray(coors, np.int64).reshape(-1, 4)
    d, h, w = (int(v) for v in shape)
    return ((c[:, 0] * d + c[:, 1]) * h + c[:, 2]) * w + c[:, 3]


def pick_collisions(keys, cap, groups=24, size=2, wrap=4, seed=0):
    """indices into the distinct `keys`: `wrap` keys whose home slot is cap - 1 (their probe run wraps past the last slot) and
    `groups` groups of `size` keys sharing one home slot each"""
    keys = np.asarray(keys, np.int64)
    home = home_slot(keys, cap)
    rng = np.random.default_rng(seed)
    last = np.nonzero(home == cap - 1)[0]
    assert len(last) >= wrap, "too few candidates with home slot cap - 1"
    out = list(rng.choice(last, wrap, replace=False))
    order = np.argsort(home, kind="stable")
    hs = home[order]
    starts = np.nonzero(np.r_[True, hs[1:] != hs[:-1]])[0]
    lens = np.diff(np.r_[starts, len(hs)])
    good = [s for s, n in zip(starts, lens) if n >= size and hs[s] != cap - 1]
    assert len(good) >= groups, "too few colliding home slots among the candidates"
    for s in rng.choice(good, groups, replace=False):
        out.extend(order[s:s + size])
    return np.array(out, np.int64)


def probe_runs(table, cap):
    """For a table read back from the device (int64 [cap]; entry key << 24 | value, empty = -1): per stored key (key, value, home,
    slot, every slot from home to slot occupied).  The last is what an open-addressing lookup needs to find the key."""
    t = np.asarray(table, np.int64).view(U64)
    occ = t != U64(0xFFFFFFFFFFFFFFFF)
    slots = np.nonzero(occ)[0]
    keys = (t[slots] >> U64(24)).astype(np.int64)
    vals = (t[slots] & U64((1 << 24) - 1)).astype(np.int64)
    home = home_slot(keys, cap)
    ok = np.array([occ[np.arange(h, h + ((s - h) % cap) + 1) % cap].all() for h, s in zip(home, slots)], bool)
    return keys, vals, home, slots, ok


# ------------------------------------------------------------------------------------------------------------ rulebooks
def out_shape(in_shape, ksize, stride, padding):
    return tuple((int(i) + 2 * p - k) // s + 1 for i, k, s, p in zip(in_shape, ksize, stride, padding))


def _lookup(index_keys, q):
    """rows of the query keys in a key list whose row i has key index_keys[i]; -1 where absent"""
    order = np.argsort(index_keys, kind="stable")
    sk = index_keys[order]
    if not len(sk):
        return np.full(len(q), -1, np.int64)
    pos = np.minimum(np.searchsorted(sk, q), len(sk) - 1)
    return np.where(sk[pos] == q, order[pos], -1)


def neighbor_table(index_coors, in_shape, out_coors, ksize, stride, padding, mut=()):
    """nbr[o, k] = row (in index_coors) of the site at out * stride - pad + k, or -1"""
    d, h, w = (int(v) for v in in_shape)
    keys = rb_key(index_coors, in_shape)
    oc = np.asarray(out_coors, np.int64).reshape(-1, 4)
    kz, ky, kx = ksize
    nbr = np.full((len(oc), kz * ky * kx), -1, np.int64)
    k = 0
    for a in range(kz):
        for b in range(ky):
            for c in range(kx):
                z = oc[:, 1] * stride[0] - padding[0] + a
                y = oc[:, 2] * stride[1] - padding[1] + b
                x = oc[:, 3] * stride[2] - padding[2] + c
                ok = np.ones(len(oc), bool)
                if "no_yz_bound" not in mut:
                    ok &= (z >= 0) & (z < d) & (y >= 0) & (y < h)
                if "no_x_bound" not in mut:
                    ok &= (x >= 0) & (x < w)
                q = ((oc[:, 0] * d + z) * h + y) * w + x
                nbr[:, k] = np.where(ok, _lookup(keys, np.where(ok, q, -1)), -1)
                k += 1
    return nbr


def strided_sites(in_coors, in_shape, ksize, stride, padding, batch, mut=()):
    """linear indices (in the output grid) of every reachable output site, ascending; and the output shape"""
    os_ = out_shape(in_shape, ksize, stride, padding)
    ic = np.asarray(in_coors, np.int64).reshape(-1, 4)
    cand = [np.zeros(0, np.int64)]
    for a in range(ksize[0]):
        for b in range(ksize[1]):
            for c in range(ksize[2]):
                n = [ic[:, 1] + padding[0] - a, ic[:, 2] + padding[1] - b, ic[:, 3] + padding[2] - c]
                ok = (n[0] >= 0) & (n[1] >= 0) & (n[2] >= 0)
                if "no_parity" not in mut:
                    for j in range(3):
                        ok &= n[j] % stride[j] == 0
                z, y, x = (n[j] // stride[j] for j in range(3))
                ok &= (z < os_[0]) & (y < os_[1]) & (x < os_[2])
                cand.append(((ic[ok, 0] * os_[0] + z[ok]) * os_[1] + y[ok]) * os_[2] + x[ok])
    return np.unique(np.concatenate(cand)), os_


def coors_of(lin, shape):
    d, h, w = (int(v) for v in shape)
    lin = np.asarray(lin, np.int64)
    x, t = lin % w, lin // w
    y, t = t % h, t // h
    z, b = t % d, t // d
    return np.stack([b, z, y, x], 1).astype(np.int32).reshape(-1, 4)


def bitmap_level(sites, nwords, max_out, mut=()):
    """The bitmap index of a strided level and its enumeration, as the device builds them: bits per 32-cell word, the exclusive prefix
    of the word popcounts (the device scan), then the ranks.  Returns (row of every site [len(sites)], -1 where the level dropped it;
    number of sites the level holds).  Row r of the level's coordinate list is the site with row r."""
    sites = np.asarray(sites, np.int64)
    word = sites >> 5
    pop = np.bincount(word, minlength=nwords).astype(np.int64) if len(sites) else np.zeros(nwords, np.int64)
    pref = np.cumsum(pop) - (0 if "inclusive" in mut else pop)
    if "lost_carry" in mut:
        start = np.arange(nwords) // SCAN_TILE * SCAN_TILE
        pref = pref - (np.cumsum(pop) - pop)[start]
    below = np.arange(len(sites)) - np.searchsorted(word, word)      # sites are ascending: set bits of the same word below
    rank = pref[word] + below
    keep = (rank < max_out) | ("untruncated" in mut)
    return np.where(keep, rank, -1), min(len(sites), max_out)


def level_coors(sites, rows, n, shape):
    """coordinate list [n, 4] of a level from the rows bitmap_level gave its sites (unset rows stay -1)"""
    out = np.full((n, 4), -1, np.int32)
    ok = (rows >= 0) & (rows < n)
    out[rows[ok]] = coors_of(sites[ok], shape)
    return out


def level_table(sites, rows, shape, out_coors, ksize, stride, padding):
    """neighbour table whose lookups go through a level's index: a site answers its row (which may exceed the level's capacity
    under "untruncated"), a dropped site answers -1"""
    keys = np.full(max(int(rows.max()) + 1, 0) if len(rows) else 0, -1, np.int64)
    keys[rows[rows >= 0]] = sites[rows >= 0]
    idx = coors_of(keys, shape)
    idx[keys < 0] = (-(1 << 20), 0, 0, 0)                      # holes: an impossible frame, never matched
    return neighbor_table(idx, shape, out_coors, ksize, stride, padding)


# ------------------------------------------------------------------------------------------------------------ voxeliser
def cells_of(points, voxel_size, range_min, grid_xyz):
    """fp32 floor((p - lo) / vs) per axis (x, y, z) and whether the point lies inside the grid (NaN and +-Inf do not)"""
    p = np.asarray(points, F32)[:, :3]
    with np.errstate(invalid="ignore"):
        cf = np.floor((p - np.asarray(range_min, F32)) / np.asarray(voxel_size, F32))
        ok = ((cf >= 0) & (cf < np.asarray(grid_xyz, F32))).all(1)
    return np.where(ok[:, None], cf, 0).astype(np.int64), ok


def voxelize_batch(clouds, voxel_size, range_min, grid_xyz, max_points, max_voxels, mut=()):
    """The batched voxeliser: per frame (voxels [m, max_points, F], coors [m, 3] zyx, num_points [m], mean [m, F]).
    Voxel order = order of first points; the frame stops at the first point that would open voxel #max_voxels (every later
    point of the frame is dropped); a voxel keeps its first max_points points; mean = fp32 sum in slot order / count."""
    nf = np.asarray(clouds[0]).shape[1] if clouds else 4
    pts = np.concatenate([np.asarray(c, F32).reshape(-1, nf) for c in clouds], 0)
    fr = np.concatenate([np.full(len(c), f, np.int64) for f, c in enumerate(clouds)])
    cells, ok = cells_of(pts, voxel_size, range_min, grid_xyz)
    key = vox_key(0 if "no_frame_key" in mut else fr, cells, grid_xyz)
    idx = np.nonzero(ok)[0]
    limit = max_voxels + (1 if "cut_off_by_one" in mut else 0)
    uk, first, inv = np.unique(key[idx], return_index=True, return_inverse=True)
    first = idx[first]                                     # first point (global index) of every distinct key
    vfr = fr[first]
    order = np.argsort(first, kind="stable")
    local = np.empty(len(uk), np.int64)
    cut = np.array([len(fr)] * len(clouds), np.int64)
    for f in range(len(clouds)):
        mine = order[vfr[order] == f]
        local[mine] = np.arange(len(mine))
        if len(mine) > limit:
            cut[f] = first[mine[limit]]
    kept_v = local < limit
    pv = inv                                               # voxel of each valid point
    live = kept_v[pv] & (idx < cut[fr[idx]])
    out = []
    for f in range(len(clouds)):
        vs_ = order[(vfr[order] == f) & kept_v[order]]
        m = len(vs_)
        slot = np.full(len(uk), -1, np.int64)
        slot[vs_] = np.arange(m)
        vox = np.zeros((m, max_points, nf), F32)
        num = np.zeros(m, np.int32)
        pi = idx[live & (slot[pv] >= 0)]
        pvv = slot[pv[live & (slot[pv] >= 0)]]
        s = np.lexsort((pi, pvv))
        pi, pvv = pi[s], pvv[s]
        start = np.searchsorted(pvv, np.arange(m))
        cnt = np.bincount(pvv, minlength=m)
        rank = np.arange(len(pi)) - start[pvv]
        if "keep_last" in mut:
            rank = rank - np.maximum(cnt[pvv] - max_points, 0)
        sel = (rank >= 0) & (rank < max_points)
        vox[pvv[sel], rank[sel]] = pts[pi[sel]]
        num[:] = np.minimum(cnt, max_points)
        coors = cells[first[vs_]][:, ::-1].astype(np.int32)
        out.append((vox, coors.reshape(-1, 3), num, voxel_mean(vox, num)))
    return out


def voxel_mean(vox, num):
    """fp32 sum over the first num slots in slot order, then one fp32 divide (what both gather kernels compute)"""
    s = np.zeros((vox.shape[0], vox.shape[2]), F32)
    for k in range(vox.shape[1]):
        s = np.where((k < num)[:, None], (s + vox[:, k]).astype(F32), s)
    with np.errstate(invalid="ignore", divide="ignore"):
        return (s / num.astype(F32)[:, None]).astype(F32)


# ------------------------------------------------------------------------------------------------------------ generators
VOXEL_SIZE = (0.05, 0.05, 0.1)
RANGE_MIN = (0.0, -40.0, -3.0)
GRID = (1408, 1600, 40)


def cell_points(cells_xyz, seed=0, nf=4, jitter=True):
    """one point inside each cell (x, y, z): near the centre, checked against the fp32 cell rule; extra features random"""
    c = np.asarray(cells_xyz, np.int64).reshape(-1, 3)
    rng = np.random.default_rng(seed)
    off = 0.5 + (rng.uniform(-0.3, 0.3, c.shape) if jitter else 0.0)
    xyz = (np.asarray(RANGE_MIN) + (c + off) * np.asarray(VOXEL_SIZE)).astype(F32)
    p = np.concatenate([xyz, rng.uniform(-1, 1, (len(c), nf - 3)).astype(F32)], 1)
    got, ok = cells_of(p, VOXEL_SIZE, RANGE_MIN, GRID)
    assert ok.all() and np.array_equal(got, c)
    return p


def random_cells(rng, n, grid=GRID):
    """n distinct cells (x, y, z)"""
    g = np.asarray(grid, np.int64)
    lin = rng.choice(int(np.prod(g)), n, replace=False)
    return np.stack([lin % g[0], lin // g[0] % g[1], lin // (g[0] * g[1])], 1)


def cut_cloud(seed, max_voxels, delta, nf=4, max_points=5):
    """max_voxels + delta distinct cells in first-appearance order; after the first point of the last cell, more points of
    cells opened earlier (dropped by the cut when delta > 0); some voxels get max_points +- 1 and 100 points"""
    rng = np.random.default_rng(seed)
    m = max_voxels + delta
    cells = random_cells(rng, m)
    rep = np.ones(m, np.int64)
    rep[: min(m, 3)] = [max_points - 1, max_points, max_points + 1][: min(m, 3)]
    if m > 3:
        rep[3] = 100
    seq = np.repeat(np.arange(m), rep)
    rng.shuffle(seq[: len(seq) // 2])                      # interleave the early voxels' points
    seq = np.concatenate([seq, rng.integers(0, max(m // 2, 1), 50)])
    return cell_points(cells[seq], seed, nf)


def clouds_with_edges(seed, nf=4):
    """a frame whose points include NaN and +-Inf coordinates and points on and just outside the range faces"""
    rng = np.random.default_rng(seed)
    p = cell_points(random_cells(rng, 300), seed, nf)
    bad = np.repeat(p[:12].copy(), 1, 0)
    bad[0, 0], bad[1, 1], bad[2, 2] = np.nan, np.nan, np.nan
    bad[3, 0], bad[4, 1], bad[5, 2] = np.inf, -np.inf, np.inf
    bad[6, 0], bad[7, 1], bad[8, 2] = -np.inf, np.inf, -np.inf
    bad[9, 0] = np.float32(70.4)                            # x = range max: cell 1408, outside
    bad[10, 1] = np.float32(-40.0001)                       # below the y range
    bad[11, 3:] = np.nan                                    # NaN payload only: kept
    out = np.concatenate([p[:100], bad, p[100:]], 0)
    return out, np.isnan(out[:, :3]).any(1)


def boundary_cloud(count, cap_tiles=(2047, 2048, 2049), seed=0, nf=4):
    """`count` points in which the first point of a new voxel sits at every listed index (< count) and every other point repeats the
    previous point's cell (scan-tile boundaries of the first-point flags)"""
    rng = np.random.default_rng(seed)
    if count == 0:
        return np.zeros((0, nf), F32)
    marks = sorted({0} | {i for i in cap_tiles if i < count} | set(rng.integers(0, count, min(count, 64)).tolist()))
    cells = random_cells(rng, len(marks))
    seq = np.zeros(count, np.int64)
    for j, s in enumerate(marks):
        seq[s:] = j
    return cell_points(cells[seq], seed, nf)


def face_sites(batch, shape, empty=(), single=(), dense=()):
    """(b, z, y, x) rows: per frame, every site whose coordinates are each in {0, 1, mid, S-2, S-1} (all faces, edges and
    corners, even and odd); frames in `empty` hold nothing, in `single` one corner, in `dense` every cell of a 4^3 corner block too"""
    rows = []
    for b in range(batch):
        if b in empty:
            continue
        if b in single:
            rows.append((b, shape[0] - 1, 0, shape[2] - 1))
            continue
        vals = [sorted({0, 1, s // 2, s - 2, s - 1} & set(range(s))) for s in shape]
        for z in vals[0]:
            for y in vals[1]:
                for x in vals[2]:
                    rows.append((b, z, y, x))
        if b in dense:
            for z in range(min(4, shape[0])):
                for y in range(min(4, shape[1])):
                    for x in range(min(4, shape[2])):
                        rows.append((b, z, y, x))
    c = np.unique(np.array(rows, np.int64).reshape(-1, 4), axis=0)
    return c[np.argsort(rb_key(c, shape), kind="stable")].astype(np.int32)


def word_sites(words, extra_words=()):
    """input x positions (along one x-line, even and odd) whose outputs land in the first, last and scan-tile-boundary words of an
    output line of 32 * words cells, for a (1, 1, 3) s2 p1 layer: input x = 2 X reaches output X, 2 X + 1 reaches X and X + 1"""
    ws = {0, 1, words - 1} | set(extra_words)
    for t in range(1, words // SCAN_TILE + 1):
        ws |= {t * SCAN_TILE - 1, t * SCAN_TILE, t * SCAN_TILE + 1}
    ws = sorted(w for w in ws if 0 <= w < words)
    xs = []
    for w in ws:
        xs += [2 * (32 * w), 2 * (32 * w + 31), 2 * (32 * w + 7) + 1]
    xs = sorted(set(x for x in xs if x < 2 * 32 * words - 1))
    return np.array(xs, np.int64)
