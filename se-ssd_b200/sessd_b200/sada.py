"""Shape-aware data augmentation (SA-DA) of SE-SSD's training frames on the device: pyramid dropout, farthest-point sparsify and pyramid
swap (reference: det3d/datasets/utils/sa_da_v2.py, pyramid_augment_v0, which Preprocess runs between the global scaling and the shuffle).

The draws are made here on the host from a numpy RandomState, with the reference's calls in the reference's order; the kernels of
csrc/sada.cu are pure functions of the points, the pyramids and the lists those draws select.  Two draws depend on the data: the swap's
``choice`` calls are sized by the per-pyramid point counts, and the shuffle after SA-DA by the frame's new size.  ``sada_frame`` therefore
reads the swap counts back once when a box is swap-selected, and the caller reads the frame's size back once before the shuffle.

Farthest-point sampling (the reference calls the external ``ifp_sample`` on the complete k = n neighbour lists of cKDTree, which makes it
exact farthest-point sampling) is pinned as: start at the pyramid's first point; each step takes the point with the largest fp64
distance to its nearest picked point, ties to the first; ``sparsity[1]`` picks in pick order (DESIGN §7).
"""
from dataclasses import dataclass

import numpy as np
import torch

from . import ops


@dataclass
class SadaConfig:
    """pyramid_augment_v0's arguments; the defaults are the car values Preprocess passes (pipelines/preprocess.py:147-151).  None turns a
    stage off, as in the reference."""
    dropout: float = 0.25                  # enable_sa_dropout
    sparsity: tuple = (0.05, 50)           # enable_sa_sparsity: (probability, points kept)
    swap: tuple = (0.1, 50)                # enable_sa_swap: (probability, points a pyramid needs)


def draw_pick(rs, k, p):
    """the dropout / sparsify draws of k boxes: ``randint(0, 6, k)`` then ``uniform(0, 1, k)``; returns (pyramid per box, box mask)"""
    idx = rs.randint(0, 6, (k,))
    return idx, rs.uniform(0, 1, (k,)) <= p


def draw_partners(rs, counts, selected, thr):
    """The swap's choices (sa_da_v2.py:131-153) given the point counts [N, 6] of the remaining pyramids and the selected boxes [N]:
    one ``choice`` per selected box with a valid pyramid (count > thr), then one per chosen pyramid over the other boxes whose same
    pyramid is valid and not chosen (none: the box itself).  Returns [(i, j, partner)] in row-major order of (i, j)."""
    counts = np.asarray(counts).reshape(-1, 6)
    selected = np.asarray(selected, bool)
    valid = counts > thr
    sel = valid * selected[:, None]
    if sel.sum() == 0:
        return []
    index_i, index_j = np.nonzero(sel)
    chosen = [rs.choice(index_j[index_i == i]) if e and (index_i == i).any() else 0 for i, e in enumerate(selected)]
    onehot = np.zeros((len(chosen), 6))
    onehot[range(len(chosen)), chosen] = 1
    mask = sel * onehot == 1
    index_i, index_j = np.nonzero(mask)
    valid[mask] = False
    partners = [rs.choice(np.where(valid[:, j])[0]) if np.where(valid[:, j])[0].shape[0] > 0 else index_i[i]
                for i, j in enumerate(index_j.tolist())]
    return [(int(i), int(j), int(q)) for i, j, q in zip(index_i, index_j, partners)]


def sada_frame(points, boxes, num_boxes, rs, cfg, stages=None):
    """SA-DA of one frame on the device.  points [N, 4] f32 (device, 16-byte aligned rows), boxes [>= num_boxes, 7] f32 (device, the
    frame's class-valid boxes after the global stages), num_boxes: their host-known count; rs: the RandomState; cfg: a SadaConfig.

    Returns (out [capacity, 4], num [1] i32 on the device): the frame's rows are out[:num].  Launches on the current stream; it waits on
    the device once, to read the swap counts back, and only when a box is swap-selected.  stages: an optional dict that receives each
    stage's (rows, count) for inspection."""
    n, K = int(points.shape[0]), int(num_boxes)
    dev = points.device
    pyr, planes = ops.sada_pyramids(boxes[:K].contiguous())
    alive = np.arange(K)
    cur, num = points, None

    def record(name):
        if stages is not None:
            stages[name] = (cur, num)

    if cfg.dropout is not None and K > 0:
        idx, drop = draw_pick(rs, K, cfg.dropout)
        ids = 6 * alive[drop] + idx[drop]
        if len(ids):
            bits, counts, _ = ops.sada_membership(cur, planes, ids, n=num)
            cur, num = ops.sada_compact(cur, bits, counts, -1, n=num)
        alive = alive[~drop]
    record("dropout")
    if cfg.sparsity is not None and len(alive) > 0:
        p, keep = cfg.sparsity
        idx, sel = draw_pick(rs, len(alive), p)
        ids = 6 * alive[sel] + idx[sel]
        if len(ids):
            rows = cur.shape[0]
            bits, counts, _ = ops.sada_membership(cur, planes, ids, n=num)
            out = torch.empty((rows + int(keep) * len(ids), 4), dtype=torch.float32, device=dev)
            _, new_num = ops.sada_compact(cur, bits, counts, int(keep), n=num, out=out)
            ops.sada_fps(cur, bits, counts, int(keep), int(keep), out, new_num, n=num)
            cur, num = out, new_num
        alive = alive[~sel]
    record("sparsify")
    if cfg.swap is not None:
        p, thr = cfg.swap
        sel = rs.uniform(0, 1, (len(alive),)) <= p
        if sel.any():
            _, counts, _ = ops.sada_membership(cur, planes, (6 * alive[:, None] + np.arange(6)).reshape(-1), n=num, with_bits=False)
            counts = counts.cpu().numpy().reshape(-1, 6)                # the read-back: the swap's choices are sized by these
            pairs = draw_partners(rs, counts, sel, thr)
            if pairs:
                ids = np.array([6 * alive[i] + j for i, j, _ in pairs] + [6 * alive[q] + j for _, j, q in pairs])
                extra = int(sum(counts[i, j] + counts[q, j] for i, j, q in pairs))
                bits, pc, d_ids = ops.sada_membership(cur, planes, ids, n=num)
                out = torch.empty((cur.shape[0] + extra, 4), dtype=torch.float32, device=dev)
                _, kept = ops.sada_compact(cur, bits, pc, -1, n=num, out=out)
                _, new_num = ops.sada_swap(cur, bits, pc, pyr, d_ids, extra, out, kept, n=num)
                cur, num = out, new_num
    record("swap")
    if num is None:
        num = torch.full((1,), n, dtype=torch.int32, device=dev)
    return cur, num
