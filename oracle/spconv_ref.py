"""CPU restatement of the sparse 3-D convolution stage (TEST INFRASTRUCTURE ONLY).

The arithmetic of this stage lives in **spconv 1.x** (third-party pip dependency of the reference,
``requirements.txt:28``, version unpinned, source NOT under /root/reference) -- PARITY UNPINNED.
What is restated here is spconv-1.x's published algorithm as the reference *configures* it:

* layer list, channel widths, kernel / stride / padding: ``det3d/models/backbones/scn.py:106-149``
* sparse shape ``grid[::-1] + [1,0,0]``, ``dense()`` and the ``view(N, C*D, H, W)``: ``scn.py:176-189``
* shape comments pinning the output-size rule ``out = floor((in + 2p - k)/s) + 1``:
  ``scn.py:113,122,134,146`` ([41,1600,1408] -> [21,800,704] -> [11,400,352] -> [5,200,176] -> [2,200,176])
* BatchNorm1d(eps=1e-3, momentum=0.01) + ReLU after every conv: ``scn.py:103-104``

spconv-1.x rules: weight layout ``[kz,ky,kx,Cin,Cout]``; a pair (i, o) exists for kernel offset k iff
``pos_i = pos_o * stride - pad + k`` (cross-correlation); SubM convs keep the input index set; regular
sparse convs output the set of all reachable in-bounds positions.  spconv's own output order is
atomics-dependent, so the *canonical* order used for parity is ascending linear index
``((b*D+z)*H+y)*W+x`` and, per kernel offset, pairs sorted by output index.
"""
import numpy as np

# (kind, cin, cout, ksize, stride, padding, indice_key)  -- scn.py:106-149
SPMIDDLE_FHD_LAYERS = [
    ("subm", None, 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm0"),
    ("subm", 16, 16, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm0"),
    ("spconv", 16, 32, (3, 3, 3), (2, 2, 2), (1, 1, 1), None),
    ("subm", 32, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm1"),
    ("subm", 32, 32, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm1"),
    ("spconv", 32, 64, (3, 3, 3), (2, 2, 2), (1, 1, 1), None),
    ("subm", 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm2"),
    ("subm", 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm2"),
    ("subm", 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm2"),
    ("spconv", 64, 64, (3, 3, 3), (2, 2, 2), (0, 1, 1), None),
    ("subm", 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm3"),
    ("subm", 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm3"),
    ("subm", 64, 64, (3, 3, 3), (1, 1, 1), (1, 1, 1), "subm3"),
    ("spconv", 64, 64, (3, 1, 1), (2, 1, 1), (0, 0, 0), None),
]


def out_shape(in_shape, ksize, stride, padding):
    return tuple((int(i) + 2 * p - k) // s + 1 for i, k, s, p in zip(in_shape, ksize, stride, padding))


def linear_index(coors, shape):
    c = coors.astype(np.int64)
    d, h, w = shape
    return ((c[:, 0] * d + c[:, 1]) * h + c[:, 2]) * w + c[:, 3]


def _lookup(sorted_keys, sorted_rows, q):
    pos = np.searchsorted(sorted_keys, q)
    pos = np.minimum(pos, len(sorted_keys) - 1) if len(sorted_keys) else pos
    hit = (sorted_keys[pos] == q) if len(sorted_keys) else np.zeros(len(q), bool)
    return np.where(hit, sorted_rows[pos] if len(sorted_keys) else -1, -1)


def neighbor_table(in_coors, in_shape, out_coors, ksize, stride, padding):
    """nbr[o, k] = row of the input voxel feeding output o through kernel offset k, or -1."""
    keys = linear_index(in_coors, in_shape)
    order = np.argsort(keys, kind="stable")
    skeys, srows = keys[order], order.astype(np.int64)
    kz, ky, kx = ksize
    nbr = np.full((out_coors.shape[0], kz * ky * kx), -1, np.int64)
    oc = out_coors.astype(np.int64)
    k = 0
    for a in range(kz):
        for b in range(ky):
            for c in range(kx):
                z = oc[:, 1] * stride[0] - padding[0] + a
                y = oc[:, 2] * stride[1] - padding[1] + b
                x = oc[:, 3] * stride[2] - padding[2] + c
                ok = (z >= 0) & (z < in_shape[0]) & (y >= 0) & (y < in_shape[1]) & (x >= 0) & (x < in_shape[2])
                q = ((oc[:, 0] * in_shape[0] + z) * in_shape[1] + y) * in_shape[2] + x
                r = _lookup(skeys, srows, np.where(ok, q, -1))
                nbr[:, k] = np.where(ok, r, -1)
                k += 1
    return nbr


def strided_out_coors(in_coors, in_shape, ksize, stride, padding):
    """Unique reachable output positions, ascending linear index (canonical order)."""
    oshape = out_shape(in_shape, ksize, stride, padding)
    ic = in_coors.astype(np.int64)
    cand = []
    for a in range(ksize[0]):
        for b in range(ksize[1]):
            for c in range(ksize[2]):
                nz = ic[:, 1] + padding[0] - a
                ny = ic[:, 2] + padding[1] - b
                nx = ic[:, 3] + padding[2] - c
                ok = (nz % stride[0] == 0) & (ny % stride[1] == 0) & (nx % stride[2] == 0)
                z, y, x = nz // stride[0], ny // stride[1], nx // stride[2]
                ok &= (nz >= 0) & (ny >= 0) & (nx >= 0) & (z < oshape[0]) & (y < oshape[1]) & (x < oshape[2])
                cand.append(((ic[:, 0] * oshape[0] + z) * oshape[1] + y)[ok] * oshape[2] + x[ok])
    keys = np.unique(np.concatenate(cand)) if cand else np.zeros((0,), np.int64)
    x = keys % oshape[2]
    t = keys // oshape[2]
    y = t % oshape[1]
    t = t // oshape[1]
    z = t % oshape[0]
    b = t // oshape[0]
    return np.stack([b, z, y, x], 1).astype(np.int32), oshape


def pairs_from_nbr(nbr):
    """Canonical rulebook: for each kernel offset, (in_idx, out_idx) sorted by out_idx."""
    out = []
    for k in range(nbr.shape[1]):
        o = np.nonzero(nbr[:, k] >= 0)[0]
        out.append((nbr[o, k].astype(np.int64), o.astype(np.int64)))
    return out


def conv_from_nbr(feat, nbr, weight, dtype=np.float64):
    """out[o] = sum_k feat[nbr[o,k]] @ W[k]; weight [K, Cin, Cout]."""
    feat = feat.astype(dtype)
    w = weight.astype(dtype)
    out = np.zeros((nbr.shape[0], w.shape[2]), dtype)
    for k in range(nbr.shape[1]):
        o = np.nonzero(nbr[:, k] >= 0)[0]
        if len(o):
            out[o] += feat[nbr[o, k]] @ w[k]
    return out


def bn_relu(x, gamma, beta, mean, var, eps=1e-3, relu=True):
    y = (x - mean) / np.sqrt(var + eps) * gamma + beta
    return np.maximum(y, 0) if relu else y


def spmiddle_forward(voxel_features, coors, batch_size, input_shape_xyz, params, dtype=np.float64, trace=None, caps=None):
    """scn.py:176-189.  params: list of dicts {weight [kz,ky,kx,Cin,Cout], gamma, beta, mean, var}.
    caps: optional per-level capacities (index = level, 1..4; None = unbounded): a strided layer keeps only the first caps[level]
    output sites in canonical order, as a capacity-bounded device level does after an overflow.
    Returns the dense BEV tensor [B, 128, 200, 176] (NCHW, channel = c*D + d)."""
    shape = tuple(int(v) for v in (np.array(input_shape_xyz)[::-1] + np.array([1, 0, 0])))
    feat = voxel_features.astype(dtype)
    cur = coors.astype(np.int32)
    books = {}
    level = 0
    for li, (kind, _cin, _cout, ks, st, pd, key) in enumerate(SPMIDDLE_FHD_LAYERS):
        p = params[li]
        w = p["weight"].reshape(-1, p["weight"].shape[3], p["weight"].shape[4])
        if kind == "subm":
            if key not in books:
                books[key] = neighbor_table(cur, shape, cur, ks, (1, 1, 1), tuple(k // 2 for k in ks))
            nbr = books[key]
        else:
            oc, oshape = strided_out_coors(cur, shape, ks, st, pd)
            level += 1
            if caps is not None and caps[level] is not None:
                oc = oc[:caps[level]]
            nbr = neighbor_table(cur, shape, oc, ks, st, pd)
            cur, shape = oc, oshape
        feat = conv_from_nbr(feat, nbr, w, dtype)
        feat = bn_relu(feat, p["gamma"], p["beta"], p["mean"], p["var"])
        if trace is not None:
            trace.append(dict(coors=cur.copy(), shape=shape, nbr=nbr, feat=feat.copy()))
    d, h, w_ = shape
    c = feat.shape[1]
    dense = np.zeros((batch_size, d, h, w_, c), dtype)
    dense[cur[:, 0], cur[:, 1], cur[:, 2], cur[:, 3]] = feat
    dense = dense.transpose(0, 4, 1, 2, 3).reshape(batch_size, c * d, h, w_)   # scn.py:186-187
    return dense


def random_params(seed, num_input_features=4):
    """Seeded random SpMiddleFHD parameters (no checkpoint is available offline)."""
    rng = np.random.default_rng(seed)
    out = []
    cin = num_input_features
    for (_kind, _c, cout, ks, _st, _pd, _key) in SPMIDDLE_FHD_LAYERS:
        fan_in = cin * ks[0] * ks[1] * ks[2]
        w = rng.standard_normal((ks[0], ks[1], ks[2], cin, cout)).astype(np.float32) * np.float32(np.sqrt(2.0 / fan_in))
        out.append(dict(weight=w,
                        gamma=(1.0 + 0.1 * rng.standard_normal(cout)).astype(np.float32),
                        beta=(0.1 * rng.standard_normal(cout)).astype(np.float32),
                        mean=(0.1 * rng.standard_normal(cout)).astype(np.float32),
                        var=(1.0 + 0.2 * rng.random(cout)).astype(np.float32)))
        cin = cout
    return out
