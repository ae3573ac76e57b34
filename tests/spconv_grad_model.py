"""numpy model of the sparse-conv weight-gradient kernels (csrc/spconv_grad.cu) and an fp64 torch restatement of SpMiddleFHD in train
mode; shared by tests/test_spconv_grad_model.py (CPU) and tests/test_gpu_spconv_grad.py.

Weight-gradient bounds (u = 2^-24).  The pairs of offset k are split into work items (offset, fixed tile range); item j of offset k sums
its pairs in tile-list order; the reduce adds the chunks' partials of the offset in ascending order from +0.

rows (fp32 fmaf chains) vs the exact fp64 result of the fp32 inputs, per element (c, n) of gW[k]:
    |got - ref| <= sum_items (P_item + 1) u M_item + chunks u M,     M_item = sum over the item's pairs of |x_c| |g_n|, M = sum_items M_item
  (a chain of P fmaf loses <= gamma_P of its magnitude; the reduce is a chain of `chunks` adds; the +1 absorbs the 1 / (1 - n u) terms).
cg (fp16 mma, split operands) vs an fp64 emulation of what it multiplies: a = (a_hi, a_lo) with x S_a = a_hi + a_lo + d, g likewise at
  S_g; emul = sum a_hi g_hi + a_hi g_lo + a_lo g_hi, / (S_a S_g).  One m16n8k16 step adds 16 exact products to the fp32 accumulator and
  loses <= 2 ulps of |C| + sum |p| (the forward's model, tests/test_gpu_spconv_ops.py), so an item with G steps (G = 2 sum over its tiles of
  ceil(count / 16): the cross accumulator takes two products per step) is off by <= CG_C 2^-23 G Ma; acc_m + acc_c adds one rounding:
    |got - emul| <= [sum_items CG_C 2^-23 (G_item + 1) Ma_item + chunks u Ma] / (S_a S_g),   Ma = sum |a_hi||g_hi| + |a_hi||g_lo| + |a_lo||g_hi|
cg vs fp64: plus the split error.  S maps the abs-max into [2^14, 2^15), so |d| <= 2^-9 <= 2^-23 amax S, and the dropped a_lo g_lo is
  below 2^-22 |x| |g| S_a S_g; with margin, per pair  + 2^-20 (amax_x |g_n| + |x_c| amax_g).
"""
import numpy as np
import torch

U = 2.0 ** -24
CG_C = 2.0
TILE = 128
ITEMS_TARGET = 4 * 132
KC = 64


def wgrad_chunks(max_out, kvol):
    """(chunks per offset, tiles per item): csrc/spconv_grad.cu wgrad_chunks"""
    nt = -(-max_out // TILE)
    c = min(-(-ITEMS_TARGET // kvol), nt)
    t = -(-nt // c)
    return -(-nt // t), t


def pow2_scale_for_bound(bound):
    e = int((np.array(bound, np.float32).view(np.uint32) >> 23) & 0xFF)
    if e in (0, 255):
        return 1.0
    return float(np.array(min(max(268 - e, 2), 252) << 23, np.uint32).view(np.float32))


def split16(v, s):
    xs = v.astype(np.float32) * np.float32(s)
    hi = xs.astype(np.float16)
    return hi, (xs - hi.astype(np.float32)).astype(np.float16)


def item_pairs(nbr, n_out, max_out):
    """{(k, chunk): [(i, o), ...]} in the order an item walks them: tiles ascending, then the tile's entries of offset k (ascending row);
    plus the item's mma step count G / 2 (sum over tiles of ceil(count / 16))"""
    kvol = nbr.shape[1]
    chunks, tpi = wgrad_chunks(max_out, kvol)
    n = min(n_out, max_out)
    nt = -(-n // TILE)
    items = {}
    for k in range(kvol):
        for c in range(chunks):
            pairs, steps = [], 0
            for t in range(c * tpi, min(nt, (c + 1) * tpi)):
                rows = np.arange(t * TILE, min(n, (t + 1) * TILE))
                o = rows[nbr[rows, k] >= 0]
                pairs += [(int(nbr[r, k]), int(r)) for r in o]
                steps += -(-len(o) // 16)
            items[(k, c)] = (pairs, steps)
    return items, chunks


class WgradCase:
    """x [n_in, Cin], g [n_out, Cout] fp32, nbr [max_out, kvol] (rows >= n_out ignored)"""

    def __init__(self, nbr, n_out, max_out, x, g):
        self.nbr, self.n_out, self.max_out, self.x, self.g = nbr, n_out, max_out, x, g
        self.kvol, self.cin, self.cout = nbr.shape[1], x.shape[1], g.shape[1]
        self.items, self.chunks = item_pairs(nbr, n_out, max_out)
        self.amax_x, self.amax_g = float(np.abs(x).max()), float(np.abs(g[:min(n_out, max_out)]).max())   # the kernel's abs-max: rows < n
        self.s_a, self.s_g = pow2_scale_for_bound(self.amax_x), pow2_scale_for_bound(self.amax_g)
        ah, al = split16(x, self.s_a)
        gh, gl = split16(g, self.s_g)
        self.ah, self.al = ah.astype(np.float64), al.astype(np.float64)
        self.gh, self.gl = gh.astype(np.float64), gl.astype(np.float64)

    def _sum(self, f, pairs):
        out = np.zeros((self.cin, self.cout))
        if pairs:
            i = np.array([p[0] for p in pairs])
            o = np.array([p[1] for p in pairs])
            out = f(i, o)
        return out

    def truth(self):
        x, g = self.x.astype(np.float64), self.g.astype(np.float64)
        return self.per_offset(lambda i, o: x[i].T @ g[o])

    def per_offset(self, f, items=None):
        items = self.items if items is None else items
        gw = np.zeros((self.kvol, self.cin, self.cout))
        for (k, _c), (pairs, _s) in items.items():
            gw[k] += self._sum(f, pairs)
        return gw

    def emul_terms(self, cross=True):
        ah, al, gh, gl = self.ah, self.al, self.gh, self.gl
        if cross:
            return lambda i, o: ah[i].T @ (gh[o] + gl[o]) + al[i].T @ gh[o]
        return lambda i, o: ah[i].T @ gh[o]

    def emul(self, cross=True, items=None):
        return self.per_offset(self.emul_terms(cross), items) / (self.s_a * self.s_g)

    def tol_rows(self):
        ax, ag = np.abs(self.x).astype(np.float64), np.abs(self.g).astype(np.float64)
        tol = np.zeros((self.kvol, self.cin, self.cout))
        tot = np.zeros_like(tol)
        for (k, _c), (pairs, _s) in self.items.items():
            m = self._sum(lambda i, o: ax[i].T @ ag[o], pairs)
            tol[k] += (len(pairs) + 1) * U * m
            tot[k] += m
        return tol + self.chunks * U * tot

    def tol_emul(self):
        ah, al, gh, gl = np.abs(self.ah), np.abs(self.al), np.abs(self.gh), np.abs(self.gl)
        tol = np.zeros((self.kvol, self.cin, self.cout))
        tot = np.zeros_like(tol)
        for (k, _c), (pairs, steps) in self.items.items():
            m = self._sum(lambda i, o: ah[i].T @ (gh[o] + gl[o]) + al[i].T @ gh[o], pairs)
            tol[k] += CG_C * 2.0 ** -23 * (2 * steps + 1) * m
            tot[k] += m
        return (tol + self.chunks * U * tot) / (self.s_a * self.s_g)

    def tol_fp64(self):
        ax, ag = np.abs(self.x).astype(np.float64), np.abs(self.g).astype(np.float64)
        split = self.per_offset(lambda i, o: self.amax_x * np.ones((self.cin, len(i))) @ ag[o] + ax[i].T @ np.full((len(i), self.cout), self.amax_g))
        return self.tol_emul() + 2.0 ** -20 * split

    # ---- negative controls: what subtly wrong kernels compute (emulation arithmetic)
    def wrong_dropped_pair(self):
        items = dict(self.items)
        key = max((kc for kc in items if items[kc][0]), key=lambda kc: len(items[kc][0]))
        pairs, s = items[key]
        items[key] = (pairs[:len(pairs) // 2] + pairs[len(pairs) // 2 + 1:], s)
        return self.emul(items=items)

    def wrong_swapped_offsets(self):
        e = self.emul()
        ks = [k for k in range(self.kvol) if np.abs(e[k]).max() > 0]
        e[[ks[0], ks[-1]]] = e[[ks[-1], ks[0]]]
        return e

    def wrong_no_cross(self):
        return self.emul(cross=False)

    def wrong_stale_slots(self):
        """a round with np % 16 != 0 reads slots [np, ceil(np / 16) 16) of its buffer still holding the pairs of the round before last (the
        rounds alternate between two buffers): what a copy that did not zero-fill those slots computes"""
        items = dict(self.items)
        for key, (pairs, s) in self.items.items():
            k, c = key
            chunks, tpi = wgrad_chunks(self.max_out, self.kvol)
            n = min(self.n_out, self.max_out)
            rounds = []
            for t in range(c * tpi, min(-(-n // TILE), (c + 1) * tpi)):
                rows = np.arange(t * TILE, min(n, (t + 1) * TILE))
                o = rows[self.nbr[rows, k] >= 0]
                tp = [(int(self.nbr[r, k]), int(r)) for r in o]
                rounds += [tp[p0:p0 + KC] for p0 in range(0, len(tp), KC)]
            for j in range(2, len(rounds)):
                npr, kp = len(rounds[j]), -(-len(rounds[j]) // 16) * 16
                stale = rounds[j - 2][npr:kp]
                if stale:
                    items[key] = (pairs + stale, s)
                    return self.emul(items=items)
        raise AssertionError("no round in this case reads a slot of the round before last")

    def wrong_reduce(self, mode):
        """one chunk's partial summed twice ('twice') or lost ('lost') in the reduce"""
        items = dict(self.items)
        key = max((kc for kc in items if items[kc][0]), key=lambda kc: len(items[kc][0]))
        pairs, s = items[key]
        items[key] = (pairs * 2 if mode == "twice" else [], s)
        return self.emul(items=items)


def ratio(got, ref, tol):
    d = np.abs(np.asarray(got, np.float64) - ref)
    r = np.divide(d, tol, out=np.where(d > 0, np.inf, 0.0), where=tol > 0)
    return float(r.max()) if r.size else 0.0


# ------------------------------------------------------------------------------------------------ fp64 restatement of the train forward
def torch_conv(feat, nbr, w):
    """out[o] = sum_k feat[nbr[o, k]] @ W[k] in torch (autograd); nbr numpy int [n_out, K], w [K, Cin, Cout]"""
    n_in = feat.shape[0]
    pad = torch.cat([feat, feat.new_zeros((1, feat.shape[1]))], 0)
    idx = torch.from_numpy(np.where(nbr >= 0, nbr, n_in).astype(np.int64))
    out = feat.new_zeros((nbr.shape[0], w.shape[2]))
    for k in range(nbr.shape[1]):
        out = out + pad[idx[:, k]] @ w[k]
    return out


def spmiddle_train_ref(feat, coors, batch_size, input_shape_xyz, params, momentum=0.01, eps=1e-3):
    """scn.py:176-189 in fp64 torch on the CPU with train-mode BatchNorm1d: params = list of dicts of fp64 tensors {weight (requires grad),
    gamma, beta (require grad), mean, var (running stats, updated in place)}.  Returns the dense [B, C*D, H, W] tensor."""
    from oracle import spconv_ref as S
    shape = tuple(int(v) for v in (np.array(input_shape_xyz)[::-1] + np.array([1, 0, 0])))
    x = feat
    cur = coors.astype(np.int32)
    books = {}
    for li, (kind, _cin, _cout, ks, st, pd, key) in enumerate(S.SPMIDDLE_FHD_LAYERS):
        p = params[li]
        w = p["weight"].reshape(-1, p["weight"].shape[3], p["weight"].shape[4])
        if kind == "subm":
            if key not in books:
                books[key] = S.neighbor_table(cur, shape, cur, ks, (1, 1, 1), tuple(k // 2 for k in ks))
            nbr = books[key]
        else:
            oc, oshape = S.strided_out_coors(cur, shape, ks, st, pd)
            nbr = S.neighbor_table(cur, shape, oc, ks, st, pd)
            cur, shape = oc, oshape
        x = torch_conv(x, nbr, w)
        x = torch.nn.functional.batch_norm(x, p["mean"], p["var"], p["gamma"], p["beta"], True, momentum, eps)
        x = torch.relu(x)
    d, h, w_ = shape
    c = x.shape[1]
    dense = x.new_zeros((batch_size, d, h, w_, c))
    idx = torch.from_numpy(cur.astype(np.int64))
    dense = dense.index_put((idx[:, 0], idx[:, 1], idx[:, 2], idx[:, 3]), x)
    return dense.permute(0, 4, 1, 2, 3).reshape(batch_size, c * d, h, w_)
