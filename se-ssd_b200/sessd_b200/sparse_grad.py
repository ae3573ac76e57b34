"""Autograd through the sparse middle encoder (SpMiddleFHD in train mode, det3d/models/backbones/scn.py:176-189).

One conv of ``middle_conv`` is one ``SparseConvFunction``; BatchNorm1d and ReLU stay the torch modules they are (batch statistics and
running-stat updates exactly as the reference), and ``dense()`` is ``DenseFunction``.  Per layer (``impl``, ``conv_impl``: runners.sparse_impl, the rule
of the inference runner):

* ``rows`` (Cin <= 16): forward on the fp32 pair-proportional kernel (spconv_rows.cu), data gradient on the same kernel with re-packed
  weights, weight gradient on the fp32 SIMT wgrad kernel;
* ``cg`` (the wider layers): the input rows are split into fp16 (hi, lo) planes (sparse_split_planes) for the tensor-core forward
  (spconv_cg.cu), the output gradient likewise for the data gradient (the forward kernel again) and the tensor-core wgrad kernel.

Data gradient through the forward kernels: a SubM layer's table is point-symmetric, so the same table / tile lists serve with
W'[k] = W[K-1-k]^T (train.subm_dgrad_weight); a strided layer runs over the transposed table nbr_t (sessd_rulebook_transpose) with W[k]^T.
Rulebooks, nbr_t and tile lists are built once per rulebook (``ConvRulebook``) and shared by the layers of an ``indice_key``."""
import torch

from . import ops
from .runners import plane_width, sparse_impl
from .train import subm_dgrad_weight

conv_impl = sparse_impl     # kernel of a training conv: the inference runner's rule, with the tensor-core kernels


class ConvRulebook:
    """The rulebook of one conv geometry on one index set: output index set, neighbour table, device row counts, and -- built on first
    use -- the forward tile lists, the transposed table and its tile lists."""

    def __init__(self, conv, x):
        import spconv
        self.skeleton, self.nbr, self.n_out_t, self.cap_out = conv.rulebook(x)
        self.n_out = int(self.skeleton.indices.shape[0])
        self.n_in = int(x.indices.shape[0])
        self.n_in_t = x._n()
        self.cap_in = max(self.n_in, 1)
        self.kvol = int(self.nbr.shape[1])
        self.subm = bool(conv.subm)
        self._tiles = self._nbr_t = self._tiles_t = None
        self._tensor_cls = spconv.SparseConvTensor

    def tiles(self):
        if self._tiles is None:
            self._tiles = ops.rulebook_tile_lists(self.nbr, self.n_out_t, self.cap_out,
                                                  ops.alloc_tile_lists(self.cap_out, self.kvol, self.nbr.device))
        return self._tiles

    def nbr_t(self):
        if self._nbr_t is None:
            self._nbr_t = ops.rulebook_transpose(self.nbr, self.n_out_t, self.cap_out, self.cap_in)
        return self._nbr_t

    def tiles_t(self):
        if self._tiles_t is None:
            self._tiles_t = ops.rulebook_tile_lists(self.nbr_t(), self.n_in_t, self.cap_in,
                                                    ops.alloc_tile_lists(self.cap_in, self.kvol, self.nbr.device))
        return self._tiles_t

    def dgrad_table(self):
        """(table, tile lists) the data gradient gathers over: the forward's own for SubM, the transposed ones for strided layers"""
        return (self.nbr, self.tiles()) if self.subm else (self.nbr_t(), self.tiles_t())

    def wrap(self, features):
        s = self.skeleton
        out = self._tensor_cls(features, s.indices, s.spatial_shape, s.batch_size)
        out._index_kind, out._index, out.indice_dict = s._index_kind, s._index, s.indice_dict
        return out


def _split(x, n_t, n):
    """fp32 rows [n, C] -> (planes [n + 1, 2 C], info {abs-max, scale}); the extra row stays zero"""
    c = int(x.shape[1])
    info = torch.zeros((2,), dtype=torch.float32, device=x.device)
    planes = ops.alloc_planes(max(n, 1), c, x.device)
    if n > 0:
        ops.absmax_rows(x, n_t, n, info[0:1])
        ops.sparse_split_planes(x, n_t, n, info, planes)
    return planes, info


class SparseConvFunction(torch.autograd.Function):
    """out [n_out, Cout] = sparse conv of feat [n_in, Cin] with weight [kz, ky, kx, Cin, Cout] (spconv layout) over ``rb``"""

    @staticmethod
    def forward(ctx, feat, weight, rb):
        kvol, cin, cout = rb.kvol, int(weight.shape[3]), int(weight.shape[4])
        impl = conv_impl(cin)
        x = feat.detach().float().contiguous()
        w = weight.detach().float().reshape(kvol, cin, cout).contiguous()
        out = torch.empty((rb.cap_out, cout), dtype=torch.float32, device=x.device)
        saved = ()
        if rb.n_out == 0 or rb.n_in == 0:
            out.zero_()
        elif impl == "rows":
            ops.spconv_forward_rows(x, rb.nbr, rb.n_out_t, rb.cap_out, w, None, None, False, out)
            saved = (feat,)
        else:
            planes, info = _split(x, rb.n_in_t, rb.n_in)
            w_h2, inv = ops.pack_weight_sp_h2(w, plane_width(cin))
            ops.spconv_forward_cg(planes, info, rb.tiles(), rb.n_out_t, rb.cap_out, w_h2, inv, None, False, 0.0, 0.0, out, None, None)
            saved = (planes, info)
        # through save_for_backward: an in-place change of the input or the weight between forward and backward raises
        ctx.save_for_backward(weight, *saved)
        ctx.rb, ctx.impl, ctx.empty = rb, impl, not saved
        return out[:rb.n_out]

    @staticmethod
    def backward(ctx, gout):
        rb, impl = ctx.rb, ctx.impl
        weight, *saved = ctx.saved_tensors
        w5 = weight.detach().float()
        kvol, cin, cout = rb.kvol, int(w5.shape[3]), int(w5.shape[4])
        gout = gout.detach().float().contiguous()
        dev = gout.device
        want_x, want_w = ctx.needs_input_grad[0], ctx.needs_input_grad[1]
        if ctx.empty:                                              # no pairs: both gradients are zero
            return (torch.zeros((rb.n_in, cin), dtype=torch.float32, device=dev) if want_x else None,
                    torch.zeros_like(w5) if want_w else None, None)
        gfeat = gw = None
        if want_x:
            table, tiles = rb.dgrad_table()
            wd = (subm_dgrad_weight(w5) if rb.subm else w5.transpose(3, 4)).reshape(kvol, cout, cin).contiguous()
            gin = torch.empty((rb.cap_in, cin), dtype=torch.float32, device=dev)
        if impl == "rows":
            if want_w:
                x = saved[0].detach().float().contiguous()
                gw = ops.spconv_wgrad_rows(x, gout, rb.tiles(), rb.n_out_t, rb.cap_out, kvol).reshape(w5.shape)
            if want_x:
                ops.spconv_forward_rows(gout, table, rb.n_in_t, rb.cap_in, wd, None, None, False, gin)
                gfeat = gin[:rb.n_in]
        else:
            g_planes, g_info = _split(gout, rb.n_out_t, rb.n_out)
            if want_w:
                planes, info = saved
                gw = ops.spconv_wgrad_cg(planes, info, g_planes, g_info, rb.tiles(), rb.n_out_t, rb.cap_out, kvol).reshape(w5.shape)
            if want_x:
                wd_h2, inv = ops.pack_weight_sp_h2(wd, plane_width(cout))
                ops.spconv_forward_cg(g_planes, g_info, tiles, rb.n_in_t, rb.cap_in, wd_h2, inv, None, False, 0.0, 0.0, gin, None, None)
                gfeat = gin[:rb.n_in]
        return gfeat, gw, None


class DenseFunction(torch.autograd.Function):
    """SparseConvTensor.dense() + view(N, C*D, H, W) (scn.py:184-187): [B, C*D, H, W] in channels-last memory, channel = c*D + d"""

    @staticmethod
    def forward(ctx, feat, indices, batch_size, spatial_shape):
        n, c = int(feat.shape[0]), int(feat.shape[1])
        grid = ops.make_grid(batch_size, spatial_shape)
        d, h, w = spatial_shape
        out = torch.empty((batch_size, h, w, c * d), dtype=torch.float32, device=feat.device)
        n_t = torch.tensor([n], dtype=torch.int32, device=feat.device)
        ops.sparse_to_dense(feat.detach().float().contiguous(), indices, n_t, max(n, 1), grid, out)
        ctx.indices, ctx.n_t, ctx.n, ctx.c, ctx.grid = indices, n_t, n, c, grid
        return out.permute(0, 3, 1, 2)

    @staticmethod
    def backward(ctx, g):
        g = g.detach().float().permute(0, 2, 3, 1).contiguous()                      # NHWC
        out = torch.zeros((max(ctx.n, 1), ctx.c), dtype=torch.float32, device=g.device)
        if ctx.n > 0:
            ops.dense_grad_gather(g, ctx.indices, ctx.n_t, ctx.n, ctx.grid, ctx.c, out)
        return out[:ctx.n], None, None, None


def sparse_conv(conv, x, rulebooks):
    """one SubMConv3d / SparseConv3d of ``x`` through SparseConvFunction; ``rulebooks`` caches the SubM rulebooks by indice_key"""
    assert conv.bias is None, "the encoder's convs have no bias (scn.py:106-149)"
    key = conv.indice_key if conv.subm else None
    rb = rulebooks.get(key) if key is not None else None
    if rb is None:
        rb = ConvRulebook(conv, x)
        if key is not None:
            rulebooks[key] = rb
    return rb.wrap(SparseConvFunction.apply(x.features, conv.weight, rb)), rb


def encoder_forward(middle_conv, x, trace=None):
    """middle_conv (spconv.SparseSequential of conv / BatchNorm1d / ReLU) on x -> SparseConvTensor; trace (a list) receives the
    ConvRulebook of every conv"""
    import spconv
    rulebooks = {}
    for m in middle_conv._modules.values():
        if isinstance(m, spconv.SparseModule):
            x, rb = sparse_conv(m, x, rulebooks)
            if trace is not None:
                trace.append(rb)
        elif x.indices.shape[0] != 0:
            x.features = m(x.features)
    return x


def dense(x):
    """[B, C*D, H, W] of a SparseConvTensor (channels-last memory), differentiable w.r.t. x.features"""
    return DenseFunction.apply(x.features, x.indices.int().contiguous(), x.batch_size, list(x.spatial_shape))
