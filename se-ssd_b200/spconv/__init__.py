"""spconv -- the slice of the spconv 1.x Python API that det3d/models/backbones/scn.py uses (scn.py:4,9,24-44,46,106-149,
182-184), backed by the sessd_b200 rulebook / gather-GEMM kernels.  spconv itself is a third-party dependency of the
reference (requirements.txt:28) whose source is not part of it; the semantics implemented here are spconv 1.x's published
ones: weight layout [kz,ky,kx,Cin,Cout], cross-correlation pairs, SubM convs keep the input index set, regular sparse convs emit
every reachable output site, ``dense()`` returns [B, C, D, H, W].  Output rows of SparseConv3d are in ascending linear index
(spconv's own order is atomics-dependent).  The modules do not build an autograd graph; SpMiddleFHD in train mode differentiates
through the same rulebooks with sessd_b200.sparse_grad.
"""
import math

import numpy as np
import torch
from torch import nn

from sessd_b200 import ops
from sessd_b200.runners import conv_out_shape

from . import utils  # noqa: F401


def _triple(v):
    return tuple(int(x) for x in v) if isinstance(v, (list, tuple)) else (int(v),) * 3


class SparseConvTensor(object):
    def __init__(self, features, indices, spatial_shape, batch_size, grid=None):
        """features [N, C] float32; indices [N, 4] int32 (batch, z, y, x); spatial_shape [D, H, W]."""
        self.features = features
        self.indices = indices
        self.spatial_shape = [int(v) for v in spatial_shape]
        self.batch_size = int(batch_size)
        self.indice_dict = {}
        self.grid = grid
        self._index_kind = None     # 0 hash over given coordinates, 1 rank bitmap (rows sorted by linear index)
        self._index = None

    @property
    def spatial_size(self):
        return int(np.prod(self.spatial_shape))

    def find_indice_pair(self, key):
        return self.indice_dict.get(key) if key is not None else None

    def _n(self):
        return torch.tensor([self.indices.shape[0]], dtype=torch.int32, device=self.indices.device)

    def _grid(self):
        return ops.make_grid(self.batch_size, self.spatial_shape)

    def _ensure_index(self):
        if self._index is None:
            idx = self.indices.int().contiguous()
            self.indices = idx
            self._index = ops.hash_build(idx, self._n(), max(idx.shape[0], 1), self._grid())
            self._index_kind = 0
        return self._index_kind, self._index

    def dense(self, channels_first=True):
        n, c = self.features.shape
        g = self._grid()
        d, h, w = self.spatial_shape
        out = torch.empty((self.batch_size, h, w, c * d), dtype=torch.float32, device=self.features.device)
        ops.sparse_to_dense(self.features.contiguous(), self.indices.int().contiguous(), self._n(), max(n, 1), g, out)
        vol = out.view(self.batch_size, h, w, c, d)
        return vol.permute(0, 3, 4, 1, 2) if channels_first else vol.permute(0, 4, 1, 2, 3)


class SparseModule(nn.Module):
    pass


class SparseSequential(SparseModule):
    """Applies SparseModules to the tensor and plain nn.Modules (BatchNorm1d, ReLU ...) to ``.features``."""

    def __init__(self, *args, **kwargs):
        super().__init__()
        for i, m in enumerate(args):
            self.add_module(str(i), m)
        for name, m in kwargs.items():
            self.add_module(name, m)

    def __getitem__(self, idx):
        return list(self._modules.values())[idx]

    def __len__(self):
        return len(self._modules)

    def forward(self, x):
        for m in self._modules.values():
            if isinstance(m, SparseModule):
                x = m(x)
            elif isinstance(x, SparseConvTensor):
                if x.indices.shape[0] != 0:
                    x.features = m(x.features)
            else:
                x = m(x)
        return x


class _SparseConvBase(SparseModule):
    def __init__(self, in_channels, out_channels, kernel_size, stride, padding, bias, subm, indice_key):
        super().__init__()
        self.in_channels, self.out_channels = in_channels, out_channels
        self.kernel_size, self.stride, self.padding = _triple(kernel_size), _triple(stride), _triple(padding)
        self.subm, self.indice_key = subm, indice_key
        self.weight = nn.Parameter(torch.empty(*self.kernel_size, in_channels, out_channels))
        self.bias = nn.Parameter(torch.empty(out_channels)) if bias else None
        self.reset_parameters()

    def reset_parameters(self):
        nn.init.kaiming_uniform_(self.weight, a=math.sqrt(5))
        if self.bias is not None:
            fan_in = self.in_channels * int(np.prod(self.kernel_size))
            bound = 1 / math.sqrt(fan_in)
            nn.init.uniform_(self.bias, -bound, bound)

    def packed_weight(self):
        return self.weight.detach().reshape(-1, self.in_channels, self.out_channels).contiguous().float()

    def rulebook(self, x):
        """The output index set of this conv on ``x`` and its neighbour table (a SubM table is shared through ``x.indice_dict`` by the
        layers of an ``indice_key``): (output SparseConvTensor without features, nbr [cap, kvol] int32, device row count [1], cap).
        Used by ``forward`` and by the training path (sessd_b200.sparse_grad)."""
        kind, index = x._ensure_index()
        n_in = x.indices.shape[0]
        kvol = int(np.prod(self.kernel_size))
        if self.subm:
            nbr = x.find_indice_pair(self.indice_key)
            if nbr is None:
                nbr = ops.subm_rulebook(x.indices, x._n(), max(n_in, 1), x._grid(), self.kernel_size, kind, index)
                if self.indice_key is not None:
                    x.indice_dict[self.indice_key] = nbr
            out = SparseConvTensor(None, x.indices, x.spatial_shape, x.batch_size)
            out._index_kind, out._index = kind, index
            n_out_t, cap = x._n(), max(n_in, 1)
        else:
            oshape = conv_out_shape(x.spatial_shape, self.kernel_size, self.stride, self.padding)
            ogrid = ops.make_grid(x.batch_size, oshape)
            cells = x.batch_size * int(np.prod(oshape))
            cap = max(1, min(cells, n_in * kvol))
            bitmap, scratch = ops.bitmap_alloc(ogrid, x.indices.device)
            ocoors = torch.empty((cap, 4), dtype=torch.int32, device=x.indices.device)
            n_out_t = torch.zeros((1,), dtype=torch.int32, device=x.indices.device)
            nbr = torch.empty((cap, kvol), dtype=torch.int32, device=x.indices.device)
            status = torch.zeros((1,), dtype=torch.int32, device=x.indices.device)
            ops.strided_rulebook(x.indices, x._n(), max(n_in, 1), x._grid(), kind, index, self.kernel_size, self.stride,
                                 self.padding, ogrid, bitmap, scratch, ocoors, n_out_t, cap, nbr, status)
            n_out = int(n_out_t.item())            # data-dependent size crosses to the host here (module-level API only)
            out = SparseConvTensor(None, ocoors[:n_out], list(oshape), x.batch_size)
            out._index_kind, out._index = 1, bitmap
            cap = max(n_out, 1)
            nbr = nbr[:cap]
        out.indice_dict = x.indice_dict
        return out, nbr, n_out_t, cap

    @torch.no_grad()
    def forward(self, x):
        assert isinstance(x, SparseConvTensor)
        out, nbr, n_out_t, cap = self.rulebook(x)
        feat = ops.spconv_forward(x.features.detach().float().contiguous(), nbr, n_out_t, cap, self.packed_weight(), None,
                                  self.bias.detach().float() if self.bias is not None else None, False)
        out.features = feat[: out.indices.shape[0]]
        return out


class SubMConv3d(_SparseConvBase):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 indice_key=None, use_hash=False):
        k = _triple(kernel_size)
        super().__init__(in_channels, out_channels, k, 1, tuple(v // 2 for v in k), bias, True, indice_key)


class SparseConv3d(_SparseConvBase):
    def __init__(self, in_channels, out_channels, kernel_size, stride=1, padding=0, dilation=1, groups=1, bias=True,
                 indice_key=None, use_hash=False):
        super().__init__(in_channels, out_channels, kernel_size, stride, padding, bias, False, indice_key)
