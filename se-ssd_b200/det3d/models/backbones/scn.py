"""SpMiddleFHD sparse middle encoder (reference: det3d/models/backbones/scn.py:92-189).

Same constructor, parameters and state-dict keys (``middle_conv.{0,3,...}.weight`` in spconv layout [kz,ky,kx,Cin,Cout],
``middle_conv.{1,4,...}`` BatchNorm1d) so reference checkpoints load.  ``forward`` runs the fused CUDA pipeline
(sessd_b200.runners.SpMiddleRunner): 8 deterministic rulebooks + 14 gather-GEMM launches with BN+ReLU in the epilogue + dense
scatter, and returns the [B, 128, 200, 176] BEV tensor in channels-last memory (logically NCHW, like the reference's
``ret.view(N, C*D, H, W)``)."""
import numpy as np
import spconv
import torch
from spconv import SparseConv3d, SubMConv3d
from torch import nn

from sessd_b200.runners import SPMIDDLE_LAYERS, SpMiddleRunner

from ..registry import BACKBONES
from ..utils import build_norm_layer


@BACKBONES.register_module
class SpMiddleFHD(nn.Module):
    def __init__(self, num_input_features=128, norm_cfg=None, name="SpMiddleFHD", **kwargs):
        super().__init__()
        self.name = name
        if norm_cfg is None:
            norm_cfg = dict(type="BN1d", eps=1e-3, momentum=0.01)
        mods, cin = [], num_input_features
        for kind, cout, ks, st, pd, key in SPMIDDLE_LAYERS:
            if kind == "subm":
                mods.append(SubMConv3d(cin, cout, ks[0], bias=False, indice_key=key))
            else:
                mods.append(SparseConv3d(cin, cout, ks, st, padding=list(pd), bias=False))
            mods.append(build_norm_layer(norm_cfg, cout)[1])
            mods.append(nn.ReLU())
            cin = cout
        self.middle_conv = spconv.SparseSequential(*mods)
        self._runner = None
        self._runner_key = None
        self._weights_key = None

    def init_weights(self, pretrained=None):
        if isinstance(pretrained, str):       # reference convention (e.g. rpn.py / resnet): a checkpoint path
            from det3d.torchie.trainer.checkpoint import load_checkpoint
            load_checkpoint(self, pretrained, strict=False)
        elif pretrained is not None:
            raise TypeError("pretrained must be a str or None")

    def _layers(self):
        out = []
        for i in range(len(SPMIDDLE_LAYERS)):
            conv, bn = self.middle_conv[3 * i], self.middle_conv[3 * i + 1]
            out.append(dict(weight=conv.weight.detach(), gamma=bn.weight.detach(), beta=bn.bias.detach(),
                            mean=bn.running_mean, var=bn.running_var, eps=float(bn.eps)))
        return out

    def forward(self, voxel_features, coors, batch_size, input_shape):
        if self.training:
            raise NotImplementedError("SpMiddleFHD: only the inference path is built (call .eval()); training is a 'next' row")
        grid_xyz = [int(v) for v in np.array(input_shape).reshape(-1)[:3]]
        coors = coors.int().contiguous()
        n = int(coors.shape[0])
        cap = max(4096, -(-n // 4096) * 4096)
        key = (int(batch_size), cap, tuple(grid_xyz), str(coors.device))
        if self._runner is None or self._runner_key != key:
            self._runner = SpMiddleRunner(int(batch_size), cap, grid_xyz, self.middle_conv[0].in_channels, coors.device)
            self._runner_key, self._weights_key = key, None
        wkey = tuple((p.data_ptr(), p._version) for p in self.parameters()) + tuple((b.data_ptr(), b._version) for b in self.buffers())
        if wkey != self._weights_key:
            self._runner.load_weights(self._layers())
            self._weights_key = wkey
        feats = voxel_features.detach().float().contiguous()
        n_dev = torch.tensor([n], dtype=torch.int32, device=coors.device)
        dense = self._runner.forward(feats, coors, n_dev)                 # NHWC [B, 200, 176, 128]
        if int(self._runner.status.item()) != 0:
            raise RuntimeError("SpMiddleFHD: active-site capacity exceeded")
        # logical NCHW, channels-last memory; a fresh tensor per call (the runner's dense buffer is overwritten by the next forward)
        return dense.permute(0, 3, 1, 2).clone()
