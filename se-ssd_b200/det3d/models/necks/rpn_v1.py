"""SSFA -- spatial-semantic feature aggregation neck (reference: det3d/models/necks/rpn_v1.py:119-235).

Identical module tree (hence identical state-dict keys: ``bottom_up_block_0.1.weight`` ...), identical constructor signature
(``logger`` is dereferenced exactly like the reference does, :212).  ``forward`` (eval mode) executes the whole neck with the
sessd_b200 kernels: 12 conv / deconv layers as NHWC implicit GEMMs on the wgmma tensor cores with BatchNorm + ReLU (+ the
deconv_0 + trans_0 residual) fused into the epilogue, and one fused kernel for the two 1-channel attention convs, their BN, the
2-way softmax and the weighted sum (:229-233)."""
from torch import nn

from sessd_b200.runners import SSFAPlanesRunner

from ..registry import NECKS
from ..utils import build_norm_layer


def _cbr(cin, cout, k, norm_cfg, stride=1, pad=None, relu=True, zero_pad=False):
    pad = k // 2 if pad is None else pad
    mods = []
    if zero_pad:                       # bottom_up_block_0 starts with ZeroPad2d(1) + an unpadded conv (:135-137)
        mods.append(nn.ZeroPad2d(1))
        pad = 0
    mods += [nn.Conv2d(cin, cout, k, stride=stride, padding=pad, bias=False), build_norm_layer(norm_cfg, cout)[1]]
    if relu:
        mods.append(nn.ReLU())
    return mods


@NECKS.register_module
class SSFA(nn.Module):
    def __init__(self, layer_nums, ds_layer_strides, ds_num_filters, us_layer_strides, us_num_filters, num_input_features,
                 norm_cfg=None, name="rpn", logger=None, **kwargs):
        super().__init__()
        self._layer_strides, self._num_filters, self._layer_nums = ds_layer_strides, ds_num_filters, layer_nums
        self._upsample_strides, self._num_upsample_filters = us_layer_strides, us_num_filters
        self._num_input_features = num_input_features
        if norm_cfg is None:
            norm_cfg = dict(type="BN", eps=1e-3, momentum=0.01)
        self._norm_cfg = norm_cfg
        S = nn.Sequential
        self.bottom_up_block_0 = S(*(_cbr(128, 128, 3, norm_cfg, zero_pad=True) + _cbr(128, 128, 3, norm_cfg) + _cbr(128, 128, 3, norm_cfg)))
        self.bottom_up_block_1 = S(*(_cbr(128, 256, 3, norm_cfg, stride=2) + _cbr(256, 256, 3, norm_cfg) + _cbr(256, 256, 3, norm_cfg)))
        self.trans_0 = S(*_cbr(128, 128, 1, norm_cfg))
        self.trans_1 = S(*_cbr(256, 256, 1, norm_cfg))
        dec = lambda: S(nn.ConvTranspose2d(256, 128, 3, stride=2, padding=1, output_padding=1, bias=False),  # noqa: E731
                        build_norm_layer(norm_cfg, 128)[1], nn.ReLU())
        self.deconv_block_0 = dec()
        self.deconv_block_1 = dec()
        self.conv_0 = S(*_cbr(128, 128, 3, norm_cfg))
        self.w_0 = S(*_cbr(128, 1, 1, norm_cfg, relu=False))
        self.conv_1 = S(*_cbr(128, 128, 3, norm_cfg))
        self.w_1 = S(*_cbr(128, 1, 1, norm_cfg, relu=False))
        logger.info("Finish RPN Initialization")
        self._runner = None
        self._runner_key = None
        self._weights_key = None

    def init_weights(self):
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.xavier_uniform_(m.weight)

    def forward(self, x):
        if self.training:
            raise NotImplementedError("SSFA: only the inference path is built (call .eval()); training is a 'next' row")
        b, c, h, w = x.shape
        key = (b, h, w, str(x.device))
        if self._runner is None or self._runner_key != key:
            self._runner = SSFAPlanesRunner(b, (h, w), x.device)
            self._runner_key, self._weights_key = key, None
        wkey = tuple((p.data_ptr(), p._version) for p in self.parameters()) + tuple((t.data_ptr(), t._version) for t in self.buffers())
        if wkey != self._weights_key:
            eps = {float(m.eps) for m in self.modules() if isinstance(m, nn.modules.batchnorm._BatchNorm)}
            assert len(eps) == 1, "SSFA: all BatchNorm layers must share one eps"
            self._runner.load_state({k: v.detach() for k, v in self.state_dict().items()}, bn_eps=eps.pop())
            self._weights_key = wkey
        x_nhwc = x.detach().float().permute(0, 2, 3, 1).contiguous()     # no copy when x is channels-last already
        out, _ = self._runner.forward(x_nhwc)
        return out.permute(0, 3, 1, 2).clone()        # fresh tensor per call: the runner buffer is overwritten by the next forward
