"""Stage runners: pre-allocated, capacity-sized device state + launch sequences for the three GPU stages
(sparse middle encoder, SSFA neck + head, post-processing).  No host synchronisation inside ``forward`` -- every
data-dependent count stays on the device -- so a whole frame can be captured in one CUDA graph (engine.py).

Layer tables mirror det3d/models/backbones/scn.py:106-149 (SpMiddleFHD) and det3d/models/necks/rpn_v1.py:135-235 (SSFA).
"""
import math

import torch
from sessd_data.layers import SPMIDDLE_LAYERS  # (kind, cout, ksize, stride, padding, indice_key)   scn.py:106-149

from . import ops

BN_EPS = 1e-3   # norm_cfg eps of both BN1d (scn.py:103) and BN2d (rpn_v1.py:131)

def conv_out_shape(shape, ksize, stride, padding):
    return tuple((int(i) + 2 * p - k) // s + 1 for i, k, s, p in zip(shape, ksize, stride, padding))


def fold_bn(gamma, beta, mean, var, eps=BN_EPS):
    scale = gamma.float() / torch.sqrt(var.float() + eps)
    shift = beta.float() - mean.float() * scale
    return scale.contiguous(), shift.contiguous()


class SpMiddleRunner:
    """SpMiddleFHD forward (scn.py:176-189): 4 SubM rulebooks + 4 strided rulebooks + 14 fused conv launches + dense()."""

    # active-site growth bounds per level relative to the level-0 capacity (uniform 20k cloud: 3.4 / 5.2 / 4.3 / 2.6)
    GROWTH = (1.0, 4.0, 6.0, 5.0, 3.0)
    SPLIT = "fp16"
    SPARSE_TC = "cg"          # tensor-core kernel of the Cin >= 32 layers: pair-proportional cp.async gather, planes written by the
                              # producing layer's epilogue (csrc/spconv_cg.cu)
    ROWS_SHAPES = ((4, 16), (16, 16), (16, 32), (32, 32))     # (Cin, Cout) whose whole weight tensor fits in shared memory
    ROWS_MAX_CIN = 16         # layers with Cin <= this run on the pair-proportional SIMT kernel (0: tensor-core kernels wherever possible)
    DENSE_GATHER = True       # dense() as one gather pass through the last level's bitmap index (False: memset + scatter)

    def __init__(self, batch, max_voxels_total, input_shape_xyz=(1408, 1600, 40), num_input_features=4, device="cuda",
                 growth=None, use_tc=True, split=None, rows_max_cin=None, sparse_tc=None, keep_f32=False):
        """use_tc: run the Cin >= 32 layers on the tensor cores (fp16 wgmma with a two-term fp16 split, csrc/spconv_cg.cu) and the
        narrow layers on the pair-proportional SIMT kernel; False = fp32 SIMT baseline for all layers.  split / sparse_tc: "fp16" / "cg",
        the only tensor-core variant."""
        self.batch, self.device = batch, torch.device(device)
        self.use_tc = bool(use_tc)
        self.split = split or self.SPLIT
        assert self.split == "fp16", "the sparse tensor-core layers use the two-term fp16 split"
        self.use_h2 = self.use_tc
        self.sparse_tc = sparse_tc or self.SPARSE_TC
        assert self.sparse_tc == "cg"
        self.keep_f32 = bool(keep_f32)      # cg layers also write their fp32 rows (tests compare per-layer features)
        # per-layer kernel: "rows" = pair-proportional fp32 SIMT (narrow layers), "cg" = pair-proportional fp16-split wgmma,
        # "simt" = the dense output-stationary fp32 baseline
        self.rows_max_cin = (self.ROWS_MAX_CIN if rows_max_cin is None else int(rows_max_cin)) if self.use_tc else 0
        self.cin0 = num_input_features
        shape = (int(input_shape_xyz[2]) + 1, int(input_shape_xyz[1]), int(input_shape_xyz[0]))   # scn.py:179
        growth = growth or self.GROWTH
        self.levels = []       # dicts: shape, cap, grid, coors, n, index_kind, index, scratch
        self.plan = []         # per layer: (kind, level_in, level_out, nbr tensor, cin, cout)
        lvl = 0
        self._add_level(shape, int(max_voxels_total), hash_index=True)
        cin = num_input_features
        subm_nbr = {}
        for li, (kind, cout, ks, st, pd, key) in enumerate(SPMIDDLE_LAYERS):
            kvol = ks[0] * ks[1] * ks[2]
            if kind == "subm":
                if key not in subm_nbr:
                    subm_nbr[key] = torch.empty((self.levels[lvl]["cap"], kvol), dtype=torch.int32, device=self.device)
                self.plan.append(dict(kind=kind, lin=lvl, lout=lvl, nbr=subm_nbr[key], cin=cin, cout=cout, ks=ks, st=st, pd=pd,
                                      key=key, first=len([p for p in self.plan if p.get("key") == key]) == 0))
            else:
                oshape = conv_out_shape(self.levels[lvl]["shape"], ks, st, pd)
                cells = batch * oshape[0] * oshape[1] * oshape[2]
                cap = min(cells, int(math.ceil(max_voxels_total * growth[lvl + 1])))
                self._add_level(oshape, cap, hash_index=False)
                nbr = torch.empty((cap, kvol), dtype=torch.int32, device=self.device)
                self.plan.append(dict(kind=kind, lin=lvl, lout=lvl + 1, nbr=nbr, cin=cin, cout=cout, ks=ks, st=st, pd=pd, key=None))
                lvl += 1
            cin = cout
        self.feats = [torch.zeros((self.levels[p["lout"]]["cap"], p["cout"]), dtype=torch.float32, device=self.device)
                      for p in self.plan]
        last = self.levels[-1]
        self.out_channels = self.plan[-1]["cout"] * last["shape"][0]
        self.dense = torch.zeros((batch, last["shape"][1], last["shape"][2], self.out_channels), dtype=torch.float32,
                                 device=self.device)
        self.status = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self.weights = None
        # fp16-split path: (hi, lo) planes of every layer output that feeds a tensor-core layer + one abs-max scalar per tensor
        self.planes = [None] * len(self.plan)
        self.amax = torch.zeros((len(self.plan) + 1,), dtype=torch.float32, device=self.device)
        for p in self.plan:
            if self.use_tc and p["cin"] <= self.rows_max_cin and (p["cin"], p["cout"]) in self.ROWS_SHAPES:
                p["impl"] = "rows"
            elif self.use_h2 and p["cin"] >= 32:
                p["impl"] = "cg"
            else:
                p["impl"] = "simt"
        for li, p in enumerate(self.plan):
            # a cg layer reads the planes its producer's epilogue writes: the pair-proportional kernels write them, the baseline does not
            assert p["impl"] != "cg" or self.plan[li - 1]["impl"] in ("rows", "cg"), "rows_max_cin too small for the tensor-core chain"
        for li, p in enumerate(self.plan[:-1]):
            if self.plan[li + 1]["impl"] == "cg":
                cp = 64 if p["cout"] > 32 else 32
                self.planes[li] = ops.alloc_planes(self.levels[p["lout"]]["cap"], cp, self.device)
                assert self.planes[li].shape[0] <= (1 << 25)
        # per-tile pair lists of every rulebook a cg layer reads (one per nbr table; a SubM rulebook is shared by its layers)
        for p in self.plan:
            p["tiles"] = None
        by_nbr = {}
        for p in self.plan:
            if p["impl"] == "cg":
                key = p["nbr"].data_ptr()
                if key not in by_nbr:
                    by_nbr[key] = ops.alloc_tile_lists(p["nbr"].shape[0], p["nbr"].shape[1], self.device)
                p["tiles"] = by_nbr[key]
        # {abs-max, plane scale} of every layer output (cg chain: written by the producing layer's epilogue)
        self.info = torch.zeros((len(self.plan), 2), dtype=torch.float32, device=self.device)

    def layer_output(self, li):
        """fp32 rows [cap, Cout] of layer li's output after forward(): the fp32 buffer when the layer wrote it, else rebuilt from the fp16
        (hi, lo) planes the next layer reads (exact: x = (hi + lo) / S) -- tests / debugging."""
        p = self.plan[li]
        nxt = self.plan[li + 1]["impl"] if li + 1 < len(self.plan) else None
        planes_only = (not self.keep_f32) and nxt == "cg" and p["impl"] in ("cg", "rows")
        if not planes_only:
            return self.feats[li]
        return ops.sparse_planes_to_float(self.planes[li][:-1], self.info[li], p["cout"])

    def _add_level(self, shape, cap, hash_index):
        grid = ops.make_grid(self.batch, shape)
        lv = dict(shape=shape, cap=cap, grid=grid, n=torch.zeros((1,), dtype=torch.int32, device=self.device))
        if hash_index:
            lv["index_kind"] = 0
            lv["index"] = torch.empty((ops.hash_capacity(cap),), dtype=torch.int64, device=self.device)
            lv["coors"] = None      # supplied by the caller
        else:
            lv["index_kind"] = 1
            lv["index"], lv["scratch"] = ops.bitmap_alloc(grid, self.device)
            lv["coors"] = torch.zeros((cap, 4), dtype=torch.int32, device=self.device)
        self.levels.append(lv)

    def load_weights(self, layers):
        """layers: 14 x dict(weight [kz,ky,kx,Cin,Cout] (spconv layout), gamma, beta, mean, var)."""
        assert len(layers) == len(self.plan)
        self.weights = []
        for p, l in zip(self.plan, layers):
            w = torch.as_tensor(l["weight"], dtype=torch.float32, device=self.device)
            assert tuple(w.shape) == (*p["ks"], p["cin"], p["cout"]), (w.shape, p)
            sc, sh = fold_bn(*[torch.as_tensor(l[k], device=self.device) for k in ("gamma", "beta", "mean", "var")], eps=float(l.get("eps", BN_EPS)))
            wp = w.reshape(-1, p["cin"], p["cout"]).contiguous()
            tc = None
            if p["impl"] == "cg":
                tiles, inv = ops.pack_weight_sp_h2(wp, 64 if p["cin"] > 32 else 32, layout="cg")
                tc = (p["impl"], tiles, (sc * inv).contiguous())
            p["gain"], p["shift_max"] = ops.conv_gain(wp, sc), float(sh.abs().max())
            self.weights.append((wp, sc, sh, tc))

    def forward(self, feat0, coors0, n0, mark=None, dense_planes=None):
        """feat0 [cap0, Cin] f32, coors0 [cap0,4] i32 (b,z,y,x), n0 [1] i32 (device).  Returns dense NHWC.
        mark: optional callable(label) invoked after every launch group (profiling scripts record a CUDA event there).
        dense_planes: (planes [2,B,H,W,C*D] fp16, info [2] f32): dense() writes the fp16 (hi, lo) planes the BEV neck reads instead
        of the fp32 map (returns the planes)."""
        mark = mark or (lambda label: None)
        assert self.weights is not None, "load_weights first"
        L0 = self.levels[0]
        assert coors0.shape[0] <= L0["cap"] or True
        cap0 = min(coors0.shape[0], L0["cap"])
        L0["coors"], L0["n_ext"] = coors0, n0
        ops.hash_build(coors0, n0, cap0, L0["grid"], L0["index"])
        mark("hash_build")
        if self.use_h2:
            self.amax.zero_()
            self.info.zero_()
        x = feat0
        for li, p in enumerate(self.plan):
            lin, lout = self.levels[p["lin"]], self.levels[p["lout"]]
            n_in = lin["n_ext"] if p["lin"] == 0 else lin["n"]
            cap_in = cap0 if p["lin"] == 0 else lin["cap"]
            if p["kind"] == "subm":
                if p["first"]:
                    ops.subm_rulebook(lin["coors"], n_in, cap_in, lin["grid"], p["ks"], lin["index_kind"], lin["index"], p["nbr"])
                    tl = next((q["tiles"] for q in self.plan if q.get("key") == p["key"] and q["tiles"] is not None), None)
                    if tl is not None:
                        ops.rulebook_tile_lists(p["nbr"], n_in, cap_in, tl)
                    mark("rulebook:%s" % p["key"])
                n_out, cap_out = n_in, cap_in
            else:
                ops.strided_rulebook(lin["coors"], n_in, cap_in, lin["grid"], lin["index_kind"], lin["index"], p["ks"], p["st"],
                                     p["pd"], lout["grid"], lout["index"], lout["scratch"], lout["coors"], lout["n"], lout["cap"],
                                     p["nbr"], self.status)
                n_out, cap_out = lout["n"], lout["cap"]
                if p["tiles"] is not None:
                    ops.rulebook_tile_lists(p["nbr"], n_out, cap_out, p["tiles"])
                mark("rulebook:sp%d" % p["lout"])
            w, sc, sh, tc = self.weights[li]
            nxt = self.plan[li + 1]["impl"] if li + 1 < len(self.plan) else None
            if p["impl"] == "rows" and nxt == "cg":
                # last SIMT layer before the tensor-core chain: writes the planes the next layer reads (scale from the bound on its output)
                ops.spconv_forward_rows_planes(x, p["nbr"], n_out, cap_out, w, sc, sh, True, self.info[li - 1, 0:1], p["gain"], p["shift_max"],
                                               self.feats[li] if self.keep_f32 else None, self.planes[li], self.info[li])
                x = self.feats[li]
            elif p["impl"] == "rows":
                need_amax = self.planes[li] is not None or (nxt == "rows" and li + 2 < len(self.plan) and self.plan[li + 2]["impl"] == "cg")
                x = ops.spconv_forward_rows(x, p["nbr"], n_out, cap_out, w, sc, sh, True, self.feats[li],
                                            self.info[li, 0:1] if need_amax else None)
            elif isinstance(tc, tuple) and tc[0] == "cg":
                last = nxt != "cg"
                ops.spconv_forward_cg(self.planes[li - 1], self.info[li - 1], p["tiles"], n_out, cap_out, tc[1], tc[2], sh, True, p["gain"],
                                      p["shift_max"], self.feats[li] if (last or self.keep_f32) else None,
                                      None if last else self.planes[li], self.info[li])
                x = self.feats[li]
            else:
                x = ops.spconv_forward(x, p["nbr"], n_out, cap_out, w, sc, sh, True, self.feats[li])
            mark("conv:%d" % li)
        last = self.levels[-1]
        if dense_planes is not None:
            assert last["index_kind"] == 1 and self.use_h2
            assert self.plan[-1]["impl"] == "cg"
            out = ops.sparse_to_dense_planes(x, last["index"], last["grid"], self.info[len(self.plan) - 1, 0:1], dense_planes[1], dense_planes[0])
            mark("dense")
            return out
        if last["index_kind"] == 1 and self.DENSE_GATHER:
            out = ops.sparse_to_dense_indexed(x, last["index"], last["grid"], self.dense)
        else:
            out = ops.sparse_to_dense(x, last["coors"], last["n"], last["cap"], last["grid"], self.dense)
        mark("dense")
        return out


# ---------------------------------------------------------------------------------------------------------------
def _pack_conv(w):
    """nn.Conv2d weight [Cout,Cin,kh,kw] -> ([kh*kw, Cin, Cout], taps (dy,dx) relative to the unpadded origin)."""
    cout, cin, kh, kw = w.shape
    packed = w.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout).contiguous()
    return packed, [(ky, kx) for ky in range(kh) for kx in range(kw)]


def _deconv_classes(w):
    """nn.ConvTranspose2d(k3,s2,p1,op1) weight [Cin,Cout,3,3] -> 4 parity classes: (py, px, packed [T,Cin,Cout], taps)."""
    out = []
    for py in (0, 1):
        for px in (0, 1):
            kys = [(1, 0)] if py == 0 else [(0, 1), (2, 0)]     # (ky, dy): iy = y + dy
            kxs = [(1, 0)] if px == 0 else [(0, 1), (2, 0)]
            taps, mats = [], []
            for ky, dy in kys:
                for kx, dx in kxs:
                    taps.append((dy, dx))
                    mats.append(w[:, :, ky, kx])
            out.append((py, px, torch.stack(mats, 0).contiguous(), taps))
    return out


def pack_head(head_sd, prefix, device, stride=24):
    """Four 1x1 head convs (mg_head_sessd.py:202-215) -> one [1,128,stride] GEMM weight + bias, channel layout
    [box 14 | cls 2 | dir 4 | iou 2 | zero pad]."""
    hw = torch.zeros((1, 128, stride), dtype=torch.float32, device=device)
    hb = torch.zeros((stride,), dtype=torch.float32, device=device)
    o = 0
    for nm, c in (("conv_box", 14), ("conv_cls", 2), ("conv_dir", 4), ("conv_iou", 2)):
        hw[0, :, o:o + c] = head_sd[prefix + nm + ".weight"].to(device, torch.float32).reshape(c, 128).t()
        hb[o:o + c] = head_sd[prefix + nm + ".bias"].to(device, torch.float32)
        o += c
    return hw.contiguous(), hb.contiguous()


class HeadRunner:
    """The fused head GEMM alone (MultiGroupHead.forward)."""

    def __init__(self, batch, hw, device="cuda", use_tc=True, stride=24):
        """use_tc: the fp16-split tensor-core conv (csrc/bevconv_p2.cu; the fp32 input is split into planes first); False = fp32 SIMT."""
        self.batch, self.h, self.w, self.stride, self.use_tc = batch, int(hw[0]), int(hw[1]), stride, use_tc
        self.out = torch.zeros((batch, self.h, self.w, stride), dtype=torch.float32, device=device)
        self.device = torch.device(device)
        self.w_simt = self.w_tc = self.bias = None
        if use_tc:
            self.x_planes = ops.alloc_bev_planes(batch, self.h, self.w, 128, self.device)
            self.info = torch.zeros((2, 2), dtype=torch.float32, device=self.device)     # {abs-max, scale} of the input / the output

    def load_state(self, head_sd, prefix=""):
        self.w_simt, self.bias = pack_head(head_sd, prefix, self.device, self.stride)
        if self.use_tc:
            planes, inv = ops.pack_weight_h2(self.w_simt, 32)
            gain = ops.conv_gain(self.w_simt, torch.ones(self.stride, device=self.device))
            self.w_tc = (planes, inv[: self.stride].contiguous(), gain, float(self.bias.abs().max()))

    def forward(self, x):
        H = (self.h, self.w)
        d = ops.conv_desc(self.batch, H, 128, H, self.stride, H, [(0, 0)], relu=False)
        if self.w_tc is not None:
            planes, scale, gain, shift_max = self.w_tc
            self.info.zero_()
            ops.absmax(x, self.info[0, 0:1])
            ops.bev_split_planes(x, self.info[0], self.x_planes)
            ops.bev_conv_p2(self.x_planes, self.info[0], planes, scale, self.bias, None, None, gain, shift_max, self.out, None, self.info[1], d)
            return self.out
        return ops.bev_conv(x, self.w_simt, None, self.bias, None, self.out, d)


class SSFARunner:
    """SSFA neck (rpn_v1.py:220-235) + the fused 128->22(+2 pad) head GEMM (mg_head_sessd.py:202-230)."""

    HEAD_STRIDE = 24

    TC_STRIDE2 = True     # run the stride-2 conv through the strided-TMA tensor-core path as well

    def __init__(self, batch, hw=(200, 176), device="cuda", use_tc=True, split="fp16"):
        """use_tc: tensor-core convs (default); False = the fp32 SIMT baseline kernels.
        split: "fp16" = two-term fp16 split (kind::f16, bevconv_h2.cu; the stride-2 conv stays on the tf32 kernel),
               "tf32" = 3xTF32 everywhere (bevconv_tc.cu)."""
        self.batch, self.h, self.w, self.device = batch, int(hw[0]), int(hw[1]), torch.device(device)
        self.use_tc = bool(use_tc)
        assert split in ("fp16", "tf32")
        self.use_h2 = self.use_tc and split == "fp16"
        self.amax = torch.zeros(16, dtype=torch.float32, device=self.device)     # per-tensor abs-max scalars (fp16 split scaling)
        h, w, h2, w2 = self.h, self.w, self.h // 2, self.w // 2
        z = lambda hh, ww, c: torch.zeros((batch, hh, ww, c), dtype=torch.float32, device=self.device)  # noqa: E731
        self.buf = dict(b0a=z(h, w, 128), b0b=z(h, w, 128), x0=z(h, w, 128), b1a=z(h2, w2, 256), b1b=z(h2, w2, 256),
                        x1=z(h2, w2, 256), t0=z(h, w, 128), t1=z(h2, w2, 256), m0=z(h, w, 128), m1=z(h, w, 128),
                        o0=z(h, w, 128), o1=z(h, w, 128), out=z(h, w, 128), head=z(h, w, self.HEAD_STRIDE))
        self.params = None

    def load_state(self, ssfa_sd, head_sd=None, head_prefix="tasks.0.", bn_eps=BN_EPS):
        """bn_eps: eps of the neck's BatchNorm2d layers (rpn_v1.py:131-132 uses 1e-3; pass the module's own value otherwise)."""
        dev = self.device
        g = lambda k: ssfa_sd[k].to(dev, torch.float32)   # noqa: E731
        P = {}

        def bn(conv_name):
            blk, idx = conv_name.rsplit(".", 1)
            b = "%s.%d" % (blk, int(idx) + 1)
            return fold_bn(g(b + ".weight"), g(b + ".bias"), g(b + ".running_mean"), g(b + ".running_var"), eps=bn_eps)

        for name, pad in (("bottom_up_block_0.1", 1), ("bottom_up_block_0.4", 1), ("bottom_up_block_0.7", 1),
                          ("bottom_up_block_1.0", 1), ("bottom_up_block_1.3", 1), ("bottom_up_block_1.6", 1),
                          ("trans_0.0", 0), ("trans_1.0", 0), ("conv_0.0", 1), ("conv_1.0", 1)):
            wp, taps = _pack_conv(g(name + ".weight"))
            P[name] = (wp, [(dy - pad, dx - pad) for dy, dx in taps]) + bn(name)
            if self.use_h2 and name != "bottom_up_block_1.0":
                planes, inv = ops.pack_weight_h2(wp, -(-wp.shape[2] // 128) * 128)
                sc_, sh_ = bn(name)
                P[name + ":h2"] = (planes, (sc_ * inv[:sc_.numel()]).contiguous(), sh_)
            elif self.use_tc and (self.TC_STRIDE2 or name != "bottom_up_block_1.0"):
                P[name + ":tc"] = ops.pack_weight_tc(wp, -(-wp.shape[2] // 128) * 128)
        for name in ("deconv_block_0.0", "deconv_block_1.0"):
            classes = _deconv_classes(g(name + ".weight"))
            P[name] = (classes,) + bn(name)
            if self.use_tc:     # one launch for the four parity classes: plain 9-tap packing of W[cin][cout][ky][kx]
                wd = g(name + ".weight")
                w9 = wd.permute(2, 3, 0, 1).reshape(9, wd.shape[0], wd.shape[1]).contiguous()
                if self.use_h2:
                    planes, inv = ops.pack_weight_h2(w9, 128)
                    sc_, sh_ = bn(name)
                    P[name + ":h2"] = (planes, (sc_ * inv[:sc_.numel()]).contiguous(), sh_)
                else:
                    P[name + ":tc"] = ops.pack_weight_tc(w9, 128)
        for name in ("w_0.0", "w_1.0"):
            sc, sh = bn(name)
            P[name] = (g(name + ".weight").reshape(-1).contiguous(), float(sc[0]), float(sh[0]))
        if head_sd is not None:
            hw, hb = pack_head(head_sd, head_prefix, dev, self.HEAD_STRIDE)
            P["head"] = (hw, hb)
            if self.use_h2:
                planes, inv = ops.pack_weight_h2(hw, 32)
                P["head:h2"] = (planes, inv.contiguous())
            elif self.use_tc:
                P["head:tc"] = ops.pack_weight_tc(hw, 32)
        self.params = P

    def _am(self, i):
        return None if i is None else self.amax[i:i + 1]

    def _conv(self, name, x, out, in_hw, out_hw, cin, cout, stride=1, relu=True, ai=None, ao=None):
        """ai / ao: slots of self.amax holding the abs-max of the input / receiving the abs-max of the output (fp16-split scaling)."""
        wp, taps, sc, sh = self.params[name]
        d = ops.conv_desc(self.batch, in_hw, cin, out_hw, cout, out_hw, taps, in_stride=stride, relu=relu)
        if (name + ":h2") in self.params:
            planes, sc2, sh2 = self.params[name + ":h2"]
            return ops.bev_conv_h2(x, planes, sc2, sh2, None, out, d, self._am(ai), self._am(ao))
        if (name + ":tc") in self.params:
            ops.bev_conv_tc(x, self.params[name + ":tc"], sc, sh, None, out, d)
        else:
            ops.bev_conv(x, wp, sc, sh, None, out, d)
        if self.use_h2 and ao is not None:
            ops.absmax(out, self._am(ao))
        return out

    def _deconv(self, name, x, out, in_hw, out_hw, cin, cout, residual=None, ai=None, ao=None):
        classes, sc, sh = self.params[name]
        if (name + ":h2") in self.params:
            planes, sc2, sh2 = self.params[name + ":h2"]
            return ops.bev_deconv_h2(x, planes, sc2, sh2, residual, out, True, self._am(ai), self._am(ao))
        tc = self.params.get(name + ":tc")
        if tc is not None:
            return ops.bev_deconv_tc(x, tc, sc, sh, residual, out, relu=True)
        for py, px, wp, taps in classes:
            d = ops.conv_desc(self.batch, in_hw, cin, out_hw, cout, in_hw, taps, in_stride=1, out_stride=2, out_off=(py, px), relu=True)
            ops.bev_conv(x, wp, sc, sh, residual, out, d)
        return out

    def forward(self, x, mark=None):
        """x NHWC [B,200,176,128] -> (neck out NHWC [B,200,176,128], head NHWC [B,200,176,24]).
        mark: optional callable(label) invoked after every layer (profiling scripts record a CUDA event there)."""
        assert self.params is not None, "load_state first"
        mark = mark or (lambda label: None)
        b = self.buf
        H, H2 = (self.h, self.w), (self.h // 2, self.w // 2)

        def conv(name, *a, **kw):
            self._conv(name, *a, **kw)
            mark("neck:" + name)

        def deconv(name, *a, **kw):
            self._deconv(name, *a, **kw)
            mark("neck:" + name)

        if self.use_h2:      # abs-max scalars: 0 x, 1 b0a, 2 b0b, 3 x0, 4 b1a, 5 b1b, 6 x1, 7 t1, 8 m0, 9 m1, 10 out
            self.amax.zero_()
            ops.absmax(x, self._am(0))
        conv("bottom_up_block_0.1", x, b["b0a"], H, H, 128, 128, ai=0, ao=1)
        conv("bottom_up_block_0.4", b["b0a"], b["b0b"], H, H, 128, 128, ai=1, ao=2)
        conv("bottom_up_block_0.7", b["b0b"], b["x0"], H, H, 128, 128, ai=2, ao=3)
        conv("bottom_up_block_1.0", b["x0"], b["b1a"], H, H2, 128, 256, stride=2, ai=3, ao=4)
        conv("bottom_up_block_1.3", b["b1a"], b["b1b"], H2, H2, 256, 256, ai=4, ao=5)
        conv("bottom_up_block_1.6", b["b1b"], b["x1"], H2, H2, 256, 256, ai=5, ao=6)
        conv("trans_0.0", b["x0"], b["t0"], H, H, 128, 128, ai=3)
        conv("trans_1.0", b["x1"], b["t1"], H2, H2, 256, 256, ai=6, ao=7)
        deconv("deconv_block_0.0", b["t1"], b["m0"], H2, H, 256, 128, residual=b["t0"], ai=7, ao=8)
        deconv("deconv_block_1.0", b["t1"], b["m1"], H2, H, 256, 128, ai=7, ao=9)
        conv("conv_0.0", b["m0"], b["o0"], H, H, 128, 128, ai=8)
        conv("conv_1.0", b["m1"], b["o1"], H, H, 128, 128, ai=9)
        w0, s0, t0 = self.params["w_0.0"]
        w1, s1, t1 = self.params["w_1.0"]
        ops.ssfa_fuse(b["o0"], b["o1"], w0, w1, s0, t0, s1, t1, b["out"])
        if self.use_h2 and "head" in self.params:
            ops.absmax(b["out"], self._am(10))
        if "head" not in self.params:
            mark("neck:fuse+head")
            return b["out"], None
        self.head(b["out"])
        mark("neck:fuse+head")
        return b["out"], b["head"]

    def bench_layer(self, name="bottom_up_block_0.4"):
        """(launch closure, kernel description) of one 3x3 128->128 layer on the buffers / abs-max slots a frame uses (valid after any
        forward): what bench.py times alone for the `roofline` object."""
        H = (self.h, self.w)
        x, out = self.buf["x0"], self.buf["b0b"]

        def launch():
            self._conv(name, x, out, H, H, 128, 128, ai=3, ao=2)

        if (name + ":h2") in self.params:
            kern = "bev_conv_p2_kernel<.., kP2SplitF16> (fp32 input split to fp16 in shared memory, fp16 wgmma)"
        elif (name + ":tc") in self.params:
            kern = "bev_conv_p2_kernel<.., kP2SplitTf32> (3xTF32, tf32 wgmma)"
        else:
            kern = "bev_conv_kernel (fp32 SIMT)"
        return launch, kern

    def head(self, x):
        hw, hb = self.params["head"]
        H = (self.h, self.w)
        d = ops.conv_desc(self.batch, H, 128, H, self.HEAD_STRIDE, H, [(0, 0)], relu=False)
        if "head:h2" in self.params:
            planes, inv = self.params["head:h2"]
            return ops.bev_conv_h2(x, planes, inv, hb, None, self.buf["head"], d, self._am(10), None)
        if "head:tc" in self.params:
            return ops.bev_conv_tc(x, self.params["head:tc"], None, hb, None, self.buf["head"], d)
        return ops.bev_conv(x, hw, None, hb, None, self.buf["head"], d)


# ---------------------------------------------------------------------------------------------------------------
class SSFAPlanesRunner:
    """SSFA neck (rpn_v1.py:220-235) + the fused 128->22(+2 pad) head GEMM (mg_head_sessd.py:202-230) on csrc/bevconv_p2.cu:
    activations travel between the layers as fp16 (hi, lo) planes written by the producing epilogue (the main loops are pure
    TMA -> wgmma).  14 launches per forward: 13 convs (the stride-2 conv included)
    + the attention fusion; + abs-max and split when the input arrives as fp32 (module API) instead of planes (FrameEngine)."""

    HEAD_STRIDE = 24
    # info slots (each {abs-max, scale}); the whole table is zeroed once per forward
    SLOT = dict(x=0, b0a=1, b0b=2, x0=3, b1a=4, b1b=5, x1=6, t1=7, m0=8, m1=9, out=10, t0=11, o0=12, o1=13, head=14)

    def __init__(self, batch, hw=(200, 176), device="cuda"):
        self.batch, self.h, self.w, self.device = batch, int(hw[0]), int(hw[1]), torch.device(device)
        h, w, h2, w2 = self.h, self.w, self.h // 2, self.w // 2
        pl = lambda hh, ww, c: ops.alloc_bev_planes(batch, hh, ww, c, self.device)     # noqa: E731
        z = lambda hh, ww, c: torch.zeros((batch, hh, ww, c), dtype=torch.float32, device=self.device)  # noqa: E731
        self.planes = dict(x=pl(h, w, 128), b0a=pl(h, w, 128), b0b=pl(h, w, 128), x0=pl(h, w, 128), b1a=pl(h2, w2, 256), b1b=pl(h2, w2, 256),
                           x1=pl(h2, w2, 256), t1=pl(h2, w2, 256), m0=pl(h, w, 128), m1=pl(h, w, 128), out=pl(h, w, 128))
        self.buf = dict(t0=z(h, w, 128), o0=z(h, w, 128), o1=z(h, w, 128), out=z(h, w, 128), head=z(h, w, self.HEAD_STRIDE))
        self.info = torch.zeros((16, 2), dtype=torch.float32, device=self.device)
        self.params = None

    def _info(self, name):
        return self.info[self.SLOT[name]]

    def load_state(self, ssfa_sd, head_sd=None, head_prefix="tasks.0.", bn_eps=BN_EPS):
        dev = self.device
        g = lambda k: ssfa_sd[k].to(dev, torch.float32)   # noqa: E731
        P = {}

        def bn(conv_name):
            blk, idx = conv_name.rsplit(".", 1)
            b = "%s.%d" % (blk, int(idx) + 1)
            return fold_bn(g(b + ".weight"), g(b + ".bias"), g(b + ".running_mean"), g(b + ".running_var"), eps=bn_eps)

        def pack(name, wp, taps, cout_pad):
            sc, sh = bn(name)
            planes, inv = ops.pack_weight_h2(wp, cout_pad)
            P[name] = dict(w=planes, taps=taps, scale=(sc * inv[:sc.numel()]).contiguous(), shift=sh.contiguous(),
                           gain=ops.conv_gain(wp, sc), shift_max=float(sh.abs().max()))

        for name, pad in (("bottom_up_block_0.1", 1), ("bottom_up_block_0.4", 1), ("bottom_up_block_0.7", 1), ("bottom_up_block_1.0", 1),
                          ("bottom_up_block_1.3", 1), ("bottom_up_block_1.6", 1), ("trans_0.0", 0), ("trans_1.0", 0), ("conv_0.0", 1),
                          ("conv_1.0", 1)):
            wp, taps = _pack_conv(g(name + ".weight"))
            pack(name, wp, [(dy - pad, dx - pad) for dy, dx in taps], -(-wp.shape[2] // 128) * 128)
        for name in ("deconv_block_0.0", "deconv_block_1.0"):       # plain 9-tap packing of W[cin][cout][ky][kx]
            wd = g(name + ".weight")
            pack(name, wd.permute(2, 3, 0, 1).reshape(9, wd.shape[0], wd.shape[1]).contiguous(), None, 128)
        for name in ("w_0.0", "w_1.0"):
            sc, sh = bn(name)
            P[name] = (g(name + ".weight").reshape(-1).contiguous(), float(sc[0]), float(sh[0]))
        if head_sd is not None:
            hw, hb = pack_head(head_sd, head_prefix, dev, self.HEAD_STRIDE)
            planes, inv = ops.pack_weight_h2(hw, 32)
            P["head"] = dict(w=planes, taps=[(0, 0)], scale=inv[: self.HEAD_STRIDE].contiguous(), shift=hb.contiguous(),
                             gain=ops.conv_gain(hw, torch.ones(self.HEAD_STRIDE, device=dev)), shift_max=float(hb.abs().max()))
        self.params = P

    def _conv(self, name, src, dst, in_hw, out_hw, cin, cout, stride=1, relu=True, f32=None):
        """src: name of the input planes; dst: name of the output planes (or None); f32: name of an fp32 output buffer (or None)"""
        q = self.params[name]
        d = ops.conv_desc(self.batch, in_hw, cin, out_hw, cout, out_hw, q["taps"], in_stride=stride, relu=relu)
        out_name = dst if dst is not None else f32
        ops.bev_conv_p2(self.planes[src], self._info(src), q["w"], q["scale"], q["shift"], None, None, q["gain"], q["shift_max"],
                        self.buf[f32] if f32 is not None else None, self.planes[dst] if dst is not None else None, self._info(out_name), d)

    def _deconv(self, name, src, dst, residual=None):
        q = self.params[name]
        ops.bev_deconv_p2(self.planes[src], self._info(src), q["w"], q["scale"], q["shift"], self.buf[residual] if residual else None,
                          self._info(residual) if residual else None, q["gain"], q["shift_max"], None, self.planes[dst], self._info(dst), True)

    def forward(self, x=None, mark=None):
        """x: NHWC fp32 [B,200,176,128] (converted to planes here) or None when self.planes['x'] / info slot 'x' were filled by the
        producer (FrameEngine: dense() writes the planes directly).  Returns (neck out NHWC fp32, head NHWC fp32 [B,200,176,24])."""
        assert self.params is not None, "load_state first"
        mark = mark or (lambda label: None)
        H, H2 = (self.h, self.w), (self.h // 2, self.w // 2)
        if x is not None:
            self.info.zero_()
            ops.absmax(x, self.info[0, 0:1])
            ops.bev_split_planes(x, self.info[0], self.planes["x"])

        def conv(name, *a, **kw):
            self._conv(name, *a, **kw)
            mark("neck:" + name)

        conv("bottom_up_block_0.1", "x", "b0a", H, H, 128, 128)
        conv("bottom_up_block_0.4", "b0a", "b0b", H, H, 128, 128)
        conv("bottom_up_block_0.7", "b0b", "x0", H, H, 128, 128)
        conv("bottom_up_block_1.0", "x0", "b1a", H, H2, 128, 256, stride=2)
        conv("bottom_up_block_1.3", "b1a", "b1b", H2, H2, 256, 256)
        conv("bottom_up_block_1.6", "b1b", "x1", H2, H2, 256, 256)
        conv("trans_0.0", "x0", None, H, H, 128, 128, f32="t0")
        conv("trans_1.0", "x1", "t1", H2, H2, 256, 256)
        self._deconv("deconv_block_0.0", "t1", "m0", residual="t0")
        mark("neck:deconv_block_0.0")
        self._deconv("deconv_block_1.0", "t1", "m1")
        mark("neck:deconv_block_1.0")
        conv("conv_0.0", "m0", None, H, H, 128, 128, f32="o0")
        conv("conv_1.0", "m1", None, H, H, 128, 128, f32="o1")
        w0, s0, t0 = self.params["w_0.0"]
        w1, s1, t1 = self.params["w_1.0"]
        ops.ssfa_fuse_planes(self.buf["o0"], self.buf["o1"], w0, w1, s0, t0, s1, t1, self.buf["out"], self._info("o0"), self._info("o1"),
                             self._info("out"), self.planes["out"])
        if "head" not in self.params:
            mark("neck:fuse+head")
            return self.buf["out"], None
        self.head()
        mark("neck:fuse+head")
        return self.buf["out"], self.buf["head"]

    def head(self):
        H = (self.h, self.w)
        self._conv("head", "out", None, H, H, 128, self.HEAD_STRIDE, relu=False, f32="head")
        return self.buf["head"]

    def activation(self, name):
        """fp32 NHWC view of an intermediate tensor (tests): planes are converted back with their scale"""
        if name in self.buf:
            return self.buf[name]
        return ops.planes_to_float(self.planes[name], self._info(name))

    def bench_layer(self, name="bottom_up_block_0.4"):
        H = (self.h, self.w)

        def launch():
            self._conv(name, "x0", "b0b", H, H, 128, 128)

        return launch, "bev_conv_p2_kernel (fp16 wgmma from pre-split fp16 planes, two-term split)"
