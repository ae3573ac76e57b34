"""Stage runners: pre-allocated, capacity-sized device state + launch sequences for the three GPU stages
(sparse middle encoder, SSFA neck + head, post-processing).  No host synchronisation inside ``forward`` -- every
data-dependent count stays on the device -- so a whole frame can be captured in one CUDA graph (engine.py).

Layer tables mirror det3d/models/backbones/scn.py:106-149 (SpMiddleFHD) and det3d/models/necks/rpn_v1.py:135-235 (SSFA).
"""
import itertools
import math

import torch
from sessd_data.layers import SPMIDDLE_LAYERS  # (kind, cout, ksize, stride, padding, indice_key)   scn.py:106-149
from sessd_data.layers import SSFA_LAUNCHES, ssfa_extents

from . import ops

BN_EPS = 1e-3   # norm_cfg eps of both BN1d (scn.py:103) and BN2d (rpn_v1.py:131)

def conv_out_shape(shape, ksize, stride, padding):
    return tuple((int(i) + 2 * p - k) // s + 1 for i, k, s, p in zip(shape, ksize, stride, padding))


def fold_bn(gamma, beta, mean, var, eps=BN_EPS):
    scale = gamma.float() / torch.sqrt(var.float() + eps)
    shift = beta.float() - mean.float() * scale
    return scale.contiguous(), shift.contiguous()


def sparse_impl(cin, use_tc=True):
    """kernel of a sparse conv with cin input channels.  use_tc: "rows" (pair-proportional fp32 SIMT, csrc/spconv_rows.cu) up to 16
    channels, "cg" (pair-proportional gather + fp16 wgmma with a two-term fp16 split, csrc/spconv_cg.cu) above; otherwise "simt" (the
    output-stationary fp32 baseline, csrc/spconv.cu) for every layer"""
    if not use_tc:
        return "simt"
    return "rows" if cin <= 16 else "cg"


def plane_width(channels):
    """cp of the fp16 (hi, lo) planes [rows, 2 cp] of a sparse feature tensor, and of the weight tiles of the cg layer that reads them"""
    return 32 if channels <= 32 else 64


def spmiddle_plan(use_tc=True, keep_f32=False, cin0=4):
    """One record per conv of SpMiddleFHD (SPMIDDLE_LAYERS): its kernel and the operands it reads and writes.
      kind, key, ks, st, pd, cin, cout: the layer;  lin / lout: its input / output level (a strided conv opens the next level)
      rb: its rulebook, the SubM indice key or "sp<lout>" for a strided conv;  build_rb: this layer builds it (the first to use it)
      tile_lists: (with build_rb) the per-tile pair lists are made from it, because a cg layer gathers over it
      impl: "rows" / "cg" / "simt" (sparse_impl);  cp_in: width of the input planes and of the packed weight of a cg layer, None for
        the layers that read fp32 rows
      cp_out: width of the output planes the layer writes for a cg successor, or None;  out_f32: it writes fp32 rows
      out_info: it writes its {abs-max, scale} info slot: every cg layer and every layer that writes planes; a rows layer without planes
        writes only the abs-max, for a successor that derives its planes' scale from that bound"""
    plan, cin, lvl = [], cin0, 0
    for kind, cout, ks, st, pd, key in SPMIDDLE_LAYERS:
        lout = lvl if kind == "subm" else lvl + 1
        rb = key if kind == "subm" else "sp%d" % lout
        impl = sparse_impl(cin, use_tc)
        plan.append(dict(kind=kind, key=key, ks=ks, st=st, pd=pd, cin=cin, cout=cout, lin=lvl, lout=lout, rb=rb,
                         build_rb=all(p["rb"] != rb for p in plan), impl=impl, cp_in=plane_width(cin) if impl == "cg" else None))
        cin, lvl = cout, lout
    nxt = {}
    for p in reversed(plan):
        p["tile_lists"] = p["build_rb"] and any(q["impl"] == "cg" for q in plan if q["rb"] == p["rb"])
        p["cp_out"] = nxt.get("cp_in")
        p["out_f32"] = keep_f32 or p["cp_out"] is None
        p["out_info"] = p["impl"] == "cg" or p["cp_out"] is not None or (nxt.get("impl") == "rows" and nxt["cp_out"] is not None)
        nxt = p
    return plan


class SpMiddleRunner:
    """SpMiddleFHD forward (scn.py:176-189): 4 SubM rulebooks + 4 strided rulebooks + 14 fused conv launches + dense(), as laid
    out by spmiddle_plan."""

    # active-site growth bounds per level relative to the level-0 capacity (uniform 20k cloud: 3.4 / 5.2 / 4.3 / 2.6)
    GROWTH = (1.0, 4.0, 6.0, 5.0, 3.0)

    def __init__(self, batch, max_voxels_total, input_shape_xyz=(1408, 1600, 40), num_input_features=4, device="cuda",
                 growth=None, use_tc=True, keep_f32=False):
        """use_tc: the narrow layers on the pair-proportional fp32 SIMT kernel and the others on the tensor cores, activations handed
        from layer to layer as fp16 (hi, lo) planes; False = the fp32 SIMT baseline for every layer (sparse_impl).
        keep_f32: the layers that hand planes to the next one write their fp32 rows as well (tests compare per-layer features)."""
        self.batch, self.device = batch, torch.device(device)
        self.use_tc, self.keep_f32 = bool(use_tc), bool(keep_f32)
        shape = (int(input_shape_xyz[2]) + 1, int(input_shape_xyz[1]), int(input_shape_xyz[0]))   # scn.py:179
        growth = growth or self.GROWTH
        self.levels = []       # dicts: shape, cap, grid, coors, n, index_kind, index, scratch
        self._add_level(shape, int(max_voxels_total), hash_index=True)
        self.plan = spmiddle_plan(self.use_tc, self.keep_f32, num_input_features)
        rulebooks = {}         # rb -> (neighbour table, tile lists or None), shared by the layers of a SubM key
        for p in self.plan:
            if p["kind"] != "subm":
                oshape = conv_out_shape(self.levels[p["lin"]]["shape"], p["ks"], p["st"], p["pd"])
                cells = batch * oshape[0] * oshape[1] * oshape[2]
                self._add_level(oshape, min(cells, int(math.ceil(max_voxels_total * growth[p["lout"]]))), hash_index=False)
            if p["build_rb"]:
                cap, kvol = self.levels[p["lout"]]["cap"], p["ks"][0] * p["ks"][1] * p["ks"][2]
                rulebooks[p["rb"]] = (torch.empty((cap, kvol), dtype=torch.int32, device=self.device),
                                      ops.alloc_tile_lists(cap, kvol, self.device) if p["tile_lists"] else None)
            p["nbr"], p["tiles"] = rulebooks[p["rb"]]
        caps = [self.levels[p["lout"]]["cap"] for p in self.plan]
        self.feats = [torch.zeros((cap, p["cout"]), dtype=torch.float32, device=self.device) if p["out_f32"] else None
                      for p, cap in zip(self.plan, caps)]
        self.planes = [ops.alloc_planes(cap, p["cp_out"], self.device) if p["cp_out"] else None for p, cap in zip(self.plan, caps)]
        # a cg layer's tile lists address its input plane rows with 25 bits (input row << 7 | tile row)
        assert all(pl is None or pl.shape[0] <= (1 << 25) for pl in self.planes)
        last = self.levels[-1]
        self.out_channels = self.plan[-1]["cout"] * last["shape"][0]
        self.dense = torch.zeros((batch, last["shape"][1], last["shape"][2], self.out_channels), dtype=torch.float32,
                                 device=self.device)
        self.status = torch.zeros((1,), dtype=torch.int32, device=self.device)
        self.weights = None
        # {abs-max, plane scale} of every layer output (out_info)
        self.info = torch.zeros((len(self.plan), 2), dtype=torch.float32, device=self.device)

    def layer_output(self, li):
        """fp32 rows [cap, Cout] of layer li's output after forward(): the fp32 buffer when the layer wrote it, else rebuilt from the fp16
        (hi, lo) planes it wrote (exact: x = (hi + lo) / S) -- tests / debugging."""
        p = self.plan[li]
        if p["out_f32"]:
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
            p["gain"], p["shift_max"] = ops.conv_gain(wp, sc), float(sh.abs().max())
            if p["impl"] == "cg":      # fp16 (hi, lo) weight tiles; their per-channel 2^-e folds into the BN scale
                tiles, inv = ops.pack_weight_sp_h2(wp, p["cp_in"])
                self.weights.append((tiles, (sc * inv).contiguous(), sh))
            else:
                self.weights.append((wp, sc, sh))

    def forward(self, feat0, coors0, n0, mark=None, dense_planes=None):
        """feat0 [cap0, Cin] f32, coors0 [cap0,4] i32 (b,z,y,x), n0 [1] i32 (device).  Returns dense NHWC.
        mark: optional callable(label) invoked after every launch group (profiling scripts record a CUDA event there).
        dense_planes: (planes [2,B,H,W,C*D] fp16, info [2] f32): dense() writes the fp16 (hi, lo) planes the BEV neck reads instead
        of the fp32 map (returns the planes)."""
        mark = mark or (lambda label: None)
        assert self.weights is not None, "load_weights first"
        L0 = self.levels[0]
        cap0 = min(coors0.shape[0], L0["cap"])
        L0["coors"], L0["n_ext"] = coors0, n0
        ops.hash_build(coors0, n0, cap0, L0["grid"], L0["index"])
        mark("hash_build")
        if self.use_tc:
            self.info.zero_()
        x = feat0
        for li, p in enumerate(self.plan):
            lin, lout = self.levels[p["lin"]], self.levels[p["lout"]]
            n_in = lin["n_ext"] if p["lin"] == 0 else lin["n"]
            cap_in = cap0 if p["lin"] == 0 else lin["cap"]
            n_out, cap_out = (n_in, cap_in) if p["kind"] == "subm" else (lout["n"], lout["cap"])
            if p["build_rb"]:
                if p["kind"] == "subm":
                    ops.subm_rulebook(lin["coors"], n_in, cap_in, lin["grid"], p["ks"], lin["index_kind"], lin["index"], p["nbr"])
                else:
                    ops.strided_rulebook(lin["coors"], n_in, cap_in, lin["grid"], lin["index_kind"], lin["index"], p["ks"], p["st"],
                                         p["pd"], lout["grid"], lout["index"], lout["scratch"], lout["coors"], lout["n"], lout["cap"],
                                         p["nbr"], self.status)
                if p["tiles"] is not None:
                    ops.rulebook_tile_lists(p["nbr"], n_out, cap_out, p["tiles"])
                mark("rulebook:" + p["rb"])
            w, sc, sh = self.weights[li]
            out = self.feats[li]
            if p["impl"] == "rows" and p["cp_out"]:
                # the planes' scale comes from the bound on the output: the input's abs-max (info slot of layer li - 1) x gain + shift_max
                ops.spconv_forward_rows_planes(x, p["nbr"], n_out, cap_out, w, sc, sh, True, self.info[li - 1, 0:1], p["gain"], p["shift_max"],
                                               out, self.planes[li], self.info[li])
            elif p["impl"] == "rows":
                ops.spconv_forward_rows(x, p["nbr"], n_out, cap_out, w, sc, sh, True, out, self.info[li, 0:1] if p["out_info"] else None)
            elif p["impl"] == "cg":
                ops.spconv_forward_cg(self.planes[li - 1], self.info[li - 1], p["tiles"], n_out, cap_out, w, sc, sh, True, p["gain"],
                                      p["shift_max"], out, self.planes[li], self.info[li])
            else:
                ops.spconv_forward(x, p["nbr"], n_out, cap_out, w, sc, sh, True, out)
            mark("conv:%d" % li)
            x = out
        last = self.levels[-1]
        if dense_planes is not None:
            assert self.plan[-1]["out_info"], "the planes' scale needs the last layer's abs-max (use_tc)"
            out = ops.sparse_to_dense_planes(x, last["index"], last["grid"], self.info[-1, 0:1], dense_planes[1], dense_planes[0])
        else:
            out = ops.sparse_to_dense_indexed(x, last["index"], last["grid"], self.dense)
        mark("dense")
        return out


# ---------------------------------------------------------------------------------------------------------------
class RunnerCache:
    """The stage runner of an eval-mode module (SpMiddleFHD, SSFA, Head): built anew when its key (shapes, device) changes, and its
    weights reloaded when the (data_ptr, _version) of any parameter or buffer of the module changes."""

    def __init__(self):
        self.runner = self.key = self.weights = None

    def get(self, module, key, build, load):
        """the runner for ``key``: build() makes a new one, load(runner) loads the module's weights into it"""
        if self.runner is None or key != self.key:
            self.runner, self.key, self.weights = build(), key, None
        weights = tuple((t.data_ptr(), t._version) for t in itertools.chain(module.parameters(), module.buffers()))
        if weights != self.weights:
            load(self.runner)
            self.weights = weights
        return self.runner


_SSFA = {L.name: L for L in SSFA_LAUNCHES}


def conv_taps(k):
    """taps (dy, dx) of a k x k conv padded by k // 2, relative to the output pixel (times the input stride), in _pack_conv order"""
    return [(dy - k // 2, dx - k // 2) for dy in range(k) for dx in range(k)]


def _pack_conv(w):
    """nn.Conv2d weight [Cout,Cin,kh,kw] -> ([kh*kw, Cin, Cout], taps (dy,dx) relative to the unpadded origin)."""
    cout, cin, kh, kw = w.shape
    packed = w.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout).contiguous()
    return packed, [(ky, kx) for ky in range(kh) for kx in range(kw)]


def launch_weight(L, w):
    """(weight [taps, Cin, Cout], taps) of launch L from its weight in the module's layout: a conv's Conv2d weight [Cout, Cin, k, k] (the
    head's from head_weight) in the packing of _pack_conv with the taps of conv_taps; a deconv's ConvTranspose2d weight
    [Cin, Cout, 3, 3] in the plain 9-tap packing of W[cin][cout][ky][kx], taps None"""
    if L.kind == "deconv":
        return w.permute(2, 3, 0, 1).reshape(9, L.cin, L.cout).contiguous(), None
    return _pack_conv(w)[0], conv_taps(L.k)


def launch_desc(L, batch, in_hw, out_hw, taps, relu=None):
    """ConvDesc of conv launch L on a batch of its ssfa_extents (in_hw, out_hw), with the taps of launch_weight's packing and the fused
    ReLU of L unless relu says otherwise"""
    return ops.conv_desc(batch, in_hw, L.cin, out_hw, L.cout, out_hw, taps, in_stride=L.stride, relu=L.relu if relu is None else relu)


HEAD_TASK_STRIDE = _SSFA["head"].cout      # channels of one task's block in the head launch: [box 14 | cls 2 | dir 4 | iou 2 | pad 2]


def head_weight(param, prefixes=("",)):
    """The four 1x1 head convs (mg_head_sessd.py:202-215) as the module-layout weight [24, 128, 1, 1] and bias [24] of the head launch,
    channel layout [box 14 | cls 2 | dir 4 | iou 2 | zero pad].  param(name) returns a conv's tensor ("conv_box.weight"); the result is
    built with torch ops, so it keeps the autograd graph of module parameters.  Several prefixes (one per task, "tasks.0." ...): the
    tasks' blocks stacked, task t at channels 24 t ... 24 t + 23 of a [24 T, 128, 1, 1] weight."""
    ws, bs = [], []
    for p in prefixes:
        w, b = (torch.cat([param(p + c + s) for c in ("conv_box", "conv_cls", "conv_dir", "conv_iou")], 0) for s in (".weight", ".bias"))
        pad = HEAD_TASK_STRIDE - w.shape[0]
        ws += [w, w.new_zeros((pad,) + tuple(w.shape[1:]))]
        bs += [b, b.new_zeros((pad,))]
    return torch.cat(ws, 0), torch.cat(bs, 0)


def head_prefixes(prefix):
    """the task prefixes of a head state dict: one prefix ("tasks.0.") or a list of them, one per task"""
    return (prefix,) if isinstance(prefix, str) else tuple(prefix)


def pack_head(head_sd, prefix, device):
    """head_weight from a state dict; prefix: one task's key prefix or a list of them (head_prefixes)"""
    return head_weight(lambda name: head_sd[name].to(device, torch.float32), head_prefixes(prefix))


def head_launch(num_tasks=1):
    """the head launch of a head with num_tasks one-class tasks: 24 channels per task"""
    return _SSFA["head"]._replace(cout=HEAD_TASK_STRIDE * int(num_tasks))


def fold_ssfa_bn(sd, conv_name, device, eps=BN_EPS):
    """folded (scale, shift) of the BatchNorm2d that follows an SSFA conv: module blk.(i+1) of the conv blk.i (rpn_v1.py:135-210)"""
    blk, idx = conv_name.rsplit(".", 1)
    b = "%s.%d." % (blk, int(idx) + 1)
    return fold_bn(*(sd[b + k].to(device, torch.float32) for k in ("weight", "bias", "running_mean", "running_var")), eps=eps)


def pack_h2(wp, taps, scale, shift):
    """launch_weight's (weight [taps, Cin, Cout], taps) + folded BN (scale None: 1) -> the fp16-split launch parameters of bev_conv_p2 /
    _h2: weight planes, epilogue scale (BN scale x the planes' 2^-e[n]), shift, gain / shift_max of the output bound, and the taps"""
    planes, inv = ops.pack_weight_h2(wp, _cout_pad(wp.shape[2]))
    scale = torch.ones(wp.shape[2], device=wp.device) if scale is None else scale
    return dict(w=planes, scale=(scale * inv[:scale.numel()]).contiguous(), shift=shift.contiguous(), gain=ops.conv_gain(wp, scale),
                shift_max=float(shift.abs().max()), taps=taps)


def _cout_pad(cout):
    """packed weight width of a BEV conv: whole n-tiles of bev_conv_p2 (32 channels up to 32, else 128), as the skip plan assumes"""
    n_tile = 32 if cout <= 32 else 128
    return -(-cout // n_tile) * n_tile


def ssfa_weights(ssfa_sd, head_sd, head_prefix, device, bn_eps=BN_EPS):
    """yields (launch, weight [taps, Cin, Cout], taps, BN scale, BN shift) in SSFA_LAUNCHES order, weight and taps from launch_weight;
    the head (only with head_sd; head_prefix: one prefix or one per task) with scale None and its bias as the shift"""
    for L in SSFA_LAUNCHES:
        if L.name != "head":
            wp, taps = launch_weight(L, ssfa_sd[L.name + ".weight"].to(device, torch.float32))
            yield (L, wp, taps) + fold_ssfa_bn(ssfa_sd, L.name, device, bn_eps)
        elif head_sd is not None:
            w, bias = pack_head(head_sd, head_prefix, device)
            yield (L, *launch_weight(L, w), None, bias)


def ssfa_fuse_weights(ssfa_sd, device, bn_eps=BN_EPS):
    """{w_0.0 / w_1.0: (weight [128], BN scale, BN shift)} of the attention fusion's 1x1 128 -> 1 convs"""
    out = {}
    for name in ("w_0.0", "w_1.0"):
        sc, sh = fold_ssfa_bn(ssfa_sd, name, device, bn_eps)
        out[name] = (ssfa_sd[name + ".weight"].to(device, torch.float32).reshape(-1).contiguous(), float(sc[0]), float(sh[0]))
    return out


# {abs-max, scale} slot of every SSFA tensor: the neck input, the launch outputs kept as planes, the fused map, then the fp32 outputs
SSFA_SLOT = {n: i for i, n in enumerate(["x"] + [L.dst for L in SSFA_LAUNCHES if not L.f32] + ["out"] + [L.dst for L in SSFA_LAUNCHES if L.f32])}


# ---------------------------------------------------------------------------------------------------------------
class SSFAPlanesRunner:
    """SSFA neck (rpn_v1.py:220-235) + the fused 128->22(+2 pad) head GEMM (mg_head_sessd.py:202-230) on csrc/bevconv_p2.cu, one 24-channel
    block per task of a multi-task head (num_tasks one-class tasks: one 128 -> 24 T GEMM, HEAD_STRIDE = 24 T):
    activations travel between the layers as fp16 (hi, lo) planes written by the producing epilogue (the main loops are pure
    TMA -> wgmma).  14 launches per forward: 13 convs (the stride-2 conv included)
    + the attention fusion; + abs-max and split when the input arrives as fp32 (module API) instead of planes (FrameEngine).
    With skip_constant and the sparse occupancy (FrameEngine): + the skip plan's two launches and one fill launch after each conv / deconv."""

    HEAD_STRIDE = 24
    # info slots (each {abs-max, scale}); the whole table is zeroed once per forward
    SLOT = SSFA_SLOT
    # the conv / deconv launches of one forward, in the order of the skip plan's records (csrc/bevskip.cu)
    SKIP_LAUNCHES = tuple(L.name for L in SSFA_LAUNCHES)

    def __init__(self, batch, hw=(200, 176), device="cuda", skip_constant=False, num_tasks=1):
        """skip_constant: when forward() gets the occupancy of the last sparse level, run only the work items whose output can differ
        from the empty-space constant of its class and fill the others with it (bit-identical to the dense neck, csrc/bevskip.cu).
        num_tasks: tasks of the head; load_state then takes one head prefix per task"""
        self.batch, self.h, self.w, self.device = batch, int(hw[0]), int(hw[1]), torch.device(device)
        self._set_tasks(num_tasks)
        pl = lambda hw_, c: ops.alloc_bev_planes(batch, hw_[0], hw_[1], c, self.device)     # noqa: E731
        z = lambda hw_, c: torch.zeros((batch,) + hw_ + (c,), dtype=torch.float32, device=self.device)  # noqa: E731
        H, ext = (self.h, self.w), lambda L: ssfa_extents(L, self.h, self.w)[1]     # noqa: E731
        self.planes = dict(x=pl(H, 128), **{L.dst: pl(ext(L), L.cout) for L in SSFA_LAUNCHES if not L.f32}, out=pl(H, 128))
        self.buf = dict(**{L.dst: z(ext(L), L.cout) for L in SSFA_LAUNCHES[:-1] if L.f32}, out=z(H, 128), head=z(H, self.HEAD_STRIDE))
        self.info = torch.zeros((16, 2), dtype=torch.float32, device=self.device)
        self.params = None
        self.skip_constant = bool(skip_constant)
        self.skip = ops.BevSkipPlan(batch, self.h, self.w, self.device, self.HEAD_STRIDE) if self.skip_constant else None

    def _set_tasks(self, num_tasks):
        self.num_tasks = int(num_tasks)
        if self.num_tasks < 1:
            raise ValueError("num_tasks must be at least 1")
        self.head_launch = head_launch(self.num_tasks)
        self.HEAD_STRIDE = self.head_launch.cout

    def _check_prefixes(self, prefix):
        if len(head_prefixes(prefix)) != self.num_tasks:
            raise ValueError("a %d-task head needs %d head prefixes, got %r" % (self.num_tasks, self.num_tasks, prefix))

    def _info(self, name):
        return self.info[self.SLOT[name]]

    def load_state(self, ssfa_sd, head_sd=None, head_prefix="tasks.0.", bn_eps=BN_EPS):
        """bn_eps: eps of the neck's BatchNorm2d layers (rpn_v1.py:131-132 uses 1e-3; pass the module's own value otherwise)."""
        if head_sd is not None:
            self._check_prefixes(head_prefix)
        P = ssfa_fuse_weights(ssfa_sd, self.device, bn_eps)
        for L, *weight in ssfa_weights(ssfa_sd, head_sd, head_prefix, self.device, bn_eps):
            P[L.name] = pack_h2(*weight)
        self.params = P

    def _split(self, x, name):
        """zero the info slots, then split the fp32 NHWC x into the planes of tensor ``name`` and its info slot"""
        self.info.zero_()
        ops.absmax(x, self._info(name)[0:1])
        ops.bev_split_planes(x, self._info(name), self.planes[name])

    def _launch(self, L, skip=False):
        """launch L from its input planes into its output planes or fp32 buffer.  skip: run the segments of this launch's segment
        record (the stride-2 conv: the work items of its tile record), then fill the skipped segments (tiles)"""
        q = self.params[L.name]
        out_f32, out_planes = (self.buf[L.dst], None) if L.f32 else (None, self.planes[L.dst])
        resid, resid_info = (self.buf[L.residual], self._info(L.residual)) if L.residual else (None, None)
        i = self.SKIP_LAUNCHES.index(L.name)
        segs = self.skip.seg_record(i) if skip else None
        rec = self.skip.record(i) if skip and segs is None else None
        if L.kind == "conv":
            d = launch_desc(L, self.batch, *ssfa_extents(L, self.h, self.w), q["taps"])
            ops.bev_conv_p2(self.planes[L.src], self._info(L.src), q["w"], q["scale"], q["shift"], resid, resid_info, q["gain"],
                            q["shift_max"], out_f32, out_planes, self._info(L.dst), d, items=rec, segs=segs)
        else:
            ops.bev_deconv_p2(self.planes[L.src], self._info(L.src), q["w"], q["scale"], q["shift"], resid, resid_info, q["gain"],
                              q["shift_max"], out_f32, out_planes, self._info(L.dst), L.relu, items=rec, segs=segs)
        if segs is not None:
            self.skip.fill_segs(i, out_f32, out_planes, L.cout)
        elif skip:
            self.skip.fill(i, out_f32, out_planes, L.cout)

    def forward(self, x=None, mark=None, occupancy=None):
        """x: NHWC fp32 [B,200,176,128] (converted to planes here) or None when self.planes['x'] / info slot 'x' were filled by the
        producer (FrameEngine: dense() writes the planes directly).  Returns (neck out NHWC fp32, head NHWC fp32 [B,200,176,24 T]).
        occupancy: (bitmap index, grid) of the last sparse level whose dense() made the input (FrameEngine); with skip_constant, the
        launches then skip the tiles of the empty space (the input must be exactly zero wherever that level has no site)."""
        assert self.params is not None, "load_state first"
        mark = mark or (lambda label: None)
        if x is not None:
            self._split(x, "x")
        skip = self.skip_constant and occupancy is not None
        if skip:
            index, grid = occupancy
            assert (grid.batch, grid.shape[1], grid.shape[2]) == (self.batch, self.h, self.w), "occupancy of another map"
            self.skip.build(index, grid)
            mark("neck:skip_plan")
        for L in SSFA_LAUNCHES[:-1]:
            self._launch(L, skip)
            mark("neck:" + L.name)
        w0, s0, t0 = self.params["w_0.0"]
        w1, s1, t1 = self.params["w_1.0"]
        ops.ssfa_fuse_planes(self.buf["o0"], self.buf["o1"], w0, w1, s0, t0, s1, t1, self.buf["out"], self._info("o0"), self._info("o1"),
                             self._info("out"), self.planes["out"])
        if "head" not in self.params:
            mark("neck:fuse+head")
            return self.buf["out"], None
        self.head(skip=skip)
        mark("neck:fuse+head")
        return self.buf["out"], self.buf["head"]

    def head(self, skip=False):
        self._launch(self.head_launch, skip)
        return self.buf["head"]

    def activation(self, name):
        """fp32 NHWC view of an intermediate tensor (tests): planes are converted back with their scale"""
        if name in self.buf:
            return self.buf[name]
        return ops.planes_to_float(self.planes[name], self._info(name))

    def bench_layer(self, name="bottom_up_block_0.4"):
        """(launch closure, kernel description) of one 3x3 128->128 layer on the planes / info slots a frame uses (valid after any
        forward): what bench.py times alone for the `roofline` object."""

        def launch():
            self._launch(_SSFA[name]._replace(src="x0", dst="b0b"))

        return launch, "bev_conv_p2_kernel (fp16 wgmma from pre-split fp16 planes, two-term split)"


class HeadRunner(SSFAPlanesRunner):
    """The fused head GEMM alone (MultiGroupHead.forward): only the buffers of the head launch (its input planes, the info slots, its
    output), launched by SSFAPlanesRunner.head after the fp32 input is split into planes.  num_tasks > 1: every task of a MultiGroupHead
    in the one launch, task t at channels 24 t ... 24 t + 23 of the output."""

    def __init__(self, batch, hw, device="cuda", num_tasks=1):
        self.batch, self.h, self.w, self.device = batch, int(hw[0]), int(hw[1]), torch.device(device)
        self._set_tasks(num_tasks)
        self.planes = dict(out=ops.alloc_bev_planes(batch, self.h, self.w, 128, self.device))
        self.buf = dict(head=torch.zeros((batch, self.h, self.w, self.HEAD_STRIDE), dtype=torch.float32, device=self.device))
        self.info = torch.zeros((len(self.SLOT), 2), dtype=torch.float32, device=self.device)
        self.params = None

    def load_state(self, head_sd, prefix=""):
        """prefix: the key prefix of the head's convs, or one prefix per task"""
        self._check_prefixes(prefix)
        w, bias = pack_head(head_sd, prefix, self.device)
        self.params = {"head": pack_h2(*launch_weight(self.head_launch, w), None, bias)}

    def forward(self, x):
        self._split(x, "out")
        return self.head()
