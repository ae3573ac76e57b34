"""Backward of the BEV neck and head on the GPU, one operator at a time and end to end (SSFA / Head / VoxelNet in train mode).

Bounds.  Weight-gradient kernel (csrc/bevgrad.cu), after the model of tests/spconv_grad_model.py: an item of R rounds makes 4 R mma steps,
each adding two products to the cross accumulator, so it is off by <= CG_C 2^-23 (8 R + 1) of its magnitude sum M = sum |x| |g|; the
reduce adds `chunks` roundings of M; the fp16 split of x and g (abs-max into [2^14, 2^15)) adds 2^-20 (amax_x sum |g| + amax_g sum |x|).
Data gradients run the forward kernels (fp16 split of both operands, fp32 accumulation): held to 2^-17 of the magnitudes of the same
product with |g| and |W|, with amax_g and the weight's abs-max in place of either operand (the split errors).

End to end (SSFA / Head / VoxelNet in train mode) each tensor T is held to max(1e-4 max |ref_T|, PERT_K max_s |ref_T^s - ref_T|): ref
is the fp64 chain, ref^s (s < PERT_SAMPLES) the same chain with every element of every conv's output and data gradient off by up to
PERT_U times its magnitude (the same product over absolute values): the rounding model of the kernels, whose per-operator errors above
stay below 2^-24 of those magnitudes.  The second term is the conditioning of the problem: the neck's maps are mostly empty space, where
every channel holds one constant, so the train-mode BatchNorm2d of a channel normalises a spread of 5e-3 of its largest value, and an
fp32 implementation of the reference itself (cuDNN without TF32) misses fp64 by up to 1.5e-2 of max |ref| on the neck's input gradient.  Where the problem is well conditioned the 1e-4 floor (the sparse
encoder's bar) decides.
"""
import copy
import logging

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from bev_grad_model import (bg_geometry, head_params, head_ref, module_forward, ssfa_params, ssfa_train_ref, wgrad_index)
from sessd_data.layers import SSFA_LAUNCHES, ssfa_extents

pytestmark = pytest.mark.gpu
CG_C = 2.0
E2E_FLOOR = 1e-4
PERT_U = 2.0 ** -22
PERT_SAMPLES = 3
PERT_K = 2.0
_L = {L.name: L for L in SSFA_LAUNCHES}
# (id, launch whose geometry it is): 3x3 s1 128 / 256, 3x3 s2 128 -> 256 (also the deconvs' role-swapped wgrad), 1x1 128 / 256, head
WGRAD_GEOMS = ["bottom_up_block_0.4", "bottom_up_block_1.3", "bottom_up_block_1.0", "trans_0.0", "trans_1.0", "head"]


def _wgrad_case(L, b, h, w, kind, seed):
    from sessd_b200 import bev_grad, ops
    g = torch.Generator().manual_seed(seed)
    ho, wo = ((h - 1) // L.stride + 1, (w - 1) // L.stride + 1)
    x = torch.randn((b, h, w, L.cin), generator=g)
    gr = torch.randn((b, ho, wo, L.cout), generator=g) * 3.0
    if kind == "zero":
        gr.zero_()
    elif kind == "border":                     # single non-zero pixels on every border and corner: they reach the padding taps
        keep = torch.zeros((b, ho, wo, 1))
        for y, xx in ((0, 0), (0, wo - 1), (ho - 1, 0), (ho - 1, wo - 1), (0, wo // 2), (ho - 1, wo // 2), (ho // 2, 0), (ho // 2, wo - 1)):
            keep[b - 1, y, xx] = 1.0
        gr = gr * keep
    cg = bev_grad.HEAD_PAD if L.name == "head" else L.cout
    gp = F.pad(gr, (0, cg - L.cout))
    xp, xi = bev_grad.split(x.cuda())
    gpl, gi = bev_grad.split(gp.cuda())
    desc = bev_grad.conv_desc(b, (h, w), L.cin, (ho, wo), cg, L.k, L.stride)
    got = ops.bev_wgrad(xp, xi, gpl, gi, desc)
    again = ops.bev_wgrad(xp, xi, gpl, gi, desc)
    return x, gp, got, again, (ho, wo), cg


@pytest.mark.parametrize("name", WGRAD_GEOMS)
@pytest.mark.parametrize("b,h,w,kind", [(1, 13, 21, "rand"), (3, 24, 40, "rand"), (3, 17, 9, "rand"), (1, 13, 21, "zero"),
                                         (2, 11, 15, "border")])
def test_wgrad_kernel_matches_fp64(name, b, h, w, kind):
    from sessd_b200 import bev_grad
    L = _L[name]
    x, gp, got, again, out_hw, cg = _wgrad_case(L, b, h, w, kind, seed=b * 100 + h)
    torch.cuda.synchronize()
    assert torch.equal(got, again), "two runs differ"
    got = got.cpu().double()
    if kind == "zero":
        assert (got == 0).all()
        return
    taps = bev_grad.conv_taps(L.k)
    xd, gd = x.double(), gp.double()
    ref = wgrad_index(xd, gd, taps, L.stride)
    mag = wgrad_index(xd.abs(), gd.abs(), taps, L.stride)
    _nc, _groups, chunks, rpc = bg_geometry(b, out_hw, L.cin, cg, len(taps))
    split = float(xd.abs().max()) * gd.abs().sum(dim=(0, 1, 2))[None, None, :] + float(gd.abs().max()) * xd.abs().sum(dim=(0, 1, 2))[None, :, None]
    tol = (CG_C * 2.0 ** -23 * (8 * rpc + 1) + chunks * 2.0 ** -24) * mag + 2.0 ** -20 * split
    r = float(((got - ref).abs() / tol.clamp(min=1e-300)).max())
    print("wgrad %s b%d %dx%d %s: ratio %.3g, max rel %.2e" % (name, b, h, w, kind, r, float((got - ref).abs().max() / ref.abs().max())))
    assert r <= 1.0
    if cg != L.cout:
        assert (got[..., L.cout:] == 0).all()


def test_wgrad_kernel_full_map():
    """3x3 128 -> 128 on a 200 x 176 map: many chunks per tap"""
    from sessd_b200 import bev_grad
    L = _L["bottom_up_block_0.4"]
    x, gp, got, again, out_hw, cg = _wgrad_case(L, 1, 200, 176, "rand", seed=7)
    torch.cuda.synchronize()
    assert torch.equal(got, again)
    taps = bev_grad.conv_taps(3)
    ref = wgrad_index(x.double(), gp.double(), taps, 1)
    mag = wgrad_index(x.double().abs(), gp.double().abs(), taps, 1)
    _nc, _g, chunks, rpc = bg_geometry(1, out_hw, 128, 128, 9)
    split = float(x.abs().max()) * gp.double().abs().sum(dim=(0, 1, 2))[None, None, :] + float(gp.abs().max()) * x.double().abs().sum(dim=(0, 1, 2))[None, :, None]
    tol = (CG_C * 2.0 ** -23 * (8 * rpc + 1) + chunks * 2.0 ** -24) * mag + 2.0 ** -20 * split
    assert float(((got.cpu().double() - ref).abs() / tol).max()) <= 1.0


@pytest.mark.parametrize("L", SSFA_LAUNCHES, ids=[L.name for L in SSFA_LAUNCHES])
def test_function_gradients_match_fp64(L):
    """BevConvFunction on every launch: the data gradient through the forward kernels against oracle/bev_grad_ref.py, the weight (and head
    bias) gradient against autograd of the module's own op, in fp64"""
    from oracle.bev_grad_ref import conv_dgrad, deconv_dgrad
    from sessd_b200 import bev_grad
    g = torch.Generator().manual_seed(11)
    b, h, w = 2, 24, 40
    in_hw, out_hw = ssfa_extents(L, h, w)
    wshape = (L.cin, L.cout, 3, 3) if L.kind == "deconv" else (L.cout, L.cin, L.k, L.k)
    W = (torch.randn(wshape, generator=g) * 0.05).cuda().requires_grad_(True)
    bias = (torch.randn(L.cout, generator=g) * 0.1).cuda().requires_grad_(True) if L.name == "head" else None
    x = torch.relu(torch.randn((b,) + in_hw + (L.cin,), generator=g)).cuda().requires_grad_(True)
    y = bev_grad.BevConvFunction.apply(x, W, bias, L, in_hw, out_hw)
    G = torch.randn(y.shape, generator=g).cuda()
    y.backward(G)
    Wd, Gd = W.detach().cpu().double(), G.cpu().double().permute(0, 3, 1, 2)
    xd = x.detach().cpu().double().permute(0, 3, 1, 2)

    def dgrad(gg, ww):
        return deconv_dgrad(gg, ww) if L.kind == "deconv" else conv_dgrad(gg, ww, L.stride, L.k // 2)

    ref = dgrad(Gd, Wd)
    mag = dgrad(Gd.abs(), Wd.abs()) + dgrad(torch.full_like(Gd, float(Gd.abs().max())), Wd.abs()) + \
        dgrad(Gd.abs(), torch.full_like(Wd, float(Wd.abs().max())))
    gx = x.grad.cpu().double().permute(0, 3, 1, 2)
    rx = float(((gx - ref).abs() / (2.0 ** -17 * mag).clamp(min=1e-300)).max())
    # weight gradient: autograd of the module's op in fp64, with the same magnitude terms
    def wgrad(xx, gg):
        ww = Wd.clone().requires_grad_(True)
        (module_forward(L, xx, ww) * gg).sum().backward()
        return ww.grad

    refw = wgrad(xd, Gd)
    magw = wgrad(xd.abs(), Gd.abs()) + wgrad(torch.full_like(xd, float(xd.abs().max())), Gd.abs()) + \
        wgrad(xd.abs(), torch.full_like(Gd, float(Gd.abs().max())))
    rw = float(((W.grad.cpu().double() - refw).abs() / (2.0 ** -17 * magw).clamp(min=1e-300)).max())
    yref = module_forward(L, xd, Wd, None if bias is None else bias.detach().cpu().double())
    ry = float((y.detach().cpu().double().permute(0, 3, 1, 2) - yref).abs().max() / yref.abs().max())
    print("%s: dX ratio %.3g, dW ratio %.3g, fwd rel %.2e" % (L.name, rx, rw, ry))
    assert rx <= 1.0 and rw <= 1.0 and ry <= 1e-5
    if bias is not None:
        assert torch.allclose(bias.grad.cpu().double(), Gd.sum(dim=(0, 2, 3)), rtol=1e-5, atol=1e-4)


def _ring_dense(batch=2, points=5000, seed=40):
    """[batch, 128, 200, 176] dense() map of ring clouds through a randomly initialised SpMiddleFHD (train-mode forward, no grad)"""
    from det3d.models.backbones.scn import SpMiddleFHD
    from oracle import cpu as ocpu
    from sessd_b200 import synth
    feats, coors = [], []
    for b in range(batch):
        v, c, n = ocpu.points_to_voxel(synth.ring_cloud(seed + b, points), synth.VOXEL_SIZE, synth.PC_RANGE, 5, 20000)
        coors.append(np.concatenate([np.full((len(c), 1), b, np.int32), c], 1))
        feats.append((v.sum(1) / n[:, None]).astype(np.float32))
    torch.manual_seed(1)
    m = SpMiddleFHD(num_input_features=4).cuda().train()
    with torch.no_grad():
        return m(torch.from_numpy(np.concatenate(feats)).cuda(), torch.from_numpy(np.concatenate(coors)).cuda(), batch, [1408, 1600, 40])


def _neck_and_head():
    from det3d.models.bbox_heads.mg_head_sessd import Head
    from det3d.models.necks.rpn_v1 import SSFA
    torch.manual_seed(2)
    neck = SSFA([5], [1], [128], [1], [128], 128, logger=logging.getLogger("test")).cuda()
    neck.init_weights()
    head = Head(128, 14, 2, use_dir=True, num_dir=4).cuda()
    with torch.no_grad():
        for m in neck.modules():
            if isinstance(m, torch.nn.BatchNorm2d):
                m.weight.uniform_(0.5, 1.5)
                m.bias.uniform_(-0.2, 0.2)
    return neck, head


def _fresh(P):
    """new fp64 leaves with the values of P (weights / affine parameters requiring grad, running stats copied)"""
    return {n: {k: (v.detach().clone().requires_grad_(v.requires_grad)) for k, v in p.items()} for n, p in P.items()}


def _grads(P, H, prefix=""):
    """{tensor name: tensor} of the gradients and running stats of a parameter set (P: neck, H: head)"""
    out = {}
    for n, p in P.items():
        out.update({prefix + n + " gW": p["weight"].grad, prefix + n + " gamma": p["gamma"].grad, prefix + n + " beta": p["beta"].grad,
                    prefix + n + " mean": p["mean"], prefix + n + " var": p["var"]})
    for n, p in H.items():
        out.update({prefix + "head " + n + " gW": p["weight"].grad, prefix + "head " + n + " gb": p["bias"].grad})
    return out


def _check_conditioned(got, ref, perturbed_refs):
    """every tensor of ``got`` within max(E2E_FLOOR max |ref|, PERT_K max_s |perturbed_s - ref|) of ``ref``"""
    trace, worst = [], 0.0
    for k, g in got.items():
        r = ref[k].detach().double().cpu()
        err = float((g.detach().double().cpu() - r).abs().max())
        sens = max(float((ps[k].detach().double().cpu() - r).abs().max()) for ps in perturbed_refs)
        tol = max(E2E_FLOOR * float(r.abs().max()), PERT_K * sens, 1e-300)
        trace.append("%-28s err/max %.2e  sensitivity/max %.2e  ratio %.3g" % (k, err / max(float(r.abs().max()), 1e-300),
                                                                               sens / max(float(r.abs().max()), 1e-300), err / tol))
        worst = max(worst, err / tol)
    print("\n".join(trace))
    assert worst <= 1.0, "\n".join(trace)


def test_ssfa_and_head_train_match_fp64():
    """SSFA.train() + Head (train mode) on a ring-cloud dense() map, batch 2, with a fixed random upstream gradient: output, input
    gradient, every conv weight gradient, BN gamma / beta gradients and running stats, head weight and bias gradients against fp64
    autograd with train-mode BatchNorm2d (on the device), within the bounds of the module docstring; the no-grad forward is bitwise equal"""
    dense = _ring_dense()
    neck, head = _neck_and_head()
    P, H = ssfa_params(neck, "cuda"), head_params(head, "cuda")
    neck.train()
    head.train()
    with torch.no_grad():
        n2 = copy.deepcopy(neck)
        out_ng = head(n2(dense))["_packed"]
    x = dense.clone().requires_grad_(True)
    neck_out = neck(x)
    packed = head(neck_out)["_packed"]
    assert torch.equal(packed.detach(), out_ng), "no-grad train-mode forward differs from the grad-mode forward"
    R = torch.randn(packed.shape, generator=torch.Generator().manual_seed(5), dtype=torch.float64).cuda()
    (packed * R.float()).sum().backward()
    got = {"neck out": neck_out, "packed": packed, "dx": x.grad}
    got.update(_grads({n: dict(weight=_module_of(neck, n)[0].weight, gamma=_module_of(neck, n)[1].weight, beta=_module_of(neck, n)[1].bias,
                               mean=_module_of(neck, n)[1].running_mean, var=_module_of(neck, n)[1].running_var) for n in P},
                      {n: dict(weight=getattr(head, n).weight, bias=getattr(head, n).bias) for n in H}))

    def chain(perturb):
        p, h = _fresh(P), _fresh(H)
        xr = dense.detach().double().requires_grad_(True)
        ref_neck = ssfa_train_ref(xr, p, perturb=perturb)
        ref = head_ref(ref_neck, h, perturb=perturb)
        (ref * R).sum().backward()
        return dict({"neck out": ref_neck, "packed": ref, "dx": xr.grad}, **_grads(p, h))

    ref = chain(None)
    pert = [chain((PERT_U, torch.Generator(device="cuda").manual_seed(100 + s))) for s in range(PERT_SAMPLES)]
    _check_conditioned(got, ref, pert)


def _module_of(neck, name):
    """(conv, BatchNorm2d) of an SSFA conv module name"""
    blk, i = name.rsplit(".", 1)
    return getattr(neck, blk)[int(i)], getattr(neck, blk)[int(i) + 1]


def test_in_place_weight_change_between_forward_and_backward_raises():
    from sessd_b200 import bev_grad
    for name in ("bottom_up_block_0.4", "deconv_block_1.0"):
        L = _L[name]
        in_hw, out_hw = ssfa_extents(L, 16, 24)
        wshape = (L.cin, L.cout, 3, 3) if L.kind == "deconv" else (L.cout, L.cin, L.k, L.k)
        W = torch.randn(wshape, device="cuda").requires_grad_(True)
        x = torch.randn((1,) + in_hw + (L.cin,), device="cuda")
        y = bev_grad.BevConvFunction.apply(x, W, None, L, in_hw, out_hw)
        with torch.no_grad():
            W.mul_(2.0)
        with pytest.raises(RuntimeError):
            y.sum().backward()


# ------------------------------------------------------------------------------------------------------------------ end to end
def test_voxelnet_train_step_end_to_end():
    """build_detector from the config + a teacher copy, batch 2 with 5k-point ring clouds and seeded GT boxes: one batch_processor_inline
    step + loss.backward() gives every student parameter a finite gradient (non-zero on every conv); the encoder + neck + head gradients
    equal an fp64 chain fed with the same gradient of the packed head tensor within the bounds of the module docstring; an ArenaAdamW step and the EMA
    update follow, and a second step's loss is finite"""
    import os
    from det3d.models import build_detector
    from det3d.torchie import Config
    from det3d.torchie.trainer.trainer_sessd import batch_processor_inline
    from sessd_b200 import synth
    from sessd_b200.train import ArenaAdamW, ParamArena, update_ema_variables
    from spconv_grad_model import spmiddle_train_ref
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    cfg = Config.fromfile(os.path.join(root, "examples", "second", "configs", "config.py"))
    from sessd_b200 import weights
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    model.load_state_dict(weights.random_detector_state(4), strict=True)
    model = model.cuda()
    ema = copy.deepcopy(model)
    for p in ema.parameters():
        p.requires_grad_(False)
    model.train()
    ema.train()
    clouds = [synth.ring_cloud(60 + i, 5000) for i in range(2)]
    gts = []
    for i in range(2):
        gt = synth.random_boxes(70 + i, 10, spread=0.4)[0]
        gt[:, 2] = -1.0
        gts.append(gt)
    ex = synth.train_batch(cfg, clouds, gts)
    # fp64 copies of the student before the step, and the tensors the chain starts from / is fed with
    enc = [dict(weight=model.backbone.middle_conv[3 * i].weight.detach().cpu().double().requires_grad_(True),
                gamma=model.backbone.middle_conv[3 * i + 1].weight.detach().cpu().double().requires_grad_(True),
                beta=model.backbone.middle_conv[3 * i + 1].bias.detach().cpu().double().requires_grad_(True),
                mean=model.backbone.middle_conv[3 * i + 1].running_mean.detach().cpu().double().clone(),
                var=model.backbone.middle_conv[3 * i + 1].running_var.detach().cpu().double().clone())
           for i in range(len(model.backbone.middle_conv) // 3)]
    P, H = ssfa_params(model.neck, "cuda"), head_params(model.bbox_head.tasks[0], "cuda")
    seen = {}
    hooks = [model.backbone.register_forward_pre_hook(lambda m, a: seen.update(enc_in=a)),                 # hooks return None: nothing
             model.bbox_head.tasks[0].register_forward_hook(lambda m, a, o: seen.update(packed=o["_packed"]))]    # is replaced
    arena, arena_ema = ParamArena(model), ParamArena(ema, with_grad=False)
    opt = ArenaAdamW(arena, lr=1e-3)
    arena.zero_grad()
    out = batch_processor_inline(model, ema, ex, consistency_weight=1.0, train_mode=True)
    seen["packed"].retain_grad()
    out["loss"].backward()
    for h in hooks:
        h.remove()
    for name, p in model.named_parameters():
        assert p.grad is not None and bool(torch.isfinite(p.grad).all()), name
        if name.endswith("weight") and p.dim() >= 2:
            assert float(p.grad.abs().max()) > 0, name
    # fp64 chain: encoder (CPU restatement, once) -> neck + head (fp64 autograd on the device: 3 x 180 GFLOP per chain) fed with the
    # packed tensor's gradient; the neck + head part again with the rounding perturbation (see the module docstring)
    vf, coors, bs, shape = seen["enc_in"]
    dense = spmiddle_train_ref(vf.detach().cpu().double(), coors.cpu().numpy(), int(bs), list(shape), enc).cuda()
    G = seen["packed"].grad.double()

    def chain(perturb):
        p, h = _fresh(P), _fresh(H)
        (head_ref(ssfa_train_ref(dense, p, perturb=perturb), h, perturb=perturb) * G).sum().backward(retain_graph=True)
        out = _grads(p, h)
        for i, e in enumerate(enc):
            out.update({"encoder %d gW" % i: e["weight"].grad, "encoder %d gamma" % i: e["gamma"].grad, "encoder %d beta" % i: e["beta"].grad})
            for k in ("weight", "gamma", "beta"):
                e[k].grad = None
        return out

    ref = chain(None)
    pert = [chain((PERT_U, torch.Generator(device="cuda").manual_seed(200 + s))) for s in range(PERT_SAMPLES)]
    got = {}
    for i in range(len(enc)):
        conv, bn = model.backbone.middle_conv[3 * i], model.backbone.middle_conv[3 * i + 1]
        got.update({"encoder %d gW" % i: conv.weight.grad, "encoder %d gamma" % i: bn.weight.grad, "encoder %d beta" % i: bn.bias.grad})
    for name in P:
        conv, bn = _module_of(model.neck, name)
        got.update({name + " gW": conv.weight.grad, name + " gamma": bn.weight.grad, name + " beta": bn.bias.grad})
    for name in H:
        conv = getattr(model.bbox_head.tasks[0], name)
        got.update({"head " + name + " gW": conv.weight.grad, "head " + name + " gb": conv.bias.grad})
    _check_conditioned(got, ref, pert)
    opt.step()
    update_ema_variables(arena, arena_ema, 1)
    arena.zero_grad()
    out2 = batch_processor_inline(model, ema, ex, consistency_weight=1.0, train_mode=True)
    out2["loss"].backward()
    assert bool(torch.isfinite(out2["loss"]).all()) and bool(torch.isfinite(arena.grad_flat).all())
