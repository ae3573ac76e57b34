"""Fused supervised head loss (csrc/headloss.cu, C ABI sessd_head_loss) vs the reference's loss classes (tests/golden/head_loss_case.npz)
and the torch-CPU oracle; chained behind the device target assigner (assign -> loss without leaving the GPU).
Tolerances: fp32 transcendental functions (expf / log1pf / sinf) differ from torch-CPU's by a few ulp -> 2e-5 relative on the sums,
1e-5 relative (+1e-9 abs) on gradient entries."""
import os

import numpy as np
import pytest
import torch

from cases import assign_cases, head_loss_case

pytestmark = pytest.mark.gpu


def test_head_loss_and_gradient_match_reference_golden(golden_dir):
    from sessd_b200 import ops
    g = np.load(os.path.join(golden_dir, "head_loss_case.npz"))
    head, anc, labels, targets = head_loss_case()
    d = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()   # noqa: E731
    losses, grad = ops.head_loss(d(head), d(anc), d(labels), d(targets))
    torch.cuda.synchronize()
    L = losses.cpu().numpy()
    for j, k in enumerate(("cls", "loc", "dir")):
        np.testing.assert_allclose(L[:, j], g[k], rtol=2e-5)
    np.testing.assert_allclose(L[:, 3].sum() / 2, float(g["cls_pos"]), rtol=2e-5)
    np.testing.assert_allclose(L[:, 4].sum() / 2, float(g["cls_neg"]), rtol=2e-5)
    assert np.array_equal(L[:, 6], (labels > 0).sum(1).astype(np.float32)) and np.array_equal(L[:, 7], (labels == 0).sum(1).astype(np.float32))
    total = (L[:, 0].sum() + 2.0 * L[:, 1].sum() + 0.2 * L[:, 2].sum()) / 2
    np.testing.assert_allclose(total, float(g["total"]), rtol=2e-5)
    G = grad.cpu().numpy().reshape(-1, 24)
    np.testing.assert_allclose(G[g["grad_pix_idx"]], g["grad_pix"], rtol=1e-5, atol=1e-9)
    np.testing.assert_allclose(np.abs(G).sum(), float(g["grad_abs_sum"]), rtol=2e-5)
    assert not G[:, 20:].any()                                   # iou head and padding: no supervised gradient
    # deterministic: two runs are bitwise equal
    losses2, grad2 = ops.head_loss(d(head), d(anc), d(labels), d(targets))
    torch.cuda.synchronize()
    assert torch.equal(losses, losses2) and torch.equal(grad, grad2)


def test_assign_then_loss_on_device_matches_oracle():
    """GT boxes -> sessd_assign_targets -> sessd_head_loss, batch 3 incl. a frame without GT, against the torch oracle with autograd."""
    from oracle import anchors as oa, loss_ref
    from sessd_b200 import ops
    anc = oa.create_anchors_3d_range().reshape(-1, 7)
    cases = dict(assign_cases())
    gts = [cases["m12"], cases["m0"], cases["edge"]]
    B, A, M = 3, anc.shape[0], 16
    gt = np.zeros((B, M, 7), np.float32)
    num = np.zeros((B,), np.int32)
    for b, x in enumerate(gts):
        gt[b, :len(x)] = x
        num[b] = len(x)
    buf = ops.AssignBuffers(A, B, M, "cuda")
    d_anc = torch.from_numpy(anc).cuda()
    ops.assign_targets(d_anc, torch.from_numpy(gt).cuda(), torch.from_numpy(num).cuda(), buf)
    gen = torch.Generator().manual_seed(7)
    head = torch.randn(B, A // 2, 24, generator=gen) * 0.7
    losses, grad = ops.head_loss(head.cuda(), d_anc, buf.labels, buf.bbox_targets, w_loc=0.0)       # the reference's total omits loc
    torch.cuda.synchronize()
    h = head.clone().requires_grad_(True)
    o = loss_ref.head_supervised_loss(*loss_ref.split_head(h), torch.from_numpy(anc), buf.labels.cpu().long(), buf.bbox_targets.cpu())
    ((o["cls"].sum() + 0.2 * o["dir"].sum()) / B).backward()
    L = losses.cpu().numpy()
    for j, k in enumerate(("cls", "loc", "dir")):
        np.testing.assert_allclose(L[:, j], o[k].detach().numpy(), rtol=2e-5, atol=1e-7)
    assert L[1, 1] == 0.0 and L[1, 2] == 0.0 and L[1, 6] == 0.0          # the empty frame has no positives
    np.testing.assert_allclose(grad.cpu().numpy(), h.grad.numpy(), rtol=1e-5, atol=1e-9)


def test_multigrouphead_loss_supervised_from_config():
    """Config-built detector: forward -> head dict -> loss_supervised with targets from TargetAssigner.assign_batch_gpu; values equal the
    oracle with the config's loss weights (cls 1.0, loc 2.0, dir 0.2), gradient has the head tensor's shape."""
    import os as _os
    from det3d.datasets.pipelines import AssignTarget
    from det3d.models import build_detector
    from det3d.torchie import Config
    from oracle import loss_ref
    from sessd_b200 import weights
    root = _os.path.dirname(_os.path.dirname(_os.path.abspath(__file__)))
    cfg = Config.fromfile(_os.path.join(root, "examples", "second", "configs", "config.py"))
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    model.load_state_dict(weights.random_detector_state(4), strict=True)
    model = model.cuda().eval()
    at = AssignTarget(cfg=cfg.train_cfg.assigner)
    ta, ad = at.target_assigners[0], at.anchor_dicts_by_task[0]
    gts = [g for n, g in assign_cases() if n in ("m12", "m40")]
    tg = ta.assign_batch_gpu(ad, gts)
    x = torch.relu(torch.randn(2, 128, 200, 176, device="cuda"))
    preds = model.bbox_head(x)
    anchors = torch.from_numpy(ad["Car"]["anchors"].reshape(1, -1, 7)).cuda().expand(2, -1, -1)
    example = dict(anchors=[anchors], labels=[tg["labels"]], reg_targets=[tg["bbox_targets"]])
    out = model.bbox_head.loss_supervised(example, preds)
    torch.cuda.synchronize()
    packed = preds[0]["_packed"].detach().cpu().reshape(2, -1, preds[0]["_packed"].shape[-1])
    o = loss_ref.head_supervised_loss(*loss_ref.split_head(packed), anchors[0].cpu(), tg["labels"].cpu().long(), tg["bbox_targets"].cpu())
    np.testing.assert_allclose(float(out["cls_loss_reduced"]), float(o["cls"].sum() / 2), rtol=2e-5)
    np.testing.assert_allclose(float(out["loc_loss_reduced"]), float(2.0 * o["loc"].sum() / 2), rtol=2e-5)
    np.testing.assert_allclose(float(out["dir_loss_reduced"]), float(0.2 * o["dir"].sum() / 2), rtol=2e-5)
    assert out["grad_head"].shape == preds[0]["_packed"].shape and bool(torch.isfinite(out["grad_head"]).all())

