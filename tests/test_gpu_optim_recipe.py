"""The reference's optimiser recipe on the device: the deterministic gradient norm (sessd_grad_sqnorm) and the AdamW step with the clip
and the teacher EMA fused in (sessd_adamw_clip_ema_step), over the SE-SSD student arena (~3.8 M parameters), against the torch chain
of optim_case.torch_recipe_step (pinned to the reference's own trajectory by tests/test_optim_recipe.py), without a host
synchronisation, resumable from a checkpoint bit for bit, and continuing the reference-written checkpoint of the fixture."""
import copy
import os

import numpy as np
import pytest
import torch

import optim_case as OC

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _voxelnet(seed=0):
    from det3d.models import build_detector
    from det3d.torchie import Config
    cfg = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    torch.manual_seed(seed)
    return build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg).cuda()


def _student_teacher(seed=0):
    from sessd_b200.train import ParamArena
    stu = _voxelnet(seed)
    tea = copy.deepcopy(stu)
    with torch.no_grad():
        for p in tea.parameters():
            p.add_(0.01)
    return stu, tea, ParamArena(stu), ParamArena(tea, with_grad=False)


def _seeded_grads(arena, step, scale):
    """unit-normal gradients times ``scale`` on every parameter view (the padding between views stays zero)"""
    g = torch.Generator(device="cuda").manual_seed(1000 + step)
    for p, off in zip(arena.params, arena.offsets):
        arena.grad_flat[off:off + p.numel()].copy_(torch.randn(p.numel(), device="cuda", generator=g) * scale)


SCALES = [0.004, 0.05, 0.01, 0.03, 0.002, 0.1]       # the arena's ~1950 * scale: below 35, above, ...


def test_grad_norm_is_the_fp64_norm_and_deterministic():
    from sessd_b200.train import grad_norm
    _stu, _tea, arena, _ = _student_teacher()
    for step, scale in enumerate((0.004, 0.05)):
        _seeded_grads(arena, step, scale)
        out1 = grad_norm(arena.grad_flat, OC.MAX_NORM)
        out2 = grad_norm(arena.grad_flat, OC.MAX_NORM)
        assert torch.equal(out1, out2)
        total = float(out1[0])
        ref64 = float(torch.linalg.vector_norm(arena.grad_flat.double()))
        assert abs(total - ref64) <= np.spacing(np.float32(ref64))
        twin = [p.grad.detach().clone().requires_grad_(False) for p in arena.params]
        holders = [torch.nn.Parameter(torch.zeros_like(t)) for t in twin]
        for h, t in zip(holders, twin):
            h.grad = t
        ref = float(torch.nn.utils.clip_grad_norm_(holders, OC.MAX_NORM))
        assert total == pytest.approx(ref, rel=1e-6)
        coef = torch.clamp((torch.tensor(total, device="cuda") + 1e-6).reciprocal() * OC.MAX_NORM, max=1.0)   # clip_grad_norm_'s arithmetic
        assert float(out1[1]) == float(coef)
        assert (float(out1[1]) < 1.0) == (total > OC.MAX_NORM)


def test_no_clip_no_ema_call_equals_the_old_entry_and_fused_ema_equals_axpby():
    from sessd_b200.train import ArenaAdamW, update_ema_variables
    _s1, _t1, a1, e1 = _student_teacher()
    _s2, _t2, a2, e2 = _student_teacher()
    o1, o2 = ArenaAdamW(a1, lr=1e-3, betas=(0.93, 0.99)), ArenaAdamW(a2, lr=1e-3, betas=(0.93, 0.99))
    for step in range(3):
        _seeded_grads(a1, step, 0.004)
        _seeded_grads(a2, step, 0.004)
        g_before = a2.grad_flat.clone()
        o1.step()                                                    # sessd_adamw_step
        update_ema_variables(a1, e1, step)                           # sessd_axpby
        norm = o2.step(max_grad_norm=OC.MAX_NORM, ema=e2, global_step=step)
        assert float(norm) < OC.MAX_NORM
        for x, y in ((a1.flat, a2.flat), (o1.exp_avg, o2.exp_avg), (o1.exp_avg_sq, o2.exp_avg_sq), (e1.flat, e2.flat), (g_before, a2.grad_flat)):
            assert torch.equal(x, y)


def _run_recipe(stu_arena, tea_arena, opt, sched, steps, scales):
    for i in steps:
        sched.step(i)
        _seeded_grads(stu_arena, i, scales[i % len(scales)])
        opt.step(max_grad_norm=OC.MAX_NORM, ema=tea_arena, global_step=i)


def test_thirty_one_cycle_steps_match_the_torch_chain():
    from det3d.solver import OneCycle
    from sessd_b200.train import ArenaAdamW
    stu, tea, arena, arena_t = _student_teacher()
    params = [p.detach().clone().requires_grad_(True) for p in stu.parameters()]
    teacher = [p.detach().clone() for p in tea.parameters()]
    adam = torch.optim.Adam(params, lr=0.0, betas=(0.9, 0.99), weight_decay=0)
    opt = ArenaAdamW(arena, weight_decay=OC.WD)
    sched = OneCycle(opt, 30, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START)
    clipped = 0
    for i in range(30):
        sched.step(i)
        _seeded_grads(arena, i, SCALES[i % len(SCALES)])
        for q, p in zip(params, arena.params):
            q.grad = p.grad.detach().clone()
        want = OC.torch_recipe_step(params, teacher, adam, opt.lr, opt.mom, i)
        got = opt.step(max_grad_norm=OC.MAX_NORM, ema=arena_t, global_step=i)
        assert float(got) == pytest.approx(float(want), rel=1e-6)
        clipped += float(want) > OC.MAX_NORM
        for k, (q, p, e, t) in enumerate(zip(params, arena.params, teacher, arena_t.params)):
            off, n = arena.offsets[k], p.numel()
            for name, x, y in (("param", p, q), ("grad", p.grad, q.grad), ("teacher", t, e),
                               ("exp_avg", opt.exp_avg[off:off + n].view_as(p), adam.state[q]["exp_avg"]),
                               ("exp_avg_sq", opt.exp_avg_sq[off:off + n].view_as(p), adam.state[q]["exp_avg_sq"])):
                assert torch.allclose(x, y, rtol=2e-5, atol=1e-7), (name, i, k, float((x - y).abs().max()))
    assert 0 < clipped < 30


def test_clipped_ema_step_never_synchronises_and_replays_from_a_cuda_graph():
    from sessd_b200.train import ArenaAdamW
    _s1, _t1, a1, e1 = _student_teacher()
    _s2, _t2, a2, e2 = _student_teacher()
    o1, o2 = ArenaAdamW(a1, lr=2e-3, betas=(0.9, 0.99)), ArenaAdamW(a2, lr=2e-3, betas=(0.9, 0.99))
    for a in (a1, a2):
        _seeded_grads(a, 0, 0.05)
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        norm = o1.step(max_grad_norm=OC.MAX_NORM, ema=e1, global_step=7)
    finally:
        torch.cuda.set_sync_debug_mode("default")
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        norm2 = o2.step(max_grad_norm=OC.MAX_NORM, ema=e2, global_step=7)
    g.replay()
    torch.cuda.synchronize()
    assert float(norm) > OC.MAX_NORM and torch.equal(norm, norm2)
    for x, y in ((a1.flat, a2.flat), (a1.grad_flat, a2.grad_flat), (o1.exp_avg, o2.exp_avg), (o1.exp_avg_sq, o2.exp_avg_sq), (e1.flat, e2.flat)):
        assert torch.equal(x, y)


def test_resume_from_a_checkpoint_is_bit_identical(tmp_path):
    from det3d.solver import OneCycle
    from det3d.torchie.trainer import load_checkpoint, save_checkpoint
    from sessd_b200.train import ArenaAdamW, ParamArena
    stu, tea, arena, arena_t = _student_teacher()
    opt = ArenaAdamW(arena, weight_decay=OC.WD)
    _run_recipe(arena, arena_t, opt, OneCycle(opt, 20, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START), range(20), SCALES)

    stu1, tea1, arena1, arena1_t = _student_teacher()
    opt1 = ArenaAdamW(arena1, weight_decay=OC.WD)
    _run_recipe(arena1, arena1_t, opt1, OneCycle(opt1, 20, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START), range(10), SCALES)
    f, f_ema = str(tmp_path / "epoch_1.pth"), str(tmp_path / "epoch_1_ema.pth")
    save_checkpoint(stu1, f, optimizer=opt1, meta={"iter": 10})
    save_checkpoint(tea1, f_ema)
    torch.cuda.synchronize()

    stu2, tea2 = _voxelnet(seed=5), _voxelnet(seed=6)
    ck = load_checkpoint(stu2, f, map_location="cpu", strict=True)
    load_checkpoint(tea2, f_ema, map_location="cpu", strict=True)
    arena2, arena2_t = ParamArena(stu2), ParamArena(tea2, with_grad=False)
    opt2 = ArenaAdamW(arena2, weight_decay=OC.WD)
    opt2.load_state_dict(ck["optimizer"])
    assert opt2.steps == 10 and ck["meta"]["iter"] == 10
    _run_recipe(arena2, arena2_t, opt2, OneCycle(opt2, 20, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START), range(10, 20), SCALES)
    for x, y in ((arena.flat, arena2.flat), (opt.exp_avg, opt2.exp_avg), (opt.exp_avg_sq, opt2.exp_avg_sq), (arena_t.flat, arena2_t.flat),
                 (arena.grad_flat, arena2.grad_flat)):
        assert torch.equal(x, y)


def test_reference_checkpoint_continues_the_reference_trajectory(golden_dir):
    """The fixture's reference-written checkpoint (after 10 one-cycle steps), loaded and stepped 10 more times on the device with the
    fixture's gradients, follows the reference's recorded trajectory; the OptimizerHook takes the same fused path."""
    from det3d.solver import OneCycle
    from det3d.torchie.trainer import load_state_dict
    from det3d.torchie.trainer.hooks import OptimizerHook
    from sessd_b200.train import ArenaAdamW, ParamArena
    gold = np.load(os.path.join(golden_dir, "optim_recipe.npz"))
    model = OC.optim_model(seed=42).cuda()
    ck = OC.reference_checkpoint(gold)
    assert load_state_dict(model, ck["state_dict"], strict=True) == []
    teacher = OC.optim_model(seed=43).cuda()
    arena, arena_t = ParamArena(model), ParamArena(teacher, with_grad=False)
    sizes = [p.numel() for p in arena.params]
    starts = np.cumsum([0] + sizes)
    k0 = OC.CKPT_STEP - 1
    for j, (off, n) in enumerate(zip(arena.offsets, sizes)):
        arena_t.flat[off:off + n].copy_(torch.from_numpy(gold["traj_teacher"][k0][starts[j]:starts[j + 1]]))
    opt = ArenaAdamW(arena, weight_decay=OC.WD)
    opt.load_state_dict(ck["optimizer"])
    sched = OneCycle(opt, OC.STEPS, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START)

    class Runner:
        pass
    hook, runner = OptimizerHook(grad_clip=dict(max_norm=OC.MAX_NORM, norm_type=2)), Runner()
    runner.model, runner.optimizer = model, opt
    for i in range(OC.CKPT_STEP, OC.STEPS):
        sched.step(i)
        if i % 2:
            for j, (off, n) in enumerate(zip(arena.offsets, sizes)):
                arena.grad_flat[off:off + n].copy_(torch.from_numpy(gold["traj_grad_in"][i][starts[j]:starts[j + 1]]))
            opt.step(max_grad_norm=OC.MAX_NORM, ema=arena_t, global_step=i)
        else:                                                            # the hook: backward of a loss whose gradient is the fixture's
            w = [torch.from_numpy(gold["traj_grad_in"][i][starts[j]:starts[j + 1]]).cuda().view_as(p) for j, p in enumerate(arena.params)]
            runner.outputs = dict(loss=sum((p * g).sum() for p, g in zip(arena.params, w)))
            hook.after_train_iter(runner)
            from sessd_b200.train import update_ema_variables
            update_ema_variables(arena, arena_t, i)
        for key, buf in (("param", arena.flat), ("grad", arena.grad_flat), ("exp_avg", opt.exp_avg), ("exp_avg_sq", opt.exp_avg_sq),
                         ("teacher", arena_t.flat)):
            got = torch.cat([buf[off:off + n] for off, n in zip(arena.offsets, sizes)]).cpu().numpy()
            np.testing.assert_allclose(got, gold["traj_" + key][i], rtol=2e-5, atol=1e-7, err_msg="%s, step %d" % (key, i))
