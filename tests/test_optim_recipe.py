"""The reference's optimiser recipe on the host side (CPU): the one-cycle schedule mirror, the torch restatement the GPU tests compare
against, the reference optimiser's parameter order, and torch-Adam-format optimiser state -- all pinned to tests/golden/optim_recipe.npz,
written by the reference's own code (tests/golden/make_optim_golden.py)."""
import os

import numpy as np
import pytest
import torch

import optim_case as OC

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Stub:
    lr, mom = 0.0, 0.0


@pytest.fixture(scope="module")
def gold(golden_dir):
    return np.load(os.path.join(golden_dir, "optim_recipe.npz"))


def _voxelnet():
    from det3d.models import build_detector
    from det3d.torchie import Config
    cfg = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    return cfg, build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)


@pytest.mark.parametrize("total", OC.SCHEDULE_TOTALS)
def test_one_cycle_equals_the_reference_schedule(gold, total):
    from det3d.solver import OneCycle
    s = _Stub()
    sched = OneCycle(s, total, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START)
    assert [s.lr, s.mom] == gold["sched%d_init" % total].tolist()
    lrs, moms = [], []
    for i in range(total):
        sched.step(i)
        lrs.append(s.lr)
        moms.append(s.mom)
    assert np.array_equal(np.array(lrs), gold["sched%d_lr" % total])
    assert np.array_equal(np.array(moms), gold["sched%d_mom" % total])


def test_torch_restatement_reproduces_the_reference_trajectory(gold):
    from det3d.solver import OneCycle
    model = OC.optim_model()
    params = list(model.parameters())
    teacher = [p.detach().clone() for p in params]
    adam = torch.optim.Adam(params, lr=0.0, betas=(0.9, 0.99), weight_decay=0, foreach=False)
    s = _Stub()
    sched = OneCycle(s, OC.STEPS, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START)
    flat = lambda ts: torch.cat([t.detach().reshape(-1) for t in ts]).numpy()          # noqa: E731
    for i in range(OC.STEPS):
        sched.step(i)
        for p, g in zip(params, OC.step_gradients(model, i)):
            p.grad = g
        assert np.array_equal(flat([p.grad for p in params]), gold["traj_grad_in"][i])
        norm = OC.torch_recipe_step(params, teacher, adam, s.lr, s.mom, i)
        assert (s.lr, s.mom) == (gold["traj_lr"][i], gold["traj_mom"][i])
        assert float(norm) == pytest.approx(gold["traj_norm"][i], rel=1e-6)
        for key, got in (("grad", [p.grad for p in params]), ("param", params), ("teacher", teacher),
                         ("exp_avg", [adam.state[p]["exp_avg"] for p in params]), ("exp_avg_sq", [adam.state[p]["exp_avg_sq"] for p in params])):
            np.testing.assert_allclose(flat(got), gold["traj_" + key][i], rtol=1e-6, atol=1e-9, err_msg="%s, step %d" % (key, i))
    assert 0 < int((gold["traj_norm"] > OC.MAX_NORM).sum()) < OC.STEPS           # the trajectory both clips and does not


def test_param_arena_records_the_reference_optimizer_order(gold):
    from sessd_b200.train import ParamArena
    _cfg, net = _voxelnet()
    names = [n for n, _ in net.named_parameters()]
    arena = ParamArena(net, with_grad=False)
    order = [names[i] for g in arena.optim_groups for i in g]
    assert order == gold["voxelnet_order"].tolist()
    assert sorted(order) == sorted(names)                                     # every parameter, once
    toy = OC.optim_model()
    toy_names = [n for n, _ in toy.named_parameters()]
    toy_arena = ParamArena(toy)
    assert [toy_names[i] for g in toy_arena.optim_groups for i in g] == gold["toy_order"].tolist()
    assert [len(g) for g in toy_arena.optim_groups] == [8, 6]                 # four conv / linear layers, then three BatchNorms


def test_reference_checkpoint_optimizer_state_loads_into_the_arena_layout(gold, tmp_path):
    from det3d.torchie.trainer import load_checkpoint, load_state_dict, save_checkpoint
    from sessd_b200.train import ArenaAdamW, ParamArena
    ck = OC.reference_checkpoint(gold)
    ref_sd = ck["optimizer"]
    assert ck["meta"]["iter"] == OC.CKPT_STEP and all(type(s["step"]) is int for s in ref_sd["state"].values())
    model = OC.optim_model(seed=99)
    assert load_state_dict(model, ck["state_dict"], strict=True) == []
    arena = ParamArena(model)
    opt = ArenaAdamW(arena, weight_decay=OC.WD)
    opt.load_state_dict(ck["optimizer"])
    k = OC.CKPT_STEP - 1
    assert opt.steps == OC.CKPT_STEP and isinstance(opt.steps, int)
    assert (opt.lr, opt.mom, opt.betas[1]) == (gold["traj_lr"][k], gold["traj_mom"][k], 0.99) and opt.weight_decay == OC.WD
    # parameter j of model.parameters() sits at arena.offsets[j]: the fixture's moments (in that order) land there
    sizes = [p.numel() for p in arena.params]
    starts = np.cumsum([0] + sizes)
    for j, (off, n) in enumerate(zip(arena.offsets, sizes)):
        for key, buf in (("exp_avg", opt.exp_avg), ("exp_avg_sq", opt.exp_avg_sq), ("param", arena.flat)):
            np.testing.assert_array_equal(buf[off:off + n].numpy(), gold["traj_" + key][k][starts[j]:starts[j + 1]])
    # state_dict() writes the same torch-Adam layout back, and save_checkpoint / load_checkpoint carry it
    mine = opt.state_dict()
    assert [g["params"] for g in mine["param_groups"]] == [g["params"] for g in ref_sd["param_groups"]]
    for g in mine["param_groups"]:
        assert (g["weight_decay"], g["amsgrad"], g["eps"]) == (0, False, 1e-8)
    for i, s in ref_sd["state"].items():
        assert int(mine["state"][i]["step"]) == s["step"]
        assert torch.equal(mine["state"][i]["exp_avg"], s["exp_avg"]) and torch.equal(mine["state"][i]["exp_avg_sq"], s["exp_avg_sq"])
    f = str(tmp_path / "ours.pth")
    save_checkpoint(model, f, optimizer=opt, meta={"iter": OC.CKPT_STEP})
    fresh = ArenaAdamW(ParamArena(OC.optim_model(seed=5)))
    fresh.load_state_dict(load_checkpoint(OC.optim_model(seed=6), f, map_location="cpu")["optimizer"])
    assert fresh.steps == OC.CKPT_STEP and torch.equal(fresh.exp_avg, opt.exp_avg) and torch.equal(fresh.exp_avg_sq, opt.exp_avg_sq)


def test_optimizer_state_is_checked_against_the_model(gold):
    from sessd_b200.train import ArenaAdamW, ParamArena
    opt = ArenaAdamW(ParamArena(OC.optim_model()))
    assert opt.state_dict()["state"] == {}                                    # torch keeps no state before the first step
    sd = OC.reference_checkpoint(gold)["optimizer"]
    bad = dict(sd, param_groups=[sd["param_groups"][0], dict(sd["param_groups"][1], params=sd["param_groups"][1]["params"][:-1])])
    with pytest.raises(ValueError):
        opt.load_state_dict(bad)
    uneven = dict(sd, state={i: dict(s, step=s["step"] + (i == 0)) for i, s in sd["state"].items()})
    with pytest.raises(ValueError):
        opt.load_state_dict(uneven)
    with pytest.raises(NotImplementedError):
        ArenaAdamW(ParamArena(OC.optim_model()), amsgrad=True)
    opt.mom = 0.91
    assert opt.betas == (0.91, 0.99) and opt.mom == 0.91


def test_build_one_cycle_optimizer_and_scheduler_from_the_config(gold):
    from det3d.torchie.apis import _create_learning_rate_scheduler, build_one_cycle_optimizer
    _cfg, net = _voxelnet()
    arena, opt = build_one_cycle_optimizer(net, OC.OPTIMIZER)
    assert arena.numel >= sum(p.numel() for p in net.parameters()) and opt.arena is arena
    assert (opt.weight_decay, opt.betas[1], opt.eps) == (0.01, 0.99, 1e-8)
    total = OC.SCHEDULE_TOTALS[-1]
    sched = _create_learning_rate_scheduler(opt, OC.LR_CONFIG, total)
    assert [opt.lr, opt.mom] == gold["sched%d_init" % total].tolist()
    for i in (0, 1, int(0.4 * total) - 1, int(0.4 * total), total - 1):
        sched.step(i)
        assert (opt.lr, opt.mom) == (gold["sched%d_lr" % total][i], gold["sched%d_mom" % total][i])


def test_optimizer_hooks_keep_torch_clipping_for_other_optimizers():
    """OptimizerHook (reference hooks/optimizer.py:35-62) and DistOptimizerHook clip with torch's clip_grad_norm_ when the optimiser is
    not an ArenaAdamW over the model's arena (here: torch SGD on the CPU)."""
    from det3d.torchie.trainer.hooks import OptimizerHook
    model, twin = OC.optim_model(), OC.optim_model()
    x = torch.randn(7, 6)

    class Runner:
        pass
    r = Runner()
    r.model, r.optimizer = model, torch.optim.SGD(model.parameters(), lr=0.1)
    r.outputs = dict(loss=(model[4](x) * 40.0).square().sum())
    OptimizerHook(grad_clip=dict(max_norm=OC.MAX_NORM, norm_type=2)).after_train_iter(r)
    sgd = torch.optim.SGD(twin.parameters(), lr=0.1)
    (twin[4](x) * 40.0).square().sum().backward()
    assert float(torch.nn.utils.clip_grad_norm_(twin.parameters(), OC.MAX_NORM)) > OC.MAX_NORM
    sgd.step()
    for p, q in zip(model.parameters(), twin.parameters()):
        assert torch.equal(p, q)
