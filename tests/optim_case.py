"""The small model and gradient sequence of tests/golden/optim_recipe.npz (tests/golden/make_optim_golden.py): BatchNorm layers between
plain ones, so the reference optimiser's BatchNorm group and parameter order differ from ``model.parameters()``, and gradients scaled so
that some steps exceed the clip threshold of 35 and some do not."""
import torch
from torch import nn

STEPS = 20
CKPT_STEP = 10            # the reference checkpoint in the fixture is written after this many steps
MAX_NORM = 35.0
LR_MAX, MOMS, DIV_FACTOR, PCT_START, WD = 0.003, [0.95, 0.85], 10.0, 0.4, 0.01
# the reference config's optimiser entries (examples/second/configs/config.py:257-260 of the reference)
OPTIMIZER = dict(type="adam", amsgrad=0.0, wd=WD, fixed_wd=True, moving_average=False)
LR_CONFIG = dict(type="one_cycle", lr_max=LR_MAX, moms=MOMS, div_factor=DIV_FACTOR, pct_start=PCT_START)
SCHEDULE_TOTALS = (10, 101, 37080)


def optim_model(seed=3):
    torch.manual_seed(seed)
    return nn.Sequential(nn.Conv2d(3, 8, 3), nn.BatchNorm2d(8), nn.ReLU(),
                         nn.Sequential(nn.Conv1d(8, 6, 1), nn.BatchNorm1d(6)), nn.Linear(6, 5), nn.BatchNorm1d(5), nn.Linear(5, 4))


def gradient_scales():
    """per-step factor on a unit-variance gradient; the model's ~500 parameters give norms of roughly 22 * scale"""
    return [0.5, 4.0, 1.0, 3.0, 0.2, 2.5, 1.2, 6.0, 0.8, 1.5, 5.0, 0.3, 2.0, 1.0, 8.0, 0.6, 1.7, 3.5, 0.9, 4.5]


def step_gradients(model, step, seed=11):
    """the seeded gradient of every parameter (model.parameters() order) at ``step``"""
    g = torch.Generator().manual_seed(seed * 1000 + step)
    s = gradient_scales()[step]
    return [s * torch.randn(p.shape, generator=g) for p in model.parameters()]


def torch_recipe_step(params, teacher, adam, lr, mom, global_step, max_norm=MAX_NORM, wd=WD):
    """One step of the reference recipe restated in plain torch (the chain the GPU tests compare ArenaAdamW against, itself pinned to
    the fixture): clip_grad_norm_ -> p *= 1 - wd * lr (true_wd, bn_wd) -> torch.optim.Adam(betas=(mom, 0.99), weight_decay=0) -> teacher
    EMA with alpha = min(1 - 1 / (global_step + 1), 0.999).  ``adam`` is a torch.optim.Adam over ``params``.  Returns the total norm."""
    norm = torch.nn.utils.clip_grad_norm_(params, max_norm=max_norm, norm_type=2)
    for g in adam.param_groups:
        g["lr"], g["betas"] = lr, (mom, g["betas"][1])
    with torch.no_grad():
        for p in params:
            p.mul_(1 - wd * lr)
    adam.step()
    alpha = min(1 - 1 / (global_step + 1), 0.999)
    with torch.no_grad():
        for e, p in zip(teacher, params):
            e.mul_(alpha).add_(p, alpha=1 - alpha)
    return norm


def reference_checkpoint(gold):
    """The checkpoint the reference's save_checkpoint(model, f, optimizer=OptimWrapper) wrote after CKPT_STEP steps, as torch.load returns
    it, rebuilt from the ``ckpt_*`` arrays of tests/golden/optim_recipe.npz: {"meta", "state_dict", "optimizer": torch Adam's state_dict
    with an int ``step`` per parameter}."""
    import json
    from collections import OrderedDict
    groups = json.loads(str(gold["ckpt_param_groups"]))
    for g in groups:
        g["betas"] = tuple(g["betas"])
    state = {}
    for i in (i for g in groups for i in g["params"]):
        if "ckpt_step_%d" % i in gold.files:
            state[i] = {"step": int(gold["ckpt_step_%d" % i]), "exp_avg": torch.from_numpy(gold["ckpt_exp_avg_%d" % i]),
                        "exp_avg_sq": torch.from_numpy(gold["ckpt_exp_avg_sq_%d" % i])}
    sd = OrderedDict((k, torch.from_numpy(gold["ckpt_state_dict_%d" % j])) for j, k in enumerate(gold["ckpt_state_dict_keys"].tolist()))
    return {"meta": json.loads(str(gold["ckpt_meta"])), "state_dict": sd, "optimizer": {"state": state, "param_groups": groups}}
