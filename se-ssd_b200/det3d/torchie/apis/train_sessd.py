"""The optimiser and learning-rate schedule the SE-SSD training run builds (reference: det3d/torchie/apis/train_sessd.py:169-175,275-283
and det3d/builder.py:191-220), on the flat parameter arena: one fused clip / AdamW / EMA pass per step (sessd_b200.train).  The
``train_detector`` / ``Trainer`` loop itself is not mirrored."""
from sessd_b200.train import ArenaAdamW, ParamArena

from ...solver import learning_schedules_fastai as lsf


def build_one_cycle_optimizer(model, optimizer_config):
    """The reference's fastai ``OptimWrapper(Adam, betas=(0.9, 0.99), wd=cfg.wd, true_wd=True, bn_wd=True)`` at lr 3e-3, over ``model``'s
    parameters re-homed into a ParamArena.  Returns (arena, optimizer); the one-cycle schedule then sets lr and mom every step."""
    if optimizer_config.get("amsgrad", False):
        raise NotImplementedError("amsgrad is not implemented (the SE-SSD config trains with amsgrad=0)")
    if not optimizer_config.get("fixed_wd", False):
        raise NotImplementedError("only the decoupled weight decay of fixed_wd=True (the SE-SSD config) is implemented")
    arena = ParamArena(model)
    return arena, ArenaAdamW(arena, lr=3e-3, betas=(0.9, 0.99), weight_decay=optimizer_config["wd"])


def _create_learning_rate_scheduler(optimizer, lr_config, total_steps):
    """``lr_config`` of type ``one_cycle`` (examples/second/configs/config.py:259)  ->  OneCycle over ``total_steps`` =
    total_epochs * len(loader)."""
    if lr_config["type"] != "one_cycle":
        raise NotImplementedError("learning-rate schedule %r: only one_cycle is implemented" % (lr_config["type"],))
    return lsf.OneCycle(optimizer, total_steps, lr_config["lr_max"], list(lr_config["moms"]), lr_config["div_factor"], lr_config["pct_start"])
