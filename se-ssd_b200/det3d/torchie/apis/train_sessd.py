"""The SE-SSD training run (reference: det3d/torchie/apis/train_sessd.py:169-175,253-323 and det3d/builder.py:191-220):
``train_detector`` builds the device loaders, the optimiser and learning-rate schedule on the flat parameter arena (one fused clip /
AdamW / EMA pass per step, sessd_b200.train), the teacher and the Trainer, and runs it."""
import copy
import logging

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


def build_loaders(dataset, cfg, twin=True):
    """the device loaders of ``dataset`` = [train, (unlabelled,) val] without the unlabelled one: ``cfg.data.samples_per_gpu`` frames per
    batch, random streams from ``cfg.seed`` (0 when unset); ``twin`` as kitti_loader.DeviceLoader takes it"""
    from det3d.datasets import build_dataloader
    datasets = list(dataset) if isinstance(dataset, (list, tuple)) else [dataset]
    if len(datasets) == 3:
        datasets = [datasets[0], datasets[2]]
    seed = cfg.get("seed") or 0
    return [build_dataloader(ds, cfg.data.samples_per_gpu, cfg.data.workers_per_gpu, dist=False, cfg=cfg, seed=seed, twin=twin)
            for ds in datasets]


def train_detector(model, dataset, cfg, distributed=False, validate=False, logger=None):
    """Train ``model`` on ``dataset`` = [train, (unlabelled,) val] as the reference's train_detector does, single-GPU, and return the
    final validation's results dict (None without a val phase).

    The teacher is a deep copy of the student whose parameters live in a ParamArena without gradients.  Every loader batches
    ``cfg.data.samples_per_gpu`` frames and draws from ``cfg.seed`` (0 when unset).  With ``my_paras.enable_ssl`` the reference also
    builds an unlabelled dataset but never draws from it (its merge is commented out, trainer_sessd.py:334-339): it is accepted and not
    iterated here."""
    from ..trainer.trainer_sessd import Trainer, batch_processor_inline
    if distributed:
        raise NotImplementedError("distributed training is not implemented")
    loaders = build_loaders(dataset, cfg)
    model = model.cuda()
    model_ema = copy.deepcopy(model)
    for p in model_ema.parameters():
        p.requires_grad_(False)
    model_ema._arena = ParamArena(model_ema, with_grad=False)
    if cfg.lr_config.type not in ("one_cycle",):
        raise NotImplementedError("learning-rate schedule %r: only one_cycle is implemented" % (cfg.lr_config.type,))
    _, optimizer = build_one_cycle_optimizer(model, cfg.optimizer)
    lr_scheduler = _create_learning_rate_scheduler(optimizer, cfg.lr_config, cfg.total_epochs * len(loaders[0]))
    trainer = Trainer(model, model_ema, batch_processor_inline, optimizer, lr_scheduler, cfg.work_dir,
                      getattr(logging, str(cfg.get("log_level", "INFO"))), logger)
    trainer.register_training_hooks(None, cfg.optimizer_config, cfg.checkpoint_config, cfg.log_config)
    if cfg.get("resume_from"):
        trainer.resume(cfg.resume_from)
    elif cfg.get("load_from") and cfg.my_paras.get("enable_ssl", False):
        trainer.load_checkpoint_from_scratch(cfg.load_from)
    return trainer.run(loaders, cfg.workflow, cfg.total_epochs)
