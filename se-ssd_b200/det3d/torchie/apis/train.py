"""The single-model training run (reference: det3d/torchie/apis/train.py:140-158, 253-300): CIA-SSD pre-training, the supervised stage
whose checkpoint SE-SSD's ``load_from`` starts both its teacher and its student from.  ``train_detector`` builds the device loaders
(student-only batches), the one-cycle AdamW on the flat parameter arena and the single-model Trainer, and runs it."""
import logging

from .train_sessd import _create_learning_rate_scheduler, build_loaders, build_one_cycle_optimizer


def batch_processor(model, data, train_mode, device=None, hooks=None, **kwargs):
    """One step on a collated batch (apis/train.py:140-158 and Trainer.batch_processor_inline): the model's CIA-SSD loss, flattened for
    logging.  ``hooks`` (optional callable taking the reference's hook names) stands in for ``Trainer.call_hook``.  Returns the
    reference's ``dict(loss, log_vars, num_samples)`` in train mode, the detections otherwise."""
    import torch

    from ..trainer.trainer_sessd import example_to_device, parse_second_losses
    call = hooks if hooks is not None else (lambda name: None)
    example = example_to_device(data, torch.cuda.current_device() if device is None else device, non_blocking=False)
    call("after_data_to_device")
    if not train_mode:
        return model(example, return_loss=False)
    losses = model(example, return_loss=True, stage="ciassd")
    call("after_forward")
    loss, log_vars = parse_second_losses(losses)
    call("after_parse_loss")
    return dict(loss=loss, log_vars=log_vars, num_samples=len(example["anchors"][0]))


def with_default_nms(test_cfg, nms_type="rotate_weighted_nms"):
    """``test_cfg`` with ``nms.nms_type`` set to DI-NMS when the config names none, as the CIA-SSD head hard-codes it
    (mg_head_ciassd.py:774); a copy, the config itself is left as it is"""
    import copy
    cfg = copy.deepcopy(test_cfg)
    nms = cfg["nms"]
    if nms.get("nms_type") is None:
        nms["nms_type"] = nms_type
    return cfg


def train_detector(model, dataset, cfg, distributed=False, validate=False, logger=None):
    """Train ``model`` on ``dataset`` = [train, (val)] without a teacher, single-GPU, and return the final validation's results dict
    (None without a val phase).

    Every loader batches ``cfg.data.samples_per_gpu`` frames and draws from ``cfg.seed`` (0 when unset); training batches carry the
    student's branch only.  Each step clips the gradient at ``cfg.optimizer_config.grad_clip`` and runs AdamW as one ArenaAdamW pass.
    ``cfg.resume_from`` restores the model, the optimiser, the epoch and the iteration; ``cfg.load_from`` (SE-SSD's start point) is
    ignored here.  Validation runs DI-NMS unless ``test_cfg.nms.nms_type`` names another NMS."""
    from ..trainer.trainer import Trainer
    if distributed:
        raise NotImplementedError("distributed training is not implemented")
    loaders = build_loaders(dataset, cfg, twin=False)
    model = model.cuda()
    model.test_cfg = with_default_nms(model.test_cfg)
    if cfg.lr_config.type not in ("one_cycle",):
        raise NotImplementedError("learning-rate schedule %r: only one_cycle is implemented" % (cfg.lr_config.type,))
    _, optimizer = build_one_cycle_optimizer(model, cfg.optimizer)
    lr_scheduler = _create_learning_rate_scheduler(optimizer, cfg.lr_config, cfg.total_epochs * len(loaders[0]))
    trainer = Trainer(model, batch_processor, optimizer, lr_scheduler, cfg.work_dir, getattr(logging, str(cfg.get("log_level", "INFO"))),
                      logger)
    trainer.register_training_hooks(None, cfg.optimizer_config, cfg.checkpoint_config, cfg.log_config)
    if cfg.get("load_from"):
        trainer.logger.info("load_from %s is ignored: pre-training starts from the model's own initialisation", cfg.load_from)
    if cfg.get("resume_from"):
        trainer.resume(cfg.resume_from)
    return trainer.run(loaders, cfg.workflow, cfg.total_epochs)
