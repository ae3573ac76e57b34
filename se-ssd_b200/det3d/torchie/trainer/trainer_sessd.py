"""The SE-SSD trainer (reference: det3d/torchie/trainer/trainer_sessd.py): the epoch loop with the teacher / student step, validation,
checkpoints and resume, the consistency-weight ramp and the teacher's exponential moving average (one kernel launch over the flat
parameter arenas, sessd_b200.train).  Over an ArenaAdamW and a teacher ParamArena the gradient clip, the AdamW update and the teacher
EMA run as one fused device pass per step."""
import logging
import os
import os.path as osp
import sys
import time
from collections import OrderedDict

import numpy as np

from sessd_b200 import train as _train


def sigmoid_rampup(current_epoch, max_epochs=1, rampup_length=15.0):
    """consistency-weight ramp exp(-5 (1 - t)^2), t = clip(epoch, 0, 15) / 15 (trainer_sessd.py:302-309); 1.0 when max_epochs == 0"""
    if max_epochs == 0:
        return 1.0
    phase = 1.0 - float(np.clip(current_epoch, 0.0, rampup_length)) / rampup_length
    return float(np.exp(-5.0 * phase * phase))


def update_ema_variables(model, ema_model, global_step):
    """ema = alpha ema + (1 - alpha) param with alpha = min(1 - 1 / (global_step + 1), 0.999) (trainer_sessd.py:315-318); ``model`` and
    ``ema_model`` are ParamArenas (or modules carrying one as ``._arena``)."""
    a = getattr(model, "_arena", model)
    b = getattr(ema_model, "_arena", ema_model)
    return _train.update_ema_variables(a, b, global_step)


# ---------------------------------------------------------------------------------------------------------------- per-step host logic
_LIST_KEYS = frozenset(b + s for b in ("anchors", "anchors_mask", "reg_targets", "reg_weights", "labels") for s in ("", "_raw"))
_TENSOR_KEYS = frozenset(b + s for b in ("voxels", "bev_map", "coordinates", "num_points", "points", "num_voxels") for s in ("", "_raw"))


def example_to_device(example, device, non_blocking=False):
    """Move one collated batch to ``device`` with the reference's key classes (trainer_sessd.py:20-38): per-task lists of tensors, plain
    tensors, the ``calib`` dict of tensors; everything else (metadata, shapes, transformation dicts) is passed through untouched."""
    import torch
    out = {}
    for key, val in example.items():
        if key in _LIST_KEYS:
            out[key] = [t.to(device, non_blocking=non_blocking) for t in val]
        elif key in _TENSOR_KEYS:
            out[key] = val.to(device, non_blocking=non_blocking)
        elif key == "calib":
            out[key] = {k: (v.to(device, non_blocking=non_blocking) if isinstance(v, torch.Tensor) else v) for k, v in val.items()}
        else:
            out[key] = val
    return out


def parse_second_losses(losses):
    """key -> [per-task value] dict of ``MultiGroupHead.loss``  ->  (total loss tensor, log_vars of python numbers) with the reference's
    three value shapes (trainer_sessd.py:40-51): per-code lists (``loc_loss_elem*``), the one-element consistency tensors, scalars."""
    from collections import OrderedDict
    num = lambda v: float(v.detach()) if hasattr(v, "detach") else float(v)            # noqa: E731
    log_vars = OrderedDict()
    for name, values in losses.items():
        if name in ("loc_loss_elem", "loc_loss_elem_ema"):
            log_vars[name] = [[num(e) for e in per_task] for per_task in values]
        elif name in ("consistency_loss", "consistency_loss_ema"):
            log_vars[name] = [num(e) for e in values[0].detach().cpu().reshape(-1)]
        else:
            log_vars[name] = [num(v) for v in values]
    return sum(losses["loss"]), log_vars


def batch_processor_inline(model, model_ema, data, consistency_weight, train_mode, device=None, hooks=None):
    """One student / teacher step on a collated batch (trainer_sessd.py:250-275): teacher forward on the raw copy of the frames, student
    forward with the teacher's predictions, ``loss += consistency_weight * consistency_loss``, losses flattened for logging.  ``hooks``
    (optional callable taking the reference's hook names) stands in for ``Trainer.call_hook``.  Returns the reference's
    ``dict(loss, log_vars, num_samples)`` in train mode, the detections otherwise."""
    import torch
    call = hooks if hooks is not None else (lambda name: None)
    example = example_to_device(data, torch.cuda.current_device() if device is None else device, non_blocking=False)
    call("after_data_to_device")
    if not train_mode:
        return model(example, return_loss=False)
    preds_ema = model_ema(example, is_ema=[True, None])
    losses = model(example, is_ema=[False, preds_ema], return_loss=True)
    losses["loss"][0] = losses["loss"][0] + losses["consistency_loss"][0][0] * consistency_weight
    call("after_forward")
    loss, log_vars = parse_second_losses(losses)
    call("after_parse_loss")
    return dict(loss=loss, log_vars=log_vars, num_samples=len(example["anchors"][0]))


def merge_label_unlabel_data(data_batch, data_batch_unlabel):
    """Concatenate a labelled and an unlabelled collated batch for the semi-supervised mode (trainer_sessd.py:275-300), key class by key
    class: tensors with a batch-id column (``points`` / ``coordinates`` + ``_raw``) get the unlabelled frame ids shifted behind the labelled
    ones; per-voxel / per-frame tensors are concatenated; ``metadata`` lists and the ``calib`` tensors likewise; per-task target lists
    are concatenated when the unlabelled batch carries them; other keys present in both are joined with ``np.concatenate``;
    ``ssl_labeled`` marks the supervised frames.  Returns a new dict (the reference edits ``data_batch`` in place)."""
    import torch
    n_lab = int(data_batch["points"][-1, 0].item()) + 1
    n_unl = int(data_batch_unlabel["points"][-1, 0].item()) + 1
    batch_id_keys = ("coordinates", "points", "coordinates_raw", "points_raw")
    cat_keys = frozenset(b + s for b in ("voxels", "num_points", "num_gt", "voxel_labels", "num_voxels") for s in ("", "_raw"))
    merged = {}
    for key, val in data_batch.items():
        other = data_batch_unlabel.get(key)
        if other is None:
            merged[key] = val
        elif key in batch_id_keys:
            shifted = other.clone()
            shifted[:, 0] += n_lab
            merged[key] = torch.cat([val, shifted], 0)
        elif key in cat_keys:
            merged[key] = torch.cat([val, other], 0)
        elif key == "metadata":
            merged[key] = list(val) + list(other)
        elif key == "calib":
            merged[key] = {k: torch.cat([v, other[k]], 0) for k, v in val.items()}
        elif key in _LIST_KEYS:
            merged[key] = [torch.cat([val[0], other[0]], 0)] + list(val[1:])
        else:
            merged[key] = np.concatenate([val, other], axis=0)
    flag = torch.zeros(n_lab + n_unl, dtype=torch.int32)
    flag[:n_lab] = 1
    merged["ssl_labeled"] = flag
    return merged


# ---------------------------------------------------------------------------------------------------------------- the loop
class Trainer:
    """The reference's Trainer with its SE-SSD semantics, single-GPU.  ``batch_processor`` has batch_processor_inline's signature.
    ``register_training_hooks`` takes the config's optimizer / checkpoint / log entries in place of the reference's hook objects."""

    def __init__(self, model, model_ema, batch_processor, optimizer=None, lr_scheduler=None, work_dir=None, log_level=logging.INFO,
                 logger=None):
        assert callable(batch_processor)
        self.model, self.model_ema, self.batch_processor = model, model_ema, batch_processor
        self.optimizer, self.lr_scheduler = optimizer, lr_scheduler
        self.work_dir = None if work_dir is None else osp.abspath(work_dir)
        if self.work_dir is not None:
            os.makedirs(self.work_dir, exist_ok=True)
        self.timestamp = time.strftime("%Y%m%d_%H%M%S", time.localtime())
        self.logger = logger if logger is not None else self.init_logger(self.work_dir, log_level)
        self.optimizer_config, self.checkpoint_config, self.log_config = {}, {}, None
        self.mode, self.data_loader, self.outputs = None, None, None
        self._epoch = self._iter = self._inner_iter = self._max_epochs = self._max_iters = 0

    epoch = property(lambda self: self._epoch)
    iter = property(lambda self: self._iter)
    inner_iter = property(lambda self: self._inner_iter)
    max_epochs = property(lambda self: self._max_epochs)
    max_iters = property(lambda self: self._max_iters)

    def init_logger(self, log_dir=None, level=logging.INFO):
        """a logger writing to stderr and, with a work dir, to ``<work_dir>/<timestamp>.log``"""
        logger = logging.getLogger("det3d.trainer.%x" % id(self))
        logger.setLevel(level)
        logger.propagate = False
        fmt = logging.Formatter("%(asctime)s - %(levelname)s - %(message)s")
        handlers = [logging.StreamHandler(sys.stderr)]
        if log_dir:
            handlers.append(logging.FileHandler(osp.join(log_dir, "%s.log" % self.timestamp), "w"))
        for h in handlers:
            h.setFormatter(fmt)
            h.setLevel(level)
            logger.addHandler(h)
        return logger

    def register_training_hooks(self, lr_config, optimizer_config=None, checkpoint_config=None, log_config=None):
        if lr_config is not None:
            raise NotImplementedError("lr_config hooks: the one-cycle schedule is passed to the Trainer as lr_scheduler")
        self.optimizer_config = dict(optimizer_config or {})
        self.checkpoint_config = dict(checkpoint_config or {})
        self.log_config = log_config

    def current_lr(self):
        return [self.optimizer.lr]

    # ------------------------------------------------------------------------------------------------ train / val
    def _fused(self):
        """the teacher's ParamArena when clip, AdamW and EMA can run as one ArenaAdamW pass, else None"""
        from .hooks.optimizer import _owns_gradients
        ema = getattr(self.model_ema, "_arena", None)
        clip = self.optimizer_config.get("grad_clip")
        if not isinstance(ema, _train.ParamArena) or (clip is not None and clip.get("norm_type", 2) != 2):
            return None
        return ema if _owns_gradients(self.optimizer, self.model.parameters()) else None

    def _step(self, global_step):
        ema = self._fused()
        if ema is not None:
            clip = self.optimizer_config.get("grad_clip")
            self.optimizer.zero_grad()
            self.outputs["loss"].backward()
            self.optimizer.step(max_grad_norm=None if clip is None else clip["max_norm"], ema=ema, global_step=global_step)
            return
        from .hooks.optimizer import OptimizerHook
        OptimizerHook(self.optimizer_config.get("grad_clip")).after_train_iter(self)
        update_ema_variables(self.model, self.model_ema, global_step)

    def train(self, data_loader, data_loader_unlabel=None, epoch=None, **kwargs):
        """One epoch (trainer_sessd.py:320-360).  ``data_loader_unlabel`` is accepted and not drawn from: the reference's merge of
        unlabelled batches is commented out."""
        self.model_ema.train()
        self.model.train()
        consistency_weight = 1.0 * sigmoid_rampup(self.epoch, self._max_epochs)
        self._train_epoch(data_loader, lambda batch: self.batch_processor(self.model, self.model_ema, batch, consistency_weight,
                                                                          train_mode=True))

    def _train_epoch(self, data_loader, process):
        """the epoch loop: per batch the schedule step, ``process(batch)`` (the batch processor's outputs), the optimiser step, the log;
        then the checkpoint"""
        self.mode, self.data_loader = "train", data_loader
        self.length = len(data_loader)
        self._max_iters = self._max_epochs * self.length
        base_step = self.epoch * self.length
        if hasattr(data_loader, "set_epoch"):
            data_loader.set_epoch(self.epoch)
        log = _LogBuffer()
        interval = self.log_config["interval"] if self.log_config else 0
        t_end = time.time()
        for i, data_batch in enumerate(data_loader):
            t_data = time.time()
            global_step = base_step + i
            if self.lr_scheduler is not None:
                self.lr_scheduler.step(global_step)
            self._inner_iter = i
            outputs = process(data_batch)
            if not isinstance(outputs, dict):
                raise TypeError("batch_processor() must return a dict")
            self.outputs = outputs
            self._step(global_step)
            self._iter += 1
            now = time.time()
            log.update(outputs["log_vars"], outputs["num_samples"], time=now - t_end, data_time=t_data - t_end)
            t_end = now
            if interval and (i + 1) % interval == 0:
                self._log_train(log)
        if self.work_dir and (self.epoch + 1) % self.checkpoint_config.get("interval", 1) == 0:
            self.save_checkpoint(self.work_dir, save_optimizer=self.checkpoint_config.get("save_optimizer", True),
                                 meta=dict(self.checkpoint_config.get("meta") or {}))
        self._epoch += 1

    def _log_train(self, log):
        avg = log.average()
        head = "Epoch [%d/%d][%d/%d]\tlr: %.5f, time: %.3f, data_time: %.3f, " % (
            self.epoch + 1, self._max_epochs, self._inner_iter + 1, self.length, self.current_lr()[0], avg.pop("time"),
            avg.pop("data_time"))
        self.logger.info(head + ", ".join("%s: %s" % (k, _fmt(v)) for k, v in avg.items()))
        log.clear()

    def val(self, data_loader, **kwargs):
        """Evaluate the student (trainer_sessd.py:362-415): predictions keyed by token, ``dataset.evaluation``, the official AP strings
        logged.  Returns the results dict."""
        self.mode, self.data_loader = "val", data_loader
        self.logger.info("work dir: %s", self.work_dir)
        result_dict, _ = data_loader.dataset.evaluation(compute_on_dataset(self.model, data_loader), output_dir=self.work_dir)
        self.logger.info("\n")
        for k, v in list(result_dict["results"].items()) + list(result_dict["results_2"].items()):
            self.logger.info("Evaluation %s: %s", k, v)
        return result_dict

    def run(self, data_loaders, workflow, max_epochs, **kwargs):
        """Train from the current epoch to ``max_epochs`` on ``data_loaders[0]``, then validate once on ``data_loaders[-1]``, the order
        of the reference's run() (trainer_sessd.py:430-470) for workflow [("train", N), ("val", 1)].  Returns the validation results,
        or None when the workflow has no val phase."""
        assert isinstance(data_loaders, list)
        self._max_epochs = max_epochs
        self.logger.info("Start running, work_dir: %s", self.work_dir)
        self.logger.info("workflow: %s, max: %d epochs", workflow, max_epochs)
        results = None
        while self.epoch < max_epochs:
            for mode, epochs in workflow:
                if mode not in ("train", "val"):
                    raise ValueError("Trainer has no method named '{}' to run an epoch".format(mode))
                for _ in range(epochs):
                    if mode == "train" and self.epoch > max_epochs:
                        return results
                    if mode == "train" and self.epoch == max_epochs:
                        return self.val(data_loaders[-1]) if len(workflow) > 1 else results
                    if mode == "val":
                        results = self.val(data_loaders[-1])
                    else:
                        self.train(data_loaders[0], epoch=self.epoch)
        return results

    # ------------------------------------------------------------------------------------------------ checkpoints
    def _checkpointed(self):
        """(model, file-name suffix) of every model a checkpoint holds: the student, then the teacher"""
        return ((self.model, ""), (self.model_ema, "_ema"))

    def save_checkpoint(self, out_dir, filename_tmpl="epoch_{}.pth", save_optimizer=True, meta=None):
        """``epoch_{n}.pth`` (student) and ``epoch_{n}_ema.pth`` (teacher), both with the optimiser state and meta = {epoch, iter} plus
        ``meta``; relative symlinks latest.pth / latest_ema.pth (trainer_sessd.py:228-248)"""
        from .checkpoint import save_checkpoint
        meta = dict(meta or {})
        meta.update(epoch=self.epoch + 1, iter=self.iter)
        stem = osp.splitext(filename_tmpl.format(self.epoch + 1))[0]
        optimizer = self.optimizer if save_optimizer else None
        for model, sfx in self._checkpointed():
            name = stem + sfx + ".pth"
            save_checkpoint(model, osp.join(out_dir, name), optimizer=optimizer, meta=meta)
            _symlink(name, osp.join(out_dir, "latest" + sfx + ".pth"))

    def load_checkpoint(self, filename, map_location="cpu", strict=False):
        """the student from ``filename``, the teacher from its ``_ema`` twin, the optimiser state"""
        from .checkpoint import load_checkpoint
        self.logger.info("load checkpoint from %s", filename)
        ckpt = load_checkpoint(self.model, filename, map_location, strict, self.logger)
        for model, sfx in self._checkpointed()[1:]:
            load_checkpoint(model, osp.splitext(filename)[0] + sfx + ".pth", map_location, strict, self.logger)
        self.optimizer.load_state_dict(ckpt["optimizer"])
        return ckpt

    def load_checkpoint_from_scratch(self, filename, map_location="cpu", strict=False):
        """student and teacher from the same checkpoint, and its optimiser state (the ``load_from`` of SE-SSD's SSL stage)"""
        from .checkpoint import load_checkpoint
        self.logger.info("load checkpoint from %s", filename)
        ckpt = load_checkpoint(self.model, filename, map_location, strict, self.logger)
        load_checkpoint(self.model_ema, filename, map_location, strict, self.logger)
        self.optimizer.load_state_dict(ckpt["optimizer"])
        return ckpt

    def resume(self, checkpoint, resume_optimizer=True, map_location="default"):
        if map_location == "default":
            import torch
            map_location = "cuda:%d" % torch.cuda.current_device() if torch.cuda.is_available() else "cpu"
        ckpt = self.load_checkpoint(checkpoint, map_location=map_location)
        self._epoch, self._iter = ckpt["meta"]["epoch"], ckpt["meta"]["iter"]
        self.logger.info("resumed epoch %d, iter %d", self.epoch, self.iter)


def compute_on_dataset(model, data_loader):
    """the model's detections on every batch of ``data_loader`` in eval mode, keyed by token, tensors on the host (tools/test.py)"""
    import torch
    model.eval()
    detections = {}
    with torch.no_grad():
        for example in data_loader:
            for output in model(example, return_loss=False):
                detections[output["metadata"]["token"]] = {k: (v if k == "metadata" else v.cpu()) for k, v in output.items()}
    return detections


def _symlink(src, dst):
    if osp.lexists(dst):
        os.remove(dst)
    os.symlink(src, dst)


def _fmt(v):
    return "%.4f" % v if np.ndim(v) == 0 else str(np.round(np.asarray(v, np.float64), 4).tolist())


class _LogBuffer:
    """averages of the logged values over the iterations since the last log line, weighted by the batch's sample count"""

    def __init__(self):
        self.clear()

    def clear(self):
        self.values, self.counts = OrderedDict(), []

    def update(self, log_vars, count, **times):
        for k, v in list(times.items()) + list(log_vars.items()):
            self.values.setdefault(k, []).append(np.asarray(v, np.float64))
        self.counts.append(count)

    def average(self):
        w = np.asarray(self.counts, np.float64)
        return OrderedDict((k, np.average(np.stack(v), axis=0, weights=w)) for k, v in self.values.items())
