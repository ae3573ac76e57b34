"""The single-model trainer (reference: det3d/torchie/trainer/trainer.py): the epoch loop of CIA-SSD pre-training, the supervised stage
that SE-SSD's teacher / student loop starts from.  It is the SE-SSD Trainer (trainer_sessd) without the teacher: the same loop, logging,
validation, checkpoint files and resume, with the gradient clip and the AdamW update as one fused device pass per step (ArenaAdamW) and
no EMA."""
import logging

from .trainer_sessd import Trainer as _TeacherStudentTrainer


class Trainer(_TeacherStudentTrainer):
    """``batch_processor(model, data, train_mode)`` has the signature of det3d.torchie.apis.train.batch_processor.  Checkpoints are
    ``epoch_{n}.pth`` with the optimiser state and meta = {epoch, iter}, and the relative symlink ``latest.pth``: the format SE-SSD's
    ``load_from`` and ``resume_from`` read."""

    def __init__(self, model, batch_processor, optimizer=None, lr_scheduler=None, work_dir=None, log_level=logging.INFO, logger=None):
        super().__init__(model, None, batch_processor, optimizer, lr_scheduler, work_dir, log_level, logger)

    def _step(self, global_step):
        from .hooks.optimizer import OptimizerHook
        OptimizerHook(self.optimizer_config.get("grad_clip")).after_train_iter(self)

    def train(self, data_loader, epoch=None, **kwargs):
        """One epoch (trainer.py:254-287)."""
        self.model.train()
        self._train_epoch(data_loader, lambda batch: self.batch_processor(self.model, batch, train_mode=True))

    def _checkpointed(self):
        return ((self.model, ""),)

    def load_checkpoint_from_scratch(self, filename, map_location="cpu", strict=False):
        raise NotImplementedError("a single-model run starts from scratch or resumes its own checkpoint")
