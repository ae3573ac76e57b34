"""Single-GPU optimiser hook of the training loop (reference: det3d/torchie/trainer/hooks/optimizer.py:35-62): zero_grad -> backward ->
clip_grad_norm_(max_norm, norm_type) -> optimizer.step.  Over an ArenaAdamW that owns the model's gradient arena, the L2 clip runs inside
the optimiser's step (one deterministic device norm, no host round trip); any other optimiser keeps torch's clip_grad_norm_."""
import torch

from sessd_b200.train import ArenaAdamW


def _owns_gradients(optimizer, params):
    """True when ``optimizer`` is an ArenaAdamW and ``params`` are exactly its arena's parameters (so the arena norm is their norm)"""
    if not isinstance(optimizer, ArenaAdamW):
        return False
    mine = optimizer.arena.params
    params = [p for p in params if p.requires_grad]
    return len(params) == len(mine) and all(p is q for p, q in zip(params, mine))


def clip_and_step(optimizer, params, grad_clip):
    """``grad_clip`` = dict(max_norm=..., norm_type=...) or None."""
    params = list(params)
    if grad_clip is not None and grad_clip.get("norm_type", 2) == 2 and _owns_gradients(optimizer, params):
        return optimizer.step(max_grad_norm=grad_clip["max_norm"])
    if grad_clip is not None:
        torch.nn.utils.clip_grad_norm_([p for p in params if p.requires_grad and p.grad is not None], **grad_clip)
    optimizer.step()


class OptimizerHook(object):
    def __init__(self, grad_clip=None):
        self.grad_clip = grad_clip

    def after_train_iter(self, trainer):
        trainer.optimizer.zero_grad()
        trainer.outputs["loss"].backward()
        clip_and_step(trainer.optimizer, trainer.model.parameters(), self.grad_clip)
