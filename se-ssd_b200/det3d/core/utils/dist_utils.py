"""Gradient all-reduce of the DDP training loop (reference: det3d/core/utils/dist_utils.py:8-57, driven from
det3d/torchie/apis/train_sessd.py:286-294).  Same entry points (``allreduce_grads``, ``DistOptimizerHook``); the GPU-native path keeps
every gradient inside one contiguous arena (sessd_b200.train.ParamArena) so the collective runs IN PLACE on one buffer -- averaged inside
NCCL over NVLink / NVSwitch -- instead of flatten -> all_reduce -> divide -> unflatten -> copy back per bucket."""
import torch
import torch.distributed as dist

from ...torchie.trainer.hooks.optimizer import clip_and_step


def _grads(params):
    return [p.grad for p in params if p.requires_grad and p.grad is not None]


def _common_arena(grads):
    """the flat tensor all gradients are views of (ParamArena.grad_flat), or None"""
    base = grads[0]._base if grads else None
    if base is None or base.dim() != 1:
        return None
    lo, hi = base.data_ptr(), base.data_ptr() + base.numel() * base.element_size()
    for g in grads:
        if g._base is not base or not (lo <= g.data_ptr() < hi):
            return None
    return base


def allreduce_grads(params, coalesce=True, bucket_size_mb=-1):
    """Average the gradients of ``params`` over the default process group.  Gradients that live in one arena are reduced in place with a
    single collective; otherwise they are packed per dtype (or per ``bucket_size_mb``) like the reference does."""
    grads = _grads(list(params))
    if not grads:
        return
    world = dist.get_world_size()
    avg = dist.ReduceOp.AVG if (grads[0].is_cuda and dist.get_backend() == "nccl") else None

    def reduce_(t):
        if avg is not None:
            dist.all_reduce(t, op=avg)
        else:
            dist.all_reduce(t)
            t.div_(world)

    arena = _common_arena(grads) if coalesce else None
    if arena is not None:
        reduce_(arena.detach())
        return
    grads = [g.detach() for g in grads]
    if not coalesce:
        for g in grads:
            reduce_(g)
        return
    buckets, limit = [], bucket_size_mb * 1024 * 1024
    for g in grads:                                   # consecutive gradients of one dtype share a bucket (optionally size-capped)
        if buckets and buckets[-1][0].dtype == g.dtype and (limit <= 0 or buckets[-1][1] + g.numel() * g.element_size() <= limit):
            buckets[-1][2].append(g)
            buckets[-1][1] += g.numel() * g.element_size()
        else:
            buckets.append([g, g.numel() * g.element_size(), [g]])
    for _first, _bytes, members in buckets:
        flat = torch.cat([g.reshape(-1) for g in members])
        reduce_(flat)
        off = 0
        for g in members:
            g.copy_(flat[off:off + g.numel()].view_as(g))
            off += g.numel()


class DistOptimizerHook(object):
    """after_train_iter: zero_grad -> backward -> allreduce_grads -> (clip) -> optimizer.step, like the reference hook.  Over an ArenaAdamW
    that owns the model's gradient arena the L2 clip runs inside its step: a deterministic norm of the all-reduced arena, identical on
    every rank (det3d.torchie.trainer.hooks.optimizer.clip_and_step)."""

    def __init__(self, grad_clip=None, coalesce=True, bucket_size_mb=-1):
        self.grad_clip, self.coalesce, self.bucket_size_mb = grad_clip, coalesce, bucket_size_mb

    def clip_grads(self, params):
        torch.nn.utils.clip_grad_norm_([p for p in params if p.requires_grad and p.grad is not None], **self.grad_clip)

    def after_train_iter(self, runner):
        runner.optimizer.zero_grad()
        runner.outputs["loss"].backward()
        allreduce_grads(runner.model.parameters(), self.coalesce, self.bucket_size_mb)
        clip_and_step(runner.optimizer, runner.model.parameters(), self.grad_clip)
