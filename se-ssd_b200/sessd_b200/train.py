"""Optimiser side of the SE-SSD training step on flat parameter arenas (SURVEY 8(f) rows 1-2; csrc/train.cu).

The reference updates the teacher parameter by parameter in Python (trainer_sessd.py:315-318), flattens and unflattens the gradients
around ``dist.all_reduce`` (dist_utils.py:8-29) and steps a fastai ``OptimWrapper`` over parameter groups.  Here a model's parameters --
and their gradients -- are views into ONE contiguous fp32 buffer each (``ParamArena``): the EMA, the gradient all-reduce (in place on the
arena: NCCL over NVLink on the device, gloo in the CPU tests) and the AdamW step are one launch / one collective each."""
import ctypes as C

import torch
import torch.distributed as dist

from ._lib import check, lib


def _p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


def _st(t):
    return C.c_void_p(torch.cuda.current_stream(t.device).cuda_stream) if t.is_cuda else C.c_void_p(0)


_BN_TYPES = (torch.nn.BatchNorm1d, torch.nn.BatchNorm2d, torch.nn.BatchNorm3d)


def _leaf_modules(m):
    children = list(m.children())
    return sum(map(_leaf_modules, children), []) if children else [m]


def _optimizer_groups(model, params):
    """Indices into ``params`` in the order of the reference optimiser's two parameter groups, split_bn_bias(get_layer_groups(model))
    (det3d/torchie/apis/train_sessd.py:161-166, det3d/solver/fastai_optim.py:14-35): the trainable parameters of the non-BatchNorm leaf
    modules, then those of the BatchNorm leaves, each in module order and without repeats."""
    index = {id(p): i for i, p in enumerate(params)}
    leaves = _leaf_modules(model)
    groups = []
    for bn in (False, True):
        mods = torch.nn.Sequential(*[c for c in leaves if isinstance(c, _BN_TYPES) == bn])
        groups.append([index[id(p)] for p in mods.parameters() if p.requires_grad])
    return groups


class ParamArena:
    """Re-homes every parameter of ``model`` into one flat fp32 buffer (``.flat``) and gives every parameter a ``.grad`` that is a view
    into a second flat buffer (``.grad_flat``).  Parameter values, names, shapes and ``state_dict()`` are unchanged; autograd accumulates
    straight into the gradient arena.  Offsets are 16-byte aligned (vector loads in the kernels).  ``optim_groups`` holds the reference
    optimiser's parameter order (indices into ``params``: non-BatchNorm group, BatchNorm group), the index space of its ``state_dict()``."""

    def __init__(self, model, with_grad=True):
        self.params = [p for p in model.parameters()]
        self.optim_groups = _optimizer_groups(model, self.params)
        assert all(p.dtype == torch.float32 for p in self.params), "fp32 master parameters"
        dev = self.params[0].device
        self.offsets, n = [], 0
        for p in self.params:
            self.offsets.append(n)
            n += (p.numel() + 3) // 4 * 4
        self.numel = n
        self.flat = torch.zeros((n,), dtype=torch.float32, device=dev)
        self.grad_flat = torch.zeros((n,), dtype=torch.float32, device=dev) if with_grad else None
        for p, off in zip(self.params, self.offsets):
            view = self.flat[off:off + p.numel()].view_as(p)
            view.copy_(p.data)
            p.data = view
            if with_grad:
                p.grad = self.grad_flat[off:off + p.numel()].view_as(p)

    def zero_grad(self):
        self.grad_flat.zero_()


def axpby(y, x, a, b):
    """y = a y + b x on flat fp32 CUDA tensors (x may be None): one kernel.  No host implementation."""
    if not y.is_cuda or (x is not None and not x.is_cuda):
        raise ValueError("sessd_b200.train.axpby: CUDA tensors only (there is no CPU path)")
    check(lib.sessd_axpby(_p(y), _p(x), float(a), float(b), int(y.numel()), _st(y)), "sessd_axpby")
    return y


def ema_alpha(global_step, max_alpha=0.999):
    """the teacher's EMA weight at ``global_step`` (trainer_sessd.py:315-316)"""
    return min(1.0 - 1.0 / (global_step + 1), max_alpha)


def update_ema_variables(model_or_arena, ema_model_or_arena, global_step, max_alpha=0.999):
    """Teacher update of trainer_sessd.py:315-318: alpha = min(1 - 1 / (global_step + 1), 0.999); ema = alpha * ema + (1 - alpha) * param.
    Both models live in ParamArenas: one launch over the flat buffers."""
    alpha = ema_alpha(global_step, max_alpha)
    if isinstance(model_or_arena, ParamArena) and isinstance(ema_model_or_arena, ParamArena):
        assert model_or_arena.numel == ema_model_or_arena.numel
        axpby(ema_model_or_arena.flat, model_or_arena.flat, alpha, 1.0 - alpha)
        return alpha
    raise TypeError("update_ema_variables: wrap both models in a ParamArena first (the update is one launch over the flat buffers)")


def allreduce_grad_arena(arena, group=None):
    """Average the gradient arena over the process group IN PLACE: one collective on one contiguous buffer (the reference's coalesced path
    builds that buffer with _flatten_dense_tensors and copies the result back tensor by tensor, dist_utils.py:20-29)."""
    world = dist.get_world_size(group)
    if world == 1:
        return arena.grad_flat
    if arena.grad_flat.is_cuda and dist.get_backend(group) == "nccl":
        dist.all_reduce(arena.grad_flat, op=dist.ReduceOp.AVG, group=group)          # averaged inside the collective (NVLink / NVSwitch)
    else:                                                                            # gloo (CPU tests of the sharding logic): sum, then scale
        dist.all_reduce(arena.grad_flat, op=dist.ReduceOp.SUM, group=group)
        arena.grad_flat.div_(world)
    return arena.grad_flat


def grad_norm_workspace(x):
    """the zero-filled workspace of grad_norm over ``x`` (the kernel leaves it zeroed again: allocate once, reuse on one stream)"""
    return torch.zeros(lib.sessd_grad_sqnorm_workspace_bytes(int(x.numel())), dtype=torch.uint8, device=x.device)


def grad_norm(x, max_norm, workspace=None):
    """[total_norm, clip_coef] of the flat fp32 CUDA tensor ``x`` as a device tensor, without a host round trip (sessd_grad_sqnorm):
    total_norm = ||x||_2 (fp64 sum, bitwise deterministic), clip_coef = min(1, max_norm / (total_norm + 1e-6)) as clip_grad_norm_."""
    if not x.is_cuda or x.dtype != torch.float32 or not x.is_contiguous():
        raise ValueError("sessd_b200.train.grad_norm: a contiguous fp32 CUDA tensor (there is no CPU path)")
    workspace = grad_norm_workspace(x) if workspace is None else workspace
    if workspace.device != x.device or workspace.numel() * workspace.element_size() < lib.sessd_grad_sqnorm_workspace_bytes(int(x.numel())):
        raise ValueError("sessd_b200.train.grad_norm: workspace too small or on another device (see grad_norm_workspace)")
    out = torch.empty(2, dtype=torch.float32, device=x.device)
    check(lib.sessd_grad_sqnorm(_p(x), int(x.numel()), float(max_norm), _p(out), _p(workspace), _st(x)), "sessd_grad_sqnorm")
    return out


class ArenaAdamW:
    """AdamW over a ParamArena in one launch per step (torch.optim.AdamW arithmetic == fastai OptimWrapper(true_wd=True, bn_wd=True) around
    Adam, det3d/solver/fastai_optim.py).  ``lr`` and ``mom`` (Adam's beta1, under fastai's name) may be changed between steps: the
    one-cycle schedule (det3d/solver/learning_schedules_fastai.py) drives both.  ``state_dict()`` / ``load_state_dict()`` use torch Adam's
    format over the reference's parameter order (``ParamArena.optim_groups``), so a run resumes, and a reference checkpoint continues."""

    def __init__(self, arena, lr=3e-3, betas=(0.9, 0.99), eps=1e-8, weight_decay=0.01, amsgrad=False):
        if amsgrad:
            raise NotImplementedError("ArenaAdamW: amsgrad is not implemented (the SE-SSD config trains with amsgrad=0)")
        self.arena, self.lr, self.betas, self.eps, self.weight_decay = arena, lr, tuple(betas), eps, weight_decay
        self.exp_avg = torch.zeros_like(arena.flat)
        self.exp_avg_sq = torch.zeros_like(arena.flat)
        self.steps = 0
        self._norm_workspace = None

    @property
    def mom(self):
        return self.betas[0]

    @mom.setter
    def mom(self, value):
        self.betas = (value, self.betas[1])

    def step(self, max_grad_norm=None, ema=None, global_step=None):
        """One AdamW step.  ``max_grad_norm``: first clip the gradient arena to that L2 norm, as clip_grad_norm_(params, max_grad_norm)
        does (det3d/torchie/trainer/hooks/optimizer.py:35-62); the clipped gradient is left in the arena.  ``ema`` (the teacher's
        ParamArena) with ``global_step``: update the teacher from the new parameters in the same pass (trainer_sessd.py:315-318).  One norm
        launch when clipping, then one update launch; the host never waits for the device.  Returns the total gradient norm as a 0-d
        device tensor when clipping, else None."""
        a = self.arena
        if not a.flat.is_cuda:
            raise ValueError("ArenaAdamW: CUDA arenas only (there is no CPU path)")
        if ema is not None and (global_step is None or ema.numel != a.numel):
            raise ValueError("ArenaAdamW.step: ema must be a ParamArena of the same layout, given with the global_step of its alpha")
        self.steps += 1
        st = _st(a.flat)
        args = (_p(a.flat), _p(a.grad_flat), _p(self.exp_avg), _p(self.exp_avg_sq), int(a.numel), float(self.lr), float(self.betas[0]),
                float(self.betas[1]), float(self.eps), float(self.weight_decay), int(self.steps))
        if max_grad_norm is None and ema is None:
            check(lib.sessd_adamw_step(*args, st), "sessd_adamw_step")
            return None
        norm = None
        if max_grad_norm is not None:
            if self._norm_workspace is None:
                self._norm_workspace = grad_norm_workspace(a.grad_flat)
            norm = grad_norm(a.grad_flat, max_grad_norm, self._norm_workspace)          # [total_norm, clip_coef]
        alpha = ema_alpha(global_step) if ema is not None else 0.0
        check(lib.sessd_adamw_clip_ema_step(*args, _p(norm[1:]) if norm is not None else C.c_void_p(0),
                                            _p(ema.flat if ema is not None else None), float(alpha), st), "sessd_adamw_clip_ema_step")
        return None if norm is None else norm[0]

    def zero_grad(self):
        self.arena.zero_grad()

    def _groups(self):
        """per reference parameter group: (state index, parameter, arena offset) in the reference optimiser's order"""
        a, i, out = self.arena, 0, []
        for members in a.optim_groups:
            out.append([(i + j, a.params[k], a.offsets[k]) for j, k in enumerate(members)])
            i += len(members)
        return out

    def state_dict(self):
        """torch.optim.Adam's state_dict over the reference's two parameter groups (the ``"optimizer"`` entry of its checkpoints): per
        index ``step``, ``exp_avg``, ``exp_avg_sq`` shaped like the parameter.  The weight decay is applied outside Adam (true_wd), so the
        groups carry weight_decay=0."""
        state, groups = {}, []
        for members in self._groups():
            for i, p, off in members:
                if self.steps > 0:
                    n = p.numel()
                    state[i] = {"step": torch.tensor(float(self.steps)), "exp_avg": self.exp_avg[off:off + n].view_as(p).clone(),
                                "exp_avg_sq": self.exp_avg_sq[off:off + n].view_as(p).clone()}
            groups.append({"lr": float(self.lr), "betas": tuple(float(b) for b in self.betas), "eps": float(self.eps), "weight_decay": 0, "amsgrad": False,
                           "params": [i for i, _, _ in members]})
        return {"state": state, "param_groups": groups}

    def load_state_dict(self, state_dict):
        """Inverse of state_dict(); also reads a reference-written ``"optimizer"`` entry, whose ``step`` is an int (torch 1.x)."""
        groups, state = state_dict["param_groups"], state_dict["state"]
        layout = self._groups()
        if [len(g["params"]) for g in groups] != [len(m) for m in layout]:
            raise ValueError("optimizer state: parameter groups of %s parameters, this model has %s"
                             % ([len(g["params"]) for g in groups], [len(m) for m in layout]))
        if any(g.get("amsgrad", False) for g in groups):
            raise NotImplementedError("ArenaAdamW: amsgrad is not implemented")
        m, v, steps = torch.zeros_like(self.exp_avg), torch.zeros_like(self.exp_avg_sq), set()
        for g, members in zip(groups, layout):
            for j, (_i, p, off) in zip(g["params"], members):
                s = state.get(j)
                if s is None:                           # torch keeps no state for a parameter that never stepped
                    steps.add(0)
                    continue
                if tuple(s["exp_avg"].shape) != tuple(p.shape) or tuple(s["exp_avg_sq"].shape) != tuple(p.shape):
                    raise ValueError("optimizer state %d: shape %s, parameter %s" % (j, tuple(s["exp_avg"].shape), tuple(p.shape)))
                steps.add(int(s["step"]))
                m[off:off + p.numel()].copy_(s["exp_avg"].reshape(-1))
                v[off:off + p.numel()].copy_(s["exp_avg_sq"].reshape(-1))
        if len(steps) > 1:
            raise ValueError("optimizer state: per-parameter step counts %s differ; the arena keeps one" % sorted(steps))
        self.exp_avg.copy_(m)
        self.exp_avg_sq.copy_(v)
        self.steps = steps.pop() if steps else 0
        self.lr, self.betas, self.eps = groups[0]["lr"], tuple(groups[0]["betas"]), groups[0]["eps"]


# ------------------------------------------------------------------------------------------------- data gradients through the forward kernels
def subm_dgrad_weight(w):
    """SubMConv3d weight [kz, ky, kx, Cin, Cout] (spconv layout, scn.py:106-131)  ->  [kz, ky, kx, Cout, Cin] such that the FORWARD sparse conv
    over the SAME rulebook / tile lists, fed with d loss / d out, yields d loss / d in:  W'[k] = W[K-1-k]^T.  (A SubM layer's neighbour
    table is point-symmetric -- nbr_t[i, k] = nbr[i, K-1-k] -- so the data gradient needs neither a transposed rulebook nor a new kernel;
    pinned on the CPU by tests/test_train_step.py against oracle/spconv_grad_ref.py, which is pinned to dense autograd.)"""
    return w.flip(0, 1, 2).transpose(3, 4).contiguous()


def conv2d_s1_dgrad_weight(w):
    """Conv2d weight [Cout, Cin, k, k] of a stride-1 neck layer  ->  [Cin, Cout, k, k], taps flipped: the stride-1 conv (pad k - 1 - p) that
    maps d loss / d out to d loss / d in (rpn_v1.py:135-210 layers bottom_up_block_0.*, bottom_up_block_1.3 / .6, conv_0, conv_1, trans_*)."""
    return w.flip(2, 3).transpose(0, 1).contiguous()
