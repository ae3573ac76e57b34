"""Generate tests/golden/optim_recipe.npz by running the REFERENCE's own optimiser recipe on the
CPU: fastai's OneCycle (det3d/solver/learning_schedules_fastai.py), OptimWrapper(torch.optim.Adam, betas=(mom, 0.99), wd=0.01,
true_wd=True, bn_wd=True) over split_bn_bias(get_layer_groups(model)) (det3d/solver/fastai_optim.py, det3d/torchie/apis/train_sessd.py:
161-175), clip_grad_norm_(max_norm=35) before each step (det3d/torchie/trainer/hooks/optimizer.py:35-62), the teacher EMA after it
(det3d/torchie/trainer/trainer_sessd.py:315-318), and the reference's save_checkpoint(model, f, optimizer=wrapper).

    python tests/golden/make_optim_golden.py

Recorded: the OneCycle lr / mom at every step for total_steps in optim_case.SCHEDULE_TOTALS; 20 steps on optim_case.optim_model() with
optim_case.step_gradients() (lr, mom, total norm, clipped gradient, parameters, both moments, teacher after each step, flattened in
model.parameters() order); the reference optimiser's parameter order for that model and for the VoxelNet this repository builds from
examples/second/configs/config.py (parameter names); and the contents of the checkpoint the reference's save_checkpoint writes after
optim_case.CKPT_STEP steps, read back from that file and stored as ``ckpt_*`` arrays (optim_case.reference_checkpoint rebuilds the dict
torch.load returns; the per-parameter ``step`` comes back as a Python int, as torch 1.x, which the reference runs on, writes it).
"""
import ast
import collections
import collections.abc
import copy
import importlib.util
import json
import os
import sys
import tempfile
from functools import partial

import numpy as np
import torch
from torch import nn

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path[:0] = [HERE, os.path.join(ROOT, "tests"), os.path.join(ROOT, "se-ssd_b200")]
import optim_case as OC  # noqa: E402
from make_checkpoint_golden import load_reference_checkpoint_module  # noqa: E402


def load_by_path(name, rel):
    spec = importlib.util.spec_from_file_location(name, os.path.join(REF, rel))
    m = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(m)
    return m


def reference_layer_groups():
    """flatten_model / get_layer_groups of det3d/torchie/apis/train_sessd.py, taken from the file (its module imports apex and datasets)"""
    src = open(os.path.join(REF, "det3d/torchie/apis/train_sessd.py")).read()
    fns = [n for n in ast.parse(src).body if isinstance(n, ast.FunctionDef) and n.name in ("flatten_model", "get_layer_groups")]
    ns = {"nn": nn}
    exec(compile(ast.Module(body=fns, type_ignores=[]), "train_sessd.py", "exec"), ns)
    return ns["get_layer_groups"]


class Stub:
    lr, mom = 0.0, 0.0


def main():
    collections.Iterable = collections.abc.Iterable          # fastai_optim.py imports it from collections (removed in Python 3.10)
    lsf = load_by_path("ref_lsf", "det3d/solver/learning_schedules_fastai.py")
    fo = load_by_path("ref_fastai_optim", "det3d/solver/fastai_optim.py")
    get_layer_groups = reference_layer_groups()
    out = {}

    for total in OC.SCHEDULE_TOTALS:
        s = Stub()
        sched = lsf.OneCycle(s, total, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START)
        out["sched%d_init" % total] = np.array([s.lr, s.mom], np.float64)
        lrs, moms = [], []
        for i in range(total):
            sched.step(i)
            lrs.append(s.lr)
            moms.append(s.mom)
        out["sched%d_lr" % total] = np.array(lrs, np.float64)
        out["sched%d_mom" % total] = np.array(moms, np.float64)

    def order_names(model):
        ids = {id(p): n for n, p in model.named_parameters()}
        return [ids[id(p)] for g in fo.split_bn_bias(get_layer_groups(model)) for p in g.parameters() if p.requires_grad]

    from det3d.models import build_detector
    from det3d.torchie import Config
    cfg = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    out["voxelnet_order"] = np.array(order_names(build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)))

    ref_ckpt = load_reference_checkpoint_module()                # stubs det3d: after this repository's det3d has built the VoxelNet
    model = OC.optim_model()
    teacher = copy.deepcopy(model)
    out["toy_order"] = np.array(order_names(model))
    out["init_params"] = torch.cat([p.detach().reshape(-1) for p in model.parameters()]).numpy()
    wrapper = fo.OptimWrapper.create(partial(torch.optim.Adam, betas=(0.9, 0.99), amsgrad=False), 3e-3, get_layer_groups(model),
                                     wd=OC.WD, true_wd=True, bn_wd=True)
    sched = lsf.OneCycle(wrapper, OC.STEPS, OC.LR_MAX, OC.MOMS, OC.DIV_FACTOR, OC.PCT_START)
    flat = lambda ts: torch.cat([t.detach().reshape(-1) for t in ts]).numpy().copy()          # noqa: E731
    rec = {k: [] for k in ("lr", "mom", "norm", "grad_in", "grad", "param", "exp_avg", "exp_avg_sq", "teacher")}
    for i in range(OC.STEPS):
        sched.step(i)
        wrapper.zero_grad()
        for p, g in zip(model.parameters(), OC.step_gradients(model, i)):
            p.grad = g.clone()
        rec["grad_in"].append(flat([p.grad for p in model.parameters()]))
        norm = nn.utils.clip_grad_norm_(filter(lambda p: p.requires_grad, model.parameters()), max_norm=OC.MAX_NORM, norm_type=2)
        wrapper.step()
        alpha = min(1 - 1 / (i + 1), 0.999)                    # Trainer.update_ema_variables(model, model_ema, global_step=i)
        for e, p in zip(teacher.parameters(), model.parameters()):
            e.data.mul_(alpha).add_(p.data, alpha=1 - alpha)
        rec["lr"].append(wrapper.lr)
        rec["mom"].append(wrapper.mom)
        rec["norm"].append(float(norm))
        rec["grad"].append(flat([p.grad for p in model.parameters()]))
        rec["param"].append(flat(model.parameters()))
        rec["exp_avg"].append(flat([wrapper.opt.state[p]["exp_avg"] for p in model.parameters()]))
        rec["exp_avg_sq"].append(flat([wrapper.opt.state[p]["exp_avg_sq"] for p in model.parameters()]))
        rec["teacher"].append(flat(teacher.parameters()))
        if i + 1 == OC.CKPT_STEP:
            with tempfile.TemporaryDirectory() as d:
                path = os.path.join(d, "epoch_1.pth")
                ref_ckpt.save_checkpoint(model, path, optimizer=wrapper, meta={"epoch": 1, "iter": OC.CKPT_STEP})
                ck = torch.load(path, weights_only=False)
            out["ckpt_meta"] = np.array(json.dumps(ck["meta"]))
            out["ckpt_state_dict_keys"] = np.array(list(ck["state_dict"]))
            for j, v in enumerate(ck["state_dict"].values()):
                out["ckpt_state_dict_%d" % j] = v.numpy()
            groups = [{k: (list(v) if isinstance(v, tuple) else v) for k, v in g.items()} for g in ck["optimizer"]["param_groups"]]
            out["ckpt_param_groups"] = np.array(json.dumps(groups, default=float))          # lr is a numpy scalar there
            for j, st in ck["optimizer"]["state"].items():
                out["ckpt_step_%d" % j] = np.array(int(st["step"]), np.int64)
                out["ckpt_exp_avg_%d" % j] = st["exp_avg"].numpy()
                out["ckpt_exp_avg_sq_%d" % j] = st["exp_avg_sq"].numpy()
    for k, v in rec.items():
        out["traj_" + k] = np.array(v, np.float64 if k in ("lr", "mom", "norm") else np.float32)
    clipped = int(sum(n > OC.MAX_NORM for n in rec["norm"]))
    assert 0 < clipped < OC.STEPS, clipped
    np.savez_compressed(os.path.join(HERE, "optim_recipe.npz"), **out)
    print("wrote optim_recipe.npz (%d of %d steps clipped)" % (clipped, OC.STEPS))


if __name__ == "__main__":
    main()
