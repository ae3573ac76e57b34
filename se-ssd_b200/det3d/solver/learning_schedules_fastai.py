"""The one-cycle learning-rate and momentum schedule of SE-SSD training (reference: det3d/solver/learning_schedules_fastai.py:7-100,
fastai's ``OneCycle``).  ``step(global_step)`` sets ``optimizer.lr`` and ``optimizer.mom`` before every iteration
(det3d/torchie/trainer/trainer_sessd.py:339-341); with ``sessd_b200.train.ArenaAdamW`` the momentum is Adam's beta1 of that step.  The
arithmetic and the phase boundaries (``int(start * total_step)``) are the reference's, so the values are equal, not close."""
from functools import partial

import numpy as np


class LRSchedulerStep(object):
    """Piecewise schedule: ``lr_phases`` / ``mom_phases`` are ``(start fraction, f(pct))`` pairs; at ``step`` the last phase that has
    started sets the value, with pct = (step - start) / (end - start) over that phase's integer step range."""

    def __init__(self, fai_optimizer, total_step, lr_phases, mom_phases):
        self.optimizer = fai_optimizer
        self.total_step = total_step
        self.lr_phases = self._phases(lr_phases, total_step)
        assert self.lr_phases[0][0] == 0
        self.mom_phases = self._phases(mom_phases, total_step)
        if self.mom_phases:
            assert self.mom_phases[0][0] == 0

    @staticmethod
    def _phases(phases, total_step):
        out = []
        for i, (start, func) in enumerate(phases):
            if not callable(func):
                raise TypeError("schedule phases take callables f(pct)")
            begin = int(start * total_step)
            end = int(phases[i + 1][0] * total_step) if i < len(phases) - 1 else total_step
            assert not out or out[-1][0] < begin
            out.append((begin, end, func))
        return out

    def step(self, step):
        lrs = [func((step - start) / (end - start)) for start, end, func in self.lr_phases if step >= start]
        if lrs:
            self.optimizer.lr = lrs[-1]
        moms = [func((step - start) / (end - start)) for start, end, func in self.mom_phases if step >= start]
        if moms:
            self.optimizer.mom = moms[-1]


def annealing_cos(start, end, pct):
    "Cosine anneal from `start` to `end` as pct goes from 0.0 to 1.0."
    cos_out = np.cos(np.pi * pct) + 1
    return end + (start - end) / 2 * cos_out


class OneCycle(LRSchedulerStep):
    """lr: cosine from lr_max / div_factor up to lr_max over the first ``pct_start`` of the steps, then down to lr_max / div_factor / 1e4;
    mom: cosine from moms[0] down to moms[1], then back.  Construction sets lr = lr_max / div_factor and mom = moms[0]."""

    def __init__(self, fai_optimizer, total_step, lr_max, moms, div_factor, pct_start):
        self.lr_max = lr_max
        self.moms = moms
        self.div_factor = div_factor
        self.pct_start = pct_start
        low_lr = self.lr_max / self.div_factor
        lr_phases = ((0, partial(annealing_cos, low_lr, self.lr_max)), (self.pct_start, partial(annealing_cos, self.lr_max, low_lr / 1e4)))
        mom_phases = ((0, partial(annealing_cos, *self.moms)), (self.pct_start, partial(annealing_cos, *self.moms[::-1])))
        fai_optimizer.lr, fai_optimizer.mom = low_lr, self.moms[0]
        super().__init__(fai_optimizer, total_step, lr_phases, mom_phases)
