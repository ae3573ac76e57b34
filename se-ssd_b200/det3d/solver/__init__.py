from .learning_schedules_fastai import LRSchedulerStep, OneCycle, annealing_cos

__all__ = ["LRSchedulerStep", "OneCycle", "annealing_cos"]
