from .optimizer import OptimizerHook

__all__ = ["OptimizerHook"]
