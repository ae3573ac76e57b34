from .train_sessd import _create_learning_rate_scheduler, build_one_cycle_optimizer, train_detector

__all__ = ["build_one_cycle_optimizer", "train_detector"]
