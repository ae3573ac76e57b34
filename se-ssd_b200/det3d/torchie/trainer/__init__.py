from .checkpoint import load_checkpoint, load_state_dict, save_checkpoint, weights_to_cpu

from .trainer_sessd import Trainer, sigmoid_rampup, update_ema_variables

__all__ = ["load_checkpoint", "load_state_dict", "save_checkpoint", "weights_to_cpu", "Trainer", "sigmoid_rampup", "update_ema_variables"]
