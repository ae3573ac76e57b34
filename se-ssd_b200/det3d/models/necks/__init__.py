"""BEV necks on the hot path: the SSFA block of SE-SSD (runs on csrc/bevconv_p2.cu through sessd_b200.runners.SSFAPlanesRunner)."""
from .rpn_v1 import SSFA

__all__ = ["SSFA"]
