"""Seeded model parameters: re-export of sessd_data.weights (the generators live in the library-free package)."""
from sessd_data.weights import *  # noqa: F401,F403
from sessd_data.weights import (SSFA_CONVS, add_task_heads, bench_detector_state, kitti_car_anchors,  # noqa: F401
                                random_detector_state, split_detector_state, task_anchors)
