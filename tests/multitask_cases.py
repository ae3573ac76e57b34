"""Three-class (Car, Pedestrian, Cyclist) variants of the reference config for the multi-class inference tests: three one-class
tasks, each with its own anchor size and z.  Values: Pedestrian 0.6 x 0.8 x 1.73 and Cyclist 0.6 x 1.76 x 1.73 (w, l, h) on the
z = -0.6 plane; Car as in the single-class config."""
import copy
import json
import os

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF_CFG = os.path.join(ROOT, "tests", "golden", "reference_config.json")
NAMES = ["Car", "Pedestrian", "Cyclist"]
TASKS = [dict(num_class=1, class_names=[n]) for n in NAMES]
SIZES = {"Car": ([1.6, 3.9, 1.56], -1.0), "Pedestrian": ([0.6, 0.8, 1.73], -0.6), "Cyclist": ([0.6, 1.76, 1.73], -0.6)}
GENERATORS = [dict(type="anchor_generator_range", sizes=SIZES[n][0], anchor_ranges=[0, -40.0, SIZES[n][1], 70.4, 40.0, SIZES[n][1]],
                   rotations=[0, 1.57], matched_threshold=0.6, unmatched_threshold=0.45, class_name=n) for n in NAMES]


def three_class(d):
    """a copy of a plain config dict with every tasks / anchor_generators / class_names entry replaced by the three-class ones"""
    d = copy.deepcopy(d)

    def walk(x):
        if isinstance(x, dict):
            for k in list(x):
                if k == "tasks":
                    x[k] = copy.deepcopy(TASKS)
                elif k == "anchor_generators":
                    x[k] = copy.deepcopy(GENERATORS)
                elif k == "class_names":
                    x[k] = list(NAMES)
                else:
                    walk(x[k])
        elif isinstance(x, list):
            for v in x:
                walk(v)
    walk(d)
    return d


def three_class_config(data_root):
    """the reference config (as tests.test_kitti_train.reference_config builds it) with three one-class tasks"""
    from det3d.torchie import Config
    from sessd_b200.kitti_train import override_data_root
    d = three_class(json.load(open(REF_CFG)))
    ours = Config.fromfile(os.path.join(ROOT, "examples", "second", "configs", "config.py"))
    d["model"]["neck"]["logger"] = ours.model.neck.logger
    d["model"]["bbox_head"]["box_coder"] = ours.model.bbox_head.box_coder
    return override_data_root(Config(d), data_root)
