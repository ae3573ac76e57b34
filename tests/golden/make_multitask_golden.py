"""Generate tests/golden/anchors_multitask.npz: the Car, Pedestrian and Cyclist anchors of a three-task KITTI config, from the
REFERENCE's own AnchorGeneratorRange and TargetAssigner.generate_anchors_dict, loaded where they lie as make_golden.py loads them.

Run once where the reference tree exists (``python tests/golden/make_multitask_golden.py``); the tests read only the .npz."""
import os
import sys

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
import make_golden as mg  # noqa: E402

# (class, sizes w/l/h, z of the anchor plane): one one-class task each
CLASSES = (("Car", (1.6, 3.9, 1.56), -1.0), ("Pedestrian", (0.6, 0.8, 1.73), -0.6), ("Cyclist", (0.6, 1.76, 1.73), -0.6))


def gen():
    bn = mg._load("det3d.core.bbox.box_np_ops", "det3d/core/bbox/box_np_ops.py")
    sys.modules["det3d.core.bbox"].box_np_ops = bn
    bt = mg._load("det3d.core.bbox.box_torch_ops", "det3d/core/bbox/box_torch_ops.py")
    sys.modules["det3d.core.bbox"].box_torch_ops = bt
    rs = mg._load("det3d.core.bbox.region_similarity", "det3d/core/bbox/region_similarity.py")
    bc = mg._load("det3d.core.bbox.box_coders", "det3d/core/bbox/box_coders.py")
    ag_mod = mg._load("det3d.core.anchor.anchor_generator", "det3d/core/anchor/anchor_generator.py")
    mg._load("det3d.core.anchor.target_ops_v2", "det3d/core/anchor/target_ops_v2.py")
    ta_mod = mg._load("det3d.core.anchor.target_assigner", "det3d/core/anchor/target_assigner.py")
    out = {}
    for name, sizes, z in CLASSES:
        ag = ag_mod.AnchorGeneratorRange(anchor_ranges=[0, -40.0, z, 70.4, 40.0, z], sizes=list(sizes), rotations=[0, 1.57],
                                         velocities=None, class_name=name, match_threshold=0.6, unmatch_threshold=0.45)
        ta = ta_mod.TargetAssigner(box_coder=bc.GroundBox3dCoderTorch(linear_dim=False, vec_encode=False, n_dim=7),
                                   anchor_generators=[ag], region_similarity_calculator=rs.NearestIouSimilarity(),
                                   positive_fraction=None, sample_size=512)
        a = ta.generate_anchors_dict([1, 200, 176])[name]["anchors"]
        a = np.ascontiguousarray(a.reshape(-1, 7), np.float32)
        # the whole array by its hash (bit for bit), plus its first and last rows readable
        out[name + "_sha"], out[name + "_head"], out[name + "_tail"] = mg.sha(a), a[:704].copy(), a[-704:].copy()
        out[name + "_shape"] = np.asarray(a.shape)
        print(name, a.shape, a.dtype)
    np.savez_compressed(os.path.join(HERE, "anchors_multitask.npz"), **out)


if __name__ == "__main__":
    mg.install_det3d_shims()
    gen()
