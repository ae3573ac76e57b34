"""String -> object builders used by the config file and the data pipeline (reference: det3d/builder.py:26-35, 38-65, 409-442,
445-500).  ``build_box_coder`` is called INSIDE examples/second/configs/config.py (config.py:5,69)."""
from det3d.core.anchor.anchor_generator import AnchorGeneratorRange
from det3d.core.bbox import region_similarity
from det3d.core.bbox.box_coders import GroundBox3dCoderTorch
from det3d.core.input.voxel_generator import VoxelGenerator


def build_voxel_generator(voxel_config):
    return VoxelGenerator(voxel_size=voxel_config.VOXEL_SIZE, point_cloud_range=voxel_config.RANGE,
                          max_num_points=voxel_config.MAX_POINTS_NUM_PER_VOXEL, max_voxels=20000)


def build_similarity_metric(similarity_config):
    kind = similarity_config.type
    if kind == "nearest_iou_similarity":
        return region_similarity.NearestIouSimilarity()
    raise ValueError("unknown / unsupported similarity type %r (the SE-SSD config uses nearest_iou_similarity)" % kind)


def build_box_coder(box_coder_config):
    kind = box_coder_config["type"]
    if kind == "ground_box3d_coder":
        return GroundBox3dCoderTorch(box_coder_config["linear_dim"], box_coder_config["encode_angle_vector"],
                                     n_dim=box_coder_config.get("n_dim", 9), norm_velo=box_coder_config.get("norm_velo", False))
    raise ValueError("unknown box_coder type")


def build_anchor_generator(anchor_config):
    velocities = anchor_config.velocities if "velocities" in anchor_config else None
    if anchor_config.type == "anchor_generator_range":
        return AnchorGeneratorRange(sizes=anchor_config.sizes, anchor_ranges=anchor_config.anchor_ranges,
                                    rotations=anchor_config.rotations, velocities=velocities,
                                    match_threshold=anchor_config.matched_threshold,
                                    unmatch_threshold=anchor_config.unmatched_threshold, class_name=anchor_config.class_name)
    raise ValueError(" unknown anchor generator type")


def build_db_preprocess(db_prep_config, logger=None):
    """reference det3d/builder.py:67-77"""
    from det3d.core.sampler import preprocess as prep
    cfg = db_prep_config
    if "filter_by_difficulty" in cfg:
        return prep.DBFilterByDifficulty(cfg["filter_by_difficulty"], logger=logger)
    elif "filter_by_min_num_points" in cfg:
        return prep.DBFilterByMinNumPoint(cfg["filter_by_min_num_points"], logger=logger)
    raise ValueError("unknown database prep type")


def build_dbsampler(cfg, logger=None, random_state=None):
    """reference det3d/builder.py:378-405: the filters in config order, the info pickle, DataBaseSamplerV2.  The database files are read
    relative to the pickle's directory unless ``sample_all`` is given another root; random_state defaults to the np.random module.
    ``global_random_rotation_range_per_object`` is read and ignored, as in sample_ops_v2."""
    import os
    import pickle

    import numpy as np

    from det3d.core.sampler import DataBasePreprocessor, DataBaseSamplerV2
    prepors = [build_db_preprocess(c, logger=logger) for c in cfg["db_prep_steps"]]
    grot_range = list(cfg["global_random_rotation_range_per_object"]) or None
    if cfg["gt_aug_with_context"] > 0.0:
        raise NotImplementedError("gt_aug_with_context > 0 is not supported (the SE-SSD car config does not use it)")
    with open(cfg["db_info_path"], "rb") as f:
        db_infos = pickle.load(f)
    sampler = DataBaseSamplerV2(db_infos, cfg["sample_groups"], DataBasePreprocessor(prepors), cfg["rate"], grot_range, logger=logger,
                                gt_random_drop=cfg["gt_random_drop"], gt_aug_with_context=cfg["gt_aug_with_context"],
                                gt_aug_similar_type=cfg["gt_aug_similar_type"],
                                random_state=np.random if random_state is None else random_state)
    sampler.root_path = os.path.dirname(os.path.abspath(cfg["db_info_path"]))
    return sampler
