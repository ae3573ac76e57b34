"""Result-annotation constructors of the KITTI mirror (reference det3d/datasets/kitti/kitti_common.py:879-913)."""
from sessd_b200.kitti_eval import empty_anno


def get_start_result_anno():
    """Empty per-key lists that a frame's detections are appended to."""
    return {k: [] for k in ("name", "truncated", "occluded", "alpha", "bbox", "dimensions", "location", "rotation_y", "score")}


def empty_result_anno():
    """The annotation of a frame without detections: zero-length arrays, [0, 4] / [0, 3] for the box fields."""
    return empty_anno()


# ------------------------------------------------------------------------------------------------ data preparation (kitti_common.py:56-209,
# 364-450, 733-770, 824-859): thin calls into sessd_b200.kitti_prep, which reads each sweep once and tests membership on the device
def get_label_anno(label_path):
    from sessd_b200 import kitti_prep
    return kitti_prep.get_label_anno(label_path)


def add_difficulty_to_annos(info):
    from sessd_b200 import kitti_prep
    return kitti_prep.add_difficulty_to_annos(info)


def get_kitti_image_info(path, training=True, label_info=True, velodyne=False, calib=False, image_ids=7481, extend_matrix=True,
                         num_worker=8, relative_path=True, with_imageshape=True):
    """Info records of the listed frames; image_shape comes from the PNG header."""
    from sessd_b200 import kitti_prep
    if not isinstance(image_ids, list):
        image_ids = list(range(image_ids))
    return [kitti_prep.image_info(path, i, training, label_info, velodyne, calib, extend_matrix, relative_path, with_imageshape)
            for i in image_ids]


def _calculate_num_points_in_gt(data_path, infos, relative_path, remove_outside=True, num_features=4):
    """Sets annos["num_points_in_gt"] of every info in place (int32, -1 for the DontCare rows)."""
    from sessd_b200 import kitti_prep
    if num_features != 4:
        raise NotImplementedError("KITTI sweeps have 4 features per point")
    kitti_prep.prepare(data_path, infos, relative_path, count=True, remove_outside=remove_outside)


def create_kitti_info_file(data_path, save_path=None, relative_path=True, imageset_dir=None):
    """kitti_infos_{train,val,trainval,test}.pkl; the split files are read from imageset_dir (default <data_path>/ImageSets)."""
    import pickle
    from pathlib import Path

    from sessd_b200 import kitti_prep
    imageset_dir = Path(imageset_dir) if imageset_dir is not None else Path(data_path) / "ImageSets"
    save_path = Path(save_path) if save_path is not None else Path(data_path)
    ids = {s: kitti_prep.imageset_ids(imageset_dir, s) for s in ("train", "val", "test")}
    train = get_kitti_image_info(data_path, True, True, True, True, ids["train"], relative_path=relative_path)
    _calculate_num_points_in_gt(data_path, train, relative_path)
    val = get_kitti_image_info(data_path, True, True, True, True, ids["val"], relative_path=relative_path)
    _calculate_num_points_in_gt(data_path, val, relative_path)
    test = get_kitti_image_info(data_path, False, False, True, True, ids["test"], relative_path=relative_path)
    for name, obj in (("kitti_infos_train.pkl", train), ("kitti_infos_val.pkl", val), ("kitti_infos_trainval.pkl", train + val),
                      ("kitti_infos_test.pkl", test)):
        with open(save_path / name, "wb") as f:
            pickle.dump(obj, f)


def _create_reduced_point_cloud(data_path, info_path, save_path=None, back=False):
    """velodyne_reduced/*.bin: the points of each frame of the info file inside its image frustum."""
    import pickle

    from sessd_b200 import kitti_prep
    if back:
        raise NotImplementedError("the mirrored (back=True) reduced point clouds are not supported")
    with open(info_path, "rb") as f:
        infos = pickle.load(f)
    kitti_prep.prepare(data_path, infos, True, reduce=True, reduced_save_path=save_path)


def create_reduced_point_cloud(data_path, train_info_path=None, val_info_path=None, test_info_path=None, save_path=None, with_back=False):
    from pathlib import Path
    if with_back:
        raise NotImplementedError("the mirrored (with_back) reduced point clouds are not supported")
    for p, name in ((train_info_path, "kitti_infos_train.pkl"), (val_info_path, "kitti_infos_val.pkl"), (test_info_path, "kitti_infos_test.pkl")):
        _create_reduced_point_cloud(data_path, p if p is not None else Path(data_path) / name, save_path)
