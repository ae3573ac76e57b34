"""The KITTI GT database (reference: det3d/datasets/utils/create_gt_database.py): one `.bin` of box-relative points per labelled object
and dbinfos_train.pkl, as DataBaseSamplerV2.load_database reads them.  A thin call into sessd_b200.kitti_prep; the points come from the
reduced sweep when it exists (LoadPointCloudFromFile), the membership runs on the device."""
import pickle
from pathlib import Path


def create_groundtruth_database(dataset_class_name, data_path, info_path=None, used_classes=None, db_path=None, dbinfo_path=None,
                                relative_path=True, add_rgb=False, lidar_only=False, bev_only=False, coors_range=None,
                                gt_aug_with_context=-1.0, **kwargs):
    from sessd_b200 import kitti_prep
    if dataset_class_name != "KITTI":
        raise NotImplementedError("only the KITTI database is supported")
    if gt_aug_with_context > 0.0:
        raise NotImplementedError("the enlarged GT database (gt_aug_with_context > 0) is not supported")
    root = Path(data_path)
    db_path = Path(db_path) if db_path is not None else root / "gt_database"
    dbinfo_path = Path(dbinfo_path) if dbinfo_path is not None else root / "dbinfos_train.pkl"
    with open(info_path, "rb") as f:
        infos = pickle.load(f)
    infos = [dict(i, point_cloud=dict(i["point_cloud"], velodyne_path=_loaded_path(root, i["point_cloud"]["velodyne_path"])))
             for i in infos]
    db = kitti_prep._DbWriter(db_path, used_classes, relative_path)
    kitti_prep.prepare(root, infos, False, remove_outside=False, db=db)
    db.dump(dbinfo_path)


def _loaded_path(root, velodyne_path):
    """the file LoadPointCloudFromFile reads: the reduced sweep when it exists, else the raw one (absolute)"""
    p = Path(velodyne_path)
    if not p.is_absolute():
        p = root / velodyne_path
    reduced = p.parent.parent / (p.parent.stem + "_reduced") / p.name
    return str(reduced if reduced.exists() else p)
