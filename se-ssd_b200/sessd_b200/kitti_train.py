"""Train SE-SSD on a prepared KITTI tree (reference: tools/train.py).

    python -m sessd_b200.kitti_train CONFIG [--pretrain] [--work-dir DIR] [--data-root DIR] [--resume-from CKPT] [--load-from CKPT]
                                            [--seed N] [--total-epochs N]

CONFIG is the SE-SSD config file (examples/second/configs/config.py of the reference, unchanged).  ``--data-root`` is the KITTI
``object`` directory prepared by ``python -m sessd_b200.kitti_prep``: it replaces the directory of every ``root_path``, ``info_path`` and
``db_info_path`` in the config.  ``--resume-from`` is relative to the work dir unless absolute.  Checkpoints (``epoch_{n}.pth`` and
``epoch_{n}_ema.pth``) and the log go to the work dir; the final validation's R11 / R40 strings are logged.

SE-SSD trains in two stages.  ``--pretrain`` runs the first, CIA-SSD pre-training: one model, the supervised CIA-SSD loss, the config's
pipeline and optimiser, checkpoints ``epoch_{n}.pth`` only; the config's ``load_from`` is ignored.  The second stage (no ``--pretrain``)
is the teacher / student loop; with ``my_paras.enable_ssl`` it starts both models from ``load_from``, which ``--load-from`` sets (a path
as given, e.g. the first stage's ``latest.pth``)."""
import os
import sys

_PATH_KEYS = ("root_path", "info_path", "db_info_path")


def override_data_root(cfg, data_root):
    """point every data path of the config at ``data_root``: root_path becomes it, info / db-info pickles keep their file names"""
    root = os.path.abspath(data_root)

    def walk(node):
        if isinstance(node, dict):
            for k in list(node.keys()):
                if k in _PATH_KEYS and isinstance(node[k], str):
                    node[k] = root if k == "root_path" else os.path.join(root, os.path.basename(node[k]))
                else:
                    walk(node[k])
        elif isinstance(node, (list, tuple)):
            for v in node:
                walk(v)
    for key in ("data", "db_sampler", "train_preprocessor"):
        if key in cfg:
            walk(cfg[key])
    return cfg


def load_config(path, data_root=None):
    from det3d.torchie import Config
    cfg = Config.fromfile(path)
    return override_data_root(cfg, data_root) if data_root else cfg


def build_datasets(cfg, pretrain=False):
    """[train, (unlabelled, when my_paras.enable_ssl and not pretrain), (val, when the workflow has a val phase)] as tools/train.py
    builds them"""
    from det3d.datasets import build_dataset
    datasets = [build_dataset(cfg.data.train)]
    if not pretrain and cfg.get("my_paras", {}).get("enable_ssl", False):
        datasets.append(build_dataset(cfg.data.train_unlabel_val))
    if len(cfg.workflow) == 2:
        datasets.append(build_dataset(cfg.data.val))
    return datasets


def train(cfg, pretrain=False):
    """build the detector and datasets of ``cfg`` and run the SE-SSD train_detector, or with ``pretrain`` the single-model (CIA-SSD)
    one; returns the final validation's results"""
    from det3d import __version__
    from det3d.models import build_detector
    if pretrain:
        from det3d.torchie.apis.train import train_detector
    else:
        from det3d.torchie.apis import train_detector
    model = build_detector(cfg.model, train_cfg=cfg.train_cfg, test_cfg=cfg.test_cfg)
    datasets = build_datasets(cfg, pretrain)
    if cfg.get("checkpoint_config") is not None:
        cfg.checkpoint_config.meta = dict(det3d_version=__version__, config=cfg.text, CLASSES=datasets[0].CLASSES)
    model.CLASSES = datasets[0].CLASSES
    return train_detector(model, datasets, cfg)


def main(argv=None):
    import argparse
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("config")
    ap.add_argument("--work-dir", default=None)
    ap.add_argument("--data-root", default=None)
    ap.add_argument("--pretrain", action="store_true", help="the first stage: CIA-SSD pre-training of one model")
    ap.add_argument("--resume-from", default=None)
    ap.add_argument("--load-from", default=None, help="checkpoint the SE-SSD stage starts teacher and student from")
    ap.add_argument("--seed", type=int, default=None)
    ap.add_argument("--total-epochs", type=int, default=None)
    a = ap.parse_args(argv)
    cfg = load_config(a.config, a.data_root)
    if a.work_dir is not None:
        cfg.work_dir = a.work_dir
    if a.resume_from is not None:
        cfg.resume_from = os.path.join(cfg.work_dir, a.resume_from)
    if a.load_from is not None:
        cfg.load_from = os.path.abspath(a.load_from)
    if a.seed is not None:
        cfg.seed = a.seed
    if a.total_epochs is not None:
        cfg.total_epochs = a.total_epochs
    train(cfg, a.pretrain)


if __name__ == "__main__":
    sys.exit(main())
