"""Evaluate an SE-SSD checkpoint on the KITTI validation split (reference: tools/test.py).

    python -m sessd_b200.kitti_test CONFIG CHECKPOINT [--data-root DIR] [--out predictions.pkl]

Runs the detector over ``data.val`` in batches built on the device, prints the official R11 and R40 AP strings, and with ``--out``
pickles the predictions (token -> box3d_lidar, scores, label_preds, metadata, tensors on the host)."""
import pickle
import sys


def evaluate(cfg, checkpoint):
    """(results dict, predictions) of ``checkpoint`` on cfg.data.val"""
    from det3d.datasets import build_dataloader, build_dataset
    from det3d.models import build_detector
    from det3d.torchie.trainer import load_checkpoint
    from det3d.torchie.trainer.trainer_sessd import compute_on_dataset
    dataset = build_dataset(cfg.data.val)
    loader = build_dataloader(dataset, cfg.data.samples_per_gpu, cfg.data.workers_per_gpu, dist=False, cfg=cfg)
    model = build_detector(cfg.model, train_cfg=None, test_cfg=cfg.test_cfg)
    load_checkpoint(model, checkpoint, map_location="cpu")
    predictions = compute_on_dataset(model.cuda(), loader)
    results, _ = dataset.evaluation(predictions)
    return results, predictions


def main(argv=None):
    import argparse

    from .kitti_train import load_config
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("config")
    ap.add_argument("checkpoint")
    ap.add_argument("--data-root", default=None)
    ap.add_argument("--out", default=None)
    a = ap.parse_args(argv)
    results, predictions = evaluate(load_config(a.config, a.data_root), a.checkpoint)
    if a.out:
        with open(a.out, "wb") as f:
            pickle.dump(predictions, f)
    for k, v in list(results["results"].items()) + list(results["results_2"].items()):
        print("Evaluation %s: %s" % (k, v))


if __name__ == "__main__":
    sys.exit(main())
