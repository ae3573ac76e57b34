"""Batches of KITTI frames built on the device (reference: det3d/datasets/loader/build_loader.py, a torch DataLoader over the dataset
with collate_kitti).

The host reads frames (``dataset[i]``: one ``np.fromfile``, the boxes in the lidar frame, the calibration frustum) on one reader thread,
one batch ahead of the device.  Every per-point stage then runs on the device:

* train mode: ``augment.launch_train_batch`` -- GT-AUG, per-object noise, global flip / rotation / scaling, SA-DA with the car values
  the reference's Preprocess hard-codes, the shuffle, both voxelisations and both target assignments;
* val / test mode: the reference's test pipeline (Preprocess with shuffle_points=False leaves the points as read, Voxelization,
  AssignTarget's anchors, Reformat) and collate_kitti: the clouds go up in one copy and ``ops.voxelize`` fills ``ops.VoxelBuffers``.

Random streams: everything random in epoch ``e`` -- the frame order, the augmentation RandomState and the GT-AUG class streams -- is a
function of ``(seed, e)`` (``epoch_streams``, ``restart_sampler``), so an epoch needs no saved RNG state and a resumed run draws what the
uninterrupted run drew.  The reference draws from each DataLoader worker's ``np.random``, which cannot be reproduced."""
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import torch

from . import augment, ops
from .sada import SadaConfig


def epoch_streams(seed, epoch, num_frames, shuffle=True):
    """(frame order, augmentation RandomState) of epoch ``epoch``"""
    order = np.random.RandomState([seed, epoch, 0]).permutation(num_frames) if shuffle else np.arange(num_frames)
    return order, np.random.RandomState([seed, epoch, 1])


def restart_sampler(db_sampler, rs):
    """Point every GT-AUG class stream at ``rs`` and restart it from a fresh shuffle of its objects (BatchSampler._reset), so the
    streams of an epoch depend on that epoch's ``rs`` alone.  The database stays on the device."""
    db_sampler._set_random_state(rs)
    for s in db_sampler._sampler_dict.values():
        s._indices = np.arange(s._example_num)
        s._reset()


class DeviceLoader:
    """Iterable of ``example`` dicts whose tensors are on ``device``; ``len()`` batches per epoch (the last one partial).  The dataset's
    mode (its pipeline's Preprocess mode) chooses the train or the val / test batch.  Train mode shuffles the frames; val / test mode keeps the info order (predictions are keyed by token, so the order does not change a result).
    Each ``iter()`` runs epoch ``self.epoch`` and advances it; ``set_epoch`` chooses the epoch, as a resumed run does.
    twin=False: training batches carry the student's branch only (no ``*_raw`` keys), as single-model (CIA-SSD) training reads them."""

    def __init__(self, dataset, batch_size, cfg, seed=0, device=None, twin=True):
        self.dataset, self.batch_size, self.cfg, self.seed, self.twin = dataset, int(batch_size), cfg, int(seed), bool(twin)
        self.device = torch.device("cuda", torch.cuda.current_device()) if device is None else torch.device(device)
        self.train = dataset.mode == "train"
        self.epoch = 0
        self.db_sampler = None
        if self.train and not dataset.labeled:
            raise NotImplementedError("unlabelled training frames are not batched (the reference never draws from that loader)")
        if self.train and cfg.get("db_sampler") is not None and cfg.db_sampler.get("enable", False):
            from det3d.builder import build_dbsampler
            self.db_sampler = build_dbsampler(cfg.db_sampler, random_state=np.random.RandomState([self.seed]))
            self.db_sampler.device_database(self.device)

    def __len__(self):
        return -(-len(self.dataset) // self.batch_size)

    def set_epoch(self, epoch):
        self.epoch = int(epoch)

    def __iter__(self):
        epoch = self.epoch
        self.epoch += 1
        order, rs = epoch_streams(self.seed, epoch, len(self.dataset), shuffle=self.train)
        if self.db_sampler is not None:
            restart_sampler(self.db_sampler, rs)
        batches = [order[i:i + self.batch_size] for i in range(0, len(order), self.batch_size)]
        if not batches:
            return
        with ThreadPoolExecutor(max_workers=1) as reader:
            nxt = reader.submit(self._read, batches[0])
            for k in range(len(batches)):
                frames = nxt.result()
                if k + 1 < len(batches):
                    nxt = reader.submit(self._read, batches[k + 1])
                yield self.train_batch(frames, rs) if self.train else self.val_batch(frames)

    def _read(self, idxs):
        return [self.dataset[int(i)] for i in idxs]

    def train_batch(self, frames, rs):
        """the collated training batch of ``frames`` (dataset items), drawing from ``rs``"""
        lidar = [f["lidar"] for f in frames]
        pending = augment.launch_train_batch(self.cfg, [l["points"] for l in lidar], [l["gt_boxes"] for l in lidar],
                                             [l["gt_names"] for l in lidar], rs, device=self.device, db_sampler=self.db_sampler,
                                             sa_da=SadaConfig(), twin=self.twin)
        ex = pending.example()
        ex["metadata"] = [f["metadata"] for f in frames]
        return ex

    def val_batch(self, frames):
        """the collated evaluation batch of ``frames``: the keys the model's eval forward and MultiGroupHead.predict read"""
        from det3d.torchie.parallel import collate_kitti
        st = augment._static_eval(self.cfg, self.device)
        B = len(frames)
        clouds = [np.asarray(f["lidar"]["points"], np.float32).reshape(-1, 4) for f in frames]
        off = np.zeros(B + 1, np.int32)
        off[1:] = np.cumsum([len(c) for c in clouds])
        buf, layout = augment._pack([np.concatenate(clouds), off])
        d_pts, d_off = augment._unpack(torch.from_numpy(buf).pin_memory().to(self.device, non_blocking=True), layout)
        vox = ops.VoxelBuffers(st["vcfg"], B, max(int(off[-1]), 1), self.device)
        ops.voxelize(d_pts, d_off, vox)
        ex = augment.voxel_example(st, vox, B, int(vox.num_voxels[B].item()))          # the one read-back
        calib = collate_kitti([{"calib": f["calib"]} for f in frames])["calib"]
        ex["calib"] = {k: v.to(self.device) for k, v in calib.items()}
        ex["metadata"] = [f["metadata"] for f in frames]
        return ex


def build_dataloader(dataset, batch_size, workers_per_gpu, num_gpus=1, dist=False, cfg=None, seed=0, twin=True, **kwargs):
    """The reference's loader entry point.  ``cfg`` (the loaded config) carries the augmentation, voxeliser, assigner and db_sampler
    values; ``seed`` the random streams.  ``workers_per_gpu`` is accepted for the reference's signature: one reader thread reads ahead,
    the rest of the work is on the device.  ``twin``: see DeviceLoader.  Multi-GPU loading (dist=True) is not implemented."""
    if dist or num_gpus != 1:
        raise NotImplementedError("distributed / multi-GPU loading is not implemented")
    if cfg is None:
        raise ValueError("build_dataloader needs the loaded config (cfg=...): the batches are built from its stage values")
    return DeviceLoader(dataset, batch_size, cfg, seed, twin=twin)
