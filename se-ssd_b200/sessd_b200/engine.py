"""FrameEngine: the whole per-frame hot path (points -> detections) as ONE CUDA graph per batch of frames.

    host points (pinned) --H2D--> voxelise(+VFE mean) -> 8 rulebooks + 14 sparse convs -> dense -> SSFA (16 conv launches)
    -> head GEMM -> score/top-k/decode/rotated NMS/finalize --D2H--> detections (pinned)

Reference call stack being replaced: tools/test.py:121-142 -> VoxelNet.forward (detectors/voxelnet_sessd.py:18-43) with
voxelisation moved from the DataLoader workers (datasets/pipelines/preprocess.py:196-232) onto the GPU.  The reference
syncs with the host >= 3 times per frame; this engine syncs once (when the caller asks for the results).
Frames are independent: multi-GPU = one engine per rank on its own shard of frames, no collective (bench.py).

A multi-class detector (MultiGroupHead with T one-class tasks, e.g. Car, Pedestrian, Cyclist) runs with ``num_tasks=T``: one head GEMM
writes the T tasks' 24-channel blocks and one post-processing pass handles every (frame, task) slot; ``label_preds`` is the task.
"""
import numpy as np
import torch

from . import ops, synth
from .runners import HEAD_TASK_STRIDE, SpMiddleRunner, SSFAPlanesRunner


class FrameEngine:
    def __init__(self, batch=1, max_points_per_frame=32768, voxel_size=synth.VOXEL_SIZE, pc_range=synth.PC_RANGE,
                 max_points_per_voxel=5, max_voxels=20000, device="cuda", post_kwargs=None, growth=None, skip_constant=True, num_tasks=1):
        """skip_constant: the neck computes only the tiles whose receptive field reaches a LiDAR site or the map border and fills the
        rest with their bit-identical empty-space constant (runners.SSFAPlanesRunner).
        num_tasks: one-class tasks of the head (load_weights then takes one anchor array per task); post_kwargs apply to every task"""
        self.batch, self.device = int(batch), torch.device(device)
        self.max_points = int(max_points_per_frame) * self.batch
        self.vcfg = ops.make_voxel_cfg(voxel_size, pc_range, max_points_per_voxel, max_voxels)
        self.grid_xyz = [int(self.vcfg.grid[j]) for j in range(3)]
        dev = self.device
        # I/O staging (pinned host <-> device)
        self.h_points = torch.zeros((self.max_points, 4), dtype=torch.float32).pin_memory()
        self.h_off = torch.zeros((self.batch + 1,), dtype=torch.int32).pin_memory()
        self.d_points = torch.zeros((self.max_points, 4), dtype=torch.float32, device=dev)
        self.d_off = torch.zeros((self.batch + 1,), dtype=torch.int32, device=dev)
        self.vox = ops.VoxelBuffers(self.vcfg, self.batch, self.max_points, dev, with_mean=True)
        self.middle = SpMiddleRunner(self.batch, self.batch * max_voxels, self.grid_xyz, 4, dev, growth=growth)
        self.num_tasks = int(num_tasks)
        self.neck = SSFAPlanesRunner(self.batch, (self.grid_xyz[1] // 8, self.grid_xyz[0] // 8), dev, skip_constant=skip_constant,
                                     num_tasks=self.num_tasks)
        self.anchors = None
        pk = dict(batch=self.batch, head_stride=self.neck.HEAD_STRIDE, num_tasks=self.num_tasks, task_stride=HEAD_TASK_STRIDE)
        pk.update(post_kwargs or {})
        self.pcfg = ops.make_post_cfg(**pk)
        self.post = ops.PostBuffers(self.pcfg, dev)
        P = ops.post_capacity(self.pcfg)
        # packed result block (written by post_finalize_kernel, or post_merge_kernel for several tasks): [B,P,8] = box 7 | score;
        # meta [B, 8+P] = count, candidates, pre-NMS, NMS-selected, voxels, capacity status, 0, 0, anchor index of every returned
        # detection into the tasks' concatenated anchors; P = tasks x the per-task capacity
        self.d_result = torch.zeros((self.batch, P, 8), dtype=torch.float32, device=dev)
        self.h_result = torch.zeros((self.batch, P, 8), dtype=torch.float32).pin_memory()
        self.d_meta = torch.zeros((self.batch, 8 + P), dtype=torch.int32, device=dev)
        self.h_meta = torch.zeros((self.batch, 8 + P), dtype=torch.int32).pin_memory()
        self.frustum = None
        self.graph = None
        self.graph_dev = None
        self.stream = torch.cuda.Stream(device=dev)

    # ---------------------------------------------------------------------------------------------- weights
    def load_weights(self, middle_layers, ssfa_state, head_state, anchors, head_prefix="tasks.0."):
        """anchors: [A, 7] of a one-task head, or a list of the T tasks' [A, 7] arrays (task_anchors); with several tasks every
        ``tasks.{t}.`` head of head_state is loaded (head_prefix is then ignored)"""
        if isinstance(anchors, (list, tuple)):
            if len(anchors) != self.num_tasks:
                raise ValueError("%d anchor arrays for a %d-task engine" % (len(anchors), self.num_tasks))
            arr = np.stack([np.asarray(a, np.float32).reshape(-1, 7) for a in anchors])
            if self.num_tasks > 1:
                head_prefix = ["tasks.%d." % t for t in range(self.num_tasks)]
        elif self.num_tasks != 1:
            raise ValueError("a %d-task engine takes a list of per-task anchor arrays" % self.num_tasks)
        else:
            arr = np.asarray(anchors, np.float32)
        self.middle.load_weights(middle_layers)
        self.neck.load_state(ssfa_state, head_state, head_prefix)
        self.anchors = torch.as_tensor(arr.reshape(-1, 7)).to(self.device).contiguous()
        assert self.anchors.shape[0] == self.num_tasks * self.pcfg.num_anchors
        self.graph = None

    # ---------------------------------------------------------------------------------------------- device pipeline
    def _device_pipeline(self):
        """All launches of one batch of frames on the current stream (capturable)."""
        ops.voxelize(self.d_points, self.d_off, self.vox)
        head = self.sparse_and_neck()
        ops.postprocess_packed(head, self.anchors, self.frustum, self.post, self.d_result, self.d_meta,
                               self.vox.num_voxels[:self.batch], self.middle.status)

    def sparse_and_neck(self, mark=None):
        """sparse encoder + dense() + neck + head on the current stream; returns the head map.  mark(label) is called after every
        launch group (profiling).  dense() writes the fp16 (hi, lo) planes of the neck input directly."""
        n0 = self.vox.num_voxels[self.batch:self.batch + 1]
        self.neck.info.zero_()
        self.middle.forward(self.vox.mean, self.vox.coors, n0, mark=mark, dense_planes=(self.neck.planes["x"], self.neck.info[0]))
        last = self.middle.levels[-1]
        _, head = self.neck.forward(None, mark=mark, occupancy=(last["index"], last["grid"]))
        return head

    def _step_body(self):
        self.d_points.copy_(self.h_points, non_blocking=True)
        self.d_off.copy_(self.h_off, non_blocking=True)
        self._device_pipeline()
        self.h_result.copy_(self.d_result, non_blocking=True)
        self.h_meta.copy_(self.d_meta, non_blocking=True)

    def capture(self):
        """Warm up once eagerly, then capture H2D + pipeline + D2H into a CUDA graph."""
        with torch.cuda.stream(self.stream):
            self._step_body()
            self.stream.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.stream):
                self._step_body()
        self.graph = g
        return g

    def capture_device_only(self):
        """Graph of the device pipeline alone (inputs already in d_points / d_off): bench.py's HBM-resident `value` loop."""
        with torch.cuda.stream(self.stream):
            self._device_pipeline()
            self.stream.synchronize()
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=self.stream):
                self._device_pipeline()
        self.graph_dev = g
        return g

    # ---------------------------------------------------------------------------------------------- host API
    def stage(self, clouds):
        """Copy a list of ``batch`` numpy point clouds [N_i,4] into the pinned staging buffers."""
        assert len(clouds) == self.batch
        off = 0
        hp = self.h_points.numpy()
        ho = self.h_off.numpy()
        for f, c in enumerate(clouds):
            n = c.shape[0]
            if off + n > self.max_points:
                raise ValueError("point capacity exceeded")
            hp[off:off + n] = c
            ho[f] = off
            off += n
        ho[self.batch] = off
        return off

    def launch(self):
        """Enqueue one batch (graph replay if captured).  Asynchronous."""
        if self.graph is not None:
            with torch.cuda.stream(self.stream):
                self.graph.replay()
        else:
            with torch.cuda.stream(self.stream):
                self._step_body()

    def results(self):
        """Synchronise and unpack: list of dict(box3d_lidar [K,7], scores [K], label_preds [K] (the task), anchor_index [K] (into the
        tasks' concatenated anchors))."""
        self.stream.synchronize()
        meta = self.h_meta.numpy()
        if int(meta[:, 5].max()) != 0:
            raise RuntimeError("sparse active-site capacity exceeded (status=%d); raise `growth`" % int(meta[:, 5].max()))
        return unpack_results(self.h_result.numpy(), meta, self.pcfg.num_anchors)

    def infer(self, clouds):
        self.stage(clouds)
        self.launch()
        return self.results()


def unpack_results(result, meta, num_anchors):
    """per-frame detection dicts of a packed result block [B, P, 8] (box 7 | score) and its meta [B, 8 + P] (see FrameEngine):
    label_preds = anchor index // num_anchors, the task of a detection, which is the reference's label of one-class tasks (their class
    offsets are 0, 1, 2 ...)"""
    out = []
    for f in range(result.shape[0]):
        k = int(meta[f, 0])
        idx = meta[f, 8:8 + k].astype(np.int64)
        out.append(dict(box3d_lidar=result[f, :k, :7].copy(), scores=result[f, :k, 7].copy(), label_preds=idx // int(num_anchors),
                        num_voxels=int(meta[f, 4]), num_candidates=int(meta[f, 1]), anchor_index=idx))
    return out
