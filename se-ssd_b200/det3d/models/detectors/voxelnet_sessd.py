"""VoxelNet detector with the reference's call contract (det3d/models/detectors/voxelnet_sessd.py): ``forward(example, is_ema,
return_loss)`` takes the collate_kitti batch dict (voxels, coordinates with a batch column, num_points, num_voxels, shape, anchors, calib,
metadata; ``*_raw`` twins for the teacher branch) and returns per-frame detection dicts (``return_loss=False``), the head outputs
(teacher branch) or the loss (SE-SSD's, or CIA-SSD's with ``stage="ciassd"``); every stage runs on the sessd_b200 CUDA kernels."""
from ..registry import DETECTORS
from .single_stage import SingleStageDetector

_STAGE_INPUTS = (("voxels", "voxels"), ("num_points_per_voxel", "num_points"), ("coors", "coordinates"))


@DETECTORS.register_module
class VoxelNet(SingleStageDetector):
    def __init__(self, reader, backbone, neck, bbox_head, train_cfg=None, test_cfg=None, pretrained=None):
        super().__init__(reader, backbone, neck, bbox_head, train_cfg, test_cfg, pretrained)

    def extract_feat(self, data):
        voxel_features = self.reader(data["voxels"], data["num_points_per_voxel"])
        bev = self.backbone(voxel_features, data["coors"], data["batch_size"], data["input_shape"])
        return self.neck(bev) if self.with_neck else bev

    def forward(self, example, is_ema=[False, None], return_loss=True, stage="sessd", **kwargs):
        """``stage="ciassd"``: the loss is the CIA-SSD pre-training loss (MultiGroupHead.loss_ciassd, reference
        det3d/models/detectors/voxelnet.py), which reads no ``*_raw`` keys and no teacher predictions."""
        if stage not in ("sessd", "ciassd"):
            raise ValueError("stage must be 'sessd' or 'ciassd', got %r" % (stage,))
        teacher, preds_ema = is_ema[0], is_ema[1]
        suffix = "_raw" if teacher else ""              # the teacher sees the un-augmented copy of the frame
        data = {name: example[key + suffix] for name, key in _STAGE_INPUTS}
        data["batch_size"] = len(example["num_voxels" + suffix])
        data["input_shape"] = example["shape" + suffix][0]
        preds = self.bbox_head(self.extract_feat(data))
        if teacher:
            return preds
        if not return_loss:
            return self.bbox_head.predict(example, preds, self.test_cfg)
        if stage == "ciassd":
            return self.bbox_head.loss_ciassd(example, preds)
        return self.bbox_head.loss(example, preds, preds_ema)
