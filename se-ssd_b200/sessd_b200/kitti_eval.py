"""KITTI object evaluation on the device (csrc/kitti_eval.cu through the C ABI).

Annotations are packed into flat arrays with per-frame CSR offsets; class names become small integer codes here, once, and
everything after that runs on the GPU.  `evaluate` returns, per metric, the precision / AOS / threshold arrays in the reference's
`[class, difficulty, min_overlap, 41]` layout plus the R11 / R40 averages of every curve.
"""
import ctypes as C

import numpy as np
import torch

from . import _lib

CLASS_NAMES = ("car", "pedestrian", "bicycle", "truck", "bus", "trailer", "construction_vehicle", "motorcycle", "barrier",
               "traffic_cone", "cyclist")
PERSON_SITTING, VAN = 11, 12
REC = 13
N_PTS = 41
MAX_FRAME_DT = 1024


def class_code(name):
    """Lower-cased name -> index into CLASS_NAMES, PERSON_SITTING / VAN for the neighbour classes, -1 otherwise."""
    n = str(name).lower()
    if n in CLASS_NAMES:
        return CLASS_NAMES.index(n)
    return {"person_sitting": PERSON_SITTING, "van": VAN}.get(n, -1)


def _codes(names):
    return np.array([class_code(n) for n in names], dtype=np.int32)


def _offsets(counts):
    off = np.zeros(len(counts) + 1, dtype=np.int64)
    np.cumsum(counts, out=off[1:])
    return off


def _records(anno, last):
    n = len(anno["name"])
    r = np.zeros((n, REC), dtype=np.float64)
    if n:
        r[:, 0:4] = anno["bbox"]
        r[:, 4] = anno["alpha"]
        r[:, 5:8] = anno["location"]
        r[:, 8:11] = anno["dimensions"]
        r[:, 11] = anno["rotation_y"]
        r[:, 12] = anno[last]
    return r


def pack_gt(gt_annos):
    """Host packing of ground-truth annotations (the reference's `get_label_anno` dicts)."""
    recs, codes, occ, dcs = [], [], [], []
    for a in gt_annos:
        recs.append(_records(a, "truncated"))
        codes.append(_codes(a["name"]))
        occ.append(np.asarray(a["occluded"], dtype=np.int32).reshape(-1))
        dc = np.array([n == "DontCare" or n == "ignore" for n in a["name"]], dtype=bool)
        dcs.append(np.asarray(a["bbox"], dtype=np.float64).reshape(-1, 4)[dc])
    return {"gt_off": _offsets([len(r) for r in recs]), "gt": np.concatenate(recs).reshape(-1, REC),
            "gt_code": np.concatenate(codes).astype(np.int32), "gt_occluded": np.concatenate(occ).astype(np.int32),
            "dc_off": _offsets([len(d) for d in dcs]), "dc": np.concatenate(dcs).reshape(-1, 4)}


def pack_dt(dt_annos):
    """Host packing of detection annotations (`dt_annos` as convert_detection_to_kitti_annos returns them)."""
    recs = [_records(a, "score") for a in dt_annos]
    return {"dt_off": _offsets([len(r) for r in recs]), "dt": np.concatenate(recs).reshape(-1, REC),
            "dt_code": np.concatenate([_codes(a["name"]) for a in dt_annos]).astype(np.int32)}


def _dev(x, dtype, device):
    return torch.as_tensor(np.ascontiguousarray(x), dtype=dtype).to(device)


def _rows(x, device, dtype):
    """Device copy with at least one row, so a set without boxes still passes non-null arrays (counts say it is empty)."""
    x = np.asarray(x)
    if len(x) == 0:
        x = np.zeros((1,) + x.shape[1:], dtype=x.dtype)
    return _dev(x, dtype, device)


class DeviceGT:
    """Packed ground truth on the device; it does not change between epochs, so a dataset builds it once."""

    def __init__(self, gt_annos, device="cuda"):
        h = pack_gt(gt_annos)
        self.num_frames = len(gt_annos)
        self.counts = np.diff(h["gt_off"])
        self.total = int(h["gt_off"][-1])
        self.gt_off = _dev(h["gt_off"], torch.int32, device)
        self.gt = _rows(h["gt"], device, torch.float64)
        self.gt_code = _rows(h["gt_code"], device, torch.int32)
        self.gt_occluded = _rows(h["gt_occluded"], device, torch.int32)
        self.dc_off = _dev(h["dc_off"], torch.int32, device)
        self.dc = _dev(h["dc"], torch.float64, device)


class DeviceDT:
    """Detection records on the device: frame f holds `cnt[f]` records from `off[f]`; `capacity[f]` bounds them."""

    def __init__(self, off, cnt, rec, code, capacity):
        self.off, self.cnt, self.rec, self.code = off, cnt, rec, code
        self.capacity = np.asarray(capacity, dtype=np.int64)

    @classmethod
    def from_annos(cls, dt_annos, device="cuda"):
        h = pack_dt(dt_annos)
        cap = np.diff(h["dt_off"])
        return cls(_dev(h["dt_off"], torch.int32, device), _dev(cap, torch.int32, device), _rows(h["dt"], device, torch.float64),
                   _rows(h["dt_code"], device, torch.int32), cap)


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None and t.numel() else C.c_void_p(0)


def _stream(device):
    return C.c_void_p(torch.cuda.current_stream(device).cuda_stream)


class Frames:
    """Ground truth and detections of one evaluation, with the per-frame overlap block layout."""

    def __init__(self, gt, dt):
        if gt.num_frames != len(dt.capacity):
            raise ValueError("ground truth has %d frames, detections %d" % (gt.num_frames, len(dt.capacity)))
        if gt.num_frames < 1:
            raise ValueError("no frames to evaluate")
        self.gt, self.dt = gt, dt
        blocks = dt.capacity * gt.counts
        self.ov_off_h = _offsets(blocks)
        self.ov_elems = int(self.ov_off_h[-1])
        self.max_frame_dt = int(dt.capacity.max()) if len(dt.capacity) else 0
        if self.max_frame_dt > MAX_FRAME_DT:
            raise ValueError("a frame holds %d detections; the evaluation takes at most %d" % (self.max_frame_dt, MAX_FRAME_DT))
        self.device = gt.gt_off.device
        self.ov_off = _dev(self.ov_off_h, torch.int64, self.device)
        self.struct = _lib.KittiFrames(gt.num_frames, _ptr(gt.gt_off), _ptr(gt.gt), _ptr(gt.gt_code), _ptr(gt.gt_occluded),
                                       _ptr(gt.dc_off), _ptr(gt.dc), _ptr(dt.off), _ptr(dt.cnt), _ptr(dt.rec), _ptr(dt.code),
                                       _ptr(self.ov_off))

    def overlaps(self, metric, z_axis=1, z_center=1.0):
        """Per-frame [n_dt, n_gt] fp64 overlap matrices of one metric (0 2D, 1 BEV, 2 3D), as host arrays."""
        ov = torch.zeros(max(self.ov_elems, 1), dtype=torch.float64, device=self.device)
        _lib.check(_lib.lib.sessd_kitti_overlaps(C.byref(self.struct), metric, z_axis, z_center, _ptr(ov), _stream(self.device)),
                   "sessd_kitti_overlaps")
        ov = ov.cpu().numpy()
        cnt = self.dt.cnt.cpu().numpy()
        return [ov[self.ov_off_h[f]:self.ov_off_h[f] + cnt[f] * self.gt.counts[f]].reshape(cnt[f], self.gt.counts[f])
                for f in range(self.gt.num_frames)]

    def eval_metric(self, metric, configs, min_overlaps, compute_aos, z_axis=1, z_center=1.0):
        """Device run of one metric for configs [(class code, difficulty)] with their min overlaps.  Device tensors out:
        thresholds / precision / aos [n, 41], num_thresholds [n], map [n, 4] (R11, R40 precision; R11, R40 AOS)."""
        n = len(configs)
        dev = self.device
        cfg = _dev(np.asarray(configs, dtype=np.int32).reshape(n, 2), torch.int32, dev)
        mo = _dev(np.asarray(min_overlaps, dtype=np.float64).reshape(n), torch.float64, dev)
        out = {k: torch.zeros(n, N_PTS, dtype=torch.float64, device=dev) for k in ("thresholds", "precision", "aos")}
        out["num_thresholds"] = torch.zeros(n, dtype=torch.int32, device=dev)
        out["map"] = torch.zeros(n, 4, dtype=torch.float64, device=dev)
        ws_bytes = _lib.lib.sessd_kitti_eval_workspace_bytes(self.gt.num_frames, self.gt.total, self.ov_elems, n, int(compute_aos))
        ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
        _lib.check(_lib.lib.sessd_kitti_eval(C.byref(self.struct), self.max_frame_dt, metric, z_axis, z_center, n, _ptr(cfg), _ptr(mo),
                                             int(compute_aos), self.gt.total, self.ov_elems, _ptr(out["thresholds"]),
                                             _ptr(out["num_thresholds"]), _ptr(out["precision"]), _ptr(out["aos"]), _ptr(out["map"]),
                                             _ptr(ws), C.c_size_t(ws_bytes), _stream(dev)), "sessd_kitti_eval")
        return out


def evaluate(frames, current_classes, difficultys, min_overlaps, aos_metrics=(0,), z_axis=1, z_center=1.0):
    """eval_class_v3 for all three metrics.  min_overlaps [K, 3, C] (C = len(current_classes), class codes).  Returns
    {metric: {"precision", "orientation", "thresholds": [C, D, K, 41], "map": [C, D, K, 4]}} as host arrays; AOS is computed for
    the metrics in `aos_metrics` (the reference also computes it for BEV and 3D, and never reports it)."""
    min_overlaps = np.asarray(min_overlaps, dtype=np.float64)
    K, nc, nd = min_overlaps.shape[0], len(current_classes), len(difficultys)
    outs = []
    for metric in range(3):
        configs, mo = [], []
        for m, cls in enumerate(current_classes):
            for diff in difficultys:
                for k in range(K):
                    configs.append((cls, diff))
                    mo.append(min_overlaps[k, metric, m])
        outs.append(frames.eval_metric(metric, configs, mo, metric in aos_metrics, z_axis, z_center))
    # one copy back, after all three metrics have been launched
    keys = ("precision", "aos", "thresholds", "map")
    flat = torch.cat([o[k].reshape(-1) for o in outs for k in keys]).cpu().numpy()
    res, pos = {}, 0
    for metric in range(3):
        host = {}
        for k in keys:
            n = outs[metric][k].numel()
            host[k] = flat[pos:pos + n]
            pos += n
        res[metric] = {"precision": host["precision"].reshape(nc, nd, K, N_PTS),
                       "orientation": host["aos"].reshape(nc, nd, K, N_PTS),
                       "thresholds": host["thresholds"].reshape(nc, nd, K, N_PTS),
                       "recall": np.zeros((nc, nd, K, N_PTS)),
                       "map": host["map"].reshape(nc, nd, K, 4), "min_overlaps": min_overlaps}
    return res


# ------------------------------------------------------------------------------------------------ detections -> camera annotations
def calib_rows(info):
    """[24] fp64: rows 0-2 of R0_rect . Tr_velo_to_cam (formed as the reference's lidar_to_camera forms it), rows 0-2 of P2."""
    c = info["calib"]
    m = np.asarray(c["R0_rect"]) @ np.asarray(c["Tr_velo_to_cam"])
    p2 = np.asarray(c["P2"])
    return np.concatenate([m[:3, :4].reshape(-1), p2[:3, :4].reshape(-1)]).astype(np.float64)


class DeviceCalib:
    """Per-frame calibration and image sizes of a dataset's infos, on the device."""

    def __init__(self, infos, device="cuda"):
        self.calib = _dev(np.stack([calib_rows(i) for i in infos]), torch.float64, device)
        self.image_hw = _dev(np.stack([np.asarray(i["image"]["image_shape"], dtype=np.int64)[:2] for i in infos]), torch.int32, device)


def convert_detections(dets, calib, class_names):
    """dets: per frame (box3d_lidar [n, 7], scores [n], label_preds [n]) tensors on any device.  Returns (DeviceDT, labels)
    where labels is the device tensor of kept labels (records stay in their frame's input slots)."""
    dev = calib.calib.device
    counts = np.array([int(b.shape[0]) for b, _, _ in dets], dtype=np.int64)
    off_h = _offsets(counts)
    cap = int(off_h[-1])
    F = len(dets)
    nonempty = [i for i in range(F) if counts[i]]
    if nonempty:
        boxes = torch.cat([dets[i][0].detach().to(dev, torch.float32).reshape(-1, 7) for i in nonempty]).contiguous()
        scores = torch.cat([dets[i][1].detach().to(dev, torch.float32).reshape(-1) for i in nonempty]).contiguous()
        labels = torch.cat([dets[i][2].detach().to(dev, torch.int32).reshape(-1) for i in nonempty]).contiguous()
    else:
        boxes = torch.zeros(1, 7, dtype=torch.float32, device=dev)
        scores = torch.zeros(1, dtype=torch.float32, device=dev)
        labels = torch.zeros(1, dtype=torch.int32, device=dev)
    n = max(cap, 1)
    off = _dev(off_h, torch.int32, dev)
    code_lut = _dev(_codes(class_names), torch.int32, dev)
    rec = torch.zeros(n, REC, dtype=torch.float64, device=dev)
    out_label = torch.zeros(n, dtype=torch.int32, device=dev)
    out_code = torch.zeros(n, dtype=torch.int32, device=dev)
    cnt = torch.zeros(F, dtype=torch.int32, device=dev)
    ws_bytes = _lib.lib.sessd_kitti_convert_workspace_bytes(n)
    ws = torch.empty(ws_bytes, dtype=torch.uint8, device=dev)
    _lib.check(_lib.lib.sessd_kitti_convert_detections(_ptr(boxes), _ptr(scores), _ptr(labels), _ptr(off), F, n, _ptr(calib.calib),
                                                       _ptr(calib.image_hw), _ptr(code_lut), len(class_names), _ptr(rec),
                                                       _ptr(out_label), _ptr(out_code), _ptr(cnt), _ptr(ws), C.c_size_t(ws_bytes),
                                                       _stream(dev)), "sessd_kitti_convert_detections")
    return DeviceDT(off, cnt, rec, out_code, counts), out_label


def dt_annos_from_device(dt, labels, class_names):
    """One device-to-host copy: numpy annotations (the reference's dt_annos, without metadata) from converted records."""
    n = dt.rec.shape[0]
    flat = torch.cat([dt.rec.reshape(-1), labels.to(torch.float64), dt.cnt.to(torch.float64)]).cpu().numpy()
    rec = flat[:n * REC].reshape(n, REC)
    lab = flat[n * REC:n * REC + n].astype(np.int64)
    cnt = flat[n * REC + n:].astype(np.int64)
    off = _offsets(dt.capacity)
    annos = []
    for f in range(len(cnt)):
        r = rec[off[f]:off[f] + cnt[f]]
        if cnt[f] == 0:
            annos.append(empty_anno())
            continue
        annos.append({"name": np.array([class_names[int(x)] for x in lab[off[f]:off[f] + cnt[f]]]),
                      "truncated": np.zeros(cnt[f]), "occluded": np.zeros(cnt[f], dtype=np.int64),
                      "alpha": r[:, 4].copy(), "bbox": r[:, 0:4].copy(), "dimensions": r[:, 8:11].copy(),
                      "location": r[:, 5:8].copy(), "rotation_y": r[:, 11].copy(), "score": r[:, 12].astype(np.float32)})
    return annos


def empty_anno():
    return {"name": np.array([]), "truncated": np.array([]), "occluded": np.array([]), "alpha": np.array([]),
            "bbox": np.zeros([0, 4]), "dimensions": np.zeros([0, 3]), "location": np.zeros([0, 3]), "rotation_y": np.array([]),
            "score": np.array([])}
