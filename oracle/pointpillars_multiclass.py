"""TEST INFRASTRUCTURE ONLY — not part of the product.

The multi-class PointPillars anchor (SSD) head restated in numpy fp32, and the CPU arm of a multi-class frame, for tests/
and tools/pointpillars_bench.py.  Built on the single-class restatement in oracle/pointpillars.py (anchor geometry, the
anchor mask, second_box_decode, NMS), which stays as it is; with one class everything here gives its results bit for bit.
Nothing under paddle3d_b200/ imports this module."""
import time

import numpy as np

from . import conv2d, hard_voxelize, nms, pillar_feature_net, pillar_scatter, ref_hard_voxelize_cpu
from .pointpillars import CpuPointPillars, anchor_areas, anchors_3d_stride, second_box_decode, second_trunk


# SECOND v1.5 TargetAssigner.generate_anchors / VoxelNet.predict with encode_background_as_zeros, sigmoid scores and
# use_multi_class_nms off (PARITY UNPINNED, as oracle/pointpillars.py).
def anchors_3d_stride_classes(feature_size, generators):
    """One anchors_3d_stride per class generator (dicts of sizes / strides / offsets / rotations), in label order,
    concatenated per location as SECOND's TargetAssigner.generate_anchors does: [D * H * W * R, 7], anchor
    (cell, class, size, rot)."""
    cells = int(np.prod([int(v) for v in feature_size]))
    per = [anchors_3d_stride(feature_size, g["sizes"], g["strides"], g["offsets"], g["rotations"]).reshape(cells, -1, 7)
           for g in generators]
    return np.concatenate(per, 1).reshape(-1, 7)


def anchor_head_postprocess(head, anchors, corners, coords, grid, post_center_range, area_threshold=1,
                            score_threshold=0.05, iou_threshold=0.5, pre_max=1000, post_max=300, num_classes=1):
    """VoxelNet.predict at batch 1 with class-agnostic NMS.  head [1, R (C + 9), H, W] (cls R C | box 7 R | dir 2 R
    planes, C = num_classes, channel a * K + k of each group belonging to anchor (y * W + x) * R + a); coords: the valid
    pillar coords.  An anchor's score is the max over its classes of the fp32 sigmoid, its label the first class
    reaching that max.  Returns what oracle.pointpillars.anchor_head_postprocess returns (boxes [K, 7], scores [K],
    labels [K] int64, mask, candidates, cand_boxes, cand_scores, keep), plus cand_labels (score order, first pre_max)."""
    f = np.float32
    head = np.asarray(head, f)
    C = int(num_classes)
    R, H, W = head.shape[1] // (C + 9), head.shape[2], head.shape[3]
    cls = head[0, :R * C].reshape(R, C, H, W).transpose(2, 3, 0, 1).reshape(-1, C)
    box = head[0, R * C:R * (C + 7)].reshape(R, 7, H, W).transpose(2, 3, 0, 1).reshape(-1, 7)
    dirs = head[0, R * (C + 7):].reshape(R, 2, H, W).transpose(2, 3, 0, 1).reshape(-1, 2)
    mask = anchor_areas(coords, corners, grid) > area_threshold
    with np.errstate(over="ignore"):
        sig = (f(1.0) / (f(1.0) + np.exp(-cls))).astype(f)
    score, label = sig.max(1), sig.argmax(1).astype(np.int64)   # argmax: ties to the lowest class
    idx = np.nonzero(mask & (score >= f(score_threshold)))[0]
    order = idx[np.argsort(-score[idx], kind="stable")][:pre_max]   # descending score, ties by ascending anchor index
    boxes = second_box_decode(box[order], np.asarray(anchors, f)[order])
    dir_label = dirs[order, 1] > dirs[order, 0]                     # argmax, ties to 0
    nb = boxes[:, [0, 1, 2, 4, 3, 5, 6]].copy()                      # rotate_nms_pcdet's layout, fp32 angle
    nb[:, 6] = -boxes[:, 6] - f(np.pi / 2)
    keep, nk = nms(nb, iou_threshold) if len(nb) else (np.zeros(0, np.int32), 0)
    keep = keep[:min(nk, post_max)]
    out = boxes[keep].copy()
    flip = (out[:, 6] > 0) ^ dir_label[keep]
    out[flip, 6] = out[flip, 6] + f(np.pi)
    lo, hi = np.asarray(post_center_range[:3], f), np.asarray(post_center_range[3:], f)
    ok = np.all(out[:, :3] >= lo, 1) & np.all(out[:, :3] <= hi, 1)
    return dict(boxes=out[ok], scores=score[order][keep][ok], labels=label[order][keep][ok], mask=mask,
                candidates=len(idx), cand_boxes=boxes, cand_scores=score[order], cand_labels=label[order], keep=keep)


class CpuPointPillarsMulticlass(CpuPointPillars):
    """CPU arm of a PointPillars frame with `num_classes` classes: the stages of CpuPointPillars, then the multi-class
    anchor postprocess above."""

    def __init__(self, cfg, weights, anchors, corners, grid, test_cfg, num_classes, use_ref_voxelizer=True):
        super().__init__(cfg, weights, anchors, corners, grid, test_cfg, use_ref_voxelizer)
        self.num_classes = int(num_classes)

    def run(self, points):
        cfg, w, tc = self.cfg, self.w, self.tc
        t = {}
        t0 = time.perf_counter()
        vox = ref_hard_voxelize_cpu if self.use_ref else hard_voxelize
        v, c, n, nv = vox(points, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"], cfg["max_voxels"])
        k = int(nv[0])
        coors = np.concatenate([np.zeros((k, 1), np.int32), c[:k]], 1)
        t["voxelize"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        p = w["pfn"]
        feats = pillar_feature_net(v[:k], n[:k], coors, p["weight"], p["gamma"], p["beta"], p["mean"], p["var"], p["eps"],
                                   cfg["voxel_size"], cfg["point_cloud_range"])
        t["pfn"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        nx, ny = self.grid
        bev = pillar_scatter(feats, coors, 1, ny, nx)
        t["scatter"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        h = w["head"]
        planes = conv2d(second_trunk(w, bev), h["weight"], h["bias"], 1, 0)
        t["dense"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        r = anchor_head_postprocess(planes, self.anchors, self.corners, coors, self.grid, tc["post_center_limit_range"],
                                    tc["anchor_area_threshold"], tc["nms_score_threshold"], tc["nms_iou_threshold"],
                                    tc["nms_pre_max_size"], tc["nms_post_max_size"], self.num_classes)
        t["postprocess"] = time.perf_counter() - t0
        return dict(r, planes=planes, num_voxels=k, coors=coors, times=t)
