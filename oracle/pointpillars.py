"""TEST INFRASTRUCTURE ONLY — not part of the product.

PointPillars anchor (SSD) head restated in numpy fp32, and the CPU arm of a PointPillars frame (CpuPointPillars), for
tests/ and tools/pointpillars_bench.py.  Nothing under paddle3d_b200/ imports this module."""
import time

import numpy as np

from . import (bn2d_relu, conv2d, deconv2d, hard_voxelize, nms, pillar_feature_net, pillar_scatter, ref_hard_voxelize_cpu,
               ref_lib)


# --------------------------------------------------------------------------- PointPillars anchor (SSD) head
# SECOND v1.5 box_np_ops / VoxelNet.predict restated in numpy fp32 (PARITY UNPINNED: SECOND behaviour, which the
# reference's pointpillars_xyres16 config descends from; not checked against the reference's own source).
def anchors_3d_stride(feature_size, sizes, strides, offsets, rotations):
    """create_anchors_3d_stride as one broadcast: feature_size (D, H, W) -> [D * H * W * n_sizes * n_rot, 7]
    (x, y, z, w, l, h, theta) in (z, y, x, size, rot) order, fp32."""
    f = np.float32
    D, H, W = [int(v) for v in feature_size]
    sizes = np.asarray(sizes, f).reshape(-1, 3)
    rot = np.asarray(rotations, f)
    S, R = len(sizes), len(rot)
    out = np.empty((D, H, W, S, R, 7), f)
    out[..., 0] = (np.arange(W, dtype=f) * f(strides[0]) + f(offsets[0]))[None, None, :, None, None]
    out[..., 1] = (np.arange(H, dtype=f) * f(strides[1]) + f(offsets[1]))[None, :, None, None, None]
    out[..., 2] = (np.arange(D, dtype=f) * f(strides[2]) + f(offsets[2]))[:, None, None, None, None]
    out[..., 3:6] = sizes[None, None, None, :, None, :]
    out[..., 6] = rot[None, None, None, None, :]
    return out.reshape(-1, 7)


def anchor_corners(anchors, voxel_size, pcr, grid):
    """rbbox2d_to_near_bbox + the floor / clamp of fused_get_anchors_area: [A, 4] int32 (x_min, y_min, x_max, y_max)."""
    a = np.asarray(anchors, np.float32)
    rot = a[:, 6]
    near_half_pi = np.abs(rot - np.floor(rot / np.pi + 0.5) * np.pi) > np.pi / 4   # |limit_period(rot, 0.5, pi)|
    dx = np.where(near_half_pi, a[:, 4], a[:, 3])
    dy = np.where(near_half_pi, a[:, 3], a[:, 4])
    lo_x, lo_y, hi_x, hi_y = a[:, 0] - dx / 2, a[:, 1] - dy / 2, a[:, 0] + dx / 2, a[:, 1] + dy / 2
    c = np.stack([np.floor((lo_x - pcr[0]) / voxel_size[0]), np.floor((lo_y - pcr[1]) / voxel_size[1]),
                  np.floor((hi_x - pcr[0]) / voxel_size[0]), np.floor((hi_y - pcr[1]) / voxel_size[1])], 1)
    c[:, [0, 2]] = np.clip(c[:, [0, 2]], 0, grid[0] - 1)
    c[:, [1, 3]] = np.clip(c[:, [1, 3]], 0, grid[1] - 1)
    return c.astype(np.int32)


def anchor_areas(coords, corners, grid):
    """fused_get_anchors_area on sparse_sum_for_anchors_mask(coords).cumsum(0).cumsum(1): occupied-pillar count over
    y in (y_min, y_max], x in (x_min, x_max] of each anchor.  coords [n, 4] (b, z, y, x) or [n, 3] (z, y, x)."""
    coords = np.asarray(coords)
    nx, ny = grid
    m = np.zeros((ny, nx), np.int64)
    np.add.at(m, (coords[:, -2], coords[:, -1]), 1)
    s = m.cumsum(0).cumsum(1)
    c = np.asarray(corners)
    return s[c[:, 3], c[:, 2]] - s[c[:, 3], c[:, 0]] - s[c[:, 1], c[:, 2]] + s[c[:, 1], c[:, 0]]


def second_box_decode(box, anchors):
    """second_box_decode without smooth_dim / angle vector, fp32, one rounding per operation (no fused multiply-add)."""
    f = np.float32
    box, anchors = np.asarray(box, f), np.asarray(anchors, f)
    xa, ya, za, wa, la, ha, ra = [anchors[:, k] for k in range(7)]
    xt, yt, zt, wt, lt, ht, rt = [box[:, k] for k in range(7)]
    za = za + ha * f(0.5)
    diag = np.sqrt(la * la + wa * wa)
    with np.errstate(over="ignore"):
        w, l, h = np.exp(wt) * wa, np.exp(lt) * la, np.exp(ht) * ha
    z = zt * ha + za
    return np.stack([xt * diag + xa, yt * diag + ya, z - h * f(0.5), w, l, h, rt + ra], 1).astype(f)


def anchor_head_postprocess(head, anchors, corners, coords, grid, post_center_range, area_threshold=1,
                            score_threshold=0.05, iou_threshold=0.5, pre_max=1000, post_max=300):
    """VoxelNet.predict for one class at batch 1.  head [1, 10 R, H, W] (cls R | box 7 R | dir 2 R planes, channel
    a * K + k of anchor (y * W + x) * R + a); coords: the valid pillar coords.  Returns a dict: boxes [K, 7], scores [K],
    labels [K] int64, and the intermediate results mask [A] bool, candidates (count above the threshold),
    cand_boxes / cand_scores (decoded, score order, first pre_max) and keep (indices into them, after NMS)."""
    f = np.float32
    head = np.asarray(head, f)
    R, H, W = head.shape[1] // 10, head.shape[2], head.shape[3]
    cls = head[0, :R].transpose(1, 2, 0).reshape(-1)
    box = head[0, R:8 * R].reshape(R, 7, H, W).transpose(2, 3, 0, 1).reshape(-1, 7)
    dirs = head[0, 8 * R:].reshape(R, 2, H, W).transpose(2, 3, 0, 1).reshape(-1, 2)
    mask = anchor_areas(coords, corners, grid) > area_threshold
    with np.errstate(over="ignore"):
        score = (f(1.0) / (f(1.0) + np.exp(-cls))).astype(f)
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
    return dict(boxes=out[ok], scores=score[order][keep][ok], labels=np.zeros(int(ok.sum()), np.int64), mask=mask,
                candidates=len(idx), cand_boxes=boxes, cand_scores=score[order], keep=keep)


def _layer(l, x):
    """One exported dense_head._Conv layer (dict from export_numpy): Conv2D, or Conv2DTranspose (up > 1, or a stride-1
    transposed k = 1 deblock), then BatchNorm2D + ReLU when present."""
    if l["up"] > 1 or l.get("transposed"):
        y = deconv2d(x, l["weight"], l["bias"], max(int(l["up"]), 1))
    else:
        y = conv2d(x, l["weight"], l["bias"], l["stride"], l["padding"])
    if l["bn"] is not None:
        bn = l["bn"]
        return bn2d_relu(y, bn["gamma"], bn["beta"], bn["mean"], bn["var"], bn["eps"], relu=l["relu"])
    return np.maximum(y, 0.0) if l["relu"] else y


def second_trunk(weights, bev):
    """SecondBackbone + SecondFPN on an NCHW BEV tensor: the channel concat of the deblock outputs."""
    x, feats = bev, []
    for blk in weights["blocks"]:
        for l in blk:
            x = _layer(l, x)
        feats.append(x)
    return np.concatenate([_layer(l, f) for l, f in zip(weights["deblocks"], feats)], axis=1)


class CpuPointPillars:
    """CPU arm of a PointPillars frame (pointpillars.PointPillars.export_numpy weights): hard_voxelize (the reference's
    hard_voxelize_cpu when oracle/_ref is built), PillarFeatureNet, PointPillarsScatter, the dense trunk and the SSD head
    conv through the oracle, then the anchor postprocess restated in numpy (anchor_head_postprocess)."""

    def __init__(self, cfg, weights, anchors, corners, grid, test_cfg, use_ref_voxelizer=True):
        self.cfg, self.w, self.anchors, self.corners, self.grid, self.tc = cfg, weights, anchors, corners, grid, test_cfg
        self.use_ref = use_ref_voxelizer and ref_lib("cpu") is not None

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
                                    tc["nms_pre_max_size"], tc["nms_post_max_size"])
        t["postprocess"] = time.perf_counter() - t0
        return dict(r, planes=planes, num_voxels=k, coors=coors, times=t)
