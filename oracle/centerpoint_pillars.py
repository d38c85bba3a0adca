"""TEST INFRASTRUCTURE ONLY — not part of the product.

The two-layer PillarFeatureNet of CenterPoint-pillars restated in fp64 numpy, and the CPU arm of a CenterPoint-pillars
frame, for tests/ and tools/centerpoint_pillars_bench.py.  Built on the oracle's voxelizer, scatter, dense convs
(cpu_reference.CpuDenseHead) and CenterPoint postprocess, which stay as they are.  Nothing under paddle3d_b200/ imports
this module."""
import time

import numpy as np

from . import centerpoint_postprocess, hard_voxelize, pillar_scatter, ref_hard_voxelize_cpu, ref_lib
from .cpu_reference import CpuDenseHead


def _decorate(voxels, npv, coors, voxel_size, point_cloud_range):
    """PillarFeatureNet.forward's decoration (pillar_encoder.py:167-198), as oracle.pillar_feature_net states it: features
    [N, M, F + 5] fp64, rows >= npv zeroed after the decoration."""
    v = np.asarray(voxels, np.float64)
    n, m, f = v.shape
    cnt = np.asarray(npv, np.float64).reshape(-1, 1, 1)
    pmean = v[:, :, :3].sum(1, keepdims=True) / cnt
    f_cluster = v[:, :, :3] - pmean
    vx, vy = float(voxel_size[0]), float(voxel_size[1])
    xo, yo = vx / 2 + float(point_cloud_range[0]), vy / 2 + float(point_cloud_range[1])
    c = np.asarray(coors)
    f_center = np.stack([v[:, :, 0] - (c[:, 3].reshape(-1, 1).astype(np.float32).astype(np.float64) * np.float32(vx) + np.float32(xo)),
                         v[:, :, 1] - (c[:, 2].reshape(-1, 1).astype(np.float32).astype(np.float64) * np.float32(vy) + np.float32(yo))], -1)
    feats = np.concatenate([v, f_cluster, f_center], -1)
    mask = (np.arange(m).reshape(1, -1) < np.asarray(npv).reshape(-1, 1)).astype(np.float64)
    return feats * mask[:, :, None]


def _linear_bn_relu(x, layer):
    """PFNLayer's Linear (no bias) + BatchNorm1D (eval) + ReLU on [N, M, Cin], fp64."""
    y = x @ np.asarray(layer["weight"], np.float64)
    y = (y - layer["mean"]) / np.sqrt(np.asarray(layer["var"], np.float64) + layer["eps"]) * layer["gamma"] + layer["beta"]
    return np.maximum(y, 0.0)


def pillar_feature_net2(voxels, npv, coors, layers, voxel_size, point_cloud_range):
    """PillarFeatureNet with two PFNLayers (feat_channels [64, 64]) (PARITY UNPINNED: paddle ops; restated from
    models/voxel_encoders/pillar_encoder.py PFNLayer.forward / PillarFeatureNet.forward).  voxels [N, M, F], npv [N],
    coors [N, 4] (b, z, y, x); layers: two dicts of weight ([F + 5, mid], then [2 mid, out]) / gamma / beta / mean / var
    / eps.  The decoration of oracle.pillar_feature_net; layer 1 (not last): x = ReLU(BN(feats @ W1)), output
    concat([x, tile(max over the M rows of x)]); layer 2 (last): max over the rows of ReLU(BN(. @ W2)).  Padding rows
    (>= npv, zero after the decoration) take part in both maxima: in layer 1 with the value ReLU(BN(0)), in layer 2 with
    [ReLU(BN(0)), x_max].  fp64 internally, [N, out] fp32 out."""
    x = _linear_bn_relu(_decorate(voxels, npv, coors, voxel_size, point_cloud_range), layers[0])
    x_max = x.max(1, keepdims=True)
    x = np.concatenate([x, np.repeat(x_max, x.shape[1], 1)], -1)
    return _linear_bn_relu(x, layers[1]).max(1).astype(np.float32)


class CpuCenterPointPillars:
    """CPU arm of a CenterPoint-pillars frame: the reference's hard_voxelize_cpu (oracle/_ref) when built, else the
    oracle port; pillar_feature_net2; pillar_scatter; the dense trunk and CenterHead through CpuDenseHead; the
    CenterPoint postprocess.  weights: CenterPointPillars.export_numpy()."""

    def __init__(self, cfg, weights, test_cfg, label_offsets, use_ref_voxelizer=True):
        self.cfg, self.w, self.tc, self.off = cfg, weights, test_cfg, label_offsets
        self.dense = CpuDenseHead(weights)
        self.use_ref = use_ref_voxelizer and ref_lib("cpu") is not None
        pcr, vs = cfg["point_cloud_range"], cfg["voxel_size"]
        self.grid = (int(round((pcr[3] - pcr[0]) / vs[0])), int(round((pcr[4] - pcr[1]) / vs[1])))

    def run(self, points):
        cfg, tc = self.cfg, self.tc
        t = {}
        t0 = time.perf_counter()
        vox = ref_hard_voxelize_cpu if self.use_ref else hard_voxelize
        v, c, n, nv = vox(points, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"], cfg["max_voxels"])
        k = int(nv[0])
        coors = np.concatenate([np.zeros((k, 1), np.int32), c[:k]], 1)
        t["voxelize"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        feats = pillar_feature_net2(v[:k], n[:k], coors, self.w["pfn"], cfg["voxel_size"], cfg["point_cloud_range"])
        t["pfn"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        nx, ny = self.grid
        bev = pillar_scatter(feats, coors, 1, ny, nx)
        t["scatter"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        h = self.dense.run(bev)
        t["dense"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        boxes, scores, labels, _ = centerpoint_postprocess(
            h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], cfg["voxel_size"][:2], cfg["point_cloud_range"],
            tc["post_center_limit_range"], self.off, tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
            tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
        t["postprocess"] = time.perf_counter() - t0
        return dict(boxes=boxes, scores=scores, labels=labels, head=h, feats=feats, num_voxels=k, coors=coors, times=t)
