"""TEST INFRASTRUCTURE ONLY: the CPU arm of a BEVDet4D frame (paddle3d_b200.bevdet.BEVDet4D, PARITY UNPINNED as its
CONFIG_4D) and the numpy restatements of BEVDet4D's shift_feature.

shift_feature restates BEVDet4D.shift_feature / gen_grid with F.grid_sample(bilinear, padding_mode='zeros',
align_corners=True) in fp64; shift_h16_fp32 is p3d_bev_shift_h16's fp32 evaluation order.  CpuBEVDet4D chains
oracle.lss.view_transform, pre_process (BasicBlocks through oracle.bevdet.CpuBEVDet's fp64 convs), the fp64 shift of
the previous frame's bev_feat and CpuBEVDet's encoder, head and postprocess.  Nothing under paddle3d_b200/ imports
this module."""
import time

import numpy as np

from oracle import centerpoint_postprocess
from oracle.bevdet import CpuBEVDet
from oracle.lss import view_transform


def shift_matrix(s2ke_curr, s2ke_prev, bda, grid_lower_bound, grid_interval):
    """gen_grid's tf [B, 3, 3] in fp64 from sensor2keyegos [B, N, 4, 4] of the two frames and bda [B, 3, 3]."""
    curr, prev = np.asarray(s2ke_curr, np.float64), np.asarray(s2ke_prev, np.float64)
    B = curr.shape[0]
    bda4 = np.zeros((B, 4, 4))
    bda4[:, :3, :3] = np.asarray(bda, np.float64)
    bda4[:, 3, 3] = 1.0
    l02l1 = (bda4 @ curr[:, 0]) @ np.linalg.inv(bda4 @ prev[:, 0])
    l02l1 = l02l1[:, [0, 1, 3]][:, :, [0, 1, 3]]
    f2b = np.eye(3)
    f2b[0, 0], f2b[1, 1] = grid_interval[0], grid_interval[1]
    f2b[0, 2], f2b[1, 2] = grid_lower_bound[0], grid_lower_bound[1]
    return np.linalg.inv(f2b) @ l02l1 @ f2b


def grid_sample_zeros(x, ix, iy):
    """F.grid_sample(bilinear, zeros, align_corners=True) of x [B, C, h, w] at pixel coordinates ix / iy [B, h, w] (already
    unnormalised), fp64; taps outside the image (and non-finite coordinates) contribute 0."""
    x = np.asarray(x, np.float64)
    B, C, h, w = x.shape
    out = np.zeros((B, C) + ix.shape[1:], np.float64)
    with np.errstate(invalid="ignore"):
        x0, y0 = np.floor(ix), np.floor(iy)
        for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
            tx, ty = x0 + dx, y0 + dy
            wx = (ix - x0) if dx else (x0 + 1 - ix)
            wy = (iy - y0) if dy else (y0 + 1 - iy)
            ok = (tx >= 0) & (tx <= w - 1) & (ty >= 0) & (ty <= h - 1)
            txi = np.where(ok, tx, 0).astype(np.int64)
            tyi = np.where(ok, ty, 0).astype(np.int64)
            for b in range(B):
                v = x[b][:, tyi[b], txi[b]]
                out[b] += np.where(ok[b], wx[b] * wy[b], 0.0)[None] * np.where(ok[b][None], v, 0.0)
    return out


def shift_feature(feat, s2ke_curr, s2ke_prev, bda, grid_lower_bound, grid_interval, tf=None):
    """BEVDet4D.shift_feature of feat [B, C, h, w] in fp64 (tf: a given [B, 3, 3] transform instead of the chain)."""
    feat = np.asarray(feat, np.float64)
    B, _, h, w = feat.shape
    if tf is None:
        tf = shift_matrix(s2ke_curr, s2ke_prev, bda, grid_lower_bound, grid_interval)
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    g = np.einsum("bij,jyx->biyx", tf, np.stack([xs, ys, np.ones_like(xs)]))
    nx = g[:, 0] / (w - 1.0) * 2.0 - 1.0
    ny = g[:, 1] / (h - 1.0) * 2.0 - 1.0
    return grid_sample_zeros(feat, (nx + 1) / 2 * (w - 1), (ny + 1) / 2 * (h - 1))


def shift_h16_fp32(x, tf6):
    """p3d_bev_shift_h16's arithmetic on merged fp32 values x [B, h, w, C] (NHWC) with the fp32 descriptor tf6 [B, 6], every
    operation rounded to fp32 on its own: g = (t0 x + t1 y) + t2, n = g / (w - 1) * 2 - 1, i = ((n + 1) * 0.5) * (w - 1),
    floor, weights (x1 - ix)(y1 - iy) ..., the sum ((0 + nw NW) + ne NE) + sw SW) + se SE with out-of-image taps 0."""
    f = np.float32
    x = np.asarray(x, np.float32)
    tf6 = np.asarray(tf6, np.float32).reshape(-1, 6)
    B, h, w, C = x.shape
    ys, xs = np.meshgrid(np.arange(h, dtype=np.float32), np.arange(w, dtype=np.float32), indexing="ij")
    out = np.zeros_like(x)
    wm1, hm1 = f(w - 1), f(h - 1)
    with np.errstate(invalid="ignore", over="ignore"):
        for b in range(B):
            t = tf6[b]
            gx = ((t[0] * xs).astype(f) + (t[1] * ys).astype(f)).astype(f) + t[2]
            gy = ((t[3] * xs).astype(f) + (t[4] * ys).astype(f)).astype(f) + t[5]
            nx = ((gx.astype(f) / wm1).astype(f) * f(2)).astype(f) - f(1)
            ny = ((gy.astype(f) / hm1).astype(f) * f(2)).astype(f) - f(1)
            ix = (((nx.astype(f) + f(1)).astype(f) * f(0.5)).astype(f) * wm1).astype(f)
            iy = (((ny.astype(f) + f(1)).astype(f) * f(0.5)).astype(f) * hm1).astype(f)
            x0, y0 = np.floor(ix), np.floor(iy)
            x1, y1 = (x0 + f(1)).astype(f), (y0 + f(1)).astype(f)
            dxl, dxr = (ix - x0).astype(f), (x1 - ix).astype(f)
            dyt, dyb = (iy - y0).astype(f), (y1 - iy).astype(f)
            acc = np.zeros((h, w, C), np.float32)
            for tx, ty, wt in ((x0, y0, dxr * dyb), (x1, y0, dxl * dyb), (x0, y1, dxr * dyt), (x1, y1, dxl * dyt)):
                ok = (tx >= 0) & (tx <= wm1) & (ty >= 0) & (ty <= hm1)
                v = x[b][np.where(ok, ty, 0).astype(np.int64), np.where(ok, tx, 0).astype(np.int64)]
                c = np.where(ok[..., None], (wt.astype(f)[..., None] * v).astype(f), f(0))
                acc = (acc + c).astype(f)
            out[b] = acc
    return out


class CpuBEVDet4D(CpuBEVDet):
    """CPU arm of a BEVDet4D sequence.  weights: BEVDet4D.export_numpy(); run() carries feat_prev (this frame's bev_feat)
    to the next call."""

    def __init__(self, weights, test_cfg, label_offsets):
        super().__init__(weights, test_cfg, label_offsets)
        self.feat_prev = None

    def pre_process(self, bev):
        x = bev
        for stage in self.w["pre_process"]:
            for blk in stage:
                x = self._block(blk, x)
        return x

    def run(self, cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size, s2ke_curr, bda,
            s2ke_prev=None, new_sequence=False):
        """cams: unpacked camera descriptor of this frame; s2ke_curr / s2ke_prev [1, N, 4, 4] and bda [1, 3, 3] (fp64
        matrices); new_sequence: the frame is its own adjacent frame."""
        tc, t = self.tc, {}
        t0 = time.perf_counter()
        bev, _, _ = view_transform(cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size)
        bev_feat = self.pre_process(bev)
        if new_sequence:
            prev, s2ke_prev = bev_feat, s2ke_curr
        else:
            prev = self.feat_prev
        shifted = shift_feature(prev, s2ke_curr, s2ke_prev, bda, grid_lower_bound, grid_interval).astype(np.float32)
        self.feat_prev = bev_feat
        t["view_transform_pre_shift"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        feat = self.encoder(np.concatenate([bev_feat, shifted], 1))
        t["encoder"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        h = self.heads(feat)
        t["head"] = time.perf_counter() - t0
        boxes, scores, labels, _ = centerpoint_postprocess(
            h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"], tc["point_cloud_range"],
            tc["post_center_limit_range"], self.off, tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
            tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
        return dict(bev=bev, bev_feat=bev_feat, shifted=shifted, feat=feat, head=h, boxes=boxes, scores=scores,
                    labels=labels, times=t)
