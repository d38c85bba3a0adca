"""TEST INFRASTRUCTURE ONLY: the CPU arm of a BEVDet frame (paddle3d_b200.bevdet, PARITY UNPINNED as its CONFIG) and the
numpy restatements of the bilinear upsampling.

CpuBEVDet chains oracle.lss.view_transform, the CustomResNet + FPN_LSS encoder and the CenterHead through the oracle's
dense convs (conv2d / bn2d_relu, fp64 accumulation; a BasicBlock adds its identity in fp64 before the ReLU; FPN_LSS's
bilinear in fp64), and oracle.centerpoint_postprocess.  Nothing under paddle3d_b200/ imports this module."""
import time

import numpy as np

from . import bn2d_relu, centerpoint_postprocess, conv2d
from .cpu_reference import CpuDenseHead
from .lss import view_transform


def _axis(n_in, n_out, src_fp32):
    if src_fp32:  # Paddle's GPU source coordinate: fp32(fp32(in - 1) / fp32(out - 1) * dst)
        r = np.float32(n_in - 1) / np.float32(n_out - 1) if n_out > 1 else np.float32(0.0)
        src = (r * np.arange(n_out, dtype=np.float32)).astype(np.float64)
    else:
        src = np.arange(n_out, dtype=np.float64) * ((n_in - 1) / (n_out - 1) if n_out > 1 else 0.0)
    i1 = np.minimum(np.floor(src).astype(np.int64), n_in - 1)
    i2 = np.minimum(i1 + 1, n_in - 1)
    return i1, i2, src - i1


def upsample_bilinear(x, s, src_fp32=False):
    """nn.Upsample(scale_factor=s, mode='bilinear', align_corners=True) of [B, C, h, w] in fp64.  src_fp32: at the source
    coordinates Paddle's bilinear_interp_v2 computes in fp32 (they differ from the exact ones by up to an fp32 rounding
    of the ratio times the index, a few 1e-6 pixel), the interpolation itself in fp64."""
    x = np.asarray(x, np.float64)
    _, _, h, w = x.shape
    y1, y2, ly = _axis(h, h * s, src_fp32)
    x1, x2, lx = _axis(w, w * s, src_fp32)
    lx = lx[None, None, None, :]
    top = x[:, :, y1][..., x1] * (1 - lx) + x[:, :, y1][..., x2] * lx
    bot = x[:, :, y2][..., x1] * (1 - lx) + x[:, :, y2][..., x2] * lx
    ly = ly[None, None, :, None]
    return top * (1 - ly) + bot * ly


def merge_h16(hi, lo):
    """fp16 pair -> fp32 value hi + lo' * 2^-11."""
    return (hi.astype(np.float32) + lo.astype(np.float32) * np.float32(2.0 ** -11)).astype(np.float32)


def split_h16(v):
    """fp32 -> (hi, lo') fp16 pair as the kernels split (|v| saturated at 65504)."""
    v = np.clip(np.asarray(v, np.float32), np.float32(-65504.0), np.float32(65504.0))
    hi = v.astype(np.float16)
    lo = ((v - hi.astype(np.float32)) * np.float32(2048.0)).astype(np.float16)
    return hi, lo


def upsample_bilinear_fp32(x, s):
    """p3d_upsample_bilinear_h16's arithmetic on merged fp32 values x [B, h, w, C] (NHWC), every operation rounded to fp32
    on its own: ratio = fp32(in - 1) / fp32(out - 1), src = ratio * dst, i1 = int(src), l1 = src - i1, l2 = 1 - l1,
    l2y (l2x a + l1x b) + l1y (l2x c + l1x d).  Scale 1 returns x."""
    x = np.asarray(x, np.float32)
    if s == 1:
        return x.copy()
    f = np.float32
    _, h, w, _ = x.shape

    def axis(n_in):
        n_out = n_in * s
        r = f(n_in - 1) / f(n_out - 1) if n_out > 1 else f(0.0)
        src = (r * np.arange(n_out, dtype=np.float32)).astype(np.float32)
        i1 = src.astype(np.int64)
        i2 = i1 + (i1 < n_in - 1)
        l1 = (src - i1.astype(np.float32)).astype(np.float32)
        return i1, i2, l1, (f(1.0) - l1).astype(np.float32)
    y1, y2, h1, h2 = axis(h)
    x1, x2, w1, w2 = axis(w)
    w1, w2 = w1[None, None, :, None], w2[None, None, :, None]
    top = (w2 * x[:, y1][:, :, x1]).astype(f) + (w1 * x[:, y1][:, :, x2]).astype(f)
    bot = (w2 * x[:, y2][:, :, x1]).astype(f) + (w1 * x[:, y2][:, :, x2]).astype(f)
    h1, h2 = h1[None, :, None, None], h2[None, :, None, None]
    return ((h2 * top).astype(f) + (h1 * bot).astype(f)).astype(f)


class CpuBEVDet:
    """CPU arm of a BEVDet frame.  weights: BEVDet.export_numpy(); test_cfg / label_offsets as BEVDet holds them."""

    def __init__(self, weights, test_cfg, label_offsets):
        self.w, self.tc, self.off = weights, test_cfg, label_offsets
        self.dense = CpuDenseHead(weights)

    def _conv(self, l, x):
        return self.dense._conv(l, x)

    def _block(self, blk, x):
        t = self._conv(blk["conv1"], x)
        c2 = blk["conv2"]
        y = conv2d(t, c2["weight"], c2["bias"], c2["stride"], c2["padding"])
        bn = c2["bn"]
        y = bn2d_relu(y, bn["gamma"], bn["beta"], bn["mean"], bn["var"], bn["eps"], relu=False).astype(np.float64)
        idn = x if blk["down"] is None else self._conv(blk["down"], x)
        return np.maximum(y + np.asarray(idn, np.float64), 0.0).astype(np.float32)

    def backbone(self, bev):
        """CustomResNet: the output of every stage, [B, C, H, W] fp32."""
        feats, x = [], bev
        for stage in self.w["backbone"]:
            for blk in stage:
                x = self._block(blk, x)
            feats.append(x)
        return feats

    def encoder(self, bev):
        """CustomResNet + FPN_LSS: bev [1, 80, 128, 128] -> [1, 256, 128, 128] fp32."""
        w = self.w
        feats = self.backbone(bev)
        i0, i2 = w["fpn_index"]
        cat = np.concatenate([feats[i0], upsample_bilinear(feats[i2], w["scale_factor"]).astype(np.float32)], 1)
        f0, f1, f2, f3 = w["fpn"]
        y = self._conv(f1, self._conv(f0, cat))
        if w["extra_upsample"]:
            y = upsample_bilinear(y, w["extra_upsample"]).astype(np.float32)
        return self._conv(f3, self._conv(f2, y))

    def heads(self, x):
        w, out = self.w, {}
        s = self._conv(w["shared"], x)
        for hs in w["heads"]:
            for name, a, fin in hs:
                out.setdefault(name, []).append(self._conv(fin, self._conv(a, s)))
        return out

    def run(self, cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size):
        """cams: unpacked camera descriptor (ops.bev_pool_v2.unpack_cameras); the rest as oracle.lss.view_transform."""
        tc, t = self.tc, {}
        t0 = time.perf_counter()
        bev, _, prep = view_transform(cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size)
        t["view_transform"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        feat = self.encoder(bev)
        t["encoder"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        h = self.heads(feat)
        t["head"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        boxes, scores, labels, _ = centerpoint_postprocess(
            h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"], tc["point_cloud_range"],
            tc["post_center_limit_range"], self.off, tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
            tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
        t["postprocess"] = time.perf_counter() - t0
        return dict(bev=bev, feat=feat, head=h, boxes=boxes, scores=scores, labels=labels, times=t,
                    n_intervals=0 if prep[0] is None else len(prep[3]))
