"""TEST INFRASTRUCTURE ONLY: the CPU arm of BEVDet from camera images (paddle3d_b200.bevdet.BEVDetFromImages, PARITY
UNPINNED as its CONFIG_IMG).  It lives under tests/, beside the other CPU arms added after oracle/, so nothing under
oracle/ changes.

CpuBEVDetImages runs the image half on the oracle's dense convs (oracle.conv2d: fp64 accumulation, fp32 outputs;
oracle.bn2d_relu: fp64): the ResNet stem with a fp64 max-pool, the Bottlenecks (identity added in fp64 before the ReLU),
CustomFPN with nearest upsampling (the top-down add in fp64) and the depth net; its logits and tran_feat feed
oracle.bevdet.CpuBEVDet.run unchanged."""
import time

import numpy as np

from oracle import bn2d_relu, conv2d
from oracle.bevdet import CpuBEVDet


def max_pool_3x3_s2_p1(x):
    """MaxPool2d(3, 2, 1) of [B, C, H, W] in fp64 (padding -inf: never the maximum)."""
    x = np.asarray(x, np.float64)
    b, c, h, w = x.shape
    oh, ow = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    p = np.full((b, c, h + 2, w + 2), -np.inf)
    p[:, :, 1:-1, 1:-1] = x
    out = np.full((b, c, oh, ow), -np.inf)
    for dy in range(3):
        for dx in range(3):
            out = np.maximum(out, p[:, :, dy:dy + 2 * oh - 1:2, dx:dx + 2 * ow - 1:2])
    return out


def upsample_nearest(x, size):
    """F.interpolate(x, size=size, mode='nearest') of [B, C, h, w]: source index floor(dst * h / H)."""
    _, _, h, w = x.shape
    H, W = size
    yi = np.floor(np.arange(H) * (h / H)).astype(np.int64)
    xi = np.floor(np.arange(W) * (w / W)).astype(np.int64)
    return x[:, :, yi][:, :, :, xi]


def _bn(l, y, relu):
    bn = l["bn"]
    return bn2d_relu(y, bn["gamma"], bn["beta"], bn["mean"], bn["var"], bn["eps"], relu=relu)


def _conv(l, x, relu=None):
    y = conv2d(x, l["weight"], l["bias"], l["stride"], l["padding"])
    r = l["relu"] if relu is None else relu
    if l["bn"] is not None:
        return _bn(l, y, r)
    return np.maximum(y, 0.0) if r else y


class CpuBEVDetImages:
    """CPU arm of a BEVDetFromImages frame.  weights: BEVDetFromImages.export_numpy(); test_cfg / label_offsets as the
    model holds them."""

    def __init__(self, weights, test_cfg, label_offsets):
        self.w = weights["image_encoder"]
        self.bev = CpuBEVDet(weights, test_cfg, label_offsets)

    def stem(self, imgs):
        """MaxPool(ReLU(BN(conv7x7 s2 p3))) -> [N, 64, pH, pW] fp64."""
        return max_pool_3x3_s2_p1(_conv(self.w["stem"], imgs, relu=True))

    @staticmethod
    def bottleneck(blk, x):
        t = _conv(blk["conv1"], x)
        t = _conv(blk["conv2"], t)
        c3 = blk["conv3"]
        y = _bn(c3, conv2d(t, c3["weight"], c3["bias"], c3["stride"], c3["padding"]), False).astype(np.float64)
        idn = x if blk["down"] is None else _conv(blk["down"], x)
        return np.maximum(y + np.asarray(idn, np.float64), 0.0).astype(np.float32)

    def backbone(self, imgs, stem=None):
        """Every stage's output [N, C, H, W] fp32 (stem: the stem's output, if already computed)."""
        x, feats = (self.stem(imgs) if stem is None else stem).astype(np.float32), []
        for stage in self.w["stages"]:
            for blk in stage:
                x = self.bottleneck(blk, x)
            feats.append(x)
        return feats

    def neck(self, feats):
        w = self.w
        x0, x1 = feats[w["out_indices"][0]], feats[w["out_indices"][1]]
        l1 = _conv(w["lateral"][1], x1)
        l0 = _conv(w["lateral"][0], x0).astype(np.float64) + upsample_nearest(l1, x0.shape[2:]).astype(np.float64)
        return _conv(w["fpn_conv"], l0.astype(np.float32))

    def image_encoder(self, imgs, feats=None):
        """imgs [N, 3, H, W] -> (logits [N, D, H/16, W/16], tran_feat [N, C, H/16, W/16]) fp32 (feats: backbone's output,
        if already computed)."""
        d = _conv(self.w["depth_net"], self.neck(self.backbone(imgs) if feats is None else feats))
        D, C = self.w["D"], self.w["C"]
        return np.ascontiguousarray(d[:, :D]), np.ascontiguousarray(d[:, D:D + C])

    def run(self, cams, axes, imgs, grid_lower_bound, grid_interval, grid_size, keep_feats=False):
        """CpuBEVDet.run on the image encoder's output; adds logits, tran_feat and the image encoder's time (keep_feats:
        also the stem's and every stage's output)."""
        t0 = time.perf_counter()
        stem = self.stem(imgs).astype(np.float32)
        feats = self.backbone(imgs, stem)
        logits, tran = self.image_encoder(imgs, feats)
        t = time.perf_counter() - t0
        out = self.bev.run(cams, axes, logits, tran, grid_lower_bound, grid_interval, grid_size)
        out["times"]["image_encoder"] = t
        out = dict(out, logits=logits, tran_feat=tran)
        if keep_feats:
            out.update(stem=stem, feats=feats)
        return out
