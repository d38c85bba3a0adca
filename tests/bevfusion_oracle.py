"""TEST INFRASTRUCTURE ONLY: numpy restatements of BEVFusion's new device steps (PARITY UNPINNED as
paddle3d_b200.bevfusion.CONFIG): HardVFE in fp64, the SE gate in fp64 with its fp32 scale, and Anchor3DHead's decode
(get_bboxes_single + box3d_multiclass_nms) in the reference's order.

anchor3d_decode_ref follows the reference's steps, not the kernel's: sigmoid of every class of every anchor, the max
over classes, topk over ALL anchors (the kernel ranks only the anchors that can reach the output), decode of every kept
anchor, then per class threshold, sort and NMS, then the max_num cut.  Where the reference leaves an order open
(torch.topk and sort among equal scores) this file takes the order the op defines: ties by the lower anchor index at
the nms_pre cut, by kept order within a class, by class-major order at the max_num cut.  A kept box with a non-finite
value takes part in no class's NMS (the op's rule).  Nothing under paddle3d_b200/ imports this module."""
import numpy as np

F = np.float32
PI32 = F(np.pi)
CODE = 9


# ------------------------------------------------------------------------------------------------------------ HardVFE
def hard_vfe_ref(voxels, npv, coors, layers, voxel_size, pcr):
    """HardVFE(feat_channels [mid, out], with_cluster_center, with_voxel_center, no distance) in fp64.  layers: two dicts
    of weight ([F + 6, mid], [2 mid, out]) / gamma / beta / mean / var / eps.  Returns [n, out]."""
    v = np.asarray(voxels, np.float64)
    n, M, _ = v.shape
    cnt = np.asarray(npv, np.float64)
    mean = v[:, :, :3].sum(1) / cnt[:, None]
    vs, lo = np.asarray(voxel_size, np.float64), np.asarray(pcr, np.float64)[:3]
    centre = np.asarray(coors, np.float64)[:, [3, 2, 1]] * vs + vs / 2 + lo
    x = np.concatenate([v, v[:, :, :3] - mean[:, None], v[:, :, :3] - centre[:, None]], -1)
    x = x * (np.arange(M)[None, :] < np.asarray(npv)[:, None])[..., None]
    for k, l in enumerate(layers):
        s = np.asarray(l["gamma"], np.float64) / np.sqrt(np.asarray(l["var"], np.float64) + l["eps"])
        t = np.asarray(l["beta"], np.float64) - np.asarray(l["mean"], np.float64) * s
        y = np.maximum((x @ np.asarray(l["weight"], np.float64)) * s + t, 0.0)
        if k == 0:
            x = np.concatenate([y, np.broadcast_to(y.max(1, keepdims=True), y.shape)], -1)
        else:
            return y.max(1)


# ------------------------------------------------------------------------------------------------------------ SE gate
def se_gate_ref(x, weight, bias):
    """sigmoid(W mean_hw(x) + b) in fp64 for x [B, H, W, C]: the gate [B, C]."""
    m = np.asarray(x, np.float64).mean((1, 2))
    return 1.0 / (1.0 + np.exp(-(m @ np.asarray(weight, np.float64).T + np.asarray(bias, np.float64))))


def pair_to_hilo(rows, C):
    """pixel H16 rows [n, 2C] fp16 (groups of 32 channels [hi 32 | lo' 32]) -> (hi, lo') [n, C] fp16 each."""
    g = np.asarray(rows, np.float16).reshape(-1, C // 32, 2, 32)
    return g[:, :, 0].reshape(-1, C), g[:, :, 1].reshape(-1, C)


def hilo_to_pair(hi, lo):
    n, C = hi.shape
    return np.stack([hi.reshape(n, C // 32, 32), lo.reshape(n, C // 32, 32)], 2).reshape(n, 2 * C)


def merge_h16(hi, lo):
    return (hi.astype(F) + lo.astype(F) * F(2.0 ** -11)).astype(F)


def split_h16(v):
    """fp32 -> (hi, lo') as the kernels split, and whether a value was saturated."""
    v = np.asarray(v, F)
    ovf = bool((np.abs(v) > F(65504.0)).any())
    v = np.clip(v, F(-65504.0), F(65504.0))
    hi = v.astype(np.float16)
    lo = ((v - hi.astype(F)) * F(2048.0)).astype(np.float16)
    return hi, lo, ovf


def se_scale_ref(rows, C, gate_rows):
    """p3d_se_gate_h16's scale: x = fp32(hi + lo'), x * gate (fp32, gate_rows [n, C] the row's batch gate), split again.
    Returns (new rows, overflow)."""
    hi, lo = pair_to_hilo(rows, C)
    with np.errstate(over="ignore", invalid="ignore"):
        y = (merge_h16(hi, lo) * np.asarray(gate_rows, F)).astype(F)
    h2, l2, ovf = split_h16(y)
    return hilo_to_pair(h2, l2), ovf


# ------------------------------------------------------------------------------------------------- Anchor3DHead decode
def sigmoid32(x):
    with np.errstate(over="ignore"):
        return (F(1.0) / (F(1.0) + np.exp(-np.asarray(x, F), dtype=F))).astype(F)


def limit_period32(v, offset, period=PI32):
    """mmdet3d limit_period in fp32: v - floor(v / p + offset) * p."""
    v = np.asarray(v, F)
    return (v - (np.floor((v / F(period)).astype(F) + F(offset)).astype(F) * F(period)).astype(F)).astype(F)


def split_head(head, C, R):
    """head [R (C + 11), H, W] -> per anchor (cls [A, C], reg [A, 9], dir [A, 2]), anchor (y W + x) R + a."""
    head = np.asarray(head, F)
    if head.ndim == 4:
        head = head[0]
    HW = head.shape[1] * head.shape[2]
    flat = head.reshape(head.shape[0], HW)

    def group(lo, K):
        return flat[lo:lo + R * K].reshape(R, K, HW).transpose(2, 0, 1).reshape(HW * R, K)
    return group(0, C), group(R * C, CODE), group(R * (C + CODE), 2)


def decode32(reg, anchors):
    """DeltaXYZWLHRBBoxCoder.decode with every operation rounded to fp32 (the kernel's order)."""
    reg, an = np.asarray(reg, F), np.asarray(anchors, F)
    xa, ya, za, wa, la, ha, ra = [an[:, k] for k in range(7)]
    xt, yt, zt, wt, lt, ht, rt = [reg[:, k] for k in range(7)]
    za = (za + (ha * F(0.5)).astype(F)).astype(F)
    diag = np.sqrt(((la * la).astype(F) + (wa * wa).astype(F)).astype(F)).astype(F)
    with np.errstate(over="ignore", invalid="ignore"):
        x = ((xt * diag).astype(F) + xa).astype(F)
        y = ((yt * diag).astype(F) + ya).astype(F)
        z = ((zt * ha).astype(F) + za).astype(F)
        w = (np.exp(wt, dtype=F) * wa).astype(F)
        l = (np.exp(lt, dtype=F) * la).astype(F)
        h = (np.exp(ht, dtype=F) * ha).astype(F)
        r = (rt + ra).astype(F)
        z = (z - (h * F(0.5)).astype(F)).astype(F)
        vel = (reg[:, 7:] + an[:, 7:]).astype(F)
    return np.concatenate([np.stack([x, y, z, w, l, h, r], 1), vel], 1).astype(F)


def anchor3d_decode_ref(head, anchors, C, R, nms_pre, score_thr, nms_thr, max_num, dir_offset, dir_limit_offset,
                        details=False):
    """(boxes [K, 9], scores [K], labels [K] int64); details=True adds dict(kept=anchor indices in kept order,
    per_class=[kept positions surviving NMS per class])."""
    import oracle
    cls, reg, dirl = split_head(head, C, R)
    A = cls.shape[0]
    scores = sigmoid32(cls)
    mx = scores.max(1)                                       # NaN when a class is NaN (torch.max)
    dir_label = (dirl[:, 1] > dirl[:, 0]).astype(np.int64)   # argmax, a tie to bin 0
    if A > nms_pre:                                          # torch.topk: NaN above every number, ties by the lower index
        nan = np.isnan(mx)
        kept = np.lexsort((np.arange(A), -np.where(nan, 0, mx), ~nan))[:nms_pre]
    else:
        kept = np.arange(A)
    boxes = decode32(reg[kept], anchors[kept])
    sk = scores[kept]
    finite = np.isfinite(boxes).all(1)
    out_b, out_s, out_l, per_class = [], [], [], []
    for c in range(C):
        with np.errstate(invalid="ignore"):
            idx = np.nonzero((sk[:, c] > F(score_thr)) & finite)[0]
        idx = idx[np.argsort(-sk[idx, c], kind="stable")]    # descending class score, ties by kept order
        keep = np.zeros(0, np.int64)
        if len(idx):
            k, nk = oracle.nms(boxes[idx, :7], float(nms_thr))
            keep = idx[k[:nk]]
        per_class.append(keep)
        out_b.append(boxes[keep])
        out_s.append(sk[keep, c])
        out_l.append(np.full(len(keep), c, np.int64))
    b = np.concatenate(out_b).reshape(-1, CODE).astype(F)
    s = np.concatenate(out_s).astype(F)
    lab = np.concatenate(out_l)
    dirs = dir_label[kept][np.concatenate(per_class).astype(np.int64)] if len(b) else np.zeros(0, np.int64)
    if len(b) > max_num:
        o = np.argsort(-s, kind="stable")[:max_num]
        b, s, lab, dirs = b[o], s[o], lab[o], dirs[o]
    b = b.copy()
    off = F(dir_offset)
    r = limit_period32((b[:, 6] - off).astype(F), dir_limit_offset)
    b[:, 6] = ((r + off).astype(F) + (PI32 * dirs.astype(F)).astype(F)).astype(F)
    res = (b, s, lab)
    return res + (dict(kept=kept, per_class=per_class),) if details else res


def aligned_anchors_loops(H, W, xy, sizes_z, rotations, n_custom):
    """AlignedAnchor3DRangeGenerator(align_corner=False) written as loops in its own terms: per (range, size) pair a
    [1, H, W, 1, R, 7 + n_custom] block from meshgrid(x_centres, y_centres, z_centres, rotations), concatenated along the
    size axis, flattened.  An independent restatement of paddle3d_b200.bevfusion.make_anchors for the tests."""
    blocks = []
    for size, z in sizes_z:
        xc = np.linspace(-xy, xy, W + 1)
        yc = np.linspace(-xy, xy, H + 1)
        zc = np.linspace(z, z, 2)
        xc = xc + (xc[1] - xc[0]) / 2
        yc = yc + (yc[1] - yc[0]) / 2
        zc = zc + (zc[1] - zc[0]) / 2
        blk = np.zeros((1, H, W, 1, len(rotations), 7 + n_custom))
        for iy in range(H):
            for ix in range(W):
                for ir, rot in enumerate(rotations):
                    blk[0, iy, ix, 0, ir, :7] = [xc[ix], yc[iy], zc[0], size[0], size[1], size[2], rot]
        blocks.append(blk)
    out = np.concatenate(blocks, axis=-3)
    return out.reshape(-1, 7 + n_custom).astype(F)


# ------------------------------------------------------------------------------------------------------ the CPU arm
class CpuBEVFusion:
    """CPU arm of a BEVFusion frame (weights: paddle3d_b200.bevfusion.BEVFusion.export_numpy(), cfg its config): the
    oracle's hard_voxelize, HardVFE in fp64, PointPillarsScatter, SecondTrunk; the oracle's LSS view transform and
    the camera encoder; the concat (camera first), reduc_conv, the SE gate in fp64, the head conv, and the decode
    restatement."""

    def __init__(self, weights, cfg, anchors):
        self.w, self.cfg, self.anchors = weights, cfg, anchors

    def run(self, points, cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size):
        import oracle
        from oracle.lss import view_transform
        from oracle.pointpillars import _layer, second_trunk
        w, c = self.w, self.cfg
        pts = np.asarray(points, F)
        pts = pts[np.isfinite(pts).all(1)]
        pcr, vs = c["point_cloud_range"], c["voxel_size"]
        nx, ny = int(round((pcr[3] - pcr[0]) / vs[0])), int(round((pcr[4] - pcr[1]) / vs[1]))
        if len(pts):
            v, co, n, nv = oracle.hard_voxelize(pts, vs, pcr, c["max_points"], c["max_voxels"])
            k = int(nv[0])
        else:
            k = 0
        C1 = w["vfe"][1]["weight"].shape[1]
        if k:
            coors = np.concatenate([np.zeros((k, 1), np.int32), co[:k]], 1)
            feats = hard_vfe_ref(v[:k], n[:k], coors, w["vfe"], vs, pcr).astype(F)
            bev_l = oracle.pillar_scatter(feats, coors, 1, ny, nx)
        else:
            bev_l = np.zeros((1, C1, ny, nx), F)
        lidar = second_trunk(w, bev_l)
        bev_c, _, _ = view_transform(cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size)
        x = bev_c
        for l in w["cam"]:
            x = _layer(l, x)
        fused = np.concatenate([x, lidar], 1).astype(F)
        y = _layer(w["reduc"], fused)
        gate = se_gate_ref(np.asarray(y, np.float64).transpose(0, 2, 3, 1), w["se"]["weight"], w["se"]["bias"])
        se = (np.asarray(y, np.float64) * gate[:, :, None, None]).astype(F)
        h = w["head"]
        planes = oracle.conv2d(se, h["weight"], h["bias"], 1, 0)
        t = c["test"]
        from paddle3d_b200.bevfusion import CLASSES, anchors_per_loc
        boxes, scores, labels = anchor3d_decode_ref(planes, self.anchors, len(CLASSES), anchors_per_loc(c), t["nms_pre"],
                                                    t["score_thr"], t["nms_thr"], t["max_num"], t["dir_offset"],
                                                    t["dir_limit_offset"])
        return dict(fused=fused, se=se, planes=planes, boxes=boxes, scores=scores, labels=labels, num_voxels=k)
