"""TEST INFRASTRUCTURE ONLY: numpy restatement of BEVDet's box decode (CenterHead.get_bboxes, get_task_detections,
CenterPointBBoxCoder.decode and the numba circle_nms; PARITY UNPINNED as paddle3d_b200.bevdet.TEST_CFG_BEVDET), and the
CPU arms of the BEVDet / BEVDet4D frames that end in it.

bevdet_postprocess_ref follows the reference's steps in the reference's order, not the kernel's: top-K per class, then
top-K of those, decode, score threshold and range mask after the decode, dims multiplied by nms_rescale_factor, NMS,
dims divided again, bottom centre from the divided dz, circle_nms as its double loop.  The kernel thresholds first,
selects once and writes the unscaled dims; the tests compare the two formulations.  Where the reference leaves an order
open (torch.topk and argsort among equal scores) this file takes ascending class * H*W + cell, the order the op defines.
pre_max_size is applied to circle tasks as well (the reference applies it to rotate tasks only; the op's rule).
Nothing under paddle3d_b200/ imports this module."""
import numpy as np

import oracle
from oracle.bevdet import CpuBEVDet

from bevdet4d_oracle import CpuBEVDet4D

F = np.float32


def _topk(scores, k):
    """torch.topk(scores, k) along the last axis with ties by ascending index: (values, indices)."""
    idx = np.argsort(-scores, axis=-1, kind="stable")[..., :k]
    return np.take_along_axis(scores, idx, -1), idx


def _per_task(v, t):
    return v[t] if isinstance(v, (list, tuple)) else v


def circle_nms(dets, thresh, post_max_size):
    """The numba circle_nms on dets [n, 3] = x, y, score already in descending score order (fp32 arithmetic)."""
    x1, y1 = dets[:, 0], dets[:, 1]
    ndets = len(dets)
    suppressed = np.zeros(ndets, np.int32)
    keep = []
    for i in range(ndets):
        if suppressed[i] == 1:
            continue
        keep.append(i)
        for j in range(i + 1, ndets):
            if suppressed[j] == 1:
                continue
            dist = F(F(x1[i] - x1[j]) ** 2) + F(F(y1[i] - y1[j]) ** 2)
            if dist <= thresh:
                suppressed[j] = 1
    return keep[:post_max_size]


def task_selection(hm, reg, height, dim, vel, rot, tc):
    """CenterPointBBoxCoder.decode of one task (NCHW fp32, batch 1): (boxes [n, 9] = x, y, z, dx, dy, dz, rot, vx, vy with z
    the gravity centre, scores [n], classes [n], flat class * H*W + cell index [n]) after the threshold and range masks,
    in score order."""
    hm = np.asarray(hm, F)
    _, C, H, W = hm.shape
    with np.errstate(over="ignore"):
        heat = (F(1.0) / (F(1.0) + np.exp(-hm, dtype=F))).astype(F).reshape(C, H * W)  # sigmoid, fp32
    K = min(int(tc["max_num"]), H * W)
    # _topk: per class, then over the classes' lists
    s_c, i_c = _topk(heat, K)                       # [C, K]
    s, flat = _topk(s_c.reshape(-1), K)             # [K]
    cls = flat // K
    inds = i_c.reshape(-1)[flat]
    ys, xs = (inds // W).astype(F), (inds % W).astype(F)
    g = lambda a, ch: np.asarray(a, F)[0, ch].reshape(-1)[inds]  # noqa: E731  _transpose_and_gather_feat
    osf, vs, pcr = F(tc["out_size_factor"]), np.asarray(tc["voxel_size"], F), np.asarray(tc["point_cloud_range"], F)
    xs = (((xs + g(reg, 0)).astype(F) * osf).astype(F) * vs[0]).astype(F) + pcr[0]
    ys = (((ys + g(reg, 1)).astype(F) * osf).astype(F) * vs[1]).astype(F) + pcr[1]
    with np.errstate(over="ignore"):
        dims = [np.exp(g(dim, k), dtype=F) for k in range(3)]   # norm_bbox
    r = np.arctan2(g(rot, 0), g(rot, 1)).astype(F)
    boxes = np.stack([xs, ys, g(height, 0)] + dims + [r, g(vel, 0), g(vel, 1)], 1).astype(F)
    rng = np.asarray(tc["post_center_limit_range"], F)
    mask = (s > F(tc["score_threshold"])) & (boxes[:, :3] >= rng[:3]).all(1) & (boxes[:, :3] <= rng[3:]).all(1)
    return boxes[mask], s[mask], cls[mask], (cls * (H * W) + inds)[mask]


def task_detections(boxes, scores, cls, t, tc):
    """get_task_detections of task t on the decoded boxes: indices kept, and the boxes after the scale round trip."""
    boxes = boxes.copy()
    n = min(len(boxes), int(tc["pre_max_size"]))
    post = int(tc["post_max_size"])
    if _per_task(tc["nms_type"], t) == "circle":
        keep = circle_nms(np.concatenate([boxes[:n, :2], scores[:n, None]], 1), F(_per_task(tc["min_radius"], t)), post)
        return np.asarray(keep, np.int64), boxes
    f = _per_task(tc["nms_rescale_factor"], t)
    fac = np.asarray([f[c] for c in cls] if isinstance(f, (list, tuple)) else [f] * len(cls), F).reshape(-1, 1)
    boxes[:, 3:6] = (boxes[:, 3:6] * fac).astype(F)
    keep = np.zeros(0, np.int64)
    if n:
        k, nk = oracle.nms(boxes[:n, :7], float(_per_task(tc["nms_thr"], t)))   # nms_gpu: greedy on rotated BEV IoU > thr
        keep = k[:nk][:post].astype(np.int64)
    boxes[:, 3:6] = (boxes[:, 3:6] / fac).astype(F)
    return keep, boxes


def bevdet_postprocess_ref(h, test_cfg, label_offsets, details=False):
    """h: dict name -> [per-task NCHW fp32 array].  Returns (boxes [K, 9] with z the bottom centre, scores [K], labels [K]
    int64, counts [T]); details=True adds per task (flat indices selected, indices kept among them)."""
    tc = test_cfg
    out_b, out_s, out_l, counts, det = [], [], [], [], []
    for t in range(len(h["hm"])):
        boxes, scores, cls, flat = task_selection(h["hm"][t], h["reg"][t], h["height"][t], h["dim"][t], h["vel"][t],
                                                  h["rot"][t], tc)
        keep, boxes = task_detections(boxes, scores, cls, t, tc)
        b = boxes[keep]
        b[:, 2] = b[:, 2] - b[:, 5] * F(0.5)   # get_bboxes: bottom centre, from the dz the round trip left
        out_b.append(b)
        out_s.append(scores[keep])
        out_l.append(cls[keep].astype(np.int64) + int(label_offsets[t]))
        counts.append(len(keep))
        det.append((flat, keep))
    res = (np.concatenate(out_b).astype(F).reshape(-1, 9), np.concatenate(out_s).astype(F), np.concatenate(out_l),
           np.asarray(counts, np.int32))
    return res + (det,) if details else res


class _BEVDetDecode:
    """A CPU arm whose frame ends in bevdet_postprocess_ref: the base arm runs with the Paddle op's test config (its own
    postprocess needs those keys) and the boxes are replaced by BEVDet's decode of the same head planes."""

    def __init__(self, weights, test_cfg, label_offsets):
        from paddle3d_b200.bevdet import CONFIG
        super().__init__(weights, CONFIG["test"], label_offsets)
        self.bevdet_cfg = test_cfg

    def run(self, *args, **kwargs):
        out = super().run(*args, **kwargs)
        boxes, scores, labels, _ = bevdet_postprocess_ref(out["head"], self.bevdet_cfg, self.off)
        return dict(out, boxes=boxes, scores=scores, labels=labels)


class CpuBEVDetNMS(_BEVDetDecode, CpuBEVDet):
    pass


class CpuBEVDet4DNMS(_BEVDetDecode, CpuBEVDet4D):
    pass
