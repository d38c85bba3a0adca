"""mmdet3d Anchor3DHead's box decode with per-class rotated NMS on the device — op `p3d_anchor3d_postprocess`
(include/p3d_b200.h states its six rules; PARITY UNPINNED: recalled from mmdet3d v0.17 get_bboxes_single and
box3d_multiclass_nms).  Rows are (x, y, z of the bottom centre, w, l, h, r, vx, vy)."""
import torch

from .._lib import check, lib
from .._mem import ptr, require_cuda, stream, workspace


def anchor3d_postprocess_device(head, anchors, num_classes, anchors_per_loc, nms_pre, score_thr, nms_thr, max_num,
                                dir_offset, dir_limit_offset, out=None):
    """head [1, R (C + 9 + 2), H, W] fp32 (cls | reg | dir planes), anchors [H * W * R, 9] fp32 on the device.  Sync-free:
    returns (boxes [max_num, 9], scores [max_num], labels int64 [max_num], count [1] int32) with count rows valid.
    out: those four buffers to reuse (a captured frame keeps their addresses)."""
    head = require_cuda(head, "head", torch.float32)
    anchors = require_cuda(anchors, "anchors", torch.float32)
    C, R = int(num_classes), int(anchors_per_loc)
    if head.dim() != 4 or head.shape[0] != 1 or head.shape[1] != R * (C + 9 + 2):
        raise ValueError("head must be [1, R * (C + 11), H, W], got %s" % (tuple(head.shape),))
    H, W = int(head.shape[2]), int(head.shape[3])
    if tuple(anchors.shape) != (H * W * R, 9):
        raise ValueError("anchors must be [H * W * R, 9], got %s" % (tuple(anchors.shape),))
    dev = head.device
    if out is None:
        out = (torch.empty((max_num, 9), dtype=torch.float32, device=dev),
               torch.empty((max_num,), dtype=torch.float32, device=dev),
               torch.empty((max_num,), dtype=torch.int64, device=dev),
               torch.empty((1,), dtype=torch.int32, device=dev))
    boxes, scores, labels, count = out
    L = lib()
    ws = workspace(L.p3d_anchor3d_postprocess_workspace_bytes(H, W, R, C, int(nms_pre), int(max_num)), dev, "a3d")
    check(L.p3d_anchor3d_postprocess(ptr(head), H, W, R, C, ptr(anchors), int(nms_pre), float(score_thr), float(nms_thr),
                                     int(max_num), float(dir_offset), float(dir_limit_offset), ptr(boxes), ptr(scores),
                                     ptr(labels), ptr(count), ptr(ws), ws.numel(), stream(dev)), "anchor3d_postprocess")
    return boxes, scores, labels, count


def anchor3d_postprocess(head, anchors, num_classes, anchors_per_loc, nms_pre, score_thr, nms_thr, max_num, dir_offset,
                         dir_limit_offset):
    """(boxes [K, 9] fp32, scores [K] fp32, labels [K] int64).  The only host sync is the read of K."""
    boxes, scores, labels, count = anchor3d_postprocess_device(head, anchors, num_classes, anchors_per_loc, nms_pre,
                                                               score_thr, nms_thr, max_num, dir_offset, dir_limit_offset)
    k = int(count.item())
    return boxes[:k], scores[:k], labels[:k]
