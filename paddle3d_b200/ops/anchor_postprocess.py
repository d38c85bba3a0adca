"""Anchor (SSD) head postprocess of PointPillars: SECOND v1.5 `VoxelNet.predict` at batch 1 with sigmoid scores and
class-agnostic NMS (the path the reference's SSDHead.post_process -> ops.nms_utils.rotate_nms_pcdet ports), as one
sync-free call into csrc/anchor_postprocess.cu.  The anchors and their voxel-index corners are constant per model: build
them once on the host (pointpillars.create_anchors_3d_stride / anchor_voxel_corners) and keep them on the device."""
import torch

from .._lib import check, host_floats, lib
from .._mem import ptr, require_cuda, stream, workspace


def anchor_head_postprocess_device(head, anchors, anchor_corners, coords, num_coords, grid_size, post_center_range,
                                   anchor_area_threshold=1, score_threshold=0.05, nms_iou_threshold=0.5,
                                   nms_pre_max_size=1000, nms_post_max_size=300, anchor_mask=None, sorted_out=None,
                                   num_classes=1):
    """head [1, R (C + 9), H, W] fp32 (cls R C | box 7 R | dir 2 R planes, C = num_classes; cls channel a * C + c is
    class c of anchor (y * W + x) * R + a); anchors [H * W * R, 7]; anchor_corners [A, 4] int32; coords [cap, 4]
    (b, z, y, x) int32 pillar coords with num_coords [1] int32 valid rows; grid_size (nx, ny).  An anchor scores
    max_c sigmoid(cls_c) and is labelled with the first class reaching it; NMS runs over all classes together.
    Returns capacity-sized (boxes [post_max, 7], scores [post_max], labels [post_max] int64, counts [2] int32 =
    (score-threshold candidates, rows written)), all on the device.  anchor_mask: optional uint8 [A] output;
    sorted_out: optional (boxes [pre_max, 7], scores [pre_max]) output of the decoded candidates in score order."""
    head = require_cuda(head, "head", torch.float32)
    anchors = require_cuda(anchors, "anchors", torch.float32)
    anchor_corners = require_cuda(anchor_corners, "anchor_corners", torch.int32)
    coords = require_cuda(coords, "coords", torch.int32)
    num_coords = require_cuda(num_coords, "num_coords", torch.int32)
    C = int(num_classes)
    if C < 1:
        raise ValueError("num_classes must be >= 1")
    if head.dim() != 4 or head.shape[0] != 1 or head.shape[1] % (C + 9):
        raise ValueError("head must be [1, anchors_per_loc * (num_classes + 9), H, W]")
    R, H, W = head.shape[1] // (C + 9), int(head.shape[2]), int(head.shape[3])
    A = H * W * R
    if tuple(anchors.shape) != (A, 7) or tuple(anchor_corners.shape) != (A, 4) or coords.dim() != 2 or coords.shape[1] != 4:
        raise ValueError("anchors [A, 7], anchor_corners [A, 4] and coords [n, 4] must match the head (A = %d)" % A)
    dev = head.device
    nx, ny = int(grid_size[0]), int(grid_size[1])
    pre, post = int(nms_pre_max_size), int(nms_post_max_size)
    boxes = torch.empty((post, 7), dtype=torch.float32, device=dev)
    scores = torch.empty((post,), dtype=torch.float32, device=dev)
    labels = torch.empty((post,), dtype=torch.int64, device=dev)
    counts = torch.empty((2,), dtype=torch.int32, device=dev)
    L = lib()
    nbytes = L.p3d_anchor_head_postprocess_workspace_bytes(A, nx, ny, pre)
    if not nbytes:
        raise ValueError("unsupported anchor postprocess shape: %d anchors, grid %d x %d, pre_max %d" % (A, nx, ny, pre))
    ws = workspace(nbytes, dev, "ahp")
    if anchor_mask is not None:
        anchor_mask = require_cuda(anchor_mask, "anchor_mask", torch.uint8)
    sb, ss = sorted_out if sorted_out is not None else (None, None)
    check(L.p3d_anchor_head_postprocess(ptr(head), H, W, R, C, ptr(anchors), ptr(anchor_corners), ptr(coords),
                                        ptr(num_coords), int(coords.shape[0]), nx, ny, int(anchor_area_threshold),
                                        float(score_threshold), float(nms_iou_threshold), pre, post,
                                        host_floats(post_center_range), ptr(boxes), ptr(scores), ptr(labels), ptr(counts),
                                        ptr(anchor_mask), ptr(sb), ptr(ss), ptr(ws), ws.numel(), stream(dev)),
          "anchor_head_postprocess")
    return boxes, scores, labels, counts


def anchor_head_postprocess(*args, **kwargs):
    """Same as anchor_head_postprocess_device, trimmed to the valid rows: (boxes [K, 7], scores [K], labels [K]).  The
    only host sync is the read of K."""
    boxes, scores, labels, counts = anchor_head_postprocess_device(*args, **kwargs)
    k = int(counts[-1].item())
    return boxes[:k], scores[:k], labels[:k]
