"""`paddle3d.ops.centerpoint_postprocess` mirror — op `centerpoint_postprocess`
(paddle3d/ops/centerpoint_postprocess/postprocess.cc:91-104; call site center_head.py:320-325)."""
import ctypes as C

import torch

from .._lib import check, host_floats, host_ints, lib
from .._mem import ptr, require_cuda, stream, workspace


def centerpoint_postprocess_device(hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range,
                                   num_classes, down_ratio, score_threshold, nms_iou_threshold, nms_pre_max_size,
                                   nms_post_max_size, with_velocity):
    """Sync-free form: returns worst-case-sized (bboxes, scores, labels) plus counts [T+1] on the device
    (rows per task, then total)."""
    T = len(hm)
    lists = []
    for name, lst in (("hm", hm), ("reg", reg), ("height", height), ("dim", dim), ("vel", vel), ("rot", rot)):
        if len(lst) != T:
            raise ValueError("%s must have one tensor per task" % name)
        lists.append([require_cuda(t, name, torch.float32) for t in lst])
    if lists[0][0].shape[0] != 1:
        raise ValueError("hm batch size must be 1.")  # CHECK_INPUT_BATCHSIZE, postprocess.cu:19-20,138
    dev = lists[0][0].device
    H, W = int(lists[0][0].shape[2]), int(lists[0][0].shape[3])
    dims = 9 if with_velocity else 7
    rows = T * max(int(nms_post_max_size), 1)
    bboxes = torch.empty((rows, dims), dtype=torch.float32, device=dev)
    scores = torch.empty((rows,), dtype=torch.float32, device=dev)
    labels = torch.empty((rows,), dtype=torch.int64, device=dev)
    counts = torch.empty((T + 1,), dtype=torch.int32, device=dev)
    L = lib()
    ws = workspace(L.p3d_centerpoint_postprocess_workspace_bytes(T, H, W, int(nms_pre_max_size), int(nms_post_max_size)),
                   dev, "cpp")
    PP = C.c_void_p * T
    arrs = [PP(*[t.data_ptr() for t in lst]) for lst in lists]
    hm_c = host_ints([t.shape[1] for t in lists[0]])
    check(L.p3d_centerpoint_postprocess(T, arrs[0], hm_c, arrs[1], arrs[2], arrs[3], arrs[4], arrs[5], H, W,
                                        host_floats(voxel_size), host_floats(point_cloud_range),
                                        host_floats(post_center_range), host_ints(list(num_classes)[:T]),
                                        int(down_ratio), float(score_threshold), float(nms_iou_threshold),
                                        int(nms_pre_max_size), int(nms_post_max_size), int(bool(with_velocity)),
                                        ptr(bboxes), ptr(scores), ptr(labels), ptr(counts), ptr(ws), ws.numel(),
                                        stream(dev)), "centerpoint_postprocess")
    return bboxes, scores, labels, counts


def centerpoint_postprocess_heads(h, voxel_size, point_cloud_range, test_cfg, label_offsets):
    """centerpoint_postprocess_device of a CenterHead output h = dict name -> [tensor per task], with the range limit,
    down ratio, threshold and NMS settings of test_cfg and the tasks' label offsets.  With a "vel" head the boxes have 9
    columns (x, y, z, d0, d1, d2, vx, vy, rot), without one 7."""
    tc = test_cfg
    with_velocity = "vel" in h
    return centerpoint_postprocess_device(
        h["hm"], h["reg"], h["height"], h["dim"], h["vel"] if with_velocity else h["reg"], h["rot"], voxel_size,
        point_cloud_range, tc["post_center_limit_range"], label_offsets, tc["down_ratio"], tc["score_threshold"],
        tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"], with_velocity)


def centerpoint_postprocess(hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range,
                            num_classes, down_ratio, score_threshold, nms_iou_threshold, nms_pre_max_size,
                            nms_post_max_size, with_velocity):
    """Reference signature and outputs: (bboxes [K, 9|7] fp32, scores [K] fp32, labels [K] int64).
    The only host sync is the read of K needed to give the outputs their dynamic shape."""
    bboxes, scores, labels, counts = centerpoint_postprocess_device(
        hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range, num_classes, down_ratio,
        score_threshold, nms_iou_threshold, nms_pre_max_size, nms_post_max_size, with_velocity)
    k = int(counts[-1].item())
    return bboxes[:k], scores[:k], labels[:k]
