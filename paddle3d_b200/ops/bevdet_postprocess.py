"""BEVDet's box decode on the device — op `p3d_bevdet_postprocess` (include/p3d_b200.h states its rules; PARITY UNPINNED:
recalled from BEVDet's CenterHead.get_bboxes / get_task_detections, CenterPointBBoxCoder.decode and circle_nms).  Rows are
(x, y, z of the bottom centre, dx, dy, dz, rot, vx, vy)."""
import ctypes as C

import torch

from .._lib import check, host_floats, host_ints, lib
from .._mem import ptr, require_cuda, stream, workspace

NMS_TYPES = {"rotate": 0, "circle": 1}  # P3D_BEVDET_NMS_ROTATE / P3D_BEVDET_NMS_CIRCLE


def _per_task(v, T, name):
    """A scalar for every task, or one value per task."""
    if isinstance(v, (list, tuple)):
        if len(v) != T:
            raise ValueError("%s must be a scalar or have one entry per task (%d), got %d" % (name, T, len(v)))
        return list(v)
    return [v] * T


def task_attrs(T, channels, nms_type, nms_thr, nms_rescale_factor, min_radius):
    """The op's host attribute lists from a test_cfg's values: (nms_type ints [T], nms_thr [T], min_radius [T], rescale
    [sum C_t], one factor per class).  nms_type / nms_thr / min_radius: a scalar or one entry per task;
    nms_rescale_factor: a scalar, or per task a scalar or one factor per class of the task."""
    types = []
    for t, name in enumerate(_per_task(nms_type, T, "nms_type")):
        if name not in NMS_TYPES:
            raise ValueError("nms_type[%d] = %r: the BEVDet decode has %s" % (t, name, " and ".join(sorted(NMS_TYPES))))
        types.append(NMS_TYPES[name])
    rescale = []
    for t, f in enumerate(_per_task(nms_rescale_factor, T, "nms_rescale_factor")):
        f = _per_task(f, channels[t], "nms_rescale_factor[%d]" % t)
        if any(not float(v) > 0.0 for v in f):
            raise ValueError("nms_rescale_factor[%d] must be positive, got %r" % (t, f))
        rescale += [float(v) for v in f]
    radius = [float(v) for v in _per_task(min_radius, T, "min_radius")]
    if any(not r >= 0.0 for r in radius):
        raise ValueError("min_radius must not be negative, got %r" % (radius,))
    return types, [float(v) for v in _per_task(nms_thr, T, "nms_thr")], radius, rescale


def bevdet_postprocess_device(hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range,
                              label_offsets, out_size_factor, score_threshold, max_num, pre_max_size, post_max_size,
                              nms_type, nms_thr, nms_rescale_factor, min_radius):
    """Sync-free form: returns worst-case-sized (bboxes [T * post_max_size, 9], scores, labels) plus counts [T+1] on the
    device (rows per task, then total)."""
    T = len(hm)
    lists = []
    for name, lst in (("hm", hm), ("reg", reg), ("height", height), ("dim", dim), ("vel", vel), ("rot", rot)):
        if len(lst) != T:
            raise ValueError("%s must have one tensor per task" % name)
        lists.append([require_cuda(t, name, torch.float32) for t in lst])
    if lists[0][0].shape[0] != 1:
        raise ValueError("hm batch size must be 1.")
    if len(label_offsets) < T:
        raise ValueError("label_offsets must have one entry per task")
    channels = [int(t.shape[1]) for t in lists[0]]
    types, thr, radius, rescale = task_attrs(T, channels, nms_type, nms_thr, nms_rescale_factor, min_radius)
    dev = lists[0][0].device
    H, W = int(lists[0][0].shape[2]), int(lists[0][0].shape[3])
    rows = T * max(int(post_max_size), 1)
    bboxes = torch.empty((rows, 9), dtype=torch.float32, device=dev)
    scores = torch.empty((rows,), dtype=torch.float32, device=dev)
    labels = torch.empty((rows,), dtype=torch.int64, device=dev)
    counts = torch.empty((T + 1,), dtype=torch.int32, device=dev)
    L = lib()
    hm_c = host_ints(channels)
    ws = workspace(L.p3d_bevdet_postprocess_workspace_bytes(T, hm_c, H, W, int(max_num)), dev, "bdp")
    PP = C.c_void_p * T
    arrs = [PP(*[t.data_ptr() for t in lst]) for lst in lists]
    check(L.p3d_bevdet_postprocess(T, arrs[0], hm_c, arrs[1], arrs[2], arrs[3], arrs[4], arrs[5], H, W,
                                   host_floats(voxel_size), host_floats(point_cloud_range),
                                   host_floats(post_center_range), int(out_size_factor), float(score_threshold),
                                   int(max_num), int(pre_max_size), int(post_max_size), host_ints(types), host_floats(thr),
                                   host_floats(radius), host_floats(rescale), host_ints(list(label_offsets)[:T]),
                                   ptr(bboxes), ptr(scores), ptr(labels), ptr(counts), ptr(ws), ws.numel(), stream(dev)),
          "bevdet_postprocess")
    return bboxes, scores, labels, counts


def bevdet_postprocess_heads(h, test_cfg, label_offsets):
    """bevdet_postprocess_device of a CenterHead output h = dict name -> [tensor per task] with a BEVDet test_cfg (the
    one with nms_type) and the tasks' label offsets.  test_cfg's max_per_img is accepted and not used: get_bboxes never
    reads it, the per-task post_max_size is the only cut."""
    tc = test_cfg
    return bevdet_postprocess_device(
        h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"], tc["point_cloud_range"],
        tc["post_center_limit_range"], label_offsets, tc["out_size_factor"], tc["score_threshold"], tc["max_num"],
        tc["pre_max_size"], tc["post_max_size"], tc["nms_type"], tc["nms_thr"], tc["nms_rescale_factor"], tc["min_radius"])


def bevdet_postprocess(hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range, label_offsets,
                       out_size_factor, score_threshold, max_num, pre_max_size, post_max_size, nms_type, nms_thr,
                       nms_rescale_factor, min_radius):
    """(bboxes [K, 9] fp32, scores [K] fp32, labels [K] int64).  The only host sync is the read of K needed to give the
    outputs their dynamic shape."""
    bboxes, scores, labels, counts = bevdet_postprocess_device(
        hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range, label_offsets, out_size_factor,
        score_threshold, max_num, pre_max_size, post_max_size, nms_type, nms_thr, nms_rescale_factor, min_radius)
    k = int(counts[-1].item())
    return bboxes[:k], scores[:k], labels[:k]
