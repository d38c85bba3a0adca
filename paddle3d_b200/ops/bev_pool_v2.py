"""`paddle3d.ops.bev_pool_v2` mirror — op `bev_pool_v2` (paddle3d/ops/bev_pool_v2/bev_pool.cc:111-118)."""
import numpy as np
import torch

from .._lib import check, lib
from .._mem import ptr, require_cuda, stream


def bev_pool_v2(depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_lengths, interval_starts, bev_feat_shape):
    """Argument order as the reference op (lengths BEFORE starts; call site bevdet_transformer.py:44-46).
    depth [B*N,D,H,W] fp32, feat [B*N,H,W,C] fp32, ranks int32, bev_feat_shape (B, Y, X, C) -> out fp32."""
    depth = require_cuda(depth, "depth", torch.float32)
    feat = require_cuda(feat, "feat", torch.float32)
    rd = require_cuda(ranks_depth, "ranks_depth", torch.int32)
    rf = require_cuda(ranks_feat, "ranks_feat", torch.int32)
    rb = require_cuda(ranks_bev, "ranks_bev", torch.int32)
    il = require_cuda(interval_lengths, "interval_lengths", torch.int32)
    is_ = require_cuda(interval_starts, "interval_starts", torch.int32)
    c = feat.shape[3]  # bev_pool.cc:36
    out = torch.empty(tuple(int(s) for s in bev_feat_shape), dtype=torch.float32, device=feat.device)
    check(lib().p3d_bev_pool_v2(ptr(depth), ptr(feat), ptr(rd), ptr(rf), ptr(rb), ptr(il), ptr(is_), il.shape[0], c,
                                ptr(out), out.numel(), stream(feat.device)), "bev_pool_v2")
    return out


def voxel_pooling_prepare_v2(coor, grid_lower_bound, grid_interval, grid_size):
    """LSSViewTransformer.voxel_pooling_prepare_v2 (bevdet_transformer.py:230-274) on the device, no host sync:
    coor [B, N, D, H, W, 3] fp32 -> (ranks_bev, ranks_depth, ranks_feat, interval_starts, interval_lengths, counts);
    the five rank arrays are int32 tensors of capacity B*N*D*H*W whose first counts[0] (ranks) / counts[1] (intervals)
    entries are valid (`trim` slices them like the reference returns them, at the cost of one D2H read)."""
    from .._lib import host_floats, host_ints
    from .._mem import workspace
    coor = require_cuda(coor, "coor", torch.float32)
    B, N, D, H, W, three = coor.shape
    assert three == 3
    n = B * N * D * H * W
    dev = coor.device
    outs = [torch.empty((n,), dtype=torch.int32, device=dev) for _ in range(5)]
    counts = torch.empty((2,), dtype=torch.int32, device=dev)
    L = lib()
    wsb = L.p3d_bev_pool_prepare_workspace_bytes(n)
    ws = workspace(wsb, dev, "bev_pool_prepare")
    check(L.p3d_bev_pool_prepare(ptr(coor), B, N, D, H, W, host_floats(grid_lower_bound), host_floats(grid_interval),
                                 host_ints(grid_size), ptr(outs[0]), ptr(outs[1]), ptr(outs[2]), ptr(outs[3]), ptr(outs[4]),
                                 ptr(counts), ptr(ws), wsb, stream(dev)), "bev_pool_prepare")
    return outs[0], outs[1], outs[2], outs[3], outs[4], counts


def trim(prepared):
    """Slice the capacity-sized outputs of voxel_pooling_prepare_v2 to their valid lengths (one D2H read), in the
    reference's return order (ranks_bev, ranks_depth, ranks_feat, interval_starts, interval_lengths)."""
    rb, rd, rf, st, ln, counts = prepared
    k, m = [int(v) for v in counts.cpu()]
    if k == 0 or m == 0:
        return None, None, None, None, None
    return rb[:k], rd[:k], rf[:k], st[:m], ln[:m]


# ---------------------------------------------------------------------------------------------- LSS view transform
CAM_FLOATS = 24  # struct p3d_lss_camera: inv_post_rot[9], post_trans[3], combine[9], trans[3]


def pack_cameras(sensor2ego, cam2imgs, post_rots, post_trans, bda):
    """Host camera descriptor of p3d_lss_prepare: fp32 [B*N*24 + B*9] = the p3d_lss_camera entries of every (b, n), then
    bda [B, 3, 3] row-major.  sensor2ego [B, N, 4, 4], cam2imgs / post_rots [B, N, 3, 3], post_trans [B, N, 3], bda
    [B, 3, 3] (numpy or CPU tensors); the inverses and combine = sensor2ego[:3, :3] . inv(cam2imgs) are taken in fp64 and
    every entry is rounded to fp32 once."""
    s2e = _f64(sensor2ego)
    B, N = s2e.shape[:2]
    cams = np.empty((B, N, CAM_FLOATS), np.float64)
    cams[..., 0:9] = np.linalg.inv(_f64(post_rots)).reshape(B, N, 9)
    cams[..., 9:12] = _f64(post_trans).reshape(B, N, 3)
    cams[..., 12:21] = (s2e[..., :3, :3] @ np.linalg.inv(_f64(cam2imgs))).reshape(B, N, 9)
    cams[..., 21:24] = s2e[..., :3, 3]
    return np.concatenate([cams.reshape(-1), _f64(bda).reshape(B * 9)]).astype(np.float32)


def unpack_cameras(desc, B, N):
    """Inverse of pack_cameras: dict of fp32 inv_post_rots / combine [B, N, 3, 3], post_trans / trans [B, N, 3],
    bda [B, 3, 3]."""
    desc = np.asarray(desc, np.float32)
    cams = desc[:B * N * CAM_FLOATS].reshape(B, N, CAM_FLOATS)
    return dict(inv_post_rots=cams[..., 0:9].reshape(B, N, 3, 3), post_trans=cams[..., 9:12],
                combine=cams[..., 12:21].reshape(B, N, 3, 3), trans=cams[..., 21:24],
                bda=desc[B * N * CAM_FLOATS:].reshape(B, 3, 3))


def _f64(a):
    return np.asarray(a.detach().cpu().numpy() if isinstance(a, torch.Tensor) else a, np.float64)


# ------------------------------------------------------------------------------------- BEVDet4D's temporal alignment
SHIFT_FLOATS = 6  # rows 0 and 1 of the 3x3 BEV-pixel transform tf, row-major


def sensor2keyegos(sensor2ego, ego2global, key_ego2global):
    """BEVDet's data pipeline: the cameras of a frame in the key (current) frame's ego frame, fp64
    inv(keyego2global) . ego2global . sensor2ego.  sensor2ego / ego2global [B, N, 4, 4] of the frame; key_ego2global
    [B, N, 4, 4] of the current frame, whose camera 0 defines the key ego (the current frame gives its own sensor2ego)."""
    key = _f64(key_ego2global)[:, 0:1]
    return np.linalg.inv(key) @ _f64(ego2global) @ _f64(sensor2ego)


def shift_matrix(sensor2keyego_curr, sensor2keyego_prev, bda, grid_lower_bound, grid_interval):
    """BEVDet4D.gen_grid's tf [B, 3, 3] in fp64: bda4 = [[bda, 0], [0, 1]], c02l0 = bda4 . curr[:, 0], c12l0 = bda4 . prev[:, 0],
    l02l1 = (c02l0 . inv(c12l0)) restricted to (x, y, w), tf = inv(feat2bev) . l02l1 . feat2bev with feat2bev the BEV pixel
    index -> metres map (grid_interval, grid_lower_bound)."""
    curr, prev, bda = _f64(sensor2keyego_curr), _f64(sensor2keyego_prev), _f64(bda)
    B = curr.shape[0]
    bda4 = np.zeros((B, 4, 4))
    bda4[:, :3, :3] = bda
    bda4[:, 3, 3] = 1.0
    c02l0 = bda4 @ curr[:, 0]
    c12l0 = bda4 @ prev[:, 0]
    l02l1 = (c02l0 @ np.linalg.inv(c12l0))[:, [0, 1, 3]][:, :, [0, 1, 3]]
    f2b = np.array([[grid_interval[0], 0.0, grid_lower_bound[0]], [0.0, grid_interval[1], grid_lower_bound[1]],
                    [0.0, 0.0, 1.0]], np.float64)
    return np.linalg.inv(f2b) @ l02l1 @ f2b


def pack_shift(sensor2keyego_curr, sensor2keyego_prev, bda, grid_lower_bound, grid_interval):
    """Device descriptor of p3d_bev_shift_h16: fp32 [B, 6] = rows 0 and 1 of shift_matrix, computed in fp64 and rounded
    once (pack_cameras' policy).  sensor2keyego_* [B, N, 4, 4] (camera 0 is used), bda [B, 3, 3]."""
    tf = shift_matrix(sensor2keyego_curr, sensor2keyego_prev, bda, grid_lower_bound, grid_interval)
    return np.ascontiguousarray(tf[:, :2].reshape(-1, SHIFT_FLOATS)).astype(np.float32)


def bev_shift_h16(x_h16, shape, tf, C, out_h16=None, out_channels=None, out_c0=0):
    """BEVDet4D.shift_feature on pixel fp16-pair rows (p3d_bev_shift_h16): channels [0, C) of x_h16 [B*h*w, 2*in_C],
    shape = (B, h, w, in_C), sampled at tf's grid (device fp32 [B, 6] from pack_shift) into channels [out_c0, out_c0 + C)
    of out_h16 [B*h*w, 2*out_channels] (None: a new C-channel image; x_h16 itself when the channel ranges are disjoint).
    Returns out_h16."""
    from .sparse_nn import status_tensor
    x_h16 = require_cuda(x_h16, "x_h16", torch.float16)
    tf = require_cuda(tf, "tf", torch.float32)
    b, h, w, in_c = [int(v) for v in shape]
    if tf.numel() != b * SHIFT_FLOATS:
        raise ValueError("bev_shift_h16: tf has %d floats, want %d" % (tf.numel(), b * SHIFT_FLOATS))
    oc = int(out_channels or C)
    dev = x_h16.device
    if out_h16 is None:
        out_h16 = torch.empty((b * h * w, 2 * oc), dtype=torch.float16, device=dev)
    check(lib().p3d_bev_shift_h16(ptr(x_h16), b, h, w, in_c, int(C), ptr(tf), ptr(out_h16), oc, int(out_c0),
                                  ptr(status_tensor(dev)), stream(dev)), "bev_shift_h16")
    return out_h16


def lss_prepare(desc, axis_depth, axis_x, axis_y, B, N, grid_lower_bound, grid_interval, grid_size, with_coor=False):
    """get_lidar_coor + voxel_pooling_prepare_v2 in one pass (p3d_lss_prepare), no host sync.  desc: device fp32 buffer
    from pack_cameras; axis_*: device fp32 frustum axes [D] / [W] / [H].  Returns (ranks_bev, ranks_depth, ranks_feat,
    interval_starts, interval_lengths, counts) as voxel_pooling_prepare_v2 does, plus coor [B, N, D, H, W, 3] with_coor."""
    from .._lib import host_floats, host_ints
    from .._mem import workspace
    desc = require_cuda(desc, "desc", torch.float32)
    ad = require_cuda(axis_depth, "axis_depth", torch.float32)
    ax = require_cuda(axis_x, "axis_x", torch.float32)
    ay = require_cuda(axis_y, "axis_y", torch.float32)
    D, H, W = ad.numel(), ay.numel(), ax.numel()
    if desc.numel() != B * N * CAM_FLOATS + B * 9:
        raise ValueError("lss_prepare: descriptor has %d floats, want %d" % (desc.numel(), B * N * CAM_FLOATS + B * 9))
    n = B * N * D * H * W
    dev = desc.device
    outs = [torch.empty((n,), dtype=torch.int32, device=dev) for _ in range(5)]
    counts = torch.empty((2,), dtype=torch.int32, device=dev)
    coor = torch.empty((B, N, D, H, W, 3), dtype=torch.float32, device=dev) if with_coor else None
    L = lib()
    wsb = L.p3d_bev_pool_prepare_workspace_bytes(n)
    ws = workspace(wsb, dev, "bev_pool_prepare")
    bda = desc[B * N * CAM_FLOATS:]
    check(L.p3d_lss_prepare(ptr(desc), ptr(bda), ptr(ad), ptr(ax), ptr(ay), B, N, D, H, W, host_floats(grid_lower_bound),
                            host_floats(grid_interval), host_ints(grid_size), ptr(coor), ptr(outs[0]), ptr(outs[1]),
                            ptr(outs[2]), ptr(outs[3]), ptr(outs[4]), ptr(counts), ptr(ws), wsb, stream(dev)), "lss_prepare")
    res = (outs[0], outs[1], outs[2], outs[3], outs[4], counts)
    return res + (coor,) if with_coor else res


def lss_depth_feat(logits, tran_feat, depth=None, feat=None):
    """Depth softmax + permute (p3d_lss_depth_feat): logits [BN, D, H, W], tran_feat [BN, C, H, W] fp32 ->
    (depth [BN, D, H, W] = softmax over D, feat [BN, H, W, C]); depth / feat: optional preallocated outputs."""
    logits = require_cuda(logits, "logits", torch.float32)
    tran_feat = require_cuda(tran_feat, "tran_feat", torch.float32)
    BN, D, H, W = logits.shape
    C = tran_feat.shape[1]
    if tuple(tran_feat.shape) != (BN, C, H, W):
        raise ValueError("lss_depth_feat: tran_feat %s does not match logits %s" % (tuple(tran_feat.shape), tuple(logits.shape)))
    depth = torch.empty_like(logits) if depth is None else depth
    feat = torch.empty((BN, H, W, C), dtype=torch.float32, device=logits.device) if feat is None else feat
    check(lib().p3d_lss_depth_feat(ptr(logits), ptr(tran_feat), BN, D, H, W, C, ptr(depth), ptr(feat), stream(logits.device)),
          "lss_depth_feat")
    return depth, feat


def lss_depth_feat_h16(rows, shape, D, C, depth=None, feat=None):
    """lss_depth_feat from the depth net's pixel H16 rows [BN*H*W, 2*in_C], shape = (BN, H, W, in_C): channels [0, D) are
    the logits, [D, D + C) the features (p3d_lss_depth_feat_h16) -> (depth [BN, D, H, W], feat [BN, H, W, C]); depth /
    feat: optional preallocated outputs."""
    rows = require_cuda(rows, "rows", torch.float16)
    BN, H, W, in_C = [int(v) for v in shape]
    if tuple(rows.shape) != (BN * H * W, 2 * in_C):
        raise ValueError("lss_depth_feat_h16: rows %s, want (%d, %d)" % (tuple(rows.shape), BN * H * W, 2 * in_C))
    depth = torch.empty((BN, D, H, W), dtype=torch.float32, device=rows.device) if depth is None else depth
    feat = torch.empty((BN, H, W, C), dtype=torch.float32, device=rows.device) if feat is None else feat
    check(lib().p3d_lss_depth_feat_h16(ptr(rows), BN, H, W, in_C, int(D), int(C), ptr(depth), ptr(feat), stream(rows.device)),
          "lss_depth_feat_h16")
    return depth, feat


def bev_pool_v2_dev(depth, feat, prepared, bev_feat_shape, planar=False, out=None):
    """bev_pool_v2 with the interval count read on the device (p3d_bev_pool_v2_dev): `prepared` as voxel_pooling_prepare_v2
    / lss_prepare return it (untrimmed); bev_feat_shape (B, Z, Y, X, C).  planar=False -> [B, Z, Y, X, C];
    planar=True -> [B, Z * C, Y, X] (view_transform's layout, channel z * C + c)."""
    depth = require_cuda(depth, "depth", torch.float32)
    feat = require_cuda(feat, "feat", torch.float32)
    rb, rd, rf, st, ln, counts = prepared[:6]
    B, Z, Y, X, C = [int(s) for s in bev_feat_shape]
    if out is None:
        shape = (B, Z * C, Y, X) if planar else (B, Z, Y, X, C)
        out = torch.empty(shape, dtype=torch.float32, device=feat.device)
    check(lib().p3d_bev_pool_v2_dev(ptr(depth), ptr(feat), ptr(rd), ptr(rf), ptr(rb), ptr(ln), ptr(st), ptr(counts),
                                    rb.numel(), C, B, Z, Y, X, int(bool(planar)), ptr(out), stream(feat.device)),
          "bev_pool_v2_dev")
    return out


def bev_pool_v2_dev_h16(depth, feat, prepared, bev_feat_shape, out_channels=None, out=None):
    """bev_pool_v2_dev straight into pixel fp16-pair rows (p3d_bev_pool_v2_dev_h16): [B*Y*X, 2*out_channels] float16,
    channel z * C + c of a cell's row (the planar layout's channel order); out_channels defaults to Z * C rounded up to a
    multiple of 32, the padding channels are zero."""
    from .sparse_nn import status_tensor
    depth = require_cuda(depth, "depth", torch.float32)
    feat = require_cuda(feat, "feat", torch.float32)
    rb, rd, rf, st, ln, counts = prepared[:6]
    B, Z, Y, X, C = [int(s) for s in bev_feat_shape]
    oc = int(out_channels or (Z * C + 31) // 32 * 32)
    if out is None:
        out = torch.empty((B * Y * X, 2 * oc), dtype=torch.float16, device=feat.device)
    check(lib().p3d_bev_pool_v2_dev_h16(ptr(depth), ptr(feat), ptr(rd), ptr(rf), ptr(rb), ptr(ln), ptr(st), ptr(counts),
                                        rb.numel(), C, B, Z, Y, X, ptr(out), oc, ptr(status_tensor(feat.device)),
                                        stream(feat.device)), "bev_pool_v2_dev_h16")
    return out
