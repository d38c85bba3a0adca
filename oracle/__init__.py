"""TEST INFRASTRUCTURE ONLY — not part of the product.

ctypes/numpy front end of the CPU oracle (``oracle/p3d_oracle.c``) and of the reference's own
code compiled unmodified into ``oracle/_ref`` (see ``oracle/Makefile``).  Only ``tests/``,
``__graft_entry__.smoke()`` and ``bench.py``'s ``cpu_baseline`` / ``--impl reference`` legs may
import this package; nothing under ``paddle3d_b200/`` does.
"""
import ctypes as C
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB = None
_REF = {}

f32p = np.ctypeslib.ndpointer(np.float32, flags="C_CONTIGUOUS")
i32p = np.ctypeslib.ndpointer(np.int32, flags="C_CONTIGUOUS")
i64p = np.ctypeslib.ndpointer(np.int64, flags="C_CONTIGUOUS")
u64p = np.ctypeslib.ndpointer(np.uint64, flags="C_CONTIGUOUS")


def build(ref=True):
    """(Re)build the oracle library and, when a Paddle3D checkout is named by $P3D_REFERENCE, oracle/_ref."""
    subprocess.run(["make", "-s", "-C", _HERE, "oracle"] + (["ref"] if ref else []), check=True)


REF_LIBS = ("cpu", "iou3d_gpu", "cpp_gpu", "bevpool_gpu")


def ref_missing():
    """Names of the reference libraries (oracle/_ref) that are not built."""
    return [n for n in REF_LIBS if not os.path.exists(os.path.join(_HERE, "_ref", "libp3d_ref_%s.so" % n))]


def lib():
    global _LIB
    if _LIB is None:
        path = os.path.join(_HERE, "libp3d_oracle.so")
        if not os.path.exists(path):
            build(ref=False)
        _LIB = C.CDLL(path)
        _LIB.orc_box_overlap.restype = C.c_float
        _LIB.orc_iou_bev.restype = C.c_float
        _LIB.orc_sparse_conv3d.restype = C.c_int64
    return _LIB


def ref_lib(name):
    """name in {cpu, iou3d_gpu, cpp_gpu, bevpool_gpu}; returns None when not built."""
    if name not in _REF:
        path = os.path.join(_HERE, "_ref", "libp3d_ref_%s.so" % name)
        _REF[name] = C.CDLL(path) if os.path.exists(path) else None
    return _REF[name]


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _i(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _fp(a):
    return a.ctypes.data_as(C.POINTER(C.c_float))


def _ip(a):
    return a.ctypes.data_as(C.POINTER(C.c_int32))


def num_threads():
    return int(lib().orc_num_threads())


# --------------------------------------------------------------------------- voxelize
def grid_size(voxel_size, pcr):
    g = np.zeros(3, np.int32)
    lib().orc_grid_size(_fp(_f(voxel_size)), _fp(_f(pcr)), _ip(g))
    return [int(x) for x in g]  # x, y, z


def hard_voxelize(points, voxel_size, pcr, max_points, max_voxels, grid_scratch=None):
    points = _f(points)
    n, f = points.shape
    voxels = np.empty((max_voxels, max_points, f), np.float32)
    coords = np.empty((max_voxels, 3), np.int32)
    npv = np.empty((max_voxels,), np.int32)
    nv = np.zeros(1, np.int32)
    gs = None if grid_scratch is None else _ip(grid_scratch)
    rc = lib().orc_hard_voxelize(_fp(points), C.c_int64(n), f, _fp(_f(voxel_size)), _fp(_f(pcr)), max_points,
                                 max_voxels, _fp(voxels), _ip(coords), _ip(npv), _ip(nv), gs)
    assert rc == 0
    return voxels, coords, npv, nv


def ref_hard_voxelize_cpu(points, voxel_size, pcr, max_points, max_voxels):
    """The reference's own hard_voxelize_cpu (voxelize_op.cc:84-146), compiled unmodified."""
    r = ref_lib("cpu")
    points = _f(points)
    n, f = points.shape
    voxels = np.empty((max_voxels, max_points, f), np.float32)
    coords = np.empty((max_voxels, 3), np.int32)
    npv = np.empty((max_voxels,), np.int32)
    nv = np.zeros(1, np.int32)
    r.ref_hard_voxelize_cpu(_fp(points), C.c_longlong(n), f, _fp(_f(voxel_size)), _fp(_f(pcr)), max_points,
                            max_voxels, _fp(voxels), _ip(coords), _ip(npv), _ip(nv))
    return voxels, coords, npv, nv


def voxel_mean(voxels, npv, nv):
    voxels = _f(voxels)
    _, p, f = voxels.shape
    out = np.empty((nv, f), np.float32)
    lib().orc_voxel_mean(_fp(voxels), _ip(_i(npv)), nv, p, f, _fp(out))
    return out


def pillar_scatter(feats, coords, batch, ny, nx):
    feats = _f(feats)
    coords = _i(coords)
    nv, c = feats.shape
    out = np.empty((batch, c, ny, nx), np.float32)
    lib().orc_pillar_scatter(_fp(feats), _ip(coords), nv, c, batch, ny, nx, _fp(out))
    return out


# --------------------------------------------------------------------------- bev_pool
def bev_pool_v2(depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_lengths, interval_starts, bev_feat_shape,
                use_fma=False):
    depth, feat = _f(depth), _f(feat)
    c = feat.shape[-1]
    out = np.empty(tuple(bev_feat_shape), np.float32)
    lib().orc_bev_pool_v2(c, len(interval_starts), _fp(depth), _fp(feat), _ip(_i(ranks_depth)), _ip(_i(ranks_feat)),
                          _ip(_i(ranks_bev)), _ip(_i(interval_starts)), _ip(_i(interval_lengths)), _fp(out),
                          C.c_int64(out.size), int(use_fma))
    return out


def bev_pool_v2_bkwd(out_grad, depth, feat, ranks_depth, ranks_feat, ranks_bev, interval_lengths, interval_starts,
                     use_fma=False):
    out_grad, depth, feat = _f(out_grad), _f(depth), _f(feat)
    c = out_grad.shape[-1]
    dg = np.empty_like(depth)
    fg = np.empty_like(feat)
    lib().orc_bev_pool_v2_grad(c, len(interval_starts), _fp(out_grad), _fp(depth), _fp(feat), _ip(_i(ranks_depth)),
                               _ip(_i(ranks_feat)), _ip(_i(ranks_bev)), _ip(_i(interval_starts)),
                               _ip(_i(interval_lengths)), _fp(dg), C.c_int64(dg.size), _fp(fg), C.c_int64(fg.size),
                               int(use_fma))
    return dg, fg


# --------------------------------------------------------------------------- iou3d / nms
def boxes_overlap_bev(a, b):
    a, b = _f(a), _f(b)
    out = np.empty((len(a), len(b)), np.float32)
    lib().orc_boxes_overlap_bev(_fp(a), len(a), _fp(b), len(b), _fp(out))
    return out


def boxes_iou_bev(a, b):
    a, b = _f(a), _f(b)
    out = np.empty((len(a), len(b)), np.float32)
    lib().orc_boxes_iou_bev(_fp(a), len(a), _fp(b), len(b), _fp(out))
    return out


def ref_boxes_iou_bev_cpu(a, b):
    """The reference's own boxes_iou_bev_cpu (iou3d_cpu.cpp:241-264), compiled unmodified."""
    a, b = _f(a), _f(b)
    out = np.empty((len(a), len(b)), np.float32)
    ref_lib("cpu").ref_boxes_iou_bev_cpu(_fp(a), len(a), _fp(b), len(b), _fp(out))
    return out


def nms_mask(boxes, thr, normal=False):
    boxes = _f(boxes)
    n = len(boxes)
    cb = (n + 63) // 64
    mask = np.zeros((n, max(cb, 1)), np.uint64)
    lib().orc_nms_mask(_fp(boxes), n, C.c_float(thr), int(normal), mask.ctypes.data_as(C.c_void_p))
    return mask[:, :cb]


def nms(boxes, thr, normal=False):
    boxes = _f(boxes)
    n = len(boxes)
    keep = np.zeros(max(n, 1), np.int32)
    nk = lib().orc_nms(_fp(boxes), n, C.c_float(thr), int(normal), _ip(keep))
    return keep[:n], int(nk)


def voxel_pooling_prepare_v2(coor, grid_lower_bound, grid_interval, grid_size):
    """numpy restatement of LSSViewTransformer.voxel_pooling_prepare_v2
    (paddle3d/models/transformers/bevdet_transformer.py:230-274), line by line; the `argsort` (:260) is taken as a
    STABLE sort (ties keep ascending point index): Paddle's tie order is upstream and unspecified, this is the order the
    repo defines and the CUDA path reproduces.  Returns (ranks_bev, ranks_depth, ranks_feat, interval_starts,
    interval_lengths) int32, or five Nones as the reference does."""
    coor = np.asarray(coor, np.float32)
    B, N, D, H, W, _ = coor.shape
    num_points = B * N * D * H * W
    ranks_depth = np.arange(num_points, dtype=np.int64)                                   # :235
    ranks_feat = np.arange(num_points // D, dtype=np.int64).reshape(B, N, 1, H, W)         # :236-238
    ranks_feat = np.broadcast_to(ranks_feat, (B, N, D, H, W)).reshape(-1)
    lower = np.asarray(grid_lower_bound, np.float32)
    interval = np.asarray(grid_interval, np.float32)
    c = ((coor - lower) / interval)                                                        # :240-242 (fp32)
    with np.errstate(invalid="ignore"):
        c = np.trunc(c).astype(np.int64).reshape(num_points, 3)                            # :243 cast('int64'): toward zero
    batch_idx = np.repeat(np.arange(B), num_points // B)                                   # :244-246
    gx, gy, gz = [int(v) for v in grid_size]
    kept = (c[:, 0] >= 0) & (c[:, 0] < gx) & (c[:, 1] >= 0) & (c[:, 1] < gy) & (c[:, 2] >= 0) & (c[:, 2] < gz)  # :249-251
    if kept.sum() == 0:
        return None, None, None, None, None
    c, ranks_depth, ranks_feat, batch_idx = c[kept], ranks_depth[kept], ranks_feat[kept], batch_idx[kept]
    ranks_bev = batch_idx * (gz * gy * gx) + c[:, 2] * (gy * gx) + c[:, 1] * gx + c[:, 0]   # :256-259
    order = np.argsort(ranks_bev, kind="stable")                                           # :260
    ranks_bev, ranks_depth, ranks_feat = ranks_bev[order], ranks_depth[order], ranks_feat[order]
    first = np.ones(len(ranks_bev), bool)                                                  # :264-265
    first[1:] = ranks_bev[1:] != ranks_bev[:-1]
    interval_starts = np.nonzero(first)[0].astype(np.int32)                                # :266
    interval_lengths = np.zeros_like(interval_starts)                                      # :269-271
    interval_lengths[:-1] = interval_starts[1:] - interval_starts[:-1]
    interval_lengths[-1] = len(ranks_bev) - interval_starts[-1]
    return (ranks_bev.astype(np.int32), ranks_depth.astype(np.int32), ranks_feat.astype(np.int32), interval_starts,
            interval_lengths.astype(np.int32))


def cpp_nms_mask(bboxes, index, sorted_index, n_for_nms, thr):
    """Bit-matrix of the postprocess's indexed NMS (centerpoint_postprocess/iou3d_nms_kernel.cu:274-339)."""
    bboxes = _f(bboxes)
    index = _i(index)
    sorted_index = np.ascontiguousarray(sorted_index, dtype=np.int64)
    cb = (n_for_nms + 63) // 64
    mask = np.zeros((max(n_for_nms, 1), max(cb, 1)), np.uint64)
    lib().orc_cpp_nms_mask(_fp(bboxes), _ip(index), sorted_index.ctypes.data_as(C.POINTER(C.c_int64)), int(n_for_nms),
                           C.c_float(thr), int(bboxes.shape[1]), mask.ctypes.data_as(C.c_void_p))
    return mask[:n_for_nms, :cb]


# --------------------------------------------------------------------------- centerpoint_postprocess
def centerpoint_postprocess(hm, reg, height, dim, vel, rot, voxel_size, point_cloud_range, post_center_range,
                            num_classes, down_ratio, score_threshold, nms_iou_threshold, nms_pre_max_size,
                            nms_post_max_size, with_velocity):
    """Same argument list as paddle3d.ops.centerpoint_postprocess.centerpoint_postprocess
    (center_head.py:320-325); lists of per-task NCHW numpy arrays with batch 1."""
    T = len(hm)
    H, W = hm[0].shape[2], hm[0].shape[3]
    arrs = [[_f(x) for x in lst] for lst in (hm, reg, height, dim, vel, rot)]
    PP = C.POINTER(C.c_float) * T
    ptrs = [PP(*[_fp(x) for x in lst]) for lst in arrs]
    hm_c = _i([x.shape[1] for x in hm])
    dims = 9 if with_velocity else 7
    cap = T * max(nms_post_max_size, 1)
    boxes = np.zeros((cap, dims), np.float32)
    scores = np.zeros((cap,), np.float32)
    labels = np.zeros((cap,), np.int64)
    counts = np.zeros((T,), np.int32)
    k = lib().orc_centerpoint_postprocess(
        T, ptrs[0], _ip(hm_c), ptrs[1], ptrs[2], ptrs[3], ptrs[4], ptrs[5], H, W, _fp(_f(voxel_size)),
        _fp(_f(point_cloud_range)), _fp(_f(post_center_range)), _ip(_i(num_classes)), int(down_ratio),
        C.c_float(score_threshold), C.c_float(nms_iou_threshold), int(nms_pre_max_size), int(nms_post_max_size),
        int(bool(with_velocity)), _fp(boxes), _fp(scores), labels.ctypes.data_as(C.POINTER(C.c_int64)), _ip(counts))
    return boxes[:k], scores[:k], labels[:k], counts


# --------------------------------------------------------------------------- sparse conv
def sparse_conv3d(coords, feats, batch, spatial, weight, stride=(1, 1, 1), padding=(0, 0, 0), subm=False,
                  out_cap=None):
    """coords [n,4] (b,z,y,x); feats [n,Cin]; weight [kD,kH,kW,Cin,Cout]. Returns
    (out_coords, out_feats, out_spatial, pairs)."""
    coords, feats, weight = _i(coords), _f(feats), _f(weight)
    n = len(coords)
    kd, kh, kw, cin, cout = weight.shape
    ks = _i([kd, kh, kw])
    st = _i([stride] * 3 if np.isscalar(stride) else stride)
    pd = _i([padding] * 3 if np.isscalar(padding) else padding)
    if out_cap is None:
        out_cap = n if subm else n * kd * kh * kw
    oc = np.zeros((max(out_cap, 1), 4), np.int32)
    of = np.zeros((max(out_cap, 1), cout), np.float32)
    osp = np.zeros(3, np.int32)
    pairs = np.zeros(1, np.int64)
    no = lib().orc_sparse_conv3d(_ip(coords), _fp(feats), C.c_int64(n), int(batch), _ip(_i(spatial)), _fp(weight),
                                 cin, cout, _ip(ks), _ip(st), _ip(pd), int(subm), _ip(oc), _fp(of),
                                 C.c_int64(out_cap), _ip(osp), pairs.ctypes.data_as(C.POINTER(C.c_int64)))
    assert no >= 0, "oracle sparse conv failed (%d)" % no
    return oc[:no], of[:no], [int(x) for x in osp], int(pairs[0])


def sparse_to_dense_bev(coords, feats, batch, spatial):
    coords, feats = _i(coords), _f(feats)
    n, c = feats.shape
    d, h, w = spatial
    out = np.empty((batch, c * d, h, w), np.float32)
    lib().orc_sparse_to_dense_bev(_ip(coords), _fp(feats), C.c_int64(n), c, batch, d, h, w, _fp(out))
    return out


def bn_relu(x, gamma, beta, mean, var, eps, relu=True, residual=None):
    """paddle.sparse.nn.BatchNorm (eval) on values + optional residual add + ReLU, fp64 internally
    (sparse_resnet.py:95-111)."""
    y = (x.astype(np.float64) - mean) / np.sqrt(var.astype(np.float64) + eps) * gamma + beta
    if residual is not None:
        y = y + residual.astype(np.float64)
    if relu:
        y = np.maximum(y, 0.0)
    return y.astype(np.float32)


# --------------------------------------------------------------------------- dense 2-D convs (RPN / neck / head)
def conv2d(x, weight, bias=None, stride=1, padding=0):
    """x [B,Cin,H,W]; weight [Cout,Cin,kH,kW] (paddle.nn.Conv2D layout); fp64 accumulation."""
    x, weight = _f(x), _f(weight)
    b, cin, h, w = x.shape
    cout, cin2, kh, kw = weight.shape
    assert cin == cin2
    oh, ow = (h + 2 * padding - kh) // stride + 1, (w + 2 * padding - kw) // stride + 1
    out = np.empty((b, cout, oh, ow), np.float32)
    bias = _f(bias) if bias is not None else None
    lib().orc_conv2d_nchw(_fp(x), b, cin, h, w, _fp(weight), _fp(bias) if bias is not None else None, cout, kh, kw,
                          int(stride), int(padding), _fp(out))
    return out


def deconv2d(x, weight, bias=None, stride=1):
    """x [B,Cin,H,W]; weight [Cin,Cout,k,k] (paddle.nn.Conv2DTranspose layout), padding 0; fp64 accumulation."""
    x, weight = _f(x), _f(weight)
    b, cin, h, w = x.shape
    cin2, cout, k, k2 = weight.shape
    assert cin == cin2 and k == k2
    oh, ow = (h - 1) * stride + k, (w - 1) * stride + k
    out = np.empty((b, cout, oh, ow), np.float32)
    bias = _f(bias) if bias is not None else None
    lib().orc_deconv2d_nchw(_fp(x), b, cin, h, w, _fp(weight), _fp(bias) if bias is not None else None, cout, k,
                            int(stride), _fp(out))
    return out


def bn2d_relu(x, gamma, beta, mean, var, eps, relu=True):
    """paddle.nn.BatchNorm2D (eval) over axis 1 of an NCHW tensor + optional ReLU, fp64 internally."""
    sh = (1, -1, 1, 1)
    y = (x.astype(np.float64) - mean.reshape(sh)) / np.sqrt(var.astype(np.float64).reshape(sh) + eps)
    y = y * gamma.reshape(sh) + beta.reshape(sh)
    if relu:
        y = np.maximum(y, 0.0)
    return y.astype(np.float32)


# --------------------------------------------------------------------------- PillarFeatureNet (PointPillars encoder)
def pillar_feature_net(voxels, npv, coors, weight, gamma, beta, mean, var, eps, voxel_size, point_cloud_range):
    """PillarFeatureNet with one (last) PFNLayer, `legacy` flag irrelevant (PARITY UNPINNED: paddle ops; restated from
    models/voxel_encoders/pillar_encoder.py:156-210 and :81-106).  voxels [N, M, F] (x, y, z, ...), npv [N], coors [N, 4]
    (b, z, y, x); weight [F + 5, C] (paddle.nn.Linear layout, no bias).  Decoration: xyz - mean of the pillar's points,
    xy - pillar centre (coors[:, 3] * vx + vx / 2 + x_min, coors[:, 2] * vy + vy / 2 + y_min); rows >= npv are zeroed
    AFTER the decoration (:193-198) and still take part in the max (their value is ReLU(BN(0))).  fp64 internally.
    Paddle's basic slicing copies, so the in-place edit of `f_center` (:181-187) does not alias `features`."""
    v = np.asarray(voxels, np.float64)
    n, m, f = v.shape
    cnt = np.asarray(npv, np.float64).reshape(-1, 1, 1)
    pmean = v[:, :, :3].sum(1, keepdims=True) / cnt
    f_cluster = v[:, :, :3] - pmean
    vx, vy = float(voxel_size[0]), float(voxel_size[1])
    xo, yo = vx / 2 + float(point_cloud_range[0]), vy / 2 + float(point_cloud_range[1])
    c = np.asarray(coors)
    f_center = np.stack([v[:, :, 0] - (c[:, 3].reshape(-1, 1).astype(np.float32).astype(np.float64) * np.float32(vx) + np.float32(xo)),
                         v[:, :, 1] - (c[:, 2].reshape(-1, 1).astype(np.float32).astype(np.float64) * np.float32(vy) + np.float32(yo))], -1)
    feats = np.concatenate([v, f_cluster, f_center], -1)
    mask = (np.arange(m).reshape(1, -1) < np.asarray(npv).reshape(-1, 1)).astype(np.float64)
    feats = feats * mask[:, :, None]
    x = feats @ np.asarray(weight, np.float64)
    x = (x - mean) / np.sqrt(np.asarray(var, np.float64) + eps) * gamma + beta
    return np.maximum(x, 0.0).max(1).astype(np.float32)
