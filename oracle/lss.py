"""TEST INFRASTRUCTURE ONLY: numpy restatement of LSSViewTransformer's forward after the depth net
(bevdet_transformer.py:147-316, PARITY UNPINNED: restated from BEVDet's class, get_lidar_coor(sensor2ego, ego2global,
cam2imgs, post_rots, post_trans, bda) with a 3x3 bda).

get_lidar_coor comes in two forms: get_lidar_coor_fp32, the exact evaluation order of p3d_lss_prepare's kernel in fp32
(every product and sum rounded on its own), and get_lidar_coor_fp64, the reference's formula in fp64 from the raw
matrices.  view_transform chains the fp32 coordinates into the voxel_pooling_prepare_v2 and bev_pool_v2 oracles."""
import numpy as np

from . import bev_pool_v2, voxel_pooling_prepare_v2


def create_frustum(depth_cfg, input_size, downsample):
    """(d [D], x [W], y [H]) fp32: arange(*depth), linspace(0, W_in - 1, W), linspace(0, H_in - 1, H)."""
    H_in, W_in = input_size
    H, W = H_in // downsample, W_in // downsample
    d = np.arange(*depth_cfg, dtype=np.float64).astype(np.float32)
    return d, np.linspace(0, W_in - 1, W).astype(np.float32), np.linspace(0, H_in - 1, H).astype(np.float32)


def _row(m, r, v):
    """((m[r, 0] * v0 + m[r, 1] * v1) + m[r, 2] * v2) in fp32; m [B, N, 3, 3] broadcast over D, H, W."""
    c = [m[:, :, r, k][:, :, None, None, None] for k in range(3)]
    return (c[0] * v[0] + c[1] * v[1]) + c[2] * v[2]


def get_lidar_coor_fp32(cams, axes):
    """cams: unpacked descriptor (ops.bev_pool_v2.unpack_cameras, fp32); axes (d, x, y) fp32 -> [B, N, D, H, W, 3] fp32,
    bit for bit what p3d_lss_prepare computes."""
    d, x, y = [np.asarray(a, np.float32) for a in axes]
    ipr, pt, cmb, tr, bda = [np.asarray(cams[k], np.float32) for k in ("inv_post_rots", "post_trans", "combine", "trans", "bda")]
    B, N = pt.shape[:2]
    pt = pt[:, :, None, None, None, :]
    p = [x[None, None, None, None, :] - pt[..., 0], y[None, None, None, :, None] - pt[..., 1],
         d[None, None, :, None, None] - pt[..., 2]]
    q = [_row(ipr, r, p) for r in range(3)]
    s = [q[0] * q[2], q[1] * q[2], q[2]]
    tr = tr[:, :, None, None, None, :]
    e = [_row(cmb, r, s) + tr[..., r] for r in range(3)]
    bda = np.broadcast_to(bda[:, None], (B, N, 3, 3))
    o = [_row(bda, r, e) for r in range(3)]
    o = [np.broadcast_to(v, (B, N, len(d), len(y), len(x))) for v in o]
    return np.stack(o, -1).astype(np.float32)


U32 = 2.0 ** -24  # unit roundoff of fp32


def _e_add(a, b, sign=1.0):
    v = a[0] + sign * b[0]
    e = a[1] + b[1]
    return v, e + U32 * (np.abs(v) + e)


def _e_mul(a, b):
    v = a[0] * b[0]
    e = np.abs(a[0]) * b[1] + np.abs(b[0]) * a[1] + a[1] * b[1]
    return v, e + U32 * (np.abs(v) + e)


def _e_row(m, r, vec):
    c = [(m[0][:, :, r, k][:, :, None, None, None], m[1][:, :, r, k][:, :, None, None, None]) for k in range(3)]
    return _e_add(_e_add(_e_mul(c[0], vec[0]), _e_mul(c[1], vec[1])), _e_mul(c[2], vec[2]))


def get_lidar_coor_error_bound(sensor2ego, cam2imgs, post_rots, post_trans, bda, axes):
    """A priori bound on |get_lidar_coor_fp32 - exact formula| per coordinate, [B, N, D, H, W, 3] fp64: forward error
    analysis of the fp32 evaluation order (every operation rounds with relative error <= 2^-24, the errors of its
    operands propagated), starting from the descriptor's own rounding (|fp32 entry - fp64 entry| of inv(post_rots) and
    combine; the frustum axes, post_trans, the translation and bda are fp32 inputs on both sides).  Evaluated in fp64
    from the camera matrices alone, never from the fp32 result."""
    d, x, y = [np.asarray(a, np.float64) for a in axes]
    s2e, k, prot = [np.asarray(a, np.float64) for a in (sensor2ego, cam2imgs, post_rots)]
    pt, bd = np.asarray(post_trans, np.float64), np.asarray(bda, np.float64)
    B, N = s2e.shape[:2]
    ipr64 = np.linalg.inv(prot)
    cmb64 = s2e[:, :, :3, :3] @ np.linalg.inv(k)
    ipr = (ipr64, np.abs(ipr64.astype(np.float32).astype(np.float64) - ipr64))
    cmb = (cmb64, np.abs(cmb64.astype(np.float32).astype(np.float64) - cmb64))
    z = lambda a: (a, np.zeros_like(a))  # noqa: E731  (an exact input)
    ptb = pt[:, :, None, None, None, :]
    p = [_e_add(z(x[None, None, None, None, :]), z(ptb[..., 0]), -1.0), _e_add(z(y[None, None, None, :, None]), z(ptb[..., 1]), -1.0),
         _e_add(z(d[None, None, :, None, None]), z(ptb[..., 2]), -1.0)]
    q = [_e_row(ipr, r, p) for r in range(3)]
    s = [_e_mul(q[0], q[2]), _e_mul(q[1], q[2]), q[2]]
    tr = s2e[:, :, None, None, None, :3, 3]
    e = [_e_add(_e_row(cmb, r, s), z(tr[..., r])) for r in range(3)]
    bdn = z(np.broadcast_to(bd[:, None], (B, N, 3, 3)))
    o = [_e_row(bdn, r, e)[1] for r in range(3)]
    return np.stack([np.broadcast_to(v, (B, N, len(d), len(y), len(x))) for v in o], -1)


def get_lidar_coor_fp64(sensor2ego, cam2imgs, post_rots, post_trans, bda, axes):
    """The reference's formula in fp64 (frustum - post_trans, inv(post_rots), (x d, y d, d), combine, translation, bda)."""
    d, x, y = [np.asarray(a, np.float64) for a in axes]
    s2e, k, prot = [np.asarray(a, np.float64) for a in (sensor2ego, cam2imgs, post_rots)]
    ptr, bda = np.asarray(post_trans, np.float64), np.asarray(bda, np.float64)
    B, N = s2e.shape[:2]
    D, H, W = len(d), len(y), len(x)
    fr = np.stack(np.broadcast_arrays(x[None, None, :], y[None, :, None], d[:, None, None]), -1)  # D, H, W, 3
    pts = fr[None, None] - ptr[:, :, None, None, None, :]
    pts = np.einsum("bnij,bndhwj->bndhwi", np.linalg.inv(prot), pts)
    pts = np.concatenate([pts[..., :2] * pts[..., 2:3], pts[..., 2:3]], -1)
    combine = s2e[:, :, :3, :3] @ np.linalg.inv(k)
    pts = np.einsum("bnij,bndhwj->bndhwi", combine, pts) + s2e[:, :, None, None, None, :3, 3]
    return np.einsum("bij,bndhwj->bndhwi", bda, pts).reshape(B, N, D, H, W, 3)


def depth_softmax(logits):
    """softmax over axis 1 of [BN, D, H, W] as p3d_lss_depth_feat takes it: max subtracted, exp, sum in ascending d, all
    in fp32 except the exponential, which is taken in fp64 and rounded once (the kernel's expf is within 2 ulp of it)."""
    x = np.asarray(logits, np.float32)
    m = x.max(1, keepdims=True)
    e = np.exp((x - m).astype(np.float64)).astype(np.float32)
    s = np.zeros_like(e[:, 0])
    for k in range(x.shape[1]):
        s = s + e[:, k]
    return (e / s[:, None]).astype(np.float32)


def feat_permute(tran_feat):
    """[BN, C, H, W] -> [BN, H, W, C] (voxel_pooling_v2's permute)."""
    return np.ascontiguousarray(np.asarray(tran_feat, np.float32).transpose(0, 2, 3, 1))


def collapse_z(bev):
    """[B, Z, Y, X, C] pool -> [B, C * Z, Y, X]: torch.cat(bev.permute(0, 4, 1, 2, 3).unbind(dim=2), 1)."""
    bczyx = bev.transpose(0, 4, 1, 2, 3)
    return np.ascontiguousarray(np.concatenate([bczyx[:, :, z] for z in range(bczyx.shape[2])], 1))


def view_transform(cams, axes, logits, tran_feat, grid_lower_bound, grid_interval, grid_size):
    """Forward from the depth net's output -> [B, C * Z, Y, X] fp32, plus the fp32 coordinates and the prepared ranks
    (five Nones when no point is inside the grid: the BEV is then zero, as the reference's dummy tensor)."""
    coor = get_lidar_coor_fp32(cams, axes)
    B = coor.shape[0]
    depth, feat = depth_softmax(logits), feat_permute(tran_feat)
    gx, gy, gz = [int(v) for v in grid_size]
    C = feat.shape[-1]
    prep = voxel_pooling_prepare_v2(coor, grid_lower_bound, grid_interval, grid_size)
    if prep[0] is None:
        return np.zeros((B, C * gz, gy, gx), np.float32), coor, prep
    rb, rd, rf, st, ln = prep
    bev = bev_pool_v2(depth, feat, rd, rf, rb, ln, st, (B, gz, gy, gx, C), use_fma=True)
    return collapse_z(bev), coor, prep
