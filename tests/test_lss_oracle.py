"""CPU suite for the LSS view transform: the numpy oracle (oracle/lss.py) against an independent torch fp64 restatement
of get_lidar_coor in the reference's tensor shapes, the oracle frame against the existing prepare / pool oracles, the
camera descriptor packing, and the argument checks of the new entry points (no GPU needed)."""
import ctypes as C

import numpy as np
import pytest

from paddle3d_b200 import synth


def _torch_lidar_coor(rig, depth_cfg, input_size, downsample):
    """BEVDet's create_frustum + get_lidar_coor, in torch fp64 with torch.inverse / matmul in the reference's shapes."""
    import torch
    t = {k: torch.from_numpy(np.asarray(v, np.float64)) for k, v in rig.items()}
    H_in, W_in = input_size
    H, W = H_in // downsample, W_in // downsample
    d = torch.arange(*depth_cfg, dtype=torch.float).view(-1, 1, 1).expand(-1, H, W)
    D = d.shape[0]
    x = torch.linspace(0, W_in - 1, W, dtype=torch.float).view(1, 1, W).expand(D, H, W)
    y = torch.linspace(0, H_in - 1, H, dtype=torch.float).view(1, H, 1).expand(D, H, W)
    frustum = torch.stack((x, y, d), -1).double()
    s2e, cam2imgs, post_rots, post_trans, bda = t["sensor2ego"], t["cam2imgs"], t["post_rots"], t["post_trans"], t["bda"]
    B, N, _, _ = s2e.shape
    points = frustum - post_trans.view(B, N, 1, 1, 1, 3)
    points = torch.inverse(post_rots).view(B, N, 1, 1, 1, 3, 3).matmul(points.unsqueeze(-1))
    points = torch.cat((points[..., :2, :] * points[..., 2:3, :], points[..., 2:3, :]), 5)
    combine = s2e[:, :, :3, :3].matmul(torch.inverse(cam2imgs))
    points = combine.view(B, N, 1, 1, 1, 3, 3).matmul(points).squeeze(-1)
    points += s2e[:, :, :3, 3].view(B, N, 1, 1, 1, 3)
    points = bda.view(B, 1, 1, 1, 1, 3, 3).matmul(points.unsqueeze(-1)).squeeze(-1)
    return points.numpy(), (d[:, 0, 0].numpy(), x[0, 0].numpy(), y[0, :, 0].numpy())


@pytest.mark.parametrize("B,with_bda", [(1, False), (1, True), (2, False), (2, True)])
def test_lidar_coor_fp32_and_fp64_oracles_vs_torch(B, with_bda):
    from oracle import lss
    from paddle3d_b200.ops import bev_pool_v2 as bp
    rig = synth.camera_rig(11 + B, B=B, bda=with_bda)
    want, axes = _torch_lidar_coor(rig, synth.LSS_BEVDET["depth"], synth.LSS_INPUT_SIZE, synth.LSS_DOWNSAMPLE)
    assert want.shape == (B, 6, 118, 16, 44, 3)
    cams = bp.unpack_cameras(bp.pack_cameras(*synth.lss_mats(rig)), B, 6)
    got32 = lss.get_lidar_coor_fp32(cams, axes)
    got64 = lss.get_lidar_coor_fp64(*synth.lss_mats(rig), axes)
    span = want.max() - want.min()
    assert got32.dtype == np.float32
    assert np.abs(got32 - want).max() <= 1e-5 * span
    assert np.abs(got64 - want).max() <= 1e-12 * span
    # the a priori forward-error bound of the fp32 order holds everywhere, and is tight enough to mean something
    bound = lss.get_lidar_coor_error_bound(*synth.lss_mats(rig), axes)
    assert (np.abs(got32.astype(np.float64) - got64) <= bound).all()
    assert bound.max() < 1e-5 * span and (np.abs(got32.astype(np.float64) - got64) > 0.01 * bound).any()
    if not with_bda:
        assert np.array_equal(cams["bda"], np.broadcast_to(np.eye(3, dtype=np.float32), (B, 3, 3)))


def test_oracle_view_transform_chains_the_prepare_and_pool_oracles(oracle_mod):
    from oracle import lss
    from paddle3d_b200.ops import bev_pool_v2 as bp
    B, N, C = 2, 6, 8
    grid = dict(synth.LSS_BEVDET, depth=[1.0, 60.0, 3.0])
    axes = lss.create_frustum(grid["depth"], synth.LSS_INPUT_SIZE, synth.LSS_DOWNSAMPLE)
    D, H, W = len(axes[0]), len(axes[2]), len(axes[1])
    rng = np.random.default_rng(3)
    logits = rng.normal(0, 2, (B * N, D, H, W)).astype(np.float32)
    tran = rng.normal(0, 1, (B * N, C, H, W)).astype(np.float32)
    rig = synth.camera_rig(4, B=B)
    cams = bp.unpack_cameras(bp.pack_cameras(*synth.lss_mats(rig)), B, N)
    lower, interval, size = [-51.2, -51.2, -5.0], [0.8, 0.8, 8.0], [128, 128, 1]
    bev, coor, prep = lss.view_transform(cams, axes, logits, tran, lower, interval, size)
    assert bev.shape == (B, C, 128, 128) and bev.any()
    rb, rd, rf, st, ln = oracle_mod.voxel_pooling_prepare_v2(coor, lower, interval, size)
    depth = lss.depth_softmax(logits)
    np.testing.assert_allclose(depth.sum(1), 1.0, rtol=1e-5)
    pool = oracle_mod.bev_pool_v2(depth, tran.transpose(0, 2, 3, 1), rd, rf, rb, ln, st, (B, 1, 128, 128, C), use_fma=True)
    assert np.array_equal(bev, pool[:, 0].transpose(0, 3, 1, 2))
    # Z > 1: channel z * C + c, as torch.cat(bev.unbind(dim=2), 1) orders it
    bev2, _, prep2 = lss.view_transform(cams, axes, logits, tran, lower, [0.8, 0.8, 2.0], [128, 128, 4])
    rb, rd, rf, st, ln = prep2
    pool = oracle_mod.bev_pool_v2(depth, tran.transpose(0, 2, 3, 1), rd, rf, rb, ln, st, (B, 4, 128, 128, C), use_fma=True)
    assert bev2.shape == (B, 4 * C, 128, 128)
    for z in range(4):
        assert np.array_equal(bev2[:, z * C:(z + 1) * C], pool[:, z].transpose(0, 3, 1, 2))


def test_camera_descriptor_round_trip():
    from paddle3d_b200.ops import bev_pool_v2 as bp
    rig = synth.camera_rig(7, B=2)
    desc = bp.pack_cameras(*synth.lss_mats(rig))
    assert desc.dtype == np.float32 and desc.shape == (2 * 6 * 24 + 2 * 9,)
    c = bp.unpack_cameras(desc, 2, 6)
    f64 = {k: np.asarray(v, np.float64) for k, v in rig.items()}
    assert np.array_equal(c["inv_post_rots"], np.linalg.inv(f64["post_rots"]).astype(np.float32))
    assert np.array_equal(c["post_trans"], rig["post_trans"])
    assert np.array_equal(c["combine"], (f64["sensor2ego"][..., :3, :3] @ np.linalg.inv(f64["cam2imgs"])).astype(np.float32))
    assert np.array_equal(c["trans"], rig["sensor2ego"][..., :3, 3])
    assert np.array_equal(c["bda"], rig["bda"])
    # torch inputs pack to the same bits; no matrix of the rig is the identity
    import torch
    assert np.array_equal(bp.pack_cameras(*[torch.from_numpy(np.asarray(m)) for m in synth.lss_mats(rig)]), desc)
    for k in ("sensor2ego", "cam2imgs", "post_rots", "bda"):
        m = rig[k][..., :3, :3]
        assert not np.any(np.all(np.isclose(m, np.eye(3)), axis=(-2, -1))), k


def test_lss_entry_points_reject_invalid_arguments():
    """Status codes from the host checks, before any CUDA call (no GPU here)."""
    from paddle3d_b200 import _lib
    L = _lib.lib()
    p = C.c_void_p(256)
    lo, iv = _lib.host_floats([-51.2, -51.2, -5]), _lib.host_floats([0.8, 0.8, 8])
    gs = _lib.host_ints([128, 128, 1])

    def prep(cams=p, bda=p, ad=p, ax=p, ay=p, B=1, N=6, D=118, H=16, W=44, lo=lo, iv=iv, gs=gs, outs=(p,) * 6, ws=p,
             wsb=1 << 30):
        return L.p3d_lss_prepare(cams, bda, ad, ax, ay, B, N, D, H, W, lo, iv, gs, None, *outs, ws, wsb, None)
    for kw in (dict(cams=None), dict(bda=None), dict(ad=None), dict(ax=None), dict(ay=None), dict(lo=None), dict(gs=None),
               dict(outs=(p,) * 5 + (None,)), dict(outs=(None,) + (p,) * 5), dict(ws=None), dict(B=0), dict(N=-1), dict(D=0),
               dict(H=0), dict(W=0)):
        assert prep(**kw) == -1, kw
    assert prep(B=2, N=6, D=4096, H=512, W=512) == -4                        # B*N*D*H*W > 2^31 - 1
    # ranks are int32: B * X * Y * Z <= 2^31 cells.  Exactly 2^31 gets past the guard to the workspace check (1 byte:
    # P3D_ERR_WORKSPACE, before any launch); one more column is refused.
    g31, g31x = _lib.host_ints([1024, 1024, 1024]), _lib.host_ints([1025, 1024, 1024])
    assert prep(B=2, N=1, D=1, H=1, W=1, gs=g31, wsb=1) == -2
    assert prep(B=2, N=1, D=1, H=1, W=1, gs=g31x, wsb=1) == -4
    assert prep(gs=_lib.host_ints([128, 0, 1])) == -4
    assert prep(ws=C.c_void_p(260)) == -1                                    # workspace not 256-byte aligned
    # the existing coordinate entry point keeps its checks
    assert L.p3d_bev_pool_prepare(None, 1, 6, 118, 16, 44, lo, iv, gs, p, p, p, p, p, p, p, 1 << 30, None) == -1
    assert L.p3d_bev_pool_prepare(p, 2, 6, 4096, 512, 512, lo, iv, gs, p, p, p, p, p, p, p, 1 << 30, None) == -4
    assert L.p3d_bev_pool_prepare(p, 2, 1, 1, 1, 1, lo, iv, g31, p, p, p, p, p, p, p, 1, None) == -2
    assert L.p3d_bev_pool_prepare(p, 2, 1, 1, 1, 1, lo, iv, g31x, p, p, p, p, p, p, p, 1, None) == -4
    # depth softmax + permute
    df = L.p3d_lss_depth_feat
    assert df(None, p, 6, 118, 16, 44, 80, p, p, None) == -1
    assert df(p, p, 6, 118, 16, 44, 80, None, p, None) == -1
    assert df(p, p, 0, 118, 16, 44, 80, p, p, None) == -1
    assert df(p, p, 6, 118, 16, -1, 80, p, p, None) == -1
    assert df(p, p, 6, 383, 16, 44, 80, p, p, None) == -4                    # D too deep for the staged tile
    assert df(p, p, 6, 118, 16, 44, 371, p, p, None) == -4
    assert df(p, p, 1, 1 << 27, 1, 1, 80, p, p, None) == -4                  # D * 32 would overflow int
    assert df(p, p, 1, 118, 1, 1, 1 << 27, p, p, None) == -4
    # pool with the device interval count
    pd = L.p3d_bev_pool_v2_dev

    def pool(ptrs=(p,) * 8, cap=1000, c=80, B=1, Z=1, Y=128, X=128, planar=1, out=p):
        return pd(*ptrs, cap, c, B, Z, Y, X, planar, out, None)
    assert pool(ptrs=(p,) * 7 + (None,)) == -1                               # no counts
    assert pool(out=None) == -1
    assert pool(cap=-1) == -1 and pool(c=0) == -1 and pool(Y=0) == -1 and pool(planar=2) == -1
    assert pool(c=7) == -4 and pool(c=260) == -4                            # warp kernel: c % 4 == 0, c <= 256
    assert pool(out=C.c_void_p(260)) == -4                                  # float4 stores need 16-byte alignment
    assert pool(B=2, Z=1024, Y=1024, X=1025) == -4                          # B * cells > 2^31: a rank past int32
    assert pool(cap=1 << 31) == -4
    # the pixel-row form has the same cell limit (c = 4 so that Z * c fits out_C)
    ph = L.p3d_bev_pool_v2_dev_h16
    assert ph(*(p,) * 8, 1000, 4, 2, 1024, 1024, 1025, p, 4096, p, None) == -4
