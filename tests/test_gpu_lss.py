"""GPU parity of the LSS view transform: fused frustum geometry + rank preparation (p3d_lss_prepare), depth softmax +
permute (p3d_lss_depth_feat), bev_pool with the device interval count (p3d_bev_pool_v2_dev), LSSViewTransformer and the
captured LSSHotPath frame, at the BEVDet shape (6 cameras, 16 x 44 features, D = 118, C = 80) on the 128 x 128 and
200 x 200 grids."""
import ctypes as C

import numpy as np
import pytest

from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu
GRIDS = {"bevdet": synth.LSS_BEVDET, "config4": synth.LSS_C4}


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _vt(cuda, grid="bevdet", accelerate=False, C_=synth.LSS_CHANNELS):
    from paddle3d_b200.lss import LSSViewTransformer
    return LSSViewTransformer(GRIDS[grid], synth.LSS_INPUT_SIZE, synth.LSS_DOWNSAMPLE, C_, accelerate=accelerate, device=cuda)


def _inputs(vt, B, seed, N=6):
    rng = np.random.default_rng(seed)
    logits = rng.normal(0, 2, (B * N, vt.D, vt.H, vt.W)).astype(np.float32)
    tran = rng.normal(0, 1, (B * N, vt.out_channels, vt.H, vt.W)).astype(np.float32)
    return logits, tran


def _input_list(rig):
    """view_transform's input list; x only supplies B and N."""
    import torch
    B, N = rig["sensor2ego"].shape[:2]
    return [torch.zeros((B, N, 1, 1, 1)), rig["sensor2ego"], rig["ego2global"], rig["cam2imgs"], rig["post_rots"],
            rig["post_trans"], rig["bda"]]


def _cams(rig):
    from paddle3d_b200.ops import bev_pool_v2 as bp
    B, N = rig["sensor2ego"].shape[:2]
    return bp.unpack_cameras(bp.pack_cameras(*synth.lss_mats(rig)), B, N)


def _axes_np(vt):
    return tuple(a.numpy() for a in vt.axes_host)


@pytest.mark.parametrize("grid", sorted(GRIDS))
def test_coordinates_and_ranks(cuda, oracle_mod, grid):
    """coor bit-equal to the fp32 oracle; every rank that differs from the fp64 formula's belongs to a point within the
    fp32 error of a cell boundary; the five rank arrays and counts equal p3d_bev_pool_prepare fed the same coor."""
    from oracle import lss
    from paddle3d_b200.ops import bev_pool_v2 as bp
    vt = _vt(cuda, grid)
    for B, with_bda in ((1, True), (2, False)):
        rig = synth.camera_rig(21 + B, B=B, bda=with_bda)
        desc = vt.descriptor(*synth.lss_mats(rig))
        got = vt._prepare(desc, B, 6, with_coor=True)
        coor = got[6].cpu().numpy()
        want = lss.get_lidar_coor_fp32(_cams(rig), _axes_np(vt))
        assert np.array_equal(coor, want), "coor differs from the fp32 oracle"
        assert np.array_equal(coor, vt.get_lidar_coor(rig["sensor2ego"], rig["ego2global"], *synth.lss_mats(rig)[1:]).cpu().numpy())
        # ranks against the prepare of the uploaded coor, bit for bit, tails zero
        ref = bp.voxel_pooling_prepare_v2(got[6], *vt.grid_args())
        assert bool((got[5] == ref[5]).all()), "counts"
        k, m = [int(v) for v in got[5].cpu()]
        # ranks over the whole capacity; interval_starts is written up to the interval count only, in both entry points
        for g, r, name, valid in zip(got[:5], ref, ("ranks_bev", "ranks_depth", "ranks_feat", "starts", "lengths"),
                                     (None, None, None, m, None)):
            assert bool((g[:valid] == r[:valid]).all()), name
        assert k > 0 and m > 0 and not got[0][k:].any() and not got[1][k:].any() and not got[4][m:].any()
        # fp64: the kernel's rank of a point (read back from the device ranks) differs from the rank of the fp64 formula
        # only where the fp64 coordinate lies within the a priori fp32 error bound of a discontinuity of the key
        # (a nonzero integer of (coor - lower) / interval: cast('int64') truncates, so (-1, 1) all maps to cell 0)
        n = coor.size // 3
        rb_, rd_ = got[0][:k].cpu().numpy(), got[1][:k].cpu().numpy()
        key_dev = np.full(n, -1, np.int64)
        key_dev[rd_] = rb_
        c64 = lss.get_lidar_coor_fp64(*synth.lss_mats(rig), _axes_np(vt)).reshape(-1, 3)
        e_c = lss.get_lidar_coor_error_bound(*synth.lss_mats(rig), _axes_np(vt)).reshape(-1, 3)
        lo, iv, size = [np.asarray(v, np.float64) for v in vt.grid_args()]
        q64 = (c64 - lo) / iv
        e_s = e_c + lss.U32 * (np.abs(c64 - lo) + e_c)            # fl(coor - lower)
        e_q = e_s / iv + lss.U32 * (np.abs(q64) + e_s / iv) + 1e-9  # fl(. / interval); slack for the fp64 evaluation
        t = np.trunc(q64)
        inside = np.all((t >= 0) & (t < size), 1)
        bidx = np.arange(n) // (n // B)
        key64 = np.where(inside, ((bidx * size[2] + t[:, 2]) * size[1] + t[:, 1]) * size[0] + t[:, 0], -1).astype(np.int64)
        diff = np.nonzero(key_dev != key64)[0]
        r = np.round(q64[diff])
        dist = np.where(r != 0, np.abs(q64[diff] - r), 1.0 - np.abs(q64[diff]))  # to the nearest nonzero integer
        near = np.any(dist <= e_q[diff], 1)
        assert near.all(), "points off a cell boundary changed cell: %s" % diff[~near][:10]
        assert e_q.max() < 1e-3  # the bound is a small fraction of a cell, so the check above can fail
        assert len(diff) < 1e-3 * n


def test_depth_softmax_and_permute(cuda):
    from oracle import lss
    from paddle3d_b200.ops import bev_pool_v2 as bp
    vt = _vt(cuda)
    logits, tran = _inputs(vt, 2, 5)
    logits[0, :, 0, 0] = 0.0  # a flat pixel
    logits[1, :, 3, 7] = np.linspace(-80, 80, vt.D)  # a sharp one
    depth, feat = bp.lss_depth_feat(_t(cuda, logits), _t(cuda, tran))
    want = lss.depth_softmax(logits)
    got = depth.cpu().numpy()
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    # expf is within 2 ulp of the correctly rounded exponential; the quotient carries the numerator's error and the sum's,
    # and once a term differs the 118 rounded partial sums no longer round alike (6 ulp seen on an H100): at most 8 ulp,
    # and 2 ulp on 99 % of the values.  Subnormal results (the sharp pixel's tail, where expf keeps fewer bits) are compared in
    # absolute terms: below the smallest normal number.
    normal = want >= np.float32(2.0 ** -126)
    assert ulp[normal].max() <= 8, (ulp[normal].max(), want[normal][np.argmax(ulp[normal])])
    assert (ulp[normal] <= 2).mean() > 0.99  # 99.2 % on an H100
    assert np.abs(got - want)[~normal].max(initial=0.0) < 2.0 ** -126
    assert np.array_equal(feat.cpu().numpy(), lss.feat_permute(tran))


def test_pool_with_device_count_both_layouts(cuda, oracle_mod):
    import torch
    from paddle3d_b200.ops import bev_pool_v2 as bp
    for grid, b in (((128, 128, 1), (-51.2, 51.2)), ((200, 200, 1), (-50.0, 50.0))):
        d = synth.bev_pool_inputs(5, grid=grid, bounds=(b, b, (-5.0, 3.0)))
        prep = bp.voxel_pooling_prepare_v2(_t(cuda, d["coor"]), d["grid_lower_bound"], d["grid_interval"], d["grid_size"])
        rb, rd, rf, st, ln = bp.trim(prep)
        depth, feat = _t(cuda, d["depth"]), _t(cuda, d["feat"])
        B, Y, X, Cc = d["bev_feat_shape"]
        host = bp.bev_pool_v2(depth, feat, rd, rf, rb, ln, st, d["bev_feat_shape"])
        zyx = bp.bev_pool_v2_dev(depth, feat, prep, (B, 1, Y, X, Cc))
        planar = bp.bev_pool_v2_dev(depth, feat, prep, (B, 1, Y, X, Cc), planar=True)
        assert torch.equal(zyx[:, 0], host)
        assert torch.equal(planar, host.permute(0, 3, 1, 2))
        ref = oracle_mod.ref_lib("bevpool_gpu")
        if ref is not None:  # the reference's own kernel, under the conditions of test_bev_pool_v2
            out = torch.zeros(d["bev_feat_shape"], dtype=torch.float32, device=cuda)
            p = [C.c_void_p(t.data_ptr()) for t in (depth, feat, rd, rf, rb, ln, st)]
            torch.cuda.synchronize()
            ref.ref_bev_pool_v2_gpu(Cc, len(st), p[0], p[1], p[2], p[3], p[4], p[6], p[5], C.c_void_p(out.data_ptr()))
            torch.cuda.synchronize()
            assert torch.equal(out, zyx[:, 0])
    # Z > 1: channel z * C + c
    d = synth.bev_pool_inputs(6, C=16, D=30, grid=(64, 64, 4), bounds=((-40, 40), (-40, 40), (-5.0, 3.0)))
    prep = bp.voxel_pooling_prepare_v2(_t(cuda, d["coor"]), d["grid_lower_bound"], d["grid_interval"], d["grid_size"])
    depth, feat = _t(cuda, d["depth"]), _t(cuda, d["feat"])
    zyx = bp.bev_pool_v2_dev(depth, feat, prep, (1, 4, 64, 64, 16))
    planar = bp.bev_pool_v2_dev(depth, feat, prep, (1, 4, 64, 64, 16), planar=True)
    assert zyx[:, 1:].any()
    assert torch.equal(planar, torch.cat(zyx.permute(0, 4, 1, 2, 3).unbind(dim=2), 1))


@pytest.mark.parametrize("grid", sorted(GRIDS))
def test_captured_frame(cuda, oracle_mod, grid):
    """Captured frame == eager forward bit for bit, == the numpy oracle frame within the bev_pool tolerances; a new
    calibration between replays of one graph == a fresh eager run; accelerate == full frame."""
    import torch
    from oracle import lss
    from paddle3d_b200.lss import LSSHotPath
    B = 1
    vt = _vt(cuda, grid)
    rig, rig2 = synth.camera_rig(31, B=B), synth.camera_rig(32, B=B)
    logits, tran = _inputs(vt, B, 7)
    tl, tt = _t(cuda, logits), _t(cuda, tran)
    eager = vt.forward(_input_list(rig), tl, tt)
    frame = LSSHotPath(vt, B, 6, device=cuda).capture(count_nodes=True)
    assert frame.graph_nodes["kernel"] > 0
    bev, counts = frame.infer(synth.lss_mats(rig), tl, tt)
    assert torch.equal(bev, eager)
    want, _, prep = lss.view_transform(_cams(rig), _axes_np(vt), logits, tran, *vt.grid_args())
    assert counts == (len(prep[0]), len(prep[3]))
    np.testing.assert_allclose(bev.cpu().numpy(), want, rtol=1e-4, atol=1e-5)
    # the view_transform signature (softmax already taken) gives the same tensor
    depth = torch.softmax(tl, 1)
    vt_out = vt.view_transform(_input_list(rig), depth, tt)
    np.testing.assert_allclose(vt_out.cpu().numpy(), want, rtol=1e-4, atol=1e-5)
    # new calibration, same graph
    bev2, _ = frame.infer(synth.lss_mats(rig2), tl, tt)
    assert torch.equal(bev2, vt.forward(_input_list(rig2), tl, tt)) and not torch.equal(bev2, eager)
    # accelerate: ranks replayed only on a calibration change, bit-equal to the full frame
    acc = LSSHotPath(_vt(cuda, grid, accelerate=True), B, 6, device=cuda).capture()
    for r in (rig, rig, rig2, rig):
        got, _ = acc.infer(synth.lss_mats(r), tl, tt)
        full, _ = frame.infer(synth.lss_mats(r), tl, tt)
        assert torch.equal(got, full)


def test_four_lanes_equal_one(cuda):
    import torch
    from paddle3d_b200.lss import LSSHotPath
    vt = _vt(cuda)
    lanes = [LSSHotPath(vt, 1, 6, device=cuda).capture() for _ in range(4)]
    rigs = [synth.camera_rig(40 + i) for i in range(4)]
    ins = [[_t(cuda, a) for a in _inputs(vt, 1, 50 + i)] for i in range(4)]
    want = [lanes[0].infer(synth.lss_mats(rigs[i]), *ins[i])[0].clone() for i in range(4)]
    torch.cuda.synchronize()
    for rep in range(2):
        for i, lane in enumerate(lanes):
            lane.launch(synth.lss_mats(rigs[i]), *ins[i])
        torch.cuda.synchronize()
        for i, lane in enumerate(lanes):
            assert torch.equal(lane.bev, want[i]), "lane %d" % i


def test_frustum_outside_the_grid(cuda):
    """No point inside: zeros and counts (0, 0) (the reference's None ranks -> zero BEV); in a B = 2 batch whose second
    sample keeps no point, that sample is zero and the first equals its B = 1 frame."""
    import torch
    from paddle3d_b200.lss import LSSHotPath
    vt = _vt(cuda)
    far = synth.camera_rig(60, B=2)
    far["sensor2ego"][1, :, :3, 3] += np.float32(1000.0)
    one = {k: v[1:] for k, v in far.items()}
    logits, tran = _inputs(vt, 2, 9)
    f1 = LSSHotPath(vt, 1, 6, device=cuda).capture()
    bev, counts = f1.infer(synth.lss_mats(one), _t(cuda, logits[6:]), _t(cuda, tran[6:]))
    assert counts == (0, 0) and not bev.any()
    assert not vt.forward(_input_list(one), _t(cuda, logits[6:]), _t(cuda, tran[6:])).any()
    f2 = LSSHotPath(vt, 2, 6, device=cuda).capture()
    bev2, counts2 = f2.infer(synth.lss_mats(far), _t(cuda, logits), _t(cuda, tran))
    first = {k: v[:1] for k, v in far.items()}
    bev1, counts1 = f1.infer(synth.lss_mats(first), _t(cuda, logits[:6]), _t(cuda, tran[:6]))
    assert counts2 == counts1 and counts1[0] > 0
    assert not bev2[1].any() and torch.equal(bev2[0], bev1[0])
