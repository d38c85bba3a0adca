"""CPU suite: the oracle against the reference's golden vectors / the reference itself; no GPU."""
import glob
import os

import numpy as np
import pytest

from conftest import ROOT, golden
from paddle3d_b200 import synth

VOX = sorted(os.path.basename(p) for p in glob.glob(os.path.join(ROOT, "tests", "golden", "voxelize_*.npz")))


@pytest.mark.parametrize("name", VOX)
def test_voxelize_oracle_matches_reference_golden(oracle_mod, name):
    g = golden(name)
    v, c, n, nv = oracle_mod.hard_voxelize(g["points"], g["voxel_size"], g["point_cloud_range"], int(g["max_points"]),
                                           int(g["max_voxels"]))
    assert int(nv[0]) == int(g["num_voxels"][0])
    assert np.array_equal(c, g["coords"])
    assert np.array_equal(n, g["num_points_per_voxel"])
    assert np.array_equal(v, g["voxels"])


def test_iou_oracle_matches_reference_golden(oracle_mod):
    g = golden("iou_bev.npz")
    iou = oracle_mod.boxes_iou_bev(g["boxes_a"], g["boxes_b"])
    assert np.array_equal(iou, g["iou"])  # bit exact: same fp32 operations, no FMA on either side
    assert (g["iou"] > 0.05).sum() > 100


@pytest.mark.parametrize("cfg,seed", [(synth.C1, 3), (synth.C2, 4)])
def test_voxelize_oracle_matches_reference_library(oracle_mod, cfg, seed):
    if oracle_mod.ref_lib("cpu") is None:
        pytest.skip("oracle/_ref not built (no Paddle3D checkout in $P3D_REFERENCE)")
    pts = synth.lidar_cloud(cfg, seed, num_points=min(cfg["num_points"], 20000))
    a = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], 5, 3000)
    b = oracle_mod.ref_hard_voxelize_cpu(pts, cfg["voxel_size"], cfg["point_cloud_range"], 5, 3000)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)


def test_iou_oracle_matches_reference_library(oracle_mod):
    if oracle_mod.ref_lib("cpu") is None:
        pytest.skip("oracle/_ref not built")
    a = synth.random_boxes(200, 21)
    assert np.array_equal(oracle_mod.boxes_iou_bev(a, a), oracle_mod.ref_boxes_iou_bev_cpu(a, a))


def test_voxelize_edge_cases(oracle_mod):
    cfg = synth.C1
    empty = np.zeros((0, 4), np.float32)
    v, c, n, nv = oracle_mod.hard_voxelize(empty, cfg["voxel_size"], cfg["point_cloud_range"], 4, 16)
    assert nv[0] == 0 and not v.any() and not c.any() and not n.any()
    outside = np.full((10, 4), 1e6, np.float32)
    assert oracle_mod.hard_voxelize(outside, cfg["voxel_size"], cfg["point_cloud_range"], 4, 16)[3][0] == 0
    # point exactly on the upper boundary is dropped, on the lower boundary is kept (voxelize_op.cc:47-55)
    pcr = cfg["point_cloud_range"]
    pts = np.array([[pcr[0], pcr[1], pcr[2], 1.0], [pcr[3], pcr[4], pcr[5], 1.0]], np.float32)
    v, c, n, nv = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], pcr, 4, 16)
    assert nv[0] == 1 and list(c[0]) == [0, 0, 0]


def test_nms_oracle_properties(oracle_mod):
    b = synth.random_boxes(300, 5)
    keep, nk = oracle_mod.nms(b, 0.2)
    kept = b[keep[:nk]]
    iou = oracle_mod.boxes_iou_bev(kept, kept)
    np.fill_diagonal(iou, 0)
    assert (iou <= 0.2).all()  # survivors do not suppress each other
    assert keep[0] == 0  # best box always survives
    # idempotence: NMS of the survivors keeps all of them
    _, nk2 = oracle_mod.nms(kept, 0.2)
    assert nk2 == nk


def test_sparse_conv_oracle_vs_torch_dense(oracle_mod):
    """The sparse-conv restatement against a dense fp64 conv3d over the active-site mask (SURVEY.md §8c)."""
    import torch
    rng = np.random.default_rng(0)
    B, D, H, W, Cin, Cout = 2, 7, 10, 9, 5, 6
    occ = rng.random((B, D, H, W)) < 0.15
    coords = np.argwhere(occ).astype(np.int32)
    feats = rng.normal(size=(len(coords), Cin)).astype(np.float32)
    dense = np.zeros((B, Cin, D, H, W))
    dense[coords[:, 0], :, coords[:, 1], coords[:, 2], coords[:, 3]] = feats
    for subm, ks, st, pd in [(True, (3, 3, 3), (1, 1, 1), (1, 1, 1)), (False, (3, 3, 3), (2, 2, 2), (1, 1, 1)),
                             (False, (3, 3, 3), (2, 2, 2), (0, 1, 1)), (False, (3, 1, 1), (2, 1, 1), (0, 0, 0))]:
        w = rng.normal(size=ks + (Cin, Cout)).astype(np.float32)
        oc, of, osp, pairs = oracle_mod.sparse_conv3d(coords, feats, B, (D, H, W), w, st, pd, subm)
        wt = torch.from_numpy(w.astype(np.float64)).permute(4, 3, 0, 1, 2)
        ref = torch.nn.functional.conv3d(torch.from_numpy(dense), wt, stride=st, padding=(pd if not subm else (1, 1, 1))).numpy()
        act = torch.nn.functional.conv3d(torch.from_numpy(occ[:, None].astype(np.float64)),
                                         torch.ones((1, 1) + ks, dtype=torch.float64), stride=st,
                                         padding=(pd if not subm else (1, 1, 1))).numpy()[:, 0] > 0
        if subm:
            act = occ
        assert list(ref.shape[2:]) == osp
        assert len(oc) == act.sum()
        got = np.zeros_like(ref)
        got[oc[:, 0], :, oc[:, 1], oc[:, 2], oc[:, 3]] = of
        np.testing.assert_allclose(got, ref * act[:, None], rtol=1e-5, atol=1e-5)
        assert pairs > 0


@pytest.mark.parametrize("cin,cout,k,stride,pad,bias", [(7, 5, 3, 1, 1, False), (6, 9, 3, 2, 1, True), (8, 4, 1, 1, 0, False)])
def test_conv2d_oracle_vs_torch_fp64(oracle_mod, cin, cout, k, stride, pad, bias):
    """Dense RPN/head conv restatement (PARITY UNPINNED by the reference: paddle.nn.Conv2D) against an independent
    implementation: torch's CPU conv2d in fp64 on the same operands."""
    import torch
    rng = np.random.default_rng(cin * 100 + cout)
    x = rng.normal(size=(2, cin, 13, 11)).astype(np.float32)
    w = (rng.normal(size=(cout, cin, k, k)) * 0.2).astype(np.float32)
    b = rng.normal(size=(cout,)).astype(np.float32) if bias else None
    got = oracle_mod.conv2d(x, w, b, stride, pad)
    want = torch.nn.functional.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(),
                                      None if b is None else torch.from_numpy(b).double(), stride=stride, padding=pad)
    assert got.shape == tuple(want.shape)
    np.testing.assert_allclose(got, want.numpy(), rtol=1e-6, atol=1e-6)


def test_deconv2d_and_bn2d_oracle_vs_torch_fp64(oracle_mod):
    import torch
    rng = np.random.default_rng(9)
    x = rng.normal(size=(2, 6, 7, 5)).astype(np.float32)
    w = (rng.normal(size=(6, 4, 2, 2)) * 0.3).astype(np.float32)  # [Cin, Cout, k, k]
    got = oracle_mod.deconv2d(x, w, None, 2)
    want = torch.nn.functional.conv_transpose2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), stride=2)
    assert got.shape == (2, 4, 14, 10)
    np.testing.assert_allclose(got, want.numpy(), rtol=1e-6, atol=1e-6)
    g, bt, m, v = (rng.uniform(0.5, 1.5, 4), rng.normal(size=4), rng.normal(size=4), rng.uniform(0.5, 2.0, 4))
    y = oracle_mod.bn2d_relu(got, g, bt, m, v, 1e-3)
    ref = torch.nn.functional.batch_norm(want, torch.from_numpy(m), torch.from_numpy(v), torch.from_numpy(g),
                                         torch.from_numpy(bt), False, 0.0, 1e-3).clamp_min(0)
    np.testing.assert_allclose(y, ref.numpy(), rtol=1e-5, atol=1e-6)


def test_cpu_dense_head_vs_torch_fp64(oracle_mod):
    """Structure of the dense RPN / neck / head restatement (dense_head.DenseRPNHead + cpu_reference.CpuDenseHead:
    block order, stride-2 stage, 1x1 / transposed-conv neck, channel concat order, shared conv, per-task heads)
    against the same network written with torch's fp64 CPU ops."""
    import torch
    import torch.nn.functional as F
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import DenseRPNHead
    net = DenseRPNHead(in_channels=32, out_channels=(32, 64), layer_nums=(1, 2), downsample_strides=(1, 2),
                       fpn_out_channels=(32, 32), upsample_strides=(1, 2), tasks=(1, 2), share_conv_channel=32)
    net.init_weight(seed=4, device=None, randomize_bn=True)
    w = net.export_numpy()
    rng = np.random.default_rng(0)
    bev = rng.normal(size=(1, 32, 20, 28)).astype(np.float32)
    got = CpuDenseHead(w).run(bev)

    def conv(l, x):
        wt = torch.from_numpy(l["weight"]).double()
        b = None if l["bias"] is None else torch.from_numpy(l["bias"]).double()
        y = (F.conv_transpose2d(x, wt, b, stride=l["up"]) if l["up"] > 1
             else F.conv2d(x, wt, b, stride=l["stride"], padding=l["padding"]))
        if l["bn"] is not None:
            bn = {k: torch.from_numpy(np.asarray(v)).double() for k, v in l["bn"].items() if k != "eps"}
            y = F.batch_norm(y, bn["mean"], bn["var"], bn["gamma"], bn["beta"], False, 0.0, l["bn"]["eps"])
        return y.clamp_min(0) if l["relu"] else y

    x, feats = torch.from_numpy(bev).double(), []
    for blk in w["blocks"]:
        for l in blk:
            x = conv(l, x)
        feats.append(x)
    cat = torch.cat([conv(l, f) for l, f in zip(w["deblocks"], feats)], 1)
    assert cat.shape == (1, 64, 20, 28)
    s = conv(w["shared"], cat)
    for ti, hs in enumerate(w["heads"]):
        for name, a, fin in hs:
            want = conv(fin, conv(a, s)).numpy()
            g = got[name][ti]
            assert g.shape == want.shape
            np.testing.assert_allclose(g, want, rtol=2e-5, atol=2e-5)
    assert got["hm"][1].shape == (1, 2, 20, 28) and got["reg"][0].shape == (1, 2, 20, 28)


def test_pillar_feature_net_oracle_vs_torch(oracle_mod):
    """PFN restatement (PARITY UNPINNED) against the same layer written with torch fp64 ops, incl. the property that
    zeroed padding rows still take part in the max with the value ReLU(BN(0))."""
    import torch
    rng = np.random.default_rng(2)
    n, m, f, c = 50, 8, 4, 16
    vs, pcr = [0.16, 0.16, 4.0], [0.0, -39.68, -3.0, 69.12, 39.68, 1.0]
    npv = rng.integers(1, m + 1, size=n).astype(np.int32)
    coors = np.stack([np.zeros(n, np.int32), np.zeros(n, np.int32), rng.integers(0, 496, n), rng.integers(0, 432, n)], 1).astype(np.int32)
    vox = np.zeros((n, m, f), np.float32)
    for i in range(n):
        cx, cy = coors[i, 3] * vs[0] + pcr[0], coors[i, 2] * vs[1] + pcr[1]
        vox[i, :npv[i], 0] = cx + rng.uniform(0, vs[0], npv[i])
        vox[i, :npv[i], 1] = cy + rng.uniform(0, vs[1], npv[i])
        vox[i, :npv[i], 2] = rng.uniform(-3, 1, npv[i])
        vox[i, :npv[i], 3] = rng.uniform(0, 1, npv[i])
    w = rng.normal(size=(f + 5, c)).astype(np.float32)
    g, b, mu, var = rng.uniform(0.5, 1.5, c), rng.normal(size=c), rng.normal(size=c) * 0.1, rng.uniform(0.5, 1.5, c)
    got = oracle_mod.pillar_feature_net(vox, npv, coors, w, g, b, mu, var, 1e-3, vs, pcr)
    v = torch.from_numpy(vox).double()
    pm = v[:, :, :3].sum(1, keepdim=True) / torch.from_numpy(npv).double().view(-1, 1, 1)
    fc = v[:, :, :2].clone()
    fc[:, :, 0] -= torch.from_numpy(coors[:, 3]).float().view(-1, 1).double() * np.float32(vs[0]) + np.float32(vs[0] / 2 + pcr[0])
    fc[:, :, 1] -= torch.from_numpy(coors[:, 2]).float().view(-1, 1).double() * np.float32(vs[1]) + np.float32(vs[1] / 2 + pcr[1])
    feats = torch.cat([v, v[:, :, :3] - pm, fc], -1)
    mask = (torch.arange(m).view(1, -1) < torch.from_numpy(npv).view(-1, 1)).double().unsqueeze(-1)
    x = (feats * mask) @ torch.from_numpy(w).double()
    x = torch.nn.functional.batch_norm(x.transpose(1, 2), torch.from_numpy(mu), torch.from_numpy(var), torch.from_numpy(g),
                                       torch.from_numpy(b), False, 0.0, 1e-3).transpose(1, 2)
    want = x.clamp_min(0).max(1).values.numpy()
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-6)
    pad = np.maximum((0 - mu) / np.sqrt(var + 1e-3) * g + b, 0)  # what a padding row contributes
    assert (got[npv < m] >= pad.astype(np.float32) - 1e-6).all()


def test_prepare_restatement_matches_the_generator(oracle_mod):
    """oracle.voxel_pooling_prepare_v2 (line-by-line restatement of bevdet_transformer.py:230-274) against the ranks the
    synthetic-input generator builds the same way: two statements of the same algorithm must agree."""
    from paddle3d_b200 import synth
    d = synth.bev_pool_inputs(3, D=20, H=6, W=10, grid=(64, 64, 1), bounds=((-30, 30), (-30, 30), (-5, 3)))
    got = oracle_mod.voxel_pooling_prepare_v2(d["coor"], d["grid_lower_bound"], d["grid_interval"], d["grid_size"])
    for g, k in zip(got, ("ranks_bev", "ranks_depth", "ranks_feat", "interval_starts", "interval_lengths")):
        assert np.array_equal(g, d[k]), k
    assert (np.diff(got[0]) >= 0).all() and got[4].sum() == len(got[0])
