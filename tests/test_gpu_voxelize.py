"""GPU parity: hard_voxelize / voxel_mean / pillar_scatter through the C ABI vs the oracle and the
reference's golden vectors.  Bar: bit-exact (integer/index work and copied floats)."""
import glob
import os

import numpy as np
import pytest

from conftest import ROOT, golden
from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu
VOX = sorted(os.path.basename(p) for p in glob.glob(os.path.join(ROOT, "tests", "golden", "voxelize_*.npz")))


def _run(cuda, pts, vs, pcr, P, V):
    import torch
    from paddle3d_b200.ops import voxelize
    out = voxelize.hard_voxelize(torch.from_numpy(pts).to(cuda), list(vs), list(pcr), P, V)
    torch.cuda.synchronize()
    return [o.cpu().numpy() for o in out]


def _assert_same(got, want):
    names = ["voxels", "coords", "num_points_per_voxel", "num_voxels"]
    assert int(got[3][0]) == int(want[3][0])
    for n, g, w in zip(names, got, want):
        assert np.array_equal(g, w), "%s differs" % n


@pytest.mark.parametrize("name", VOX)
def test_golden(cuda, name):
    g = golden(name)
    got = _run(cuda, g["points"], g["voxel_size"], g["point_cloud_range"], int(g["max_points"]), int(g["max_voxels"]))
    _assert_same(got, [g["voxels"], g["coords"], g["num_points_per_voxel"], g["num_voxels"]])


@pytest.mark.parametrize("cfg,gen,seed,n,P,V", [
    (synth.C1, synth.uniform_cloud, 0, 1000, 32, 40000),
    (synth.C2, synth.uniform_cloud, 1, 20000, 32, 40000),
    (synth.C2, synth.lidar_cloud, 2, 20000, 32, 40000),
    (synth.C2, synth.lidar_cloud, 3, 20000, 3, 2000),       # P overflow + voxel cap
    (synth.C3, synth.lidar_cloud, 4, 300000, 10, 160000),   # full BASELINE size, realistic occupancy
    (synth.C3, synth.uniform_cloud, 5, 300000, 10, 160000), # full size, hits the 160000 cap
    (synth.C3_01, synth.lidar_cloud, 6, 300000, 10, 160000),
    (synth.C3, synth.lidar_cloud, 7, 300000, 10, 20000),    # cap binds on lidar data
])
def test_vs_oracle(cuda, oracle_mod, cfg, gen, seed, n, P, V):
    pts = gen(cfg, seed, num_points=n)
    got = _run(cuda, pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
    want = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
    _assert_same(got, want)


def test_edge_cases(cuda, oracle_mod):
    cfg = synth.C2
    vs, pcr = cfg["voxel_size"], cfg["point_cloud_range"]
    # empty input
    got = _run(cuda, np.zeros((0, 4), np.float32), vs, pcr, 4, 64)
    assert got[3][0] == 0 and not got[0].any() and not got[1].any() and not got[2].any()
    # everything outside
    got = _run(cuda, np.full((100, 4), 1e6, np.float32), vs, pcr, 4, 64)
    assert got[3][0] == 0 and not got[0].any()
    # all points in ONE cell (worst contention), more than P
    one = np.tile(np.array([[10.0, 0.0, -1.0, 0.5]], np.float32), (5000, 1))
    one[:, 3] = np.arange(5000) / 5000.0
    _assert_same(_run(cuda, one, vs, pcr, 7, 64), oracle_mod.hard_voxelize(one, vs, pcr, 7, 64))
    # boundary points, NaN / inf coordinates are dropped like the CPU kernel drops them
    pts = np.array([[pcr[0], pcr[1], pcr[2], 1], [pcr[3], pcr[4], pcr[5], 1], [np.nan, 0, 0, 1], [np.inf, 0, 0, 1],
                    [pcr[3] - 1e-4, pcr[4] - 1e-4, pcr[5] - 1e-4, 1]], np.float32)
    _assert_same(_run(cuda, pts, vs, pcr, 4, 64), oracle_mod.hard_voxelize(pts, vs, pcr, 4, 64))
    # ragged: num_point_dim 3 and 6, V*P*F not a multiple of 4
    for F in (3, 6, 5):
        p = synth.lidar_cloud(dict(cfg, point_dim=5), 9, num_points=3001)[:, :min(F, 5)]
        if F == 6:
            p = np.concatenate([p, p[:, :1]], 1)
        p = np.ascontiguousarray(p)
        _assert_same(_run(cuda, p, vs, pcr, 3, 333), oracle_mod.hard_voxelize(p, vs, pcr, 3, 333))


def test_determinism_and_properties_full_size(cuda):
    """Size-independent properties at the BASELINE size: run-to-run identical, every kept point is an input
    point of the right cell, counts sum correctly, permutation of out-of-range points changes nothing."""
    cfg = synth.C3
    pts = synth.lidar_cloud(cfg, 11)
    a = _run(cuda, pts, cfg["voxel_size"], cfg["point_cloud_range"], 10, 160000)
    b = _run(cuda, pts, cfg["voxel_size"], cfg["point_cloud_range"], 10, 160000)
    for x, y in zip(a, b):
        assert np.array_equal(x, y)
    nv = int(a[3][0])
    voxels, coords, npv = a[0][:nv], a[1][:nv], a[2][:nv]
    assert npv.min() >= 1 and npv.max() <= 10
    vs = np.asarray(cfg["voxel_size"], np.float32)
    lo = np.asarray(cfg["point_cloud_range"][:3], np.float32)
    first = voxels[:, 0, :3]
    cell = np.floor((first - lo) / vs).astype(np.int32)[:, ::-1]
    assert np.array_equal(cell, coords)
    assert len(np.unique(coords, axis=0)) == nv
    assert not a[0][nv:].any() and not a[1][nv:].any() and not a[2][nv:].any()


def test_voxelize_mean_and_voxel_mean(cuda, oracle_mod):
    import torch
    from paddle3d_b200.ops import voxelize
    cfg = synth.C3
    pts = synth.lidar_cloud(cfg, 12, num_points=120000)
    want = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], 10, 50000)
    nv = int(want[3][0])
    want_mean = oracle_mod.voxel_mean(want[0], want[2], nv)
    t = torch.from_numpy(pts).to(cuda)
    mean, coors, npv, num = voxelize.voxelize_mean(t, cfg["voxel_size"], cfg["point_cloud_range"], 10, 50000, batch_id=0)
    assert int(num.item()) == nv
    assert np.array_equal(coors.cpu().numpy()[:nv, 1:], want[1][:nv])
    assert not coors.cpu().numpy()[:, 0].any()
    assert np.array_equal(npv.cpu().numpy(), want[2])
    np.testing.assert_allclose(mean.cpu().numpy()[:nv], want_mean, rtol=1e-6, atol=1e-7)  # fp32, tolerance 1e-4 rel allowed
    assert not mean.cpu().numpy()[nv:].any()
    v, c, n, k = voxelize.hard_voxelize(t, cfg["voxel_size"], cfg["point_cloud_range"], 10, 50000)
    m2 = voxelize.voxel_mean(v, n, k)
    np.testing.assert_allclose(m2.cpu().numpy()[:nv], want_mean, rtol=1e-6, atol=1e-7)


@pytest.mark.parametrize("cfg,C", [(synth.C2, 64), (dict(synth.C2, voxel_size=[0.2, 0.2, 4.0], point_cloud_range=[-40.1, -40.1, -3, 40.1, 40.1, 1]), 7)])
def test_pillar_scatter(cuda, oracle_mod, cfg, C):
    import torch
    from paddle3d_b200.layers import PointPillarsScatter
    rng = np.random.default_rng(3)
    pts = synth.uniform_cloud(cfg, 13, num_points=20000)
    v, c, n, nv = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], 4, 40000)
    k = int(nv[0])
    coors = np.concatenate([np.zeros((k, 1), np.int32), c[:k]], 1)
    feats = rng.normal(size=(k, C)).astype(np.float32)
    layer = PointPillarsScatter(C, cfg["voxel_size"], cfg["point_cloud_range"])
    got = layer(torch.from_numpy(feats).to(cuda), torch.from_numpy(coors).to(cuda), 1).cpu().numpy()
    want = oracle_mod.pillar_scatter(feats, coors, 1, layer.ny, layer.nx)
    assert got.shape == want.shape
    assert np.array_equal(got, want)  # pure copy: bit exact
    # batch of 2 with a device-side row count smaller than the capacity
    coors2 = coors.copy()
    coors2[k // 2:, 0] = 1
    num = torch.tensor([k - 5], dtype=torch.int32, device=cuda)
    got2 = layer(torch.from_numpy(feats).to(cuda), torch.from_numpy(coors2).to(cuda), 2, num=num).cpu().numpy()
    want2 = oracle_mod.pillar_scatter(feats[:k - 5], coors2[:k - 5], 2, layer.ny, layer.nx)
    assert np.array_equal(got2, want2)


def test_pillar_feature_net(cuda, oracle_mod):
    """hard_voxelize (C2 geometry) -> PillarFeatureNet against the oracle restatement; 1e-4 relative."""
    import torch
    from paddle3d_b200.ops import pillar_encoder, voxelize
    cfg = synth.C2
    pts = synth.lidar_cloud(cfg, 4, num_points=6000)
    P, V = 32, 3000
    vox, co, npv, nv = voxelize.hard_voxelize(torch.from_numpy(pts).to(cuda), cfg["voxel_size"], cfg["point_cloud_range"], P, V)
    k = int(nv[0].item())
    coors = torch.cat([torch.zeros((V, 1), dtype=torch.int32, device=cuda), co], 1).contiguous()
    rng = np.random.default_rng(8)
    f, c = pts.shape[1], 64
    w = (rng.normal(size=(f + 5, c)) * 0.3).astype(np.float32)
    g, b, mu, var = rng.uniform(0.5, 1.5, c), rng.normal(size=c) * 0.2, rng.normal(size=c) * 0.1, rng.uniform(0.5, 1.5, c)
    got = pillar_encoder.pillar_feature_net(vox, npv, coors, torch.from_numpy(w).to(cuda), g, b, mu, var, 1e-3,
                                            cfg["voxel_size"], cfg["point_cloud_range"], num_voxels=nv)
    want = oracle_mod.pillar_feature_net(vox.cpu().numpy()[:k], npv.cpu().numpy()[:k], coors.cpu().numpy()[:k], w, g, b, mu,
                                         var, 1e-3, cfg["voxel_size"], cfg["point_cloud_range"])
    np.testing.assert_allclose(got.cpu().numpy()[:k], want, rtol=1e-4, atol=1e-4 * np.abs(want).max())
