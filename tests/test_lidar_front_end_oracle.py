"""CPU: the restatements of tests/lidar_front_end_oracle.py against fp64 and plain loops, and the argument checks of the
LiDAR front-end entry points (pillar encoders, few-channel conv, dense scatter, rows to pixel rows), which refuse before
any launch."""
import ctypes as C

import numpy as np
import pytest

import lidar_front_end_oracle as lfo
from paddle3d_b200 import synth

ERR_INVALID, ERR_WORKSPACE, ERR_UNSUPPORTED = -1, -2, -4


def _cloud(seed, n, f, cfg=synth.C3):
    """Points of a C3 cloud plus dense clusters: cells with many more points than any P, and cells with 1 point."""
    rng = np.random.default_rng(seed)
    pts = synth.lidar_cloud(dict(cfg, point_dim=min(f, 5)), seed, num_points=n)[:, :min(f, 5)]
    if f > 5:
        pts = np.concatenate([pts, rng.normal(size=(n, f - 5)).astype(np.float32)], 1)
    lo = np.asarray(cfg["point_cloud_range"][:3], np.float32)
    vs = np.asarray(cfg["voxel_size"], np.float32)
    blob = lo + vs * (np.asarray([300, 500, 20]) + rng.uniform(0.05, 0.95, (400, 3)))
    blob = np.concatenate([blob, rng.uniform(-50, 50, (400, f - 3))], 1).astype(np.float32)
    return np.ascontiguousarray(np.concatenate([pts, blob])[rng.permutation(n + 400)], np.float32)


@pytest.mark.parametrize("P,f", [(1, 4), (10, 3), (17, 5), (64, 6)])
def test_voxel_mean_restatement_within_fp64_bound(oracle_mod, P, f):
    """The fp32 slot-order mean is within P 2^-24 sum|x| / cnt + 1/2 ulp of the fp64 mean; dividing by P instead of the
    count, or dropping the last kept point, is not."""
    cfg = synth.C3
    pts = _cloud(P + f, 20000, f)
    vox, _, npv, nv = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, 30000)
    k = int(nv[0])
    got = lfo.voxel_mean_f32(vox, npv, k)
    assert not got[k:].any()
    want = lfo.voxel_mean_f64(vox, npv, k)
    bound = lfo.mean_bound(vox, npv, k, P, got)
    assert (np.abs(got[:k] - want) <= bound).all()
    assert (npv[:k] == P).any() and (npv[:k] == 1).any()
    if P > 1:
        by_p = (vox[:k].astype(np.float64).sum(1) / P).astype(np.float32)
        assert (np.abs(by_p - want) > bound).any()
        short = vox.copy()
        short[np.arange(k), npv[:k] - 1] = 0
        assert (np.abs(lfo.voxel_mean_f32(short, npv, k)[:k] - want) > bound).any()


def test_scatter_restatement_matches_a_loop():
    rng = np.random.default_rng(0)
    B, C, D, ny, nx = 3, 5, 2, 7, 9
    n_cap, n = 300, 260
    co = np.stack([rng.integers(-1, B + 1, n_cap), rng.integers(-1, D + 1, n_cap), rng.integers(-1, ny + 1, n_cap),
                   rng.integers(-1, nx + 1, n_cap)], 1).astype(np.int32)
    feats = rng.normal(size=(n_cap, C)).astype(np.float32)
    for use_z in (0, 1):
        want = np.zeros((B, C, D, ny, nx), np.float32)
        for i in range(n):
            b, z, y, x = co[i]
            z = z if use_z else 0
            if 0 <= b < B and 0 <= z < D and 0 <= y < ny and 0 <= x < nx:
                want[b, :, z, y, x] = feats[i]
        assert np.array_equal(lfo.scatter_dense(feats, co, n, B, D, ny, nx, use_z), want)


def test_rows_to_pixel_restatement_matches_a_loop():
    rng = np.random.default_rng(1)
    B, C, D, ny, nx = 2, 64, 3, 5, 6
    sites = rng.choice(B * D * ny * nx, 70, replace=False)
    co = np.stack([sites // (D * ny * nx), sites // (ny * nx) % D, sites // nx % ny, sites % nx], 1).astype(np.int32)
    co[:5, 2] = ny  # out of range: skipped
    rows = rng.integers(0, 65536, (70, 2 * C)).astype(np.uint16)
    want = np.zeros((B, ny, nx, D * 2 * C), np.uint16)
    for i in range(60):
        b, z, y, x = co[i]
        if y < ny:
            want[b, y, x, 2 * z * C:2 * (z + 1) * C] = rows[i]
    assert np.array_equal(lfo.rows_to_pixel_h16(rows, co, 60, C, B, D, ny, nx), want.reshape(B * ny * nx, -1))
    canvas = rng.normal(size=(B, C, D, ny, nx))
    zc = lfo.zc_order(canvas)
    assert np.array_equal(zc[:, 2 * C + 7], canvas[:, 7, 2])


@pytest.mark.parametrize("ksize,subm", [((3, 3, 3), True), ((1, 1, 7), True), ((1, 3, 1), True), ((1, 1, 1), True),
                                        ((2, 4, 5), False)])
def test_nbr_map_gather_matches_oracle_sparse_conv(oracle_mod, ksize, subm):
    """The neighbour map built here, gathered in fp64, is oracle.sparse_conv3d: same taps in the same weight order."""
    rng = np.random.default_rng(sum(ksize))
    spatial = (6, 12, 14)
    n = 300
    sites = rng.choice(2 * np.prod(spatial), n, replace=False)
    D, H, W = spatial
    co = np.stack([sites // (D * H * W), sites // (H * W) % D, sites // W % H, sites % W], 1).astype(np.int32)
    feats = rng.normal(size=(n, 5)).astype(np.float32)
    w = rng.normal(size=ksize + (5, 16)).astype(np.float32)
    pad = tuple(k // 2 for k in ksize) if subm else (0, 0, 0)
    oc, of, osp, _ = oracle_mod.sparse_conv3d(co, feats, 2, spatial, w, padding=pad, subm=subm)
    nbr = lfo.nbr_map(co, oc, spatial, ksize, padding=pad)
    assert (nbr >= 0).any() and ((nbr < 0).any() or nbr.shape[1] == 1)
    np.testing.assert_allclose(lfo.gather_conv_f64(feats, nbr, w), of, rtol=1e-6, atol=1e-5)


def _pfn_case(rng, far, f=4, m=32, c=64):
    n = 200
    cnt = np.concatenate([[1] * 20, [m] * 20, rng.integers(1, m + 1, n - 40)]).astype(np.int32)
    vs, pcr = [0.16, 0.16, 4.0], [0.0, -39.68, -3.0, 69.12, 39.68, 1.0]
    nx, ny = 432, 496
    xs = rng.integers(nx - 12, nx, n) if far else rng.integers(nx // 2 - 6, nx // 2 + 6, n)
    ys = rng.integers(0, 6, n) if far else rng.integers(ny // 2 - 6, ny // 2 + 6, n)
    coors = np.stack([np.zeros(n), np.zeros(n), ys, xs], 1).astype(np.int32)
    vox = np.zeros((n, m, f), np.float32)
    for i in range(n):
        x0 = pcr[0] + (xs[i] + rng.uniform(0, 1, cnt[i])) * vs[0]
        y0 = pcr[1] + (ys[i] + rng.uniform(0, 1, cnt[i])) * vs[1]
        vox[i, :cnt[i]] = np.concatenate([np.stack([x0, y0, rng.uniform(-3, 1, cnt[i])], 1),
                                          rng.uniform(0, 1, (cnt[i], f - 3))], 1)
    w = (rng.normal(size=(f + 5, c)) * 0.3).astype(np.float32)
    g, b = rng.uniform(0.5, 1.5, c), rng.normal(size=c) * 0.2
    mu, var = rng.normal(size=c) * 0.1, rng.uniform(0.5, 1.5, c)
    return vox, cnt, coors, w, (g, b, mu, var, 1e-3), vs, pcr


def _pfn_f32(vox, cnt, coors, w, scale, shift, vs, pcr):
    """The one-layer kernel in fp32 numpy (products and sums rounded separately: the bound covers FMA or not)."""
    f32 = np.float32
    n, m, f = vox.shape
    mean = (vox[:, :, :3].sum(1, dtype=np.float32) / cnt[:, None].astype(f32)).astype(f32)
    xo, yo = f32(f32(vs[0]) / 2 + f32(pcr[0])), f32(f32(vs[1]) / 2 + f32(pcr[1]))
    cx = (coors[:, 3].astype(f32) * f32(vs[0]) + xo).astype(f32)
    cy = (coors[:, 2].astype(f32) * f32(vs[1]) + yo).astype(f32)
    feats = np.concatenate([vox, vox[:, :, :3] - mean[:, None], (vox[:, :, :2] - np.stack([cx, cy], 1)[:, None])], -1)
    feats = feats.astype(f32) * (np.arange(m)[None, :] < cnt[:, None])[:, :, None].astype(f32)
    acc = np.zeros((n, m, w.shape[1]), f32)
    for d in range(f + 5):
        acc = (acc + (feats[:, :, d:d + 1] * w[d]).astype(f32)).astype(f32)
    return np.maximum((acc * scale + shift).astype(f32), 0).max(1)


@pytest.mark.parametrize("far", [False, True])
def test_pfn_bound_covers_an_fp32_restatement(oracle_mod, far):
    """pfn_bound holds for an fp32 restatement of the kernel near the origin and at the far edge of the grid (x ~ 69 m,
    where the decoration subtracts values that agree to ~0.1 m), and stays far below 1e-4 of the output's scale."""
    rng = np.random.default_rng(7 + far)
    vox, cnt, coors, w, bn, vs, pcr = _pfn_case(rng, far)
    g, b, mu, var, eps = bn
    s = (g / np.sqrt(var + eps)).astype(np.float32)
    t = (b - mu * (g / np.sqrt(var + eps))).astype(np.float32)
    got = _pfn_f32(vox, cnt, coors, w, s, t, vs, pcr)
    want = oracle_mod.pillar_feature_net(vox, cnt, coors, w, g, b, mu, var, eps, vs, pcr)
    bound = lfo.pfn_bound(vox, cnt, coors, w, s, t, vs, pcr)
    err = np.abs(got.astype(np.float64) - want)
    assert (err <= bound).all(), float((err / bound).max())
    assert bound.max() < 1e-5 * np.abs(want).max()  # not vacuous


def test_entry_points_refuse_before_launch():
    from paddle3d_b200 import _lib
    L = _lib.lib()
    p = C.c_void_p(256)  # non-null, 256-byte aligned dummy address: every call below returns before touching it
    vs, pcr = _lib.host_floats([0.2, 0.2, 8.0]), _lib.host_floats([-51.2, -51.2, -5.0, 51.2, 51.2, 3.0])
    # one-layer pillar encoder: more than 64 points per pillar, more than 8 point features
    assert L.p3d_pillar_feature_net(p, p, p, None, 10, 65, 4, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert L.p3d_pillar_feature_net(p, p, p, None, 10, 64, 9, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert L.p3d_pillar_feature_net(p, p, p, None, 10, 64, 8, 0, p, p, p, vs, pcr, p, None) == ERR_INVALID
    assert L.p3d_pillar_feature_net(p, p, p, None, 0, 64, 8, 64, p, p, p, vs, pcr, p, None) == 0  # nothing to do
    # two-layer encoder: the same limits, and a first layer wider than 64 channels
    pfn2 = L.p3d_pillar_feature_net2
    assert pfn2(p, p, p, None, 10, 20, 5, 65, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert pfn2(p, p, p, None, 10, 65, 5, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert pfn2(p, p, p, None, 10, 20, 9, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    # few-channel conv with fp16-pair rows: the weights of all taps must fit 40 KB of shared memory
    sc = L.p3d_sparse_conv_small_cin_h16
    assert sc(p, p, None, 100, 41, 8, 32, p, None, None, 0, p, None, None, None) == ERR_UNSUPPORTED
    assert sc(p, p, None, 100, 27, 9, 16, p, None, None, 0, p, None, None, None) == ERR_UNSUPPORTED
    assert sc(p, p, None, 100, 27, 4, 24, p, None, None, 0, p, None, None, None) == ERR_UNSUPPORTED
    assert sc(p, p, None, 100, 27, 4, 16, p, None, None, 0, None, None, None, None) == ERR_INVALID  # no output
    assert sc(p, p, None, 100, 27, 4, 16, p, None, None, 0, C.c_void_p(264), None, None, None) == ERR_INVALID
    # dense scatter: a workspace one byte short, misaligned coordinates
    need = L.p3d_scatter_dense_workspace_bytes(3, 5, 33, 17)
    assert need >= 3 * 5 * 33 * 17 * 4
    assert L.p3d_scatter_dense(p, p, None, 10, 9, 3, 5, 33, 17, 1, p, p, need - 1, None) == ERR_WORKSPACE
    assert L.p3d_scatter_dense(p, C.c_void_p(260), None, 10, 9, 3, 5, 33, 17, 1, p, p, need, None) == ERR_INVALID
    # rows to pixel rows: C a multiple of 32 only
    assert L.p3d_sparse_rows_to_pixel_h16(p, p, None, 10, 48, 2, 2, 8, 8, p, None) == ERR_INVALID
    # fused voxelize + mean: a workspace one byte short
    ws = L.p3d_hard_voxelize_workspace_bytes(1000, 20, 500)
    assert L.p3d_voxelize_mean(p, 1000, 4, vs, pcr, 20, 500, 0, p, p, p, p, p, ws - 1, None) == ERR_WORKSPACE
