"""GPU: the LiDAR front-end kernels between the point cloud and the first dense image, at their edges, through the C ABI:
voxelize_mean / voxel_mean (csrc/voxelize.cu), the one-layer pillar encoder (csrc/pillar_encoder.cu), the dense scatter
and sparse rows to pixel rows (csrc/scatter.cu), the few-channel input conv and the unfused sparse epilogue
(csrc/sparse_conv.cu).  References: oracle.hard_voxelize (bit-exact), the fp32 / numpy restatements of
tests/lidar_front_end_oracle.py (bit-exact), and the fp64 oracles (oracle.pillar_feature_net, oracle.sparse_conv3d +
oracle.bn_relu) at rel_check 1e-4 or an a-priori bound.  Outputs are pre-filled with sentinels wherever the kernel must
either write every element or leave rows beyond the device count untouched."""
import numpy as np
import pytest

import lidar_front_end_oracle as lfo
from paddle3d_b200 import synth
from parity import rel_check

pytestmark = pytest.mark.gpu


def _t(a, cuda):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _num(n, cuda):
    import torch
    return torch.tensor([n], dtype=torch.int32, device=cuda)


def _lib():
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    return lib(), check, ptr, stream


def _bits(a):
    a = np.ascontiguousarray(a)
    return a.view({4: np.uint32, 2: np.uint16}[a.dtype.itemsize])


# ================================================================================================= 1. voxelize_mean
def _crafted_cloud(P, F, seed, n=20000, cfg=synth.C3):
    """A LiDAR cloud plus cells on the top slab of the grid (which the cloud does not reach) holding more than
    max(4P, 32) points, exactly P, P + 1 and 1 point, and points with NaN / inf coordinates; rows shuffled so that every
    cell's points arrive interleaved."""
    rng = np.random.default_rng(seed)
    pts = synth.lidar_cloud(dict(cfg, point_dim=5), seed, num_points=n)
    pts = np.concatenate([pts, rng.normal(size=(n, 3)).astype(np.float32)], 1)[:, :F]
    lo = np.asarray(cfg["point_cloud_range"][:3], np.float64)
    vs = np.asarray(cfg["voxel_size"], np.float64)
    gz = int(round((cfg["point_cloud_range"][5] - cfg["point_cloud_range"][2]) / vs[2]))
    big = max(4 * P, 32) + 5
    counts = [big, big + 40, P, P, P + 1, P + 1, 1, 1, 1, 3 * P + 2]
    extra = []
    for j, c in enumerate(counts):
        cell = np.asarray([100 + 37 * j, 200 + 11 * j, gz - 1])
        xyz = lo + vs * (cell + rng.uniform(0.05, 0.95, (c, 3)))
        extra.append(np.concatenate([xyz, rng.normal(scale=20.0, size=(c, F - 3))], 1))
    bad = np.asarray([[np.nan, 0, 0], [0, np.nan, 0], [0, 0, np.nan], [np.inf, 0, 0], [-np.inf, 0, 0], [0, 0, np.inf]])
    extra.append(np.concatenate([bad, np.ones((len(bad), F - 3))], 1))
    pts = np.concatenate([pts] + [e.astype(np.float32) for e in extra])
    return np.ascontiguousarray(pts[rng.permutation(len(pts))], np.float32)


def _voxelize_mean(cuda, pts, cfg, P, V, batch_id):
    """p3d_voxelize_mean with every output pre-filled with a sentinel."""
    import torch
    from paddle3d_b200._lib import host_floats
    L, check, ptr, stream = _lib()
    n, F = pts.shape
    mean = torch.full((V, F), float("nan"), device=cuda)
    coors = torch.full((V, 4), -7, dtype=torch.int32, device=cuda)
    npv = torch.full((V,), -7, dtype=torch.int32, device=cuda)
    nv = torch.full((1,), -7, dtype=torch.int32, device=cuda)
    ws = torch.empty(max(L.p3d_hard_voxelize_workspace_bytes(n, P, V), 256), dtype=torch.uint8, device=cuda)
    tp = _t(pts, cuda) if n else torch.empty((0, F), device=cuda)
    check(L.p3d_voxelize_mean(ptr(tp), n, F, host_floats(cfg["voxel_size"]), host_floats(cfg["point_cloud_range"]), P, V,
                              batch_id, ptr(mean), ptr(coors), ptr(npv), ptr(nv), ptr(ws), ws.numel(), stream(cuda)),
          "voxelize_mean")
    torch.cuda.synchronize()
    return mean.cpu().numpy(), coors.cpu().numpy(), npv.cpu().numpy(), int(nv.item())


def _check_voxelize_mean(cuda, oracle_mod, pts, cfg, P, V, batch_id, name):
    import torch
    from paddle3d_b200.ops import voxelize
    vs, pcr = cfg["voxel_size"], cfg["point_cloud_range"]
    vox, co, npv, nv = oracle_mod.hard_voxelize(pts, vs, pcr, P, V)
    k = int(nv[0])
    mean, coors4, npv_g, k_g = _voxelize_mean(cuda, pts, cfg, P, V, batch_id)
    assert k_g == k
    assert np.array_equal(npv_g, npv)
    assert (coors4[:k, 0] == batch_id).all()
    assert np.array_equal(coors4[:k, 1:], co[:k])
    assert not coors4[k:].any()
    want = lfo.voxel_mean_f32(vox, npv, k)
    assert np.array_equal(_bits(mean), _bits(want)), "%s: mean differs from the fp32 slot-order restatement" % name
    if k:
        err = np.abs(mean[:k].astype(np.float64) - lfo.voxel_mean_f64(vox, npv, k))
        assert (err <= lfo.mean_bound(vox, npv, k, P, mean)).all()
    # voxel_mean on hard_voxelize's padded outputs: the same bits (its sum adds the zero padding, which changes nothing)
    if len(pts):
        v, _, n_g, nv_g = voxelize.hard_voxelize(_t(pts, cuda), vs, pcr, P, V)
        m2 = voxelize.voxel_mean(v, n_g, nv_g)
        assert np.array_equal(_bits(m2.cpu().numpy()), _bits(mean))
        if k == V:  # every capacity row is live: a device count above capacity, and none at all, change nothing
            for num in (_num(V + 5, cuda), None):
                assert np.array_equal(_bits(voxelize.voxel_mean(v, n_g, num).cpu().numpy()), _bits(mean))
        torch.cuda.synchronize()
    return k, npv


@pytest.mark.parametrize("F", [3, 4, 5, 6])
@pytest.mark.parametrize("P", [1, 10, 16, 17, 20, 32, 64])
def test_voxelize_mean_crafted(cuda, oracle_mod, P, F):
    """Both slot paths (P <= 16 records arrivals, P > 16 cascades every point), voxels with more than max(4P, 32)
    points, exactly P, P + 1 and 1; batch_id 0 and 3; max_voxels binding and not."""
    cfg = synth.C3
    pts = _crafted_cloud(P, F, seed=P * 10 + F)
    k, npv = _check_voxelize_mean(cuda, oracle_mod, pts, cfg, P, 60000, 3 if (P + F) % 2 else 0, "P%d F%d" % (P, F))
    assert k < 60000 and (npv[:k] == P).any() and (npv[:k] == 1).any()
    k2, _ = _check_voxelize_mean(cuda, oracle_mod, pts, cfg, P, k // 3, 0 if (P + F) % 2 else 3, "P%d F%d V" % (P, F))
    assert k2 == k // 3


def test_voxelize_mean_empty_and_outside(cuda, oracle_mod):
    cfg = synth.C3
    for P in (10, 20):
        _check_voxelize_mean(cuda, oracle_mod, np.zeros((0, 4), np.float32), cfg, P, 64, 3, "empty")
        out = np.full((500, 4), 1e4, np.float32)
        out[::2, 0] = np.nan
        out[1::4, 2] = -np.inf
        k, _ = _check_voxelize_mean(cuda, oracle_mod, out, cfg, P, 64, 3, "outside")
        assert k == 0


@pytest.mark.parametrize("cfg", [synth.C3, synth.C3_01], ids=["C3", "C3_01"])
def test_voxelize_mean_bench_frame(cuda, oracle_mod, cfg):
    """The first kernel of the benchmarked frame at its size: 300k points, P = 10, V = 160000."""
    pts = synth.lidar_cloud(cfg, 21)
    _check_voxelize_mean(cuda, oracle_mod, pts, cfg, 10, 160000, 0, "bench")


# ================================================================================================= 2. pillar encoder
PFN_GEOM = dict(voxel_size=[0.16, 0.16, 4.0], point_cloud_range=[0.0, -39.68, -3.0, 69.12, 39.68, 1.0])  # 432 x 496


def _pfn_pillars(f, m, seed, cap=330, n=300):
    """Pillars with 1 and with M points and counts in between; half at the grid's far corners (x ~ 69 m, |y| ~ 39 m),
    half near the middle; rows n .. cap are capacity rows (with valid contents, for the count-above-capacity case)."""
    rng = np.random.default_rng(seed)
    vs, pcr = PFN_GEOM["voxel_size"], PFN_GEOM["point_cloud_range"]
    cnt = np.concatenate([[1] * 20, [m] * 20, rng.integers(1, m + 1, cap - 40)]).astype(np.int32)
    far = rng.random(cap) < 0.5
    xs = np.where(far, rng.integers(420, 432, cap), rng.integers(200, 232, cap))
    ys = np.where(far, np.where(rng.random(cap) < 0.5, rng.integers(0, 12, cap), rng.integers(484, 496, cap)),
                  rng.integers(230, 266, cap))
    coors = np.stack([np.zeros(cap), np.zeros(cap), ys, xs], 1).astype(np.int32)
    vox = np.zeros((cap, m, f), np.float32)
    for i in range(cap):
        x = pcr[0] + (xs[i] + rng.uniform(0, 1, cnt[i])) * vs[0]
        y = pcr[1] + (ys[i] + rng.uniform(0, 1, cnt[i])) * vs[1]
        vox[i, :cnt[i]] = np.concatenate([np.stack([x, y, rng.uniform(-3, 1, cnt[i])], 1),
                                          rng.uniform(0, 1, (cnt[i], f - 3))], 1)
    return vox, cnt, coors, n


def _pfn_params(f, c, seed):
    """BN with large positive shifts on a third of the channels: there a padding row's ReLU(shift) is the maximum of
    pillars whose rows all project below it."""
    rng = np.random.default_rng(seed)
    w = (rng.normal(size=(f + 5, c)) * 0.3).astype(np.float32)
    g, mu, var = rng.uniform(0.5, 1.5, c), rng.normal(size=c) * 0.1, rng.uniform(0.5, 1.5, c)
    b = np.where(np.arange(c) % 3 == 0, rng.uniform(3.0, 6.0, c), rng.normal(size=c) * 0.2)
    return w, (g, b, mu, var, 1e-3)


def _pfn_abi(cuda, vox, npv, coors, num, cap, w, s, t, out):
    from paddle3d_b200._lib import host_floats
    L, check, ptr, stream = _lib()
    m, f = vox.shape[1], vox.shape[2]
    rc = L.p3d_pillar_feature_net(ptr(vox), ptr(npv), ptr(coors), ptr(num), cap, m, f, w.shape[1], ptr(w), ptr(s),
                                  ptr(t), host_floats(PFN_GEOM["voxel_size"]), host_floats(PFN_GEOM["point_cloud_range"]),
                                  ptr(out), stream(cuda))
    check(rc, "pillar_feature_net")


@pytest.mark.parametrize("m", [1, 20, 32, 64])
@pytest.mark.parametrize("f", [3, 4, 5, 8])
def test_pillar_feature_net_one_layer(cuda, oracle_mod, f, m):
    """p3d_pillar_feature_net for C in {1, 7, 64, 65, 128, 200} (64- and 128-thread launches, channels wrapping over
    the block): the fp64 oracle at rel_check 1e-4, and within pfn_bound element by element; rows beyond the device
    count keep a sentinel; a count above capacity computes every capacity row; n_cap = 0 writes nothing."""
    import torch
    from paddle3d_b200.ops import pillar_encoder as pe
    vox, cnt, coors, n = _pfn_pillars(f, m, seed=f * 100 + m)
    cap = len(cnt)
    dv, dn, dc = _t(vox, cuda), _t(cnt, cuda), _t(coors, cuda)
    vs, pcr = PFN_GEOM["voxel_size"], PFN_GEOM["point_cloud_range"]
    for c in (1, 7, 64, 65, 128, 200):
        w, (g, b, mu, var, eps) = _pfn_params(f, c, seed=c + f + m)
        s, t = pe.fold_bn(g, b, mu, var, eps, cuda)
        dw = _t(w, cuda)
        want = oracle_mod.pillar_feature_net(vox, cnt, coors, w, g, b, mu, var, eps, vs, pcr)
        bound = lfo.pfn_bound(vox, cnt, coors, w, s.cpu().numpy(), t.cpu().numpy(), vs, pcr)
        out = torch.full((cap, c), 7.0, device=cuda)
        _pfn_abi(cuda, dv, dn, dc, _num(n, cuda), cap, dw, s, t, out)
        got = out.cpu().numpy()
        assert (got[n:] == 7.0).all(), "rows beyond the device count were written"
        rel_check("pfn1 F%d M%d C%d" % (f, m, c), got[:n], want[:n], rtol=1e-4)
        err = np.abs(got[:n].astype(np.float64) - want[:n])
        assert (err <= bound[:n]).all(), "F%d M%d C%d: %.3g x the a-priori bound" % (f, m, c, (err / bound[:n]).max())
        if m > 1 and c >= 64:  # the padding rows' ReLU(shift) decides some maxima: the checks above saw them
            t_np = t.cpu().numpy()
            assert ((cnt[:n] < m)[:, None] & (want[:n] == np.float32(np.maximum(t_np, 0))) & (t_np > 1.0)).any()
        # the wrapper (zero-filled output, count on the device) gives the same bits
        ref = pe.pillar_feature_net(dv, dn, dc, dw, g, b, mu, var, eps, vs, pcr, num_voxels=_num(n, cuda), folded=(s, t))
        assert torch.equal(ref[:n], out[:n])
        # a device count above capacity: every capacity row
        out2 = torch.full((cap, c), 7.0, device=cuda)
        _pfn_abi(cuda, dv, dn, dc, _num(cap + 9, cuda), cap, dw, s, t, out2)
        rel_check("pfn1 F%d M%d C%d all" % (f, m, c), out2.cpu().numpy(), want, rtol=1e-4)
        assert torch.equal(out2[:n], out[:n])
        # n_cap = 0: nothing to do, nothing written
        out3 = torch.full((1, c), 7.0, device=cuda)
        _pfn_abi(cuda, dv, dn, dc, _num(n, cuda), 0, dw, s, t, out3)
        torch.cuda.synchronize()
        assert bool((out3 == 7.0).all())


# ================================================================================================= 3. dense scatter
def _coords(rng, n, batch, D, ny, nx, dup_frac=0.3, bad=True):
    """(b, z, y, x) rows in random batch order, a fraction of them repeating an earlier cell, and (bad=True) rows with
    each of the four fields out of range, negative and at / beyond the bound."""
    base = np.stack([rng.integers(0, batch, n), rng.integers(0, D, n), rng.integers(0, ny, n), rng.integers(0, nx, n)],
                    1).astype(np.int32)
    dup = rng.random(n) < dup_frac
    base[dup] = base[rng.integers(0, n, int(dup.sum()))]
    if bad:
        bounds = (batch, D, ny, nx)
        for field in range(4):
            for val in (-1, -1000, bounds[field], bounds[field] + 5):
                i = rng.integers(0, n)
                base[i, field] = val
    return base


SCATTER_GEOMS = [  # (batch, D, ny, nx, use_z): S = D ny nx
    (3, 1, 16, 24, 0),    # vector path, 3 tiles
    (3, 1, 7, 9, 0),      # S = 63: scalar path, one partial tile
    (3, 2, 5, 12, 1),     # S = 120: vector path, one partial tile
    (2, 5, 11, 13, 1),    # S = 715: scalar path, partial last tile
    (3, 5, 16, 20, 1),    # S = 1600: vector path
    (2, 5, 8, 8, 0),      # z not read: every row lands in slice 0
]


@pytest.mark.parametrize("C", [1, 3, 8, 9, 64, 65, 130])
@pytest.mark.parametrize("geom", SCATTER_GEOMS, ids=lambda g: "B%dD%d_%dx%d_z%d" % g)
def test_scatter_dense(cuda, geom, C):
    """p3d_scatter_dense against the numpy canvas, bit for bit, on a NaN-poisoned output: duplicate cells (the later
    row wins), rows of three batches interleaved, out-of-range fields skipped, device counts None, 0, below and above
    capacity; a workspace one byte short is refused."""
    import torch
    L, check, ptr, stream = _lib()
    batch, D, ny, nx, use_z = geom
    rng = np.random.default_rng(C * 7 + D)
    cap = 400
    co = _coords(rng, cap, batch, D, ny, nx)
    feats = rng.normal(size=(cap, C)).astype(np.float32)
    feats[::17] = -0.0
    dco, dfe = _t(co, cuda), _t(feats, cuda)
    need = L.p3d_scatter_dense_workspace_bytes(batch, D, ny, nx)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    for num in (None, 0, 321, cap + 50):
        n = cap if num is None else min(num, cap)
        out = torch.full((batch, C, D, ny, nx), float("nan"), device=cuda)
        dnum = None if num is None else _num(num, cuda)  # every device argument stays referenced until the launch
        check(L.p3d_scatter_dense(ptr(dfe), ptr(dco), ptr(dnum), cap, C, batch, D, ny,
                                  nx, use_z, ptr(out), ptr(ws), need, stream(cuda)), "scatter_dense")
        want = lfo.scatter_dense(feats, co, n, batch, D, ny, nx, use_z)
        assert np.array_equal(_bits(out.cpu().numpy()), _bits(want)), "count %s" % num
    assert L.p3d_scatter_dense(ptr(dfe), ptr(dco), None, cap, C, batch, D, ny, nx, use_z, ptr(out), ptr(ws), need - 1,
                               stream(cuda)) == -2


def test_scatter_dense_partially_occupied_groups(cuda):
    """Every pattern of occupied cells in a group of four (the vector path's unit) on one row of the canvas."""
    import torch
    L, check, ptr, stream = _lib()
    nx = 64  # 16 groups of 4 cells: group g holds the occupancy pattern g
    cells = [4 * g + j for g in range(16) for j in range(4) if (g >> j) & 1]
    co = np.asarray([[0, 0, 0, x] for x in cells], np.int32)
    feats = np.random.default_rng(5).normal(size=(len(cells), 9)).astype(np.float32)
    need = L.p3d_scatter_dense_workspace_bytes(1, 1, 2, nx)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    out = torch.full((1, 9, 1, 2, nx), float("nan"), device=cuda)
    dfe, dco = _t(feats, cuda), _t(co, cuda)
    check(L.p3d_scatter_dense(ptr(dfe), ptr(dco), None, len(co), 9, 1, 1, 2, nx, 0, ptr(out), ptr(ws),
                              need, stream(cuda)), "scatter_dense")
    assert np.array_equal(_bits(out.cpu().numpy()), _bits(lfo.scatter_dense(feats, co, len(co), 1, 1, 2, nx, 0)))


# ================================================================================================= 4. rows -> pixel rows
def _to_h16(cuda, x, C):
    import torch
    L, check, ptr, stream = _lib()
    h = torch.empty((x.shape[0], 2 * C), dtype=torch.float16, device=cuda)
    check(L.p3d_rows_convert_h16(ptr(x), 1, None, x.shape[0], C, ptr(h), None, stream(cuda)), "rows_convert_h16")
    return h


@pytest.mark.parametrize("D", [1, 2, 5])
@pytest.mark.parametrize("C", [32, 64, 128, 256])
def test_sparse_rows_to_pixel_h16(cuda, C, D):
    """p3d_sparse_rows_to_pixel_h16: each row's (hi, lo') pairs at channel z C + c of its pixel, bit for bit; pixels
    without a row all-zero pairs (the output is poisoned first); out-of-range rows skipped; device counts None, 0, below
    and above capacity.  The image equals nchw_to_pixel_h16 of the scatter_dense canvas with its channels permuted from
    (c, z) to (z, c).  Sites are unique: the kernel copies without a row map, so duplicate sites have no defined
    winner and are not a valid input."""
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    L, check, ptr, stream = _lib()
    B, ny, nx = 2, 9, 14
    rng = np.random.default_rng(C + D)
    ok = min(300, B * D * ny * nx)
    sites = rng.choice(B * D * ny * nx, ok, replace=False)
    co = np.stack([sites // (D * ny * nx), sites // (ny * nx) % D, sites // nx % ny, sites % nx], 1).astype(np.int32)
    bad = np.asarray([[-1, 0, 0, 0], [B, 0, 0, 0], [0, -1, 0, 0], [0, D, 0, 0], [0, 0, -1, 0], [0, 0, ny, 0],
                      [0, 0, 0, -1], [0, 0, 0, nx]], np.int32)
    co = np.concatenate([co, bad])[rng.permutation(ok + len(bad))]
    cap = len(co)
    feats = rng.normal(size=(cap, C)).astype(np.float32) * 10
    dco, dfe = _t(co, cuda), _t(feats, cuda)
    rows = _to_h16(cuda, dfe, C)
    rows_u16 = rows.cpu().numpy().view(np.uint16)
    for num in (None, 0, cap // 2 + 3, cap + 7):
        n = cap if num is None else min(num, cap)
        out = torch.full((B * ny * nx, 2 * D * C), float("nan"), dtype=torch.float16, device=cuda)
        dnum = None if num is None else _num(num, cuda)
        check(L.p3d_sparse_rows_to_pixel_h16(ptr(rows), ptr(dco), ptr(dnum), cap, C, B,
                                             D, ny, nx, ptr(out), stream(cuda)), "rows_to_pixel_h16")
        got = out.cpu().numpy().view(np.uint16)
        assert np.array_equal(got, lfo.rows_to_pixel_h16(rows_u16, co, n, C, B, D, ny, nx)), "count %s" % num
    # against the dense route: scatter_dense canvas [B, C, D, ny, nx] -> (z, c) channel order -> nchw_to_pixel_h16
    need = L.p3d_scatter_dense_workspace_bytes(B, D, ny, nx)
    ws = torch.empty(need, dtype=torch.uint8, device=cuda)
    canvas = torch.empty((B, C, D, ny, nx), device=cuda)
    check(L.p3d_scatter_dense(ptr(dfe), ptr(dco), None, cap, C, B, D, ny, nx, 1, ptr(canvas), ptr(ws), need, stream(cuda)),
          "scatter_dense")
    dense = dc.nchw_to_pixel_h16(canvas.permute(0, 2, 1, 3, 4).reshape(B, D * C, ny, nx).contiguous())
    assert np.array_equal(dense.cpu().numpy().view(np.uint16), got)


# ================================================================================================= 5. few-channel conv
KSIZE = {1: ((1, 1, 1), True), 3: ((1, 3, 1), True), 7: ((1, 1, 7), True), 27: ((3, 3, 3), True),
         40: ((2, 4, 5), False)}  # K = 40 at Cin 8, Cout 32 is the 40 KB weight bound


def _small_cin_case(oracle_mod, K, cin, cout, seed):
    """Random sites (missing neighbours everywhere), the oracle's conv and the neighbour map of its output sites."""
    rng = np.random.default_rng(seed)
    spatial = (6, 20, 24)
    D, H, W = spatial
    sites = rng.choice(2 * D * H * W, 900, replace=False)
    co = np.stack([sites // (D * H * W), sites // (H * W) % D, sites // W % H, sites % W], 1).astype(np.int32)
    feats = rng.normal(size=(len(co), cin)).astype(np.float32)
    ksize, subm = KSIZE[K]
    w = (rng.normal(size=ksize + (cin, cout)) / np.sqrt(K * cin)).astype(np.float32)
    pad = tuple(k // 2 for k in ksize) if subm else (0, 0, 0)
    oc, of, _, _ = oracle_mod.sparse_conv3d(co, feats, 2, spatial, w, padding=pad, subm=subm)
    nbr = lfo.nbr_map(co, oc, spatial, ksize, padding=pad)
    assert (nbr < 0).any() or K == 1
    bn = (rng.uniform(0.5, 1.5, cout), rng.normal(size=cout) * 0.3, rng.normal(size=cout) * 0.1,
          rng.uniform(0.5, 1.5, cout), 1e-3)
    return feats, w.reshape(K, cin, cout), of, nbr, bn


def _fold(bn):
    g, b, mu, var, eps = bn
    s = g / np.sqrt(var + eps)
    return s.astype(np.float32), (b - mu * s).astype(np.float32)


@pytest.mark.parametrize("K", [1, 3, 7, 27, 40])
@pytest.mark.parametrize("cin,cout", [(1, 16), (4, 16), (5, 16), (8, 16), (1, 32), (4, 32), (5, 32), (8, 32)])
def test_small_cin_conv(cuda, oracle_mod, cin, cout, K):
    """The few-channel kernel through p3d_sparse_conv_small_cin_h16 (out_f32 only, out_h16 only, both in one launch)
    and p3d_sparse_conv_gather_gemm FP32 (with a residual, scale / shift and ReLU, and bare): oracle.sparse_conv3d +
    bn_relu at rel_check 1e-4; out_h16 bit-equal to p3d_rows_convert_h16 of out_f32; rows beyond the device count
    untouched; a count above capacity computes every row."""
    import torch
    L, check, ptr, stream = _lib()
    feats, w, of, nbr, bn = _small_cin_case(oracle_mod, K, cin, cout, seed=K * 100 + cin * 10 + cout)
    n_out = len(nbr)
    n = n_out - 37  # not a multiple of the 128-row block
    s, t = _fold(bn)
    din, dnbr, dw, ds, dt = [_t(a, cuda) for a in (feats, nbr, w, s, t)]
    status = torch.zeros(1, dtype=torch.int32, device=cuda)
    tag = "small_cin Cin%d Cout%d K%d" % (cin, cout, K)
    want = oracle_mod.bn_relu(of, *bn, relu=True)

    def run(num, f32, h16, relu=1, scale=ds, shift=dt):
        check(L.p3d_sparse_conv_small_cin_h16(ptr(din), ptr(dnbr), ptr(num), n_out, K, cin, cout, ptr(dw), ptr(scale),
                                              ptr(shift), relu, ptr(f32), ptr(h16), ptr(status), stream(cuda)),
              "small_cin_h16")

    f32_only = torch.full((n_out, cout), float("nan"), device=cuda)
    run(_num(n, cuda), f32_only, None)
    got = f32_only.cpu().numpy()
    assert np.isnan(got[n:]).all()
    rel_check(tag, got[:n], want[:n])
    both_f = torch.full((n_out, cout), float("nan"), device=cuda)
    both_h = torch.full((n_out, 2 * cout), float("nan"), dtype=torch.float16, device=cuda)
    h_only = torch.full((n_out, 2 * cout), float("nan"), dtype=torch.float16, device=cuda)
    run(_num(n_out + 3, cuda), both_f, both_h)
    run(_num(n, cuda), None, h_only)
    ref_h = _to_h16(cuda, both_f, cout)
    torch.cuda.synchronize()
    rel_check(tag + " all rows", both_f.cpu().numpy(), want)
    assert np.array_equal(both_h.cpu().numpy().view(np.uint16), ref_h.cpu().numpy().view(np.uint16))
    assert np.array_equal(h_only.cpu().numpy().view(np.uint16)[:n], ref_h.cpu().numpy().view(np.uint16)[:n])
    assert np.isnan(h_only.cpu().numpy()[n:].astype(np.float32)).all()
    assert int(status.item()) == 0
    # values beyond fp16's range saturate and set the status bit
    big = _t(s * 1e6, cuda)
    run(None, None, h_only, relu=0, scale=big)
    torch.cuda.synchronize()
    assert int(status.item()) & 1
    # p3d_sparse_conv_gather_gemm FP32 dispatches the same kernel; its residual branch is reachable only this way
    res = np.random.default_rng(K).normal(size=(n_out, cout)).astype(np.float32)
    for scale, shift, residual, relu in ((ds, dt, _t(res, cuda), 1), (None, None, _t(res, cuda), 0), (ds, dt, None, 0),
                                         (None, None, None, 1), (None, None, None, 0)):
        out = torch.full((n_out, cout), float("nan"), device=cuda)
        dnum = _num(n, cuda)
        check(L.p3d_sparse_conv_gather_gemm(ptr(din), ptr(dnbr), ptr(dnum), n_out, K, cin, cout, ptr(dw),
                                            ptr(scale), ptr(shift), ptr(residual), relu, 0, ptr(out), stream(cuda)),
              "gather_gemm fp32")
        g = bn if scale is not None else (np.ones(cout), np.zeros(cout), np.zeros(cout), np.ones(cout), 0.0)
        want2 = oracle_mod.bn_relu(of, *g, relu=bool(relu), residual=res if residual is not None else None)
        got2 = out.cpu().numpy()
        assert np.isnan(got2[n:]).all()
        rel_check(tag + " gather_gemm s%d r%d relu%d" % (scale is not None, residual is not None, relu), got2[:n],
                  want2[:n])


# ================================================================================================= 6. unfused epilogue
U = 2.0 ** -24


def _affine_bound(x, scale, shift, res):
    """|fp32 - fp64| of act(x s + t + r): at most three roundings, of x s, of (x s + t) and of the sum with r, each within
    2^-24 of its result (first order: 2^-24 (3 |x s| + 2 |t| + |r|)); an FMA for x s + t drops the first.  ReLU is
    exact."""
    xs = np.abs(x * (scale if scale is not None else 1.0))
    t = np.abs(shift) if shift is not None else 0.0
    r = np.abs(res) if res is not None else 0.0
    return U * (3 * xs + 2 * t + r) * (1 + 8 * U)


@pytest.mark.parametrize("relu", [0, 1])
@pytest.mark.parametrize("with_res", [False, True])
@pytest.mark.parametrize("with_shift", [False, True])
@pytest.mark.parametrize("with_scale", [False, True])
def test_sparse_affine_act(cuda, with_scale, with_shift, with_res, relu):
    """p3d_sparse_affine_act with scale, shift, residual and ReLU each present or null: within the rounding bound of
    the fp64 value; rows beyond the device count untouched."""
    import torch
    L, check, ptr, stream = _lib()
    rng = np.random.default_rng(with_scale * 8 + with_shift * 4 + with_res * 2 + relu)
    cap, C, n = 1000, 37, 901
    x = rng.normal(size=(cap, C)).astype(np.float32) * 3
    scale = rng.uniform(-2, 2, C).astype(np.float32) if with_scale else None
    shift = rng.normal(size=C).astype(np.float32) if with_shift else None
    res = rng.normal(size=(cap, C)).astype(np.float32) * 2 if with_res else None
    dev = lambda a: _t(a, cuda) if a is not None else None  # noqa: E731
    out = torch.full((cap, C), float("nan"), device=cuda)
    dx, dnum, dscale, dshift, dres = dev(x), _num(n, cuda), dev(scale), dev(shift), dev(res)
    check(L.p3d_sparse_affine_act(ptr(dx), ptr(dnum), cap, C, ptr(dscale), ptr(dshift), ptr(dres),
                                  relu, ptr(out), stream(cuda)), "sparse_affine_act")
    got = out.cpu().numpy()
    assert np.isnan(got[n:]).all()
    want = x.astype(np.float64)
    if scale is not None:
        want = want * scale
    if shift is not None:
        want = want + shift
    if res is not None:
        want = want + res
    if relu:
        want = np.maximum(want, 0.0)
    bound = _affine_bound(x[:n].astype(np.float64), scale, shift, None if res is None else res[:n].astype(np.float64))
    err = np.abs(got[:n] - want[:n])
    assert (err <= bound).all(), float((err - bound).max())
    if relu:
        assert (want[:n] == 0).any() and (got[:n] == 0).all(where=want[:n] <= 0)


def test_sparse_nn_routes_to_the_unfused_epilogue(cuda, oracle_mod):
    """The sparse_nn layers that cannot fold into a pending conv: BatchNorm after a ReLU, add of two materialised
    tensors, ReLU of a materialised tensor; against oracle.bn_relu."""
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(11)
    cap, C, n = 700, 24, 650
    sites = rng.choice(2 * 8 * 30 * 30, cap, replace=False)
    co = np.stack([sites // 7200, sites // 900 % 8, sites // 30 % 30, sites % 30], 1).astype(np.int32)
    xv = rng.normal(size=(cap, C)).astype(np.float32)
    yv = rng.normal(size=(cap, C)).astype(np.float32)
    x = sp.sparse_coo_tensor(_t(co, cuda), _t(xv, cuda), [2, 8, 30, 30, C], num=_num(n, cuda))
    y = sp.SparseCooTensor(x.index, values=_t(yv, cuda))
    ident = (np.ones(C), np.zeros(C), np.zeros(C), np.ones(C), 0.0)
    r = sp.ReLU()(x)
    rel_check("affine relu", r.values().cpu().numpy()[:n], oracle_mod.bn_relu(xv, *ident, relu=True)[:n])
    bn = sp.BatchNorm(C, epsilon=1e-3).init_parameters(rng, cuda, randomize=True)
    z = bn(r)
    par = [bn.weight, bn.bias, bn._mean, bn._variance]
    g, b, mu, var = [p.cpu().numpy().astype(np.float64) for p in par]
    want = oracle_mod.bn_relu(np.maximum(xv, 0), g, b, mu, var, 1e-3, relu=False)
    rel_check("affine bn after relu", z.values().cpu().numpy()[:n], want[:n])
    a = sp.add(x, y)
    rel_check("affine add", a.values().cpu().numpy()[:n], oracle_mod.bn_relu(xv, *ident, relu=False, residual=yv)[:n])
