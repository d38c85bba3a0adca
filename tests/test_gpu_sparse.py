"""GPU parity: sparse conv (rulebook + gather-GEMM) and SparseResNet3D through the C ABI vs the oracle.
Tolerance: 1e-4 relative (fp32), BASELINE.json north_star.  PARITY UNPINNED by the reference (the
arithmetic is PaddlePaddle's); the oracle restatement is itself checked against dense fp64 conv3d in
tests/test_oracle.py."""
import os

import numpy as np
import pytest

from paddle3d_b200 import synth
from parity import rel_check

pytestmark = pytest.mark.gpu

# 0 fp32 CUDA cores, 1 wgmma on fp32 rows, 2 wgmma on tf32 split rows, 4 wgmma on fp16-pair rows (default);
# 3 = the slower TMA-gather variant of 2, kept for the record (P3D_EXPERIMENTAL=1)
PRECISIONS = [0, 1, 2, 4] + ([3] if os.environ.get("P3D_EXPERIMENTAL") == "1" else [])


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _dense(coords, feats, B, sp):
    out = np.zeros((B,) + tuple(sp) + (feats.shape[1],), np.float32)
    out[coords[:, 0], coords[:, 1], coords[:, 2], coords[:, 3]] = feats
    return out


def _rand_sites(rng, B, D, H, W, p):
    occ = rng.random((B, D, H, W)) < p
    c = np.argwhere(occ).astype(np.int32)
    rng.shuffle(c, axis=0)
    return c


@pytest.mark.parametrize("precision", PRECISIONS)
@pytest.mark.parametrize("subm,ks,st,pd,cin,cout", [
    (True, 3, 1, 1, 5, 16), (True, 3, 1, 1, 16, 16), (True, 3, 1, 1, 64, 64), (True, 3, 1, 1, 128, 128),
    (False, 3, 2, 1, 16, 32), (False, 3, 2, [0, 1, 1], 64, 128), (False, (3, 1, 1), (2, 1, 1), 0, 128, 128),
    (True, 3, 1, 1, 7, 9),
])
def test_single_conv(cuda, oracle_mod, precision, subm, ks, st, pd, cin, cout):
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(cin * 131 + cout)
    B, D, H, W = 2, 11, 40, 37
    coords = _rand_sites(rng, B, D, H, W, 0.08)
    feats = rng.normal(size=(len(coords), cin)).astype(np.float32)
    cls = sp.SubmConv3D if subm else sp.Conv3D
    conv = cls(cin, cout, ks, st, padding=pd, bias_attr=True)
    conv.init_parameters(rng, cuda)
    conv.precision = precision
    bn = sp.BatchNorm(cout, epsilon=1e-3).init_parameters(rng, cuda, randomize=True)
    x = sp.sparse_coo_tensor(_t(cuda, coords).t(), _t(cuda, feats), [B, D, H, W, cin])
    y = sp.ReLU()(bn(conv(x)))
    vals = y.values()
    n = y.nnz()
    got = _dense(y.index.coords.cpu().numpy()[:n], vals.cpu().numpy()[:n], B, y.index.spatial)
    w = conv.weight.cpu().numpy()
    oc, of, osp, pairs = oracle_mod.sparse_conv3d(coords, feats, B, (D, H, W), w, conv.stride, conv.padding, subm)
    of = of + conv.bias.cpu().numpy()
    of = oracle_mod.bn_relu(of, bn.weight.cpu().numpy(), bn.bias.cpu().numpy(), bn._mean.cpu().numpy(),
                            bn._variance.cpu().numpy(), 1e-3, relu=True)
    assert n == len(oc) and osp == y.index.spatial
    want = _dense(oc, of, B, osp)
    rel_check('single_conv p%d %s %d->%d' % (precision, 'subm' if subm else 'conv', cin, cout), got, want)
    if not subm:
        assert int(y.index.counters[1].item()) == 0  # no overflow
    # to_dense_bev == reference to_dense + transpose + reshape
    bev = y.to_dense_bev().cpu().numpy()
    want_bev = np.transpose(want, (0, 4, 1, 2, 3)).reshape(B, cout * osp[0], osp[1], osp[2])
    rel_check('single_conv bev', bev, want_bev)


@pytest.mark.parametrize("wm", [True, False])
@pytest.mark.parametrize("subm,ks,st,pd,cin,cout,residual", [
    (True, 3, 1, 1, 16, 16, True), (True, 3, 1, 1, 32, 32, True), (True, 3, 1, 1, 32, 32, False),
    (False, 3, 2, 1, 16, 32, False), (True, (3, 1, 1), 1, (1, 0, 0), 16, 16, False),
])
def test_narrow_layers_on_both_kernels(cuda, oracle_mod, wm, subm, ks, st, pd, cin, cout, residual):
    """The 16/32-channel layers of the fp16-pair path: register-gather warp-MMA kernel (csrc/sparse_conv_wm.cu, default)
    and the wgmma kernel (P3D_SPARSE_WM=0) against the oracle - conv + BN (+ residual) + ReLU, fp32 and H16 outputs,
    a row count that is not a multiple of 16."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(cin * 17 + cout + (5 if residual else 0))
    B, D, H, W = 2, 9, 33, 41
    coords = _rand_sites(rng, B, D, H, W, 0.11)
    if len(coords) % 16 == 0:
        coords = coords[:-3]
    feats = rng.normal(size=(len(coords), cin)).astype(np.float32)
    cls = sp.SubmConv3D if subm else sp.Conv3D
    conv = cls(cin, cout, ks, st, padding=pd, bias_attr=True).init_parameters(rng, cuda)
    conv.precision = sp.F16X3
    bn = sp.BatchNorm(cout, epsilon=1e-3).init_parameters(rng, cuda, randomize=True)
    x = sp.sparse_coo_tensor(_t(cuda, coords).t(), _t(cuda, feats), [B, D, H, W, cin])
    old = sp.NARROW_WM[0]
    sp.NARROW_WM[0] = wm
    def lazy():
        y = bn(conv(x))
        assert y._pending.wm == wm
        if residual:
            y = sp.add(y, x)
        return sp.ReLU()(y)

    try:
        y = lazy()
        vals = y.values()                      # the kernel writes fp32 rows
        vals16 = lazy().get(sp.ROWS_H16)       # the kernel writes the pair rows itself
    finally:
        sp.NARROW_WM[0] = old
    n = y.nnz()
    w = conv.weight.cpu().numpy()
    oc, of, osp, _ = oracle_mod.sparse_conv3d(coords, feats, B, (D, H, W), w, conv.stride, conv.padding, subm)
    of = oracle_mod.bn_relu(of + conv.bias.cpu().numpy(), bn.weight.cpu().numpy(), bn.bias.cpu().numpy(),
                            bn._mean.cpu().numpy(), bn._variance.cpu().numpy(), 1e-3, relu=True,
                            residual=feats if residual else None)
    assert n == len(oc)
    want = _dense(oc, of, B, osp)
    got = _dense(y.index.coords.cpu().numpy()[:n], vals.cpu().numpy()[:n], B, y.index.spatial)
    rel_check('narrow %s wm=%d %d->%d' % ('subm' if subm else 'conv', wm, cin, cout), got, want)
    if vals16 is not None:  # the pair rows the next layer would consume, converted back by the library
        back = torch.empty((y.index.cap, cout), dtype=torch.float32, device=cuda)
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        check(lib().p3d_rows_convert_h16(ptr(vals16), 0, ptr(y.index.num), y.index.cap, cout, ptr(back), None, stream(cuda)),
              "rows_convert_h16")
        got16 = _dense(y.index.coords.cpu().numpy()[:n], back.cpu().numpy()[:n], B, y.index.spatial)
        rel_check('narrow h16 rows wm=%d %d->%d' % (wm, cin, cout), got16, want)


def test_strided_overflow_is_flagged(cuda):
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(0)
    coords = _rand_sites(rng, 1, 9, 30, 30, 0.2)
    x = sp.sparse_coo_tensor(_t(cuda, coords).t(), _t(cuda, rng.normal(size=(len(coords), 16)).astype(np.float32)), [1, 9, 30, 30, 16])
    conv = sp.Conv3D(16, 16, 3, 2, padding=1, bias_attr=False).init_parameters(rng, cuda)
    conv.out_cap = 50
    y = conv(x)
    y.values()
    c = y.index.counters.cpu().numpy()
    assert c[0] == 50 and c[1] == 1 and c[2] > 50 and c[2] <= 2048


def _oracle_resnet(oracle_mod, net, coords, feats, B):
    """SparseResNet3D.forward (sparse_resnet.py:185-206) composed from oracle pieces."""
    def conv(l, c, f, sp, subm):
        w = l.weight.cpu().numpy()
        oc, of, osp, pairs = oracle_mod.sparse_conv3d(c, f, B, sp, w, l.stride, l.padding, subm)
        if l.bias is not None:
            of = of + l.bias.cpu().numpy()
        return oc, of, osp, pairs

    def bn(l, f, relu, residual=None):
        return oracle_mod.bn_relu(f, l.weight.cpu().numpy(), l.bias.cpu().numpy(), l._mean.cpu().numpy(),
                                  l._variance.cpu().numpy(), l.epsilon, relu=relu, residual=residual)

    def block(b, c, f, sp):
        _, o, _, p1 = conv(b.conv1, c, f, sp, True)
        o = bn(b.bn1, o, True)
        _, o, _, p2 = conv(b.conv2, c, o, sp, True)
        return bn(b.bn2, o, True, residual=f), p1 + p2

    sp_ = net.sparse_shape
    pairs = []
    c, f, _, p = conv(net.conv_input[0], coords, feats, sp_, True)
    pairs.append(p)
    f = bn(net.conv_input[1], f, True)
    for b in net.blocks0:
        f, p = block(b, c, f, sp_)
        pairs.append(p)
    for down, blocks in net.stages:
        c, f, sp_, p = conv(down[0], c, f, sp_, False)
        pairs.append(p)
        f = bn(down[1], f, True)
        for b in blocks:
            f, p = block(b, c, f, sp_)
            pairs.append(p)
    c, f, sp_, p = conv(net.extra_conv[0], c, f, sp_, False)
    pairs.append(p)
    f = bn(net.extra_conv[1], f, True)
    return oracle_mod.sparse_to_dense_bev(c, f, B, sp_), pairs


@pytest.mark.parametrize("precision", PRECISIONS)
def test_sparse_resnet3d_small(cuda, oracle_mod, precision):
    """Whole 21-conv backbone on a reduced grid (41 x 176 x 176 -> 2 x 22 x 22), lidar-like occupancy."""
    from paddle3d_b200.layers import SparseResNet3D
    cfg = dict(synth.C3, point_cloud_range=[-6.6, -6.6, -5.0, 6.6, 6.6, 3.0])
    pts = synth.lidar_cloud(dict(cfg, point_cloud_range=[-20, -20, -5, 20, 20, 3]), 5, num_points=40000)
    v, c, n, nv = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], 10, 20000)
    k = int(nv[0])
    assert k > 3000
    feats = oracle_mod.voxel_mean(v, n, k)
    coors = np.concatenate([np.zeros((k, 1), np.int32), c[:k]], 1)
    net = SparseResNet3D(5, cfg["voxel_size"], cfg["point_cloud_range"]).init_weight(seed=3, device=cuda, randomize_bn=True)
    net.set_precision(precision)
    assert net.sparse_shape == [41, 176, 176]
    got = net(_t(cuda, feats), _t(cuda, coors), 1).cpu().numpy()
    want, pairs = _oracle_resnet(oracle_mod, net, coors, feats, 1)
    assert got.shape == want.shape == (1, 256, 22, 22)
    rel_check('sparse_resnet3d_small p%d' % precision, got, want)
    assert (want != 0).mean() > 0.05


@pytest.mark.parametrize("precision", PRECISIONS)
def test_sparsenet3d_small(cuda, oracle_mod, precision):
    """SparseNet3D (sparsenet.py:67-182): dense BEV output and the multi-scale sparse tensors vs the oracle."""
    from paddle3d_b200.layers import SparseNet3D
    cfg = dict(synth.C3, point_cloud_range=[-6.6, -6.6, -5.0, 6.6, 6.6, 3.0])
    pts = synth.lidar_cloud(dict(cfg, point_cloud_range=[-20, -20, -5, 20, 20, 3]), 8, num_points=30000)
    v, c, n, nv = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], 10, 20000)
    k = int(nv[0])
    feats = oracle_mod.voxel_mean(v, n, k)
    coors = np.concatenate([np.zeros((k, 1), np.int32), c[:k]], 1)
    net = SparseNet3D(5, cfg["voxel_size"], cfg["point_cloud_range"]).init_weight(seed=5, device=cuda, randomize_bn=True)
    net.set_precision(precision)
    got = net(_t(cuda, feats), _t(cuda, coors), 1)
    cc, ff, sp_ = coors, feats, net.sparse_shape
    scales = []
    for i, seq in enumerate(net.sequences()):
        conv, bn = seq[0], seq[1]
        cc, ff, sp_, _ = oracle_mod.sparse_conv3d(cc, ff, 1, sp_, conv.weight.cpu().numpy(), conv.stride, conv.padding, conv.subm)
        ff = oracle_mod.bn_relu(ff, bn.weight.cpu().numpy(), bn.bias.cpu().numpy(), bn._mean.cpu().numpy(),
                                bn._variance.cpu().numpy(), bn.epsilon)
        if i in (1, 4, 7, 10):
            scales.append((cc, ff, sp_))
    want = oracle_mod.sparse_to_dense_bev(cc, ff, 1, sp_)
    out = got["spatial_features"].cpu().numpy()
    assert out.shape == want.shape == (1, 256, 22, 22)
    # legacy tf32 paths (1, 2): errors compound over the stacked layers a little above 1e-4 on the multi-scale tensors
    rtol = 1e-4 if precision in (0, 4) else 2e-4
    rel_check('sparsenet3d_small p%d bev' % precision, out, want, rtol=rtol)
    for name, (wc, wf, wsp) in zip(["x_conv1", "x_conv2", "x_conv3", "x_conv4"], scales):
        t = got["multi_scale_3d_features"][name]
        m = t.nnz()
        assert m == len(wc) and t.index.spatial == wsp
        gd = _dense(t.index.coords.cpu().numpy()[:m], t.values().cpu().numpy()[:m], 1, wsp)
        wd = _dense(wc, wf, 1, wsp)
        rel_check('sparsenet3d_small p%d %s' % (precision, name), gd, wd, rtol=rtol)


def test_hard_voxelizer_batch2(cuda, oracle_mod):
    import torch
    from paddle3d_b200.layers import HardVoxelizer
    cfg = synth.C2
    a, b = synth.lidar_cloud(cfg, 1, num_points=5000), synth.uniform_cloud(cfg, 2, num_points=3000)
    vx = HardVoxelizer(cfg["voxel_size"], cfg["point_cloud_range"], 8, [4000, 4000])
    v, c, n = vx([_t(cuda, a), _t(cuda, b)]).trim()
    wa = oracle_mod.hard_voxelize(a, cfg["voxel_size"], cfg["point_cloud_range"], 8, 4000)
    wb = oracle_mod.hard_voxelize(b, cfg["voxel_size"], cfg["point_cloud_range"], 8, 4000)
    ka, kb = int(wa[3][0]), int(wb[3][0])
    assert v.shape[0] == ka + kb
    assert np.array_equal(v.cpu().numpy(), np.concatenate([wa[0][:ka], wb[0][:kb]]))
    cw = np.concatenate([np.concatenate([np.zeros((ka, 1), np.int32), wa[1][:ka]], 1),
                         np.concatenate([np.ones((kb, 1), np.int32), wb[1][:kb]], 1)])
    assert np.array_equal(c.cpu().numpy(), cw)
    assert np.array_equal(n.cpu().numpy(), np.concatenate([wa[2][:ka], wb[2][:kb]]))


def test_workspace_and_table_rulebook_apis_agree(cuda):
    """The scratch-workspace rulebook entry point (p3d_sparse_rulebook_subm) and the caller-owned-table one
    (p3d_sparse_table_build + p3d_sparse_rulebook_subm_t) must produce the same neighbour map."""
    import torch
    from paddle3d_b200._lib import check, host_ints, lib
    from paddle3d_b200._mem import ptr, stream
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(4)
    coords = _rand_sites(rng, 2, 9, 33, 31, 0.1)
    n = len(coords)
    x = sp.sparse_coo_tensor(_t(cuda, coords).t(), _t(cuda, rng.normal(size=(n, 16)).astype(np.float32)), [2, 9, 33, 31, 16])
    a = x.index.subm_rulebook([3, 3, 3], "k")
    L = lib()
    ws = torch.empty((L.p3d_sparse_rulebook_workspace_bytes(n, 0),), dtype=torch.uint8, device=cuda)
    b = torch.empty((n, 27), dtype=torch.int32, device=cuda)
    check(L.p3d_sparse_rulebook_subm(ptr(x.index.coords), None, n, 2, host_ints([9, 33, 31]), host_ints([3, 3, 3]), ptr(b),
                                     ptr(ws), ws.numel(), stream(cuda)), "rulebook_subm")
    assert torch.equal(a, b)
    # every entry points at the row whose coordinate is coord + offset
    nb = a.cpu().numpy()
    k = 0
    for dz in (-1, 0, 1):
        for dy in (-1, 0, 1):
            for dx in (-1, 0, 1):
                rows = np.nonzero(nb[:, k] >= 0)[0]
                assert np.array_equal(coords[nb[rows, k]], coords[rows] + np.array([0, dz, dy, dx], np.int32))
                k += 1


def test_level_rulebook_matches_separate_calls(cuda):
    """p3d_sparse_rulebook_level_t (strided map + the new level's SubM map in one launch, warp-aggregated site numbering)
    against p3d_sparse_rulebook_subm_t on the output index set, and the overflow counters of a too-small capacity."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(8)
    coords = _rand_sites(rng, 2, 11, 40, 37, 0.15)
    n = len(coords)
    x = sp.sparse_coo_tensor(_t(cuda, coords).t(), _t(cuda, rng.normal(size=(n, 16)).astype(np.float32)), [2, 11, 40, 37, 16])
    conv = sp.Conv3D(16, 32, 3, 2, padding=1, bias_attr=False).init_parameters(rng, cuda)
    conv.fuse_subm = ((3, 3, 3), "lvl")
    index, nbr = conv.build_index(x.index)
    fused = index.subm_rulebooks[("lvl", (3, 3, 3))]
    separate = index.subm_rulebook([3, 3, 3], "other")
    torch.cuda.synchronize()
    m = int(index.num.cpu().numpy()[0])
    assert m > 0 and torch.equal(fused[:m], separate[:m])
    oc = index.coords.cpu().numpy()[:m]
    assert len({tuple(r) for r in oc}) == m  # every site numbered once
    # strided map: input row at out * 2 - 1 + k
    nb = nbr.cpu().numpy()[:m]
    k = 0
    for dz in range(3):
        for dy in range(3):
            for dx in range(3):
                rows = np.nonzero(nb[:, k] >= 0)[0]
                want = oc[rows] * np.array([1, 2, 2, 2], np.int32) + np.array([0, dz - 1, dy - 1, dx - 1], np.int32)
                assert np.array_equal(coords[nb[rows, k]], want)
                k += 1
    assert (nb >= 0).sum() == sum(1 for c in coords for dz in range(3) for dy in range(3) for dx in range(3)
                                  if (c[1] + 1 - dz) % 2 == 0 and (c[2] + 1 - dy) % 2 == 0 and (c[3] + 1 - dx) % 2 == 0
                                  and 0 <= (c[1] + 1 - dz) // 2 < 6 and 0 <= (c[2] + 1 - dy) // 2 < 20
                                  and 0 <= (c[3] + 1 - dx) // 2 < 19)


def test_h16_rows_roundtrip_and_range_flag(cuda):
    """fp32 rows -> fp16 (hi, lo' = (x - hi) * 2^11) pair rows -> fp32: error <= 2^-22 |x| inside fp16's range; a value
    outside it saturates and raises bit 0 of the status word (never a silent inf)."""
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    rng = np.random.default_rng(0)
    for C in (16, 32, 128):
        x = (rng.normal(size=(1000, C)) * np.exp(rng.uniform(-8, 8, size=(1000, C)))).astype(np.float32)
        x[0, :4] = [0.0, -0.0, 65504.0, -1e-7]
        tx = _t(cuda, x)
        h = torch.empty((1000, 2 * C), dtype=torch.float16, device=cuda)
        back = torch.empty_like(tx)
        status = torch.zeros((1,), dtype=torch.int32, device=cuda)
        L = lib()
        check(L.p3d_rows_convert_h16(ptr(tx), 1, None, 1000, C, ptr(h), ptr(status), stream(cuda)), "to_h16")
        check(L.p3d_rows_convert_h16(ptr(h), 0, None, 1000, C, ptr(back), None, stream(cuda)), "from_h16")
        err = np.abs(back.cpu().numpy().astype(np.float64) - x)
        assert (err <= np.abs(x) * 2.0 ** -21 + 2.0 ** -34).all()
        assert int(status[0]) == 0
        # layout: groups of KC = min(C, 32) channels, [hi KC | lo KC]
        KC = min(C, 32)
        hh = h.cpu().numpy().reshape(1000, C // KC, 2, KC)
        assert np.array_equal(hh[:, :, 0, :].reshape(1000, C), x.astype(np.float16))
        tx[5, 3] = 1e6
        check(L.p3d_rows_convert_h16(ptr(tx), 1, None, 1000, C, ptr(h), ptr(status), stream(cuda)), "to_h16")
        assert int(status[0]) == 1


def test_lazy_fusion_does_not_mutate_its_input(cuda, oracle_mod):
    """conv -> bn -> add -> relu fold into one launch WITHOUT editing the tensors they were given (ADVICE r1): a consumer
    that kept the conv output still reads the plain convolution."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(11)
    B, D, H, W = 1, 7, 20, 21
    coords = _rand_sites(rng, B, D, H, W, 0.15)
    feats = rng.normal(size=(len(coords), 16)).astype(np.float32)
    conv = sp.SubmConv3D(16, 16, 3, padding=1, bias_attr=False).init_parameters(rng, cuda)
    conv.precision = sp.F16X3
    bn = sp.BatchNorm(16, epsilon=1e-3).init_parameters(rng, cuda, randomize=True)
    x = sp.sparse_coo_tensor(_t(cuda, coords).t(), _t(cuda, feats), [B, D, H, W, 16])
    c = conv(x)
    y = sp.ReLU()(sp.add(bn(c), x))
    assert y is not c and c._pending is not None and c._pending.scale is None and not c._pending.relu and c._pending.residual is None
    n = y.nnz()
    plain = c.values().cpu().numpy()[:n]      # the un-fused convolution
    fused = y.values().cpu().numpy()[:n]
    _, of, _, _ = oracle_mod.sparse_conv3d(coords, feats, B, (D, H, W), conv.weight.cpu().numpy(), conv.stride, conv.padding, True)
    rel_check('unfused conv kept by an earlier consumer', plain, of)
    want = oracle_mod.bn_relu(of, bn.weight.cpu().numpy(), bn.bias.cpu().numpy(), bn._mean.cpu().numpy(),
                              bn._variance.cpu().numpy(), 1e-3, relu=True, residual=feats)
    rel_check('fused conv + bn + add + relu', fused, want)
    assert plain.min() < 0 <= fused.min()
