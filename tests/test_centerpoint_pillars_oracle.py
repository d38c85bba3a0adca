"""CPU suite for CenterPoint-pillars: the fp64 restatement of the two-layer PillarFeatureNet against an independent torch
restatement of PFNLayer / PillarFeatureNet, the model's shapes and algorithmic flops, and the argument checks of
p3d_pillar_feature_net2 (no launch)."""
import numpy as np
import pytest

from paddle3d_b200 import synth


def _torch_pfn2(voxels, npv, coors, layers, voxel_size, pcr):
    """PillarFeatureNet.forward with two PFNLayers in torch fp64: decoration, mask, then per layer Linear (no bias) +
    BatchNorm1d (eval) + ReLU and the max over the points; the first layer's output is concat([x, x_max tiled])."""
    import torch
    v = torch.from_numpy(np.asarray(voxels, np.float64))
    n, m, _ = v.shape
    npv_t = torch.from_numpy(np.asarray(npv, np.int64))
    c = torch.from_numpy(np.asarray(coors, np.int64))
    points_mean = v[:, :, :3].sum(dim=1, keepdim=True) / npv_t.double().view(-1, 1, 1)
    f_cluster = v[:, :, :3] - points_mean
    f_center = torch.zeros_like(v[:, :, :2])
    vx, vy = float(voxel_size[0]), float(voxel_size[1])
    x_off, y_off = vx / 2 + float(pcr[0]), vy / 2 + float(pcr[1])
    f32 = lambda a: torch.tensor(a, dtype=torch.float32).double()  # noqa: E731  (the reference's fp32 centre terms)
    f_center[:, :, 0] = v[:, :, 0] - (c[:, 3].float().double().unsqueeze(1) * f32(vx) + f32(x_off))
    f_center[:, :, 1] = v[:, :, 1] - (c[:, 2].float().double().unsqueeze(1) * f32(vy) + f32(y_off))
    features = torch.cat([v, f_cluster, f_center], dim=-1)
    mask = (torch.arange(m).view(1, -1) < npv_t.view(-1, 1)).unsqueeze(-1).double()
    x = features * mask
    for li, l in enumerate(layers):
        lin = torch.nn.Linear(l["weight"].shape[0], l["weight"].shape[1], bias=False).double()
        bn = torch.nn.BatchNorm1d(l["weight"].shape[1], eps=l["eps"]).double().eval()
        with torch.no_grad():
            lin.weight.copy_(torch.from_numpy(np.asarray(l["weight"], np.float64).T))
            bn.weight.copy_(torch.from_numpy(np.asarray(l["gamma"], np.float64)))
            bn.bias.copy_(torch.from_numpy(np.asarray(l["beta"], np.float64)))
            bn.running_mean.copy_(torch.from_numpy(np.asarray(l["mean"], np.float64)))
            bn.running_var.copy_(torch.from_numpy(np.asarray(l["var"], np.float64)))
            y = torch.relu(bn(lin(x).permute(0, 2, 1)).permute(0, 2, 1))
        y_max = y.max(dim=1, keepdim=True)[0]
        x = y_max.squeeze(1) if li == len(layers) - 1 else torch.cat([y, y_max.repeat(1, m, 1)], dim=2)
    return x.numpy()


def _layers(rng, f, mid=32, out=64):
    ls = []
    for cin, c in ((f + 5, mid), (2 * mid, out)):
        ls.append(dict(weight=(rng.normal(size=(cin, c)) * 0.4).astype(np.float32),
                       gamma=rng.uniform(0.5, 1.5, c), beta=rng.normal(size=c) * 0.3,
                       mean=rng.normal(size=c) * 0.1, var=rng.uniform(0.5, 1.5, c), eps=1e-3))
    return ls


@pytest.mark.parametrize("f,m", [(5, 20), (4, 32)])
def test_pillar_feature_net2_oracle_vs_torch(f, m):
    """Pillars with 1, some and all M points; negative BN shifts make ReLU(BN(0)) of the padding rows the max of some
    channels in both layers, so the padding rows taking part in both maxima is checked."""
    from oracle.centerpoint_pillars import pillar_feature_net2
    rng = np.random.default_rng(11 + f)
    n = 40
    npv = np.concatenate([[1, m, m - 1, 2], rng.integers(1, m + 1, n - 4)]).astype(np.int32)
    vox = np.zeros((n, m, f), np.float32)
    for i in range(n):
        vox[i, :npv[i]] = np.concatenate([rng.normal(size=(npv[i], 3)) * [0.1, 0.1, 1.0] + [5, -3, 0],
                                          rng.uniform(size=(npv[i], f - 3))], 1)
    coors = np.stack([np.zeros(n), np.zeros(n), rng.integers(0, 512, n), rng.integers(0, 512, n)], 1).astype(np.int32)
    vs, pcr = [0.2, 0.2, 8.0], [-51.2, -51.2, -5.0, 51.2, 51.2, 3.0]
    layers = _layers(rng, f)
    got = pillar_feature_net2(vox, npv, coors, layers, vs, pcr)
    want = _torch_pfn2(vox, npv, coors, layers, vs, pcr)
    assert got.shape == (n, 64)
    np.testing.assert_allclose(got, want, rtol=1e-6, atol=1e-6 * np.abs(want).max())
    # the padding rows matter: without them (max over the real rows only) some pillars with count < M differ
    from oracle.centerpoint_pillars import _decorate, _linear_bn_relu
    x = _linear_bn_relu(_decorate(vox, npv, coors, vs, pcr), layers[0])
    real = np.arange(m)[None, :, None] < npv[:, None, None]
    x_max_real = np.where(real, x, -np.inf).max(1, keepdims=True)
    y = _linear_bn_relu(np.concatenate([x, np.repeat(x_max_real, m, 1)], -1), layers[1])
    no_pad = np.where(real, y, -np.inf).max(1)
    part = npv < m
    assert not np.allclose(no_pad[part], want[part], rtol=1e-4)


def test_model_shapes_and_flops():
    """Grid 512 x 512, feature maps 256 / 128 / 64, the 2x2 stride-2 conv / 1x1 conv / 2x2 deconv neck into 128 x 128 x
    384, 70 head planes, and the algorithmic flops of the dense part (2 x MACs, from the shapes)."""
    from paddle3d_b200.centerpoint_pillars import CONFIG, CenterPointPillars
    m = CenterPointPillars(synth.CP_PILLARS, CONFIG).init_weight(seed=0, device=None)
    assert m.grid == (512, 512)
    assert m.pfn_channels == (32, 64)
    assert [l["weight"].shape for l in m.pfn] == [(10, 32), (64, 64)]
    assert m.feat_hw == [(256, 256), (128, 128), (64, 64)]
    assert m.cat_hw == (128, 128) and m.head.fpn_channels == 384
    de = m.head.deblocks
    assert [(d.cin, d.cout, d.k, d.stride, d.up, d.transposed) for d in de] == [
        (64, 128, 2, 2, 1, False), (128, 128, 1, 1, 1, False), (256, 128, 2, 2, 2, True)]
    assert m.head_planes() == 70
    assert m.test_cfg["down_ratio"] == 4 and m.cat_hw[0] * 4 == m.grid[1]
    fl = {k: round(v / 1e9, 2) for k, v in m.flops().items()}
    assert fl == dict(backbone=72.48, fpn=2.68, head_shared=7.25, head_convmodules=43.49, head_output=1.32, head=52.06)
    assert round(sum(m.flops()[k] for k in ("backbone", "fpn", "head")) / 1e9, 1) == 127.2
    w = m.export_numpy()
    assert w["deblocks"][0]["stride"] == 2 and w["deblocks"][0]["up"] == 1 and w["deblocks"][0]["weight"].shape == (128, 64, 2, 2)


def test_cpu_dense_head_runs_the_strided_deblock():
    """CpuDenseHead runs the exported 2x2 stride-2 deblock through oracle.conv2d: a small trunk gives one concat size."""
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import DenseRPNHead
    net = DenseRPNHead(in_channels=64, out_channels=(64, 64, 64), layer_nums=(1, 1, 1), downsample_strides=(2, 2, 2),
                       fpn_out_channels=(32, 32, 32), upsample_strides=(0.5, 1, 2), tasks=(1, 2), share_conv_channel=32,
                       bev_depth=1).init_weight(seed=3, device=None)
    bev = np.random.default_rng(1).normal(size=(1, 64, 32, 32)).astype(np.float32)
    out = CpuDenseHead(net.export_numpy()).run(bev)
    assert out["hm"][0].shape == (1, 1, 8, 8) and out["hm"][1].shape == (1, 2, 8, 8)


def test_trunk_rejects_deblocks_of_different_sizes():
    from paddle3d_b200.dense_head import SecondTrunk
    t = SecondTrunk(64, (64, 128), (1, 1), (2, 2), (32, 32), (1, 1))
    sizes = [(16, 16), (8, 8)]
    assert {SecondTrunk.deblock_out_hw(d, *s) for d, s in zip(t.deblocks, sizes)} == {(16, 16), (8, 8)}


def test_pillar_feature_net2_abi_validation():
    """Argument checks of p3d_pillar_feature_net2 (they return before any launch)."""
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    L = _lib.lib()
    p = 16

    def call(**kw):
        a = dict(vox=p, npv=p, coors=p, num=None, n=10, M=20, F=5, mid=32, w1=p, s1=p, t1=p, out_c=64, w2=p, s2=p, t2=p,
                 vs=p, pcr=p, out=p)
        a.update(kw)
        return L.p3d_pillar_feature_net2(a["vox"], a["npv"], a["coors"], a["num"], a["n"], a["M"], a["F"], a["mid"],
                                         a["w1"], a["s1"], a["t1"], a["out_c"], a["w2"], a["s2"], a["t2"], a["vs"],
                                         a["pcr"], a["out"], None)
    for name in ("vox", "npv", "coors", "w1", "s1", "t1", "w2", "s2", "t2", "vs", "pcr", "out"):
        assert call(**{name: None}) == -1, name
    assert call(n=-1) == -1 and call(mid=0) == -1 and call(out_c=0) == -1
    assert call(M=65) == -4          # > 64 points per pillar
    assert call(M=0) == -4
    assert call(F=9) == -4           # > 8 values per point
    assert call(F=2) == -4
    assert call(mid=65) == -4        # first layer wider than the kernel's shared rows / registers
    assert call(n=0) == 0            # nothing to launch
