"""The CenterHead's fused path (DenseRPNHead.fused_heads): the batched ConvModule conv also runs the output convs'
tap-as-N GEMM on its staged fp16-pair tile (p3d_head_conv_p_f16) and p3d_head_tap_sum adds the taps.  Against the
layer-by-layer head and the CPU reference on small ragged images, bit-identical to the unfused path (conv image, then
p3d_head_out_conv_f16) on the full-size CenterPoint heads, and the fp16 overflow bit of the conv's pair split."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _unfused(net, s, shape, bp, dev):
    big = bp["big"]
    mid, _, _ = big(s, shape)
    return net._final_convs(mid, shape, big.cout, bp, bp["planes"], dev)


def test_fused_head_matches_per_head_and_cpu(cuda, oracle_mod):
    """Batch 2, image sides that are not multiples of the 8 x 16 conv tile or the 8 x 32 tap-sum tile, 1- and 2-class
    heat maps."""
    import torch
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import DenseRPNHead
    net = DenseRPNHead(in_channels=64, out_channels=(32, 64), layer_nums=(1, 1), downsample_strides=(1, 2),
                       fpn_out_channels=(64, 64), upsample_strides=(1, 2), tasks=(1, 2), share_conv_channel=64)
    net.init_weight(seed=12, device=cuda, randomize_bn=True)
    assert net.fused_heads(net._batched_params(cuda))
    bev = np.random.default_rng(9).normal(size=(2, 64, 26, 42)).astype(np.float32)
    got = net.forward(_t(cuda, bev))
    ref = net.forward_per_head(_t(cuda, bev))
    torch.cuda.synchronize()
    want = CpuDenseHead(net.export_numpy()).run(bev)
    for name in want:
        for g, r, w in zip(got[name], ref[name], want[name]):
            assert tuple(g.shape) == w.shape
            tol = 1e-4 * max(1.0, np.abs(w).max())
            assert np.abs(g.cpu().numpy() - w).max() <= tol, name
            assert np.abs(g.cpu().numpy() - r.cpu().numpy()).max() <= tol, name


def _bit_identical(net, bev, dev):
    import torch
    bp = net._batched_params(dev)
    assert net.fused_heads(bp)
    s, shape = net._trunk(bev)
    fused = net._tap_sum(net._heads_conv_p(s, shape, bp, dev), bp, dev)
    ref = _unfused(net, s, shape, bp, dev)
    torch.cuda.synchronize()
    assert fused.shape == ref.shape and torch.equal(fused, ref)


def test_fused_head_bit_identical_voxel_180(cuda):
    """The CenterPoint voxel head (6 tasks, 36 heads) at 180 x 180."""
    import torch
    from paddle3d_b200.dense_head import DenseRPNHead
    net = DenseRPNHead(256).init_weight(seed=1, device=cuda)
    g = torch.Generator(device=cuda).manual_seed(3)
    _bit_identical(net, torch.randn((1, 256, 180, 180), generator=g, device=cuda), cuda)


def test_fused_head_bit_identical_pillars_128(cuda):
    """The CenterPoint-pillars head at its 128 x 128 feature map."""
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillars
    m = CenterPointPillars()
    net = m.head.init_weight(seed=1, device=cuda)
    assert m.cat_hw == (128, 128)
    g = torch.Generator(device=cuda).manual_seed(4)
    _bit_identical(net, torch.randn((1, m.C, m.grid[1], m.grid[0]), generator=g, device=cuda), cuda)


def test_fused_head_overflow_bit(cuda):
    """A ConvModule output outside fp16's range raises status bit 0 in the fused conv as in the unfused one."""
    import torch
    from paddle3d_b200.dense_head import DenseRPNHead
    from paddle3d_b200.ops import dense_conv as dc
    net = DenseRPNHead(in_channels=64, out_channels=(32, 64), layer_nums=(1, 1), downsample_strides=(1, 2),
                       fpn_out_channels=(64, 64), upsample_strides=(1, 2), tasks=(1, 2), share_conv_channel=64)
    net.init_weight(seed=13, device=cuda)
    bp = net._batched_params(cuda)
    bev = _t(cuda, np.random.default_rng(2).normal(size=(1, 64, 20, 28)).astype(np.float32))
    s, shape = net._trunk(bev)
    status = dc._status(cuda)
    for overflow in (False, True):
        if overflow:
            bp["big"].dev["shift"][70] = 1e6  # channel 6 of the second head: ReLU(conv + 1e6) > 65504 everywhere
        for run in (lambda: net._tap_sum(net._heads_conv_p(s, shape, bp, cuda), bp, cuda),
                    lambda: _unfused(net, s, shape, bp, cuda)):
            torch.cuda.synchronize()
            status.zero_()
            run()
            torch.cuda.synchronize()
            assert int(status[0]) & 1 == int(overflow)
    status.zero_()
