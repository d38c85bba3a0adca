"""GPU parity of the dense 2-D conv path (RPN / neck / CenterHead, SURVEY §8f-1) against the oracle's fp64-accumulating
conv2d / deconv2d (PARITY UNPINNED by the reference: the arithmetic is paddle.nn.Conv2D / Conv2DTranspose; the oracle
is checked against torch's fp64 CPU convs in tests/test_oracle.py).  Tolerance 1e-4 relative (BASELINE.json), true
relative on the elements above 1e-2 x max (tests/parity.py).  Both kernel families: fp16-pair (default) and tf32-pair."""
import numpy as np
import pytest

from parity import rel_check

pytestmark = pytest.mark.gpu


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _merge(split, b, h, w, c):
    """pixel split rows [B*H*W, 2C] -> fp32 NCHW (hi + lo)."""
    s = split.cpu().numpy().reshape(b, h, w, 2, c)
    return (s[:, :, :, 0, :] + s[:, :, :, 1, :]).transpose(0, 3, 1, 2)


def test_nchw_to_pixel_split(cuda):
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(0)
    x = rng.normal(size=(2, 37, 9, 13)).astype(np.float32)
    s = dc.nchw_to_pixel_split(_t(cuda, x)).cpu().numpy().reshape(2, 9, 13, 2, 37)
    hi, lo = s[..., 0, :], s[..., 1, :]
    assert np.array_equal((hi.view(np.uint32) & 0x1fff), np.zeros_like(hi, np.uint32))  # tf32: 13 low bits clear
    np.testing.assert_allclose((hi + lo).transpose(0, 3, 1, 2), x, rtol=3e-7, atol=0)


@pytest.mark.parametrize("cin,cout,k,stride,pad,up,h,w", [
    (32, 64, 3, 1, 1, 1, 20, 23),     # 3x3, ragged tiles on both axes
    (64, 128, 3, 2, 1, 1, 21, 34),    # stride 2 (tensor-map element stride), odd input height
    (128, 256, 1, 1, 0, 1, 16, 16),   # 1x1, two N tiles of 128
    (64, 64, 2, 2, 0, 2, 9, 11),      # transposed conv k = s = 2
    (64, 3, 3, 1, 1, 1, 17, 19),      # head output: N tile 16, fp32 NCHW planes
    (512, 64, 3, 1, 1, 1, 12, 18),    # the shared conv's channel count (16 uses per tap)
])
def test_dense_conv_vs_oracle(cuda, oracle_mod, cin, cout, k, stride, pad, up, h, w):
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(cin + cout)
    x = rng.normal(size=(2, cin, h, w)).astype(np.float32)
    wshape = (cin, cout, k, k) if up > 1 else (cout, cin, k, k)
    wt = (rng.normal(size=wshape) / np.sqrt(cin * k * k)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    shift = rng.normal(size=cout).astype(np.float32)
    ref = (oracle_mod.deconv2d(x, wt, None, up) if up > 1 else oracle_mod.conv2d(x, wt, None, stride, pad)).astype(np.float64)
    ref = np.maximum(ref * scale.reshape(1, -1, 1, 1) + shift.reshape(1, -1, 1, 1), 0.0)
    nt = dc.n_tile_for(cout)
    packed = (dc.pack_deconv_weight if up > 1 else dc.pack_conv_weight)(_t(cuda, wt), nt)
    xs = dc.nchw_to_pixel_split(_t(cuda, x))
    want_nchw = cout % 16 != 0
    o_split, o_nchw, (b, oh, ow) = dc.dense_conv2d(xs, (2, h, w, cin), packed, cout, nt, k, stride, pad, up, _t(cuda, scale),
                                                   _t(cuda, shift), True, want_nchw=want_nchw)
    torch.cuda.synchronize()
    got = o_nchw.cpu().numpy() if want_nchw else _merge(o_split, b, oh, ow, cout)
    assert got.shape == ref.shape
    assert np.abs(got - ref).max() <= 1e-4 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("mode,m_tiles", [(0, 1), (0, 2), (1, 1), (1, 2)])
@pytest.mark.parametrize("cin,cout,k,stride,pad,up,h,w", [
    (32, 64, 3, 1, 1, 1, 20, 23),     # 3x3: haloed-tile mode (mode 0) or one box per tap (mode 1); ragged tiles
    (64, 128, 3, 2, 1, 1, 21, 34),    # stride 2 (tensor-map element stride), odd input height
    (128, 256, 1, 1, 0, 1, 16, 16),   # 1x1, two N tiles of 128
    (64, 64, 2, 2, 0, 2, 9, 11),      # transposed conv k = s = 2
    (512, 64, 3, 1, 1, 1, 12, 18),    # the shared conv's channel count
    (64, 320, 3, 1, 1, 1, 37, 19),    # batched heads: three N tiles, the last one half used; two M tiles over 37 rows
    (32, 208, 3, 1, 1, 1, 50, 61),    # last N tile partly used, many pixel tiles per N tile
    (64, 2304, 3, 1, 1, 1, 24, 16),   # the CenterHead's batched ConvModules: 18 N tiles of 128
])
def test_dense_conv_f16_vs_oracle(cuda, oracle_mod, cin, cout, k, stride, pad, up, h, w, mode, m_tiles):
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(cin + cout)
    x = rng.normal(size=(2, cin, h, w)).astype(np.float32)
    wshape = (cin, cout, k, k) if up > 1 else (cout, cin, k, k)
    wt = (rng.normal(size=wshape) / np.sqrt(cin * k * k)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    shift = rng.normal(size=cout).astype(np.float32)
    ref = (oracle_mod.deconv2d(x, wt, None, up) if up > 1 else oracle_mod.conv2d(x, wt, None, stride, pad)).astype(np.float64)
    ref = np.maximum(ref * scale.reshape(1, -1, 1, 1) + shift.reshape(1, -1, 1, 1), 0.0)
    nt = dc.n_tile_for_f16(cout)
    packed = (dc.pack_deconv_weight_f16 if up > 1 else dc.pack_conv_weight_f16)(_t(cuda, wt), nt)
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    np.testing.assert_allclose(dc.pixel_h16_to_nchw(xs, (2, h, w, cin)).cpu().numpy(), x, rtol=2.0 ** -21, atol=2.0 ** -34)
    oc = ((cout + 31) // 32) * 32
    o_h16, _, (b, oh, ow) = dc.dense_conv2d_f16(xs, (2, h, w, cin), packed, cout, nt, k, stride, pad, up, _t(cuda, scale),
                                               _t(cuda, shift), True, out_channels=oc, mode=mode, m_tiles=m_tiles)
    _, o_nchw, _ = dc.dense_conv2d_f16(xs, (2, h, w, cin), packed, cout, nt, k, stride, pad, up, _t(cuda, scale),
                                       _t(cuda, shift), True, want_nchw=True, mode=mode, m_tiles=m_tiles)
    torch.cuda.synchronize()
    got = dc.pixel_h16_to_nchw(o_h16, (b, oh, ow, oc)).cpu().numpy()[:, :cout]
    assert got.shape == ref.shape
    # 512 x 9 = 4608-term sums of random signs: the fp32 accumulation noise alone (sqrt(K) x 2^-24 of the term magnitudes)
    # exceeds 1e-4 of results below ~5 % of the maximum, for any fp32 implementation
    floor = 1e-2 if cin * k * k <= 2304 else 5e-2
    rel_check("dense f16 %d->%d k%d s%d up%d mode%d mt%d" % (cin, cout, k, stride, up, mode, m_tiles), got, ref, floor=floor,
              small_atol=2e-6 if floor == 1e-2 else 1e-5)
    rel_check("dense f16 nchw", o_nchw.cpu().numpy(), ref, floor=floor, small_atol=2e-6 if floor == 1e-2 else 1e-5)


def test_concat_offset_and_small_head(cuda, oracle_mod):
    import torch
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import DenseRPNHead
    want = None
    for f16 in (True, False):
        net = DenseRPNHead(in_channels=64, out_channels=(32, 64), layer_nums=(1, 2), downsample_strides=(1, 2),
                           fpn_out_channels=(64, 64), upsample_strides=(1, 2), tasks=(1, 2), share_conv_channel=64, f16=f16)
        net.init_weight(seed=2, device=cuda, randomize_bn=True)
        rng = np.random.default_rng(1)
        bev = rng.normal(size=(1, 64, 40, 36)).astype(np.float32)
        got = net(_t(cuda, bev))
        torch.cuda.synchronize()
        if want is None:
            want = CpuDenseHead(net.export_numpy()).run(bev)
        for name in want:
            for g, w in zip(got[name], want[name]):
                assert tuple(g.shape) == w.shape
                # head outputs (regression maps, heat-map logits): absolute 1e-4 of the value range, true relative above
                assert np.abs(g.cpu().numpy() - w).max() <= 1e-4 * max(1.0, np.abs(w).max()), name
                rel_check("small head %s f16=%s" % (name, f16), g.cpu().numpy(), w, rtol=2e-4, floor=1e-1, small_atol=1e-4)


def test_batched_head_matches_per_layer_head(cuda, oracle_mod):
    """forward (one 64 -> 36*64 conv + one launch for the output convs) against forward_per_head() and the CPU
    reference, both kernel families."""
    import torch
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import DenseRPNHead
    for f16 in (True, False):
        net = DenseRPNHead(in_channels=64, out_channels=(32, 64), layer_nums=(1, 1), downsample_strides=(1, 2),
                           fpn_out_channels=(64, 64), upsample_strides=(1, 2), tasks=(1, 2, 2), share_conv_channel=64, f16=f16)
        net.init_weight(seed=6, device=cuda, randomize_bn=True)
        rng = np.random.default_rng(3)
        bev = rng.normal(size=(1, 64, 24, 40)).astype(np.float32)
        a = net.forward_per_head(_t(cuda, bev))
        b = net.forward(_t(cuda, bev))
        torch.cuda.synchronize()
        want = CpuDenseHead(net.export_numpy()).run(bev)
        for name in want:
            for x, y, w in zip(a[name], b[name], want[name]):
                tol = 1e-4 * max(1.0, np.abs(w).max())
                assert tuple(y.shape) == w.shape
                assert np.abs(y.cpu().numpy() - w).max() <= tol, name
                assert np.abs(y.cpu().numpy() - x.cpu().numpy()).max() <= tol, name


def test_head_out_conv_tap_as_n(cuda, oracle_mod):
    """p3d_head_out_conv_f16 (9 taps in the GEMM's N dimension, virtual groups for a 4-class heat map, image sides that are
    not multiples of the 14-pixel tile, batch 2) against the CPU reference, for head widths 64, 96 (an odd number of
    32-channel groups) and 256 (two-slot activation ring)."""
    import torch
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import DenseRPNHead
    for share in (64, 96, 256):
        tasks = (1, 4, 2) if share == 64 else (1, 4)  # the wide heads: few tasks keep the CPU reference fast
        net = DenseRPNHead(in_channels=64, out_channels=(32, 64), layer_nums=(1, 1), downsample_strides=(1, 2),
                           fpn_out_channels=(64, 64), upsample_strides=(1, 2), tasks=tasks, share_conv_channel=share,
                           f16=True)
        net.init_weight(seed=11, device=cuda, randomize_bn=True)
        rng = np.random.default_rng(5)
        bev = rng.normal(size=(2, 64, 30, 44)).astype(np.float32)
        got = net.forward(_t(cuda, bev))
        torch.cuda.synchronize()
        want = CpuDenseHead(net.export_numpy()).run(bev)
        for name in want:
            for x, w in zip(got[name], want[name]):
                assert tuple(x.shape) == w.shape
                tol = 1e-4 * max(1.0, np.abs(w).max())
                assert np.abs(x.cpu().numpy() - w).max() <= tol, "%s (share %d)" % (name, share)
                rel_check("head out conv %s share %d" % (name, share), x.cpu().numpy(), w, rtol=2e-4, floor=1e-1,
                          small_atol=1e-4)
