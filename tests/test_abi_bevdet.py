"""CPU suite for BEVDet: host-side argument checks of its entry points (p3d_dense_conv2d_f16_residual,
p3d_upsample_bilinear_h16, p3d_bev_pool_v2_dev_h16; every call here is refused before it reaches the device), the
oracle's bilinear upsampling against torch, and the model's shapes and FLOP count."""
import ctypes

import numpy as np
import pytest


def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib.lib()


def test_residual_conv_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16  # 16-byte aligned host pointer, never dereferenced
    odd = p + 4
    f = L.p3d_dense_conv2d_f16_residual

    def call(res=p, res_c=64, up=1, out=p, out_c=64, c0=0, nchw=None, cout=64):
        k = up if up > 1 else 3
        return f(p, 1, 8, 8, 64, p, cout, 64, k, k, up if up > 1 else 1, 0 if up > 1 else 1, up, None, None, 1, out, out_c, c0,
                 nchw, res, res_c, 0, 0, None, None)
    assert call(res=None) == -1                  # no residual
    assert call(res=odd) == -1                   # misaligned residual
    assert call(res_c=32) == -1                  # fewer residual channels than outputs
    assert call(up=2) == -4                      # transposed conv
    assert call(nchw=p) == -4                    # fp32 planes
    assert call(out=None, nchw=p) == -4
    assert call(out_c=96, c0=16, cout=64) == -4  # output group split across two layers
    assert call(res_c=80) == -4                  # residual rows not whole 32-channel groups
    # the checks of p3d_dense_conv2d_f16 still apply: mode, channel counts
    assert f(p, 1, 8, 8, 48, p, 64, 64, 3, 3, 1, 1, 1, None, None, 1, p, 64, 0, None, p, 64, 0, 0, None, None) == -4
    assert f(p, 1, 8, 8, 64, p, 64, 64, 3, 3, 1, 1, 1, None, None, 1, p, 64, 0, None, p, 64, 2, 0, None, None) == -1


def test_residual_offset_guard():
    """The kernel addresses the residual with 32-bit byte offsets: a residual image of B * oH * oW * 4 * res_C bytes past
    0x7fffffff is refused (P3D_ERR_UNSUPPORTED), one at or below it is not, and the count is on the output's size
    (stride 2 halves each side).  Every call passes mode 2, which the conv's own argument checks refuse
    (P3D_ERR_INVALID_ARG) after the guard and before any tensor map or launch: -4 is the guard, -1 a call past it."""
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16

    def call(B, H, W, stride, res_c):
        return L.p3d_dense_conv2d_f16_residual(p, B, H, W, 64, p, 64, 64, 3, 3, stride, 1, 1, None, None, 1, p, 64, 0, None,
                                               p, res_c, 2, 0, None, None)
    limit = 0x7fffffff
    assert 2 * 2048 * 2048 * 4 * 64 == limit + 1
    assert call(2, 2048, 2048, 1, 64) == -4       # 2^23 pixels x 256 bytes
    assert call(1, 1, 2 ** 23, 1, 64) == -4       # the same bytes in one pixel row
    assert (2 ** 23 - 1) * 4 * 64 == limit + 1 - 256
    assert call(1, 1, 2 ** 23 - 1, 1, 64) == -1   # one pixel fewer: past the guard
    assert call(1, 4096, 4096, 2, 128) == -4      # 2048 x 2048 outputs x 512 bytes
    assert call(1, 4096, 4096, 2, 64) == -1       # 2^32 bytes counted on the input, 2^30 on the output
    assert 5592406 * 4 * 96 - limit == 257 and limit - 5592405 * 4 * 96 == 127
    assert call(1, 1, 5592406, 1, 96) == -4       # one pixel row of 5592406 x 384 bytes
    assert call(1, 1, 5592405, 1, 96) == -1


def test_upsample_and_pixel_pool_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    odd = p + 8
    up = L.p3d_upsample_bilinear_h16
    assert up(p, 1, 4, 4, 24, 2, p, 32, 0, None, None) == -1    # input rows of whole 32-channel groups
    assert up(p, 1, 4, 4, 48, 2, p, 64, 0, None, None) == -1
    assert up(p, 1, 4, 4, 32, 2, p, 64, 8, None, None) == -1    # out_c0 % 16
    assert up(p, 1, 4, 4, 32, 2, p, 48, 0, None, None) == -1    # out_C % 32
    assert up(p, 1, 4, 4, 32, 2, p, 32, 16, None, None) == -1   # past out_C
    assert up(p, 1, 4, 4, 32, 0, p, 32, 0, None, None) == -1    # scale
    assert up(odd, 1, 4, 4, 32, 2, p, 32, 0, None, None) == -1  # alignment
    assert up(p, 1, 4, 4, 32, 2, None, 32, 0, None, None) == -1
    pool = L.p3d_bev_pool_v2_dev_h16

    def call(feat=p, c=80, Z=1, out=p, out_c=96):
        return pool(p, feat, p, p, p, p, p, p, 100, c, 1, Z, 8, 8, out, out_c, None, None)
    assert call(out_c=80) == -1          # not a multiple of 32
    assert call(out_c=64) == -1          # narrower than Z * c
    assert call(Z=2, out_c=128) == -1
    assert call(out=None) == -1
    assert call(c=6, out_c=32) == -4     # c % 4
    assert call(feat=odd) == -4          # float4 feature loads
    assert call(out=odd) == -4


@pytest.mark.parametrize("s,h,w", [(2, 5, 7), (4, 3, 4), (1, 4, 6), (3, 1, 5)])
def test_oracle_bilinear_matches_torch(s, h, w):
    import torch
    from oracle import bevdet
    x = np.random.default_rng(s * 10 + h).normal(size=(2, 3, h, w))
    want = torch.nn.functional.interpolate(torch.from_numpy(x), scale_factor=s, mode="bilinear", align_corners=True).numpy()
    np.testing.assert_allclose(bevdet.upsample_bilinear(x, s), want, rtol=1e-12, atol=1e-12)
    # the fp32 restatement of the kernel stays within fp32 rounding of it
    got = bevdet.upsample_bilinear_fp32(x.transpose(0, 2, 3, 1).astype(np.float32), s).transpose(0, 3, 1, 2)
    np.testing.assert_allclose(got, want, rtol=1e-5, atol=1e-5)


def test_model_shapes_and_flops(oracle_mod):
    from oracle.bevdet import CpuBEVDet
    from paddle3d_b200.bevdet import BEVDet
    m = BEVDet(device="cpu").init_weight(seed=3, device=False)
    assert m.image_shape == (1, 128, 128, 96)
    fl = m.flops()
    # by hand: stage s of CustomResNet at (64 / 2^s)^2 pixels: conv1 + identity conv (cin -> cout) and three cout -> cout
    bb = 0.0
    cin = 80
    for s, cout in enumerate((160, 320, 640)):
        px = (64 >> s) ** 2
        bb += 2.0 * px * 9 * (2 * cin * cout + 3 * cout * cout)
        cin = cout
    fpn = 2.0 * 9 * (4096 * (800 * 512 + 512 * 512) + 16384 * 512 * 256) + 2.0 * 16384 * 256 * 256
    head = 2.0 * 16384 * 9 * (256 * 64 + 36 * 64 * 64 + 64 * m.head_planes())
    assert fl["backbone"] == pytest.approx(bb) and fl["fpn"] == pytest.approx(fpn) and fl["head"] == pytest.approx(head)
    assert 155e9 < fl["total"] < 170e9
    w = m.export_numpy()
    assert [[b["down"] is not None for b in st] for st in w["backbone"]] == [[True, False]] * 3
    assert w["backbone"][0][0]["conv1"]["weight"].shape == (160, 80, 3, 3)  # exported unpadded
    # the oracle encoder's shapes on a 16 x 16 BEV: stages at 8, 4, 2; the concat at 8; the output at 16
    cpu = CpuBEVDet(w, m.test_cfg, m.label_off)
    bev = np.random.default_rng(0).normal(size=(1, 80, 16, 16)).astype(np.float32)
    feats = cpu.backbone(bev)
    assert [f.shape for f in feats] == [(1, 160, 8, 8), (1, 320, 4, 4), (1, 640, 2, 2)]
    assert min(float(f.min()) for f in feats) >= 0.0  # ReLU after the residual
    out = cpu.encoder(bev)
    assert out.shape == (1, 256, 16, 16) and np.isfinite(out).all()
