"""CPU suite for BEVDet from camera images: host-side argument checks of p3d_resnet_stem_h16, p3d_upsample_nearest_h16 and
p3d_lss_depth_feat_h16 (every call here is refused before it reaches the device), the model's stage shapes, its
ValueError on an input size that is not a multiple of 32, its FLOP count and the CPU arm's shapes on a small image."""
import ctypes

import numpy as np
import pytest


def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib.lib()


def _ptrs():
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16  # 16-byte aligned host pointer, never dereferenced
    return buf, p, p + 8


def test_stem_argument_checks():
    L = _lib()
    buf, p, odd = _ptrs()
    f = L.p3d_resnet_stem_h16

    def call(x=p, B=1, H=32, W=32, w=p, s=p, t=p, out=p):
        return f(x, B, H, W, w, s, t, out, None, None)
    assert call(x=None) == -1 and call(w=None) == -1 and call(s=None) == -1 and call(t=None) == -1
    assert call(out=None) == -1
    assert call(B=0) == -1 and call(H=0) == -1 and call(W=0) == -1
    assert call(w=odd) == -1 and call(out=odd) == -1       # 16-byte loads / stores
    assert call(B=65536) == -4                             # grid z
    assert call(B=1, H=2 ** 15, W=2 ** 15) == -4           # 3 H W fp32 elements past int32
    assert L.p3d_resnet_stem_packed_weight_bytes() == 10 * 8 * 32 * 16
    assert L.p3d_resnet_stem_pack_weights(None, p, None, None) == -1
    assert L.p3d_resnet_stem_pack_weights(p, odd, None, None) == -1


def test_upsample_nearest_argument_checks():
    L = _lib()
    buf, p, odd = _ptrs()
    up = L.p3d_upsample_nearest_h16
    assert up(p, 1, 4, 4, 24, 2, p, 32, 0, None) == -1    # input rows of whole 32-channel groups
    assert up(p, 1, 4, 4, 48, 2, p, 64, 0, None) == -1
    assert up(p, 1, 4, 4, 32, 2, p, 64, 8, None) == -1    # out_c0 % 16
    assert up(p, 1, 4, 4, 32, 2, p, 48, 0, None) == -1    # out_C % 32
    assert up(p, 1, 4, 4, 32, 2, p, 32, 16, None) == -1   # past out_C
    assert up(p, 1, 4, 4, 32, 0, p, 32, 0, None) == -1    # scale
    assert up(p, 0, 4, 4, 32, 2, p, 32, 0, None) == -1
    assert up(odd, 1, 4, 4, 32, 2, p, 32, 0, None) == -1  # alignment
    assert up(p, 1, 4, 4, 32, 2, odd, 32, 0, None) == -1
    assert up(None, 1, 4, 4, 32, 2, p, 32, 0, None) == -1
    assert up(p, 1, 4, 4, 32, 2, None, 32, 0, None) == -1


def test_lss_depth_feat_h16_argument_checks():
    L = _lib()
    buf, p, odd = _ptrs()
    f = L.p3d_lss_depth_feat_h16

    def call(rows=p, BN=6, H=16, W=44, in_C=224, D=118, C=80, depth=p, feat=p):
        return f(rows, BN, H, W, in_C, D, C, depth, feat, None)
    assert call(rows=None) == -1 and call(depth=None) == -1 and call(feat=None) == -1
    assert call(rows=odd) == -1                      # 16-byte aligned rows
    assert call(in_C=208) == -1                      # rows of whole 32-channel groups
    assert call(in_C=192) == -1                      # in_C < D + C
    assert call(D=150, C=80) == -1
    assert call(D=0) == -1 and call(C=0) == -1 and call(BN=0) == -1 and call(H=0) == -1
    assert call(in_C=416, D=371, C=10) == -4         # the staged logits' shared memory
    assert call(BN=65536, H=1, W=1) == -4
    assert call(BN=6, H=1024, W=1024, in_C=224) == -4  # 32-bit row offsets


@pytest.mark.parametrize("size", [(256, 704), (128, 352)])
def test_model_stage_shapes(size):
    from paddle3d_b200.bevdet import CONFIG_IMG, BEVDetFromImages
    H, W = size
    m = BEVDetFromImages(dict(CONFIG_IMG, input_size=size), device="cpu")
    want = [(64, H // 4, W // 4), (256, H // 4, W // 4), (512, H // 8, W // 8), (1024, H // 16, W // 16),
            (2048, H // 32, W // 32), (224, H // 16, W // 16)]
    assert m.stage_shapes() == want
    enc = m.image_encoder
    assert (enc.D, enc.C, enc.out_C, enc.depth_net.cout, enc.depth_net.cout_pad) == (118, 80, 224, 198, 208)
    assert [len(s) for s in enc.stages] == [3, 4, 6, 3]
    assert [[b["down"] is not None for b in s] for s in enc.stages] == [[True] + [False] * (len(s) - 1) for s in enc.stages]
    assert [s[0]["conv2"].stride for s in enc.stages] == [1, 2, 2, 2] and all(s[0]["down"].stride == s[0]["conv2"].stride
                                                                             for s in enc.stages)
    assert len(enc.convs()) == 1 + 48 + 4 + 3 + 1
    assert (m.vt.H, m.vt.W) == (H // 16, W // 16)


@pytest.mark.parametrize("size", [(250, 704), (256, 700), (240, 688)])
def test_input_size_not_multiple_of_32(size):
    from paddle3d_b200.bevdet import CONFIG_IMG, BEVDetFromImages
    with pytest.raises(ValueError, match="multiple of 32"):
        BEVDetFromImages(dict(CONFIG_IMG, input_size=size), device="cpu")


def test_flops():
    from paddle3d_b200.bevdet import BEVDet, BEVDetFromImages
    m = BEVDetFromImages(device="cpu")
    fl = m.flops()
    assert round(fl["img_stem"] / 1e9, 2) == 5.09
    assert round(fl["img_layers"] / 1e9, 2) == 171.08
    assert round(fl["img_neck"] / 1e9, 2) == 26.58
    assert round(fl["depth_net"] / 1e9, 2) == 0.86
    assert round(fl["img_total"] / 1e9, 2) == 203.60
    assert fl["img_backbone"] == pytest.approx(fl["img_stem"] + fl["img_layers"])
    # by hand: stem 6 x 128 x 352 x 147 x 64; CustomFPN's two laterals and 3x3 conv at 16 x 44 / 8 x 22
    assert fl["img_stem"] == 2.0 * 6 * 128 * 352 * 147 * 64
    assert fl["img_neck"] == 2.0 * 6 * (704 * 1024 * 512 + 176 * 2048 * 512 + 704 * 9 * 512 * 512)
    assert fl["depth_net"] == 2.0 * 6 * 704 * 512 * 198
    base = BEVDet(device="cpu").flops()
    for k, v in base.items():
        assert fl[k] == v, k
    assert fl["frame_total"] == pytest.approx(base["total"] + fl["img_total"])


def test_cpu_arm_shapes(oracle_mod):
    """The CPU arm's image half on a 64 x 128 image (two cameras): every stage's shape, ReLU outputs non-negative, the
    logits / tran_feat split of the depth net, and its max-pool / nearest helpers against torch."""
    import torch
    import torch.nn.functional as F
    from bevdet_images_oracle import CpuBEVDetImages, max_pool_3x3_s2_p1, upsample_nearest
    from paddle3d_b200 import synth
    from paddle3d_b200.bevdet import CONFIG_IMG, BEVDetFromImages
    m = BEVDetFromImages(dict(CONFIG_IMG, input_size=(64, 128)), device="cpu").init_weight(seed=1, device=False)
    cpu = CpuBEVDetImages(m.export_numpy(), m.test_cfg, m.label_off)
    imgs = synth.camera_images(3, 2, 64, 128)
    feats = cpu.backbone(imgs)
    assert [f.shape for f in feats] == [(2, 256, 16, 32), (2, 512, 8, 16), (2, 1024, 4, 8), (2, 2048, 2, 4)]
    assert min(float(f.min()) for f in feats) >= 0.0
    logits, tran = cpu.image_encoder(imgs)
    assert logits.shape == (2, 118, 4, 8) and tran.shape == (2, 80, 4, 8) and np.isfinite(logits).all()
    x = np.random.default_rng(0).normal(size=(2, 3, 7, 9))
    np.testing.assert_array_equal(max_pool_3x3_s2_p1(x), F.max_pool2d(torch.from_numpy(x), 3, 2, 1).numpy())
    np.testing.assert_array_equal(upsample_nearest(x, (14, 18)),
                                  F.interpolate(torch.from_numpy(x), size=(14, 18), mode="nearest").numpy())
