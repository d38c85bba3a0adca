"""GPU tests of BEVDet from camera images: the fused ResNet stem against fp64, nearest upsampling of pixel fp16-pair rows
bit for bit, lss_depth_feat_h16 bit-identical to lss_depth_feat, the image encoder (and one Bottleneck of every stage)
against the fp64 CPU arm, and the captured frame (BEVDetImageHotPath: CPU arm, both decodes, eager, lanes, accelerate,
frustum outside the grid, overflow)."""
import numpy as np
import pytest

from parity import rel_check, rel_errors
from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu
BN_GAIN = 6.0 ** 0.5


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _pairs(img, B, H, W, C):
    """pixel H16 rows [B*H*W, 2*C] float16 -> (hi, lo') numpy [B, H, W, C] float16"""
    a = img.cpu().numpy().reshape(B, H, W, C // 32, 2, 32)
    return a[:, :, :, :, 0].reshape(B, H, W, C), a[:, :, :, :, 1].reshape(B, H, W, C)


def _cams(rig):
    from paddle3d_b200.ops import bev_pool_v2 as bp
    return bp.unpack_cameras(bp.pack_cameras(*synth.lss_mats(rig)), 1, 6)


# ---------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("B,H,W", [(1, 256, 704), (6, 256, 704), (1, 37, 53), (6, 37, 53), (2, 100, 150), (1, 7, 5)])
def test_stem_vs_fp64(cuda, oracle_mod, B, H, W):
    """conv 7x7 s2 p3 + BN + ReLU + MaxPool(3, 2, 1) against fp64 (oracle.conv2d, BN / ReLU / max-pool in numpy), at the
    full size, odd sizes and sizes that are not a multiple of the 32 x 64-pixel input tile."""
    import torch
    from bevdet_images_oracle import max_pool_3x3_s2_p1
    from paddle3d_b200.ops import dense_conv as dc
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(B * 1000 + H + W)
    x = synth.camera_images(H + W, B, H, W)
    wt = rng.uniform(-1, 1, (64, 3, 7, 7)).astype(np.float32) / np.float32(np.sqrt(147.0))
    scale = rng.uniform(0.5, 3.0, 64).astype(np.float32)
    shift = rng.normal(0, 0.3, 64).astype(np.float32)
    ref = oracle_mod.conv2d(x, wt, None, 2, 3).astype(np.float64)
    ref = max_pool_3x3_s2_p1(np.maximum(ref * scale.reshape(1, -1, 1, 1) + shift.reshape(1, -1, 1, 1), 0.0))
    st = sp.status_tensor(cuda)
    st.zero_()
    out, shape = dc.resnet_stem_h16(_t(cuda, x), dc.pack_stem_weight(_t(cuda, wt)), _t(cuda, scale), _t(cuda, shift))
    torch.cuda.synchronize()
    assert shape == (B,) + dc.stem_shape(H, W) + (64,) and shape[1:3] == ref.shape[2:]
    assert int(st[0]) == 0
    got = dc.pixel_h16_to_nchw(out, shape).cpu().numpy()
    rel_check("stem %dx%dx%d" % (B, H, W), got, ref, floor=1e-2, small_atol=2e-6)  # test_gpu_dense.py's floor for 147 terms
    # an input past fp16's range sets the status bit
    dc.resnet_stem_h16(_t(cuda, x * np.float32(1e5)), dc.pack_stem_weight(_t(cuda, wt)), _t(cuda, scale), _t(cuda, shift))
    torch.cuda.synchronize()
    try:
        assert int(st[0]) & 1
    finally:
        st.zero_()  # the flag is sticky per device: clear it for the tests that follow


@pytest.mark.parametrize("scale,B,h,w,C,out_C,c0", [
    (2, 6, 8, 22, 512, 512, 0),      # CustomFPN's top-down step at 256 x 704
    (2, 1, 4, 11, 512, 512, 0),      # at 128 x 352
    (3, 2, 3, 5, 64, 96, 16),        # channel offset % 32 == 16, odd factor
    (1, 2, 5, 7, 32, 64, 32),        # copy into the second group
    (4, 1, 2, 3, 96, 128, 32),
])
def test_upsample_nearest_bit_exact(cuda, scale, B, h, w, C, out_C, c0):
    """The pairs of pixel (Y / s, X / s), bit for bit; channels outside [c0, c0 + C) untouched."""
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    x = np.random.default_rng(scale * 100 + C).normal(0, 3, size=(B, C, h, w)).astype(np.float32)
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    H, W = h * scale, w * scale
    out = torch.full((B * H * W, 2 * out_C), 7.0, dtype=torch.float16, device=cuda)
    got, (b, oh, ow) = dc.upsample_nearest_h16(xs, (B, h, w, C), scale, out_h16=out, out_channels=out_C, out_c0=c0)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr() and (b, oh, ow) == (B, H, W)
    hi, lo = _pairs(xs, B, h, w, C)
    yi, xi = np.arange(H) // scale, np.arange(W) // scale
    ghi, glo = _pairs(out, B, H, W, out_C)
    assert np.array_equal(ghi[..., c0:c0 + C].view(np.int16), hi[:, yi][:, :, xi].view(np.int16))
    assert np.array_equal(glo[..., c0:c0 + C].view(np.int16), lo[:, yi][:, :, xi].view(np.int16))
    rest = np.ones(out_C, bool)
    rest[c0:c0 + C] = False
    assert (ghi[..., rest] == 7.0).all() and (glo[..., rest] == 7.0).all()


@pytest.mark.parametrize("BN,H,W,D,C,in_C", [(6, 16, 44, 118, 80, 224), (6, 8, 22, 118, 80, 224), (2, 5, 7, 59, 64, 128),
                                             (1, 3, 37, 40, 8, 64)])
def test_lss_depth_feat_h16_bit_identical(cuda, BN, H, W, D, C, in_C):
    """Bit-identical to p3d_lss_depth_feat on pixel_h16_to_nchw of the same rows (both outputs), whatever the padding
    channels hold."""
    import torch
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(D + C + H)
    x = rng.normal(0, 2, (BN, in_C, H, W)).astype(np.float32)
    x[:, :D] += np.linspace(-6, 6, D, dtype=np.float32).reshape(1, -1, 1, 1) * rng.uniform(-1, 1, (BN, 1, H, W)).astype(np.float32)
    rows = dc.nchw_to_pixel_h16(_t(cuda, x))
    merged = dc.pixel_h16_to_nchw(rows, (BN, H, W, in_C))
    want_d, want_f = bp.lss_depth_feat(merged[:, :D].contiguous(), merged[:, D:D + C].contiguous())
    depth = torch.full((BN, D, H, W), float("nan"), device=cuda)
    feat = torch.full((BN, H, W, C), float("nan"), device=cuda)
    got_d, got_f = bp.lss_depth_feat_h16(rows, (BN, H, W, in_C), D, C, depth, feat)
    torch.cuda.synchronize()
    assert got_d.data_ptr() == depth.data_ptr() and got_f.data_ptr() == feat.data_ptr()
    assert torch.equal(got_d.view(torch.int32), want_d.view(torch.int32))
    assert torch.equal(got_f.view(torch.int32), want_f.view(torch.int32))


# ---------------------------------------------------------------------------------------------------- the model
def _model(cuda, cfg=None, seed=0):
    from paddle3d_b200.bevdet import BEVDetFromImages
    return BEVDetFromImages(cfg, device=cuda).init_weight(seed=seed, bn_gain=BN_GAIN)


def _cpu_arm(m, rig, imgs, keep_feats=False):
    from bevdet_images_oracle import CpuBEVDetImages
    cpu = CpuBEVDetImages(m.export_numpy(), m.test_cfg, m.label_off)
    axes = tuple(a.numpy() for a in m.vt.axes_host)
    return dict(cpu.run(_cams(rig), axes, imgs, *m.vt.grid_args(), keep_feats=keep_feats), arm=cpu)


@pytest.fixture(scope="module")
def frame(cuda):
    """A seeded, calibrated BEVDetFromImages at 256 x 704 with its first frame's images and the CPU arm's result for them
    (computed once: ~370 GFLOP of fp64)."""
    m = _model(cuda)
    rig = synth.camera_rig(31)
    imgs = synth.camera_images(7)
    m.calibrate_heatmap_bias(synth.lss_mats(rig), _t(cuda, imgs))
    return dict(m=m, rig=rig, imgs=imgs, cpu=_cpu_arm(m, rig, imgs, keep_feats=True))


def test_image_encoder_matches_cpu_arm(cuda, frame):
    """The depth net's logits and tran_feat against the fp64 CPU arm at 256 x 704, six cameras; status 0."""
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    from paddle3d_b200.ops import sparse_nn as sp
    m, cpu = frame["m"], frame["cpu"]
    rows, shape = m.image_encoder(_t(cuda, frame["imgs"]))
    torch.cuda.synchronize()
    assert shape == (6, 16, 44, 224) and int(sp.status_tensor(cuda)[0]) == 0
    d = dc.pixel_h16_to_nchw(rows, shape).cpu().numpy()
    assert not d[:, 198:].any()
    # 56 convs in a chain, up to 4608 terms each; 3.0e-4 (logits) and 4.1e-4 (tran_feat) max_rel, 3.8e-6 / 5.0e-6 small
    # seen on an H100
    for name, g, w in (("logits", d[:, :118], cpu["logits"]), ("tran_feat", d[:, 118:198], cpu["tran_feat"])):
        e = rel_errors(g, w)
        assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 3e-5, (name, e)


@pytest.mark.parametrize("si", [0, 1, 2, 3])
def test_one_bottleneck_per_stage(cuda, frame, si):
    """The first Bottleneck of each stage (the one with the downsample identity and, from stage 1 on, stride 2) on the CPU
    arm's own input to it, against the CPU arm's Bottleneck."""
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    m, cpu = frame["m"], frame["cpu"]
    x = cpu["stem"] if si == 0 else cpu["feats"][si - 1]
    blk = m.image_encoder.stages[si][0]
    b, c, h, w = x.shape
    y, shape = m.image_encoder.bottleneck(blk, dc.nchw_to_pixel_h16(_t(cuda, x)), (b, h, w, c))
    torch.cuda.synchronize()
    got = dc.pixel_h16_to_nchw(y, shape).cpu().numpy()
    want = cpu["arm"].bottleneck(cpu["arm"].w["stages"][si][0], x)
    e = rel_errors(got, want)
    # 1.9e-5 / 2.6e-5 / 3.9e-5 / 1.1e-4 max_rel (stages 0-3; 4608 terms in stage 3's 3x3 conv) seen on an H100
    assert e["max_rel"] <= 5e-4 and e["max_small_abs_over_scale"] <= 1e-5, e


def _check_frame(oracle_mod, m, hot, got, cpu):
    from test_gpu_bevdet import _pair
    h = {k: [t.cpu().numpy() for t in v] for k, v in hot.out["head"].items()}
    # 3.1e-3 (256 x 704) and 5.3e-3 (128 x 352) max_rel seen on an H100: the image encoder's error, lifted and pooled,
    # then BEVDet's encoder and head (test_gpu_bevdet.py's frame alone: 2.1e-3)
    for name in h:
        for t, (g, w) in enumerate(zip(h[name], cpu["head"][name])):
            e = rel_errors(g, w)
            assert e["max_rel"] <= 1e-2 and e["max_small_abs_over_scale"] <= 1e-4, (name, t, e)
    tc = m.test_cfg
    r = oracle_mod.centerpoint_postprocess(h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"],
                                           tc["point_cloud_range"], tc["post_center_limit_range"], m.label_off,
                                           tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
                                           tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
    assert len(got[0]) == len(r[0]) > 0
    np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
    assert np.array_equal(got[2], r[2])
    assert abs(len(got[0]) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    assert _pair(got, cpu) >= 0.95  # 498 of 498 paired at both sizes on an H100


def test_frame_matches_cpu_arm(cuda, oracle_mod, frame):
    """Captured frame at 256 x 704: head planes within 1e-2 max_rel of the CPU arm, its postprocess equal to the oracle's
    on the frame's own planes, boxes paired with equal labels; status 0."""
    from paddle3d_b200.bevdet import BEVDetImageHotPath
    m = frame["m"]
    hot = BEVDetImageHotPath(m, device=cuda).capture(count_nodes=True)
    assert hot.graph_nodes["kernel"] > 60 and hot.graph_nodes["memcpy"] >= 6
    got = [t.clone().numpy() for t in hot.infer(synth.lss_mats(frame["rig"]), _t(cuda, frame["imgs"]))]
    assert int(hot.h_status[0]) == 0
    _check_frame(oracle_mod, m, hot, got, frame["cpu"])


def test_frame_matches_cpu_arm_small(cuda, oracle_mod):
    """The same at 128 x 352 (8 x 22 depth-net output)."""
    from paddle3d_b200.bevdet import CONFIG_IMG, BEVDetImageHotPath
    m = _model(cuda, dict(CONFIG_IMG, input_size=(128, 352)), seed=1)
    rig = synth.camera_rig(32)
    imgs = synth.camera_images(8, 6, 128, 352)
    m.calibrate_heatmap_bias(synth.lss_mats(rig), _t(cuda, imgs))
    hot = BEVDetImageHotPath(m, device=cuda).capture()
    got = [t.clone().numpy() for t in hot.infer(synth.lss_mats(rig), _t(cuda, imgs))]
    _check_frame(oracle_mod, m, hot, got, _cpu_arm(m, rig, imgs))


def test_frame_bevdet_nms(cuda, frame):
    """CONFIG_IMG_BEVDET_NMS on the same weights: the frame's rows equal BEVDet's decode (bevdet_postprocess_ref) of its
    own head planes."""
    from bevdet_postprocess_oracle import bevdet_postprocess_ref
    from paddle3d_b200.bevdet import CONFIG_IMG_BEVDET_NMS, BEVDetFromImages, BEVDetImageHotPath
    base = frame["m"]
    m = BEVDetFromImages(CONFIG_IMG_BEVDET_NMS, device=cuda)
    m.encoder, m.head, m.image_encoder = base.encoder, base.head, base.image_encoder
    hot = BEVDetImageHotPath(m, device=cuda).capture()
    got = [t.clone().numpy() for t in hot.infer(synth.lss_mats(frame["rig"]), _t(cuda, frame["imgs"]))]
    h = {k: [t.cpu().numpy() for t in v] for k, v in hot.out["head"].items()}
    r = bevdet_postprocess_ref(h, m.test_cfg, m.label_off)
    assert len(got[0]) == len(r[0]) > 0 and np.array_equal(got[2], r[2])
    np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(got[1], r[1], rtol=1e-6)


def test_captured_eager_lanes_accelerate(cuda, frame):
    """Captured == eager bit for bit with a new rig and new images on every replay; four lanes sharing the model == one
    lane; accelerate=True == the full frame."""
    import torch
    from paddle3d_b200.bevdet import BEVDetFromImages, BEVDetImageHotPath
    m = frame["m"]
    rigs = [synth.camera_rig(40 + i) for i in range(4)]
    ins = [_t(cuda, synth.camera_images(50 + i)) for i in range(4)]
    hot = BEVDetImageHotPath(m, device=cuda).capture()
    want = []
    for r, im in zip(rigs, ins):
        boxes, scores, labels, counts = m.forward_images(synth.lss_mats(r), im)
        k = int(counts[-1])
        eager = [boxes[:k].cpu(), scores[:k].cpu(), labels[:k].cpu()]
        got = [t.clone() for t in hot.infer(synth.lss_mats(r), im)]
        assert k > 0 and all(torch.equal(g, e) for g, e in zip(got, eager))
        want.append(got)
    assert not all(torch.equal(want[0][0], w[0]) for w in want[1:])
    lanes = [BEVDetImageHotPath(m, device=cuda).capture().share_model(hot) for _ in range(4)]
    for rep in range(2):
        for i, lane in enumerate(lanes):
            lane.launch(synth.lss_mats(rigs[i]), ins[i])
        for i, lane in enumerate(lanes):
            assert all(torch.equal(g, w) for g, w in zip(lane.result(), want[i])), "lane %d" % i
    acc_model = BEVDetFromImages(accelerate=True, device=cuda)
    acc_model.encoder, acc_model.head, acc_model.image_encoder = m.encoder, m.head, m.image_encoder
    acc = BEVDetImageHotPath(acc_model, device=cuda).capture()
    for i in (0, 0, 1, 0):
        got = acc.infer(synth.lss_mats(rigs[i]), ins[i])
        assert all(torch.equal(g, w) for g, w in zip(got, want[i]))


def test_frustum_outside_the_grid_and_overflow(cuda, frame):
    """A rig whose frustum misses the grid: zero pool image and status 0.  Images scaled by 1e6 raise the fp16 error."""
    import torch
    from paddle3d_b200.bevdet import BEVDetImageHotPath
    from paddle3d_b200.ops import sparse_nn as sp
    m = frame["m"]
    im = _t(cuda, frame["imgs"])
    far = synth.camera_rig(60)
    far["sensor2ego"][:, :, :3, 3] += np.float32(1000.0)
    hot = BEVDetImageHotPath(m, device=cuda).capture()
    hot.infer(synth.lss_mats(far), im)
    assert not hot.image.any() and int(hot.h_status[0]) == 0
    big = im * 1e6
    try:
        hot.launch(synth.lss_mats(frame["rig"]), big)
        with pytest.raises(RuntimeError, match="fp16"):
            hot.result()
    finally:
        torch.cuda.synchronize()
        sp.status_tensor(cuda).zero_()  # the flag is sticky per device: clear it for the tests that follow
