"""GPU tests of BEVDet: the residual epilogue of the fp16-pair dense conv against fp64, the bilinear upsampling of pixel
fp16-pair rows bit for bit against its numpy fp32 restatement, bev_pool into pixel rows, and the BEVDet frame (eager,
captured, lanes, accelerate) against the CPU arm (oracle.bevdet.CpuBEVDet)."""
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


@pytest.mark.parametrize("mode,m_tiles", [(0, 1), (0, 2), (1, 1), (1, 2)])
@pytest.mark.parametrize("cin,cout,n_tile,stride,res_extra,h,w", [
    (64, 160, 64, 1, 0, 20, 23),     # three N tiles of 64, the last half used; ragged pixel tiles
    (160, 160, 128, 1, 32, 21, 18),  # two N tiles of 128, the last a quarter used; residual rows wider than the output
    (96, 320, 64, 2, 0, 33, 30),     # stride 2 (per-tap boxes), five N tiles
    (64, 320, 128, 1, 0, 17, 40),    # three N tiles of 128, the last half used
    (64, 640, 128, 1, 0, 12, 20),    # five full N tiles
])
def test_residual_conv_vs_fp64(cuda, oracle_mod, cin, cout, n_tile, stride, res_extra, h, w, mode, m_tiles):
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(cin + cout + stride)
    B = 2
    x = rng.normal(size=(B, cin, h, w)).astype(np.float32)
    wt = (rng.normal(size=(cout, cin, 3, 3)) / np.sqrt(cin * 9)).astype(np.float32)
    scale = rng.uniform(0.5, 1.5, cout).astype(np.float32)
    shift = rng.normal(size=cout).astype(np.float32)
    oh, ow = (h + 2 - 3) // stride + 1, (w + 2 - 3) // stride + 1
    rc = cout + res_extra
    res = rng.normal(size=(B, rc, oh, ow)).astype(np.float32)
    res_h16 = dc.nchw_to_pixel_h16(_t(cuda, res))
    res_dec = dc.pixel_h16_to_nchw(res_h16, (B, oh, ow, rc)).cpu().numpy()[:, :cout].astype(np.float64)
    ref = oracle_mod.conv2d(x, wt, None, stride, 1).astype(np.float64)
    ref = np.maximum(ref * scale.reshape(1, -1, 1, 1) + shift.reshape(1, -1, 1, 1) + res_dec, 0.0)
    packed = dc.pack_conv_weight_f16(_t(cuda, wt), n_tile)
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    oc = (cout + 31) // 32 * 32
    out, _, (b, oh2, ow2) = dc.dense_conv2d_f16(xs, (B, h, w, cin), packed, cout, n_tile, 3, stride, 1, 1, _t(cuda, scale),
                                                _t(cuda, shift), True, out_channels=oc, mode=mode, m_tiles=m_tiles,
                                                residual=res_h16, res_channels=rc)
    torch.cuda.synchronize()
    assert (oh2, ow2) == (oh, ow)
    got = dc.pixel_h16_to_nchw(out, (b, oh, ow, oc)).cpu().numpy()[:, :cout]
    floor = 1e-2 if cin * 9 <= 2304 else 5e-2  # test_gpu_dense.py's floors
    rel_check("residual f16 %d->%d n%d s%d mode%d mt%d" % (cin, cout, n_tile, stride, mode, m_tiles), got, ref, floor=floor,
              small_atol=2e-6 if floor == 1e-2 else 1e-5)


@pytest.mark.parametrize("scale,B,h,w,C,out_C,c0", [
    (1, 2, 7, 9, 32, 64, 32),        # copy into the second group
    (2, 2, 5, 7, 64, 96, 16),        # odd sizes, channel offset % 32 == 16
    (4, 1, 16, 16, 640, 800, 160),   # FPN_LSS's up4 of the third stage into the concat
    (2, 1, 64, 64, 512, 512, 0),     # FPN_LSS's extra up2
    (4, 2, 3, 5, 32, 64, 16),
])
def test_upsample_bit_exact(cuda, scale, B, h, w, C, out_C, c0):
    """Bit-equal to the numpy fp32 restatement (scale 1: the input pairs), channels outside [c0, c0 + C) untouched, and
    within 1e-6 relative of the fp64 bilinear of the input values."""
    import torch
    from oracle import bevdet as ob
    from paddle3d_b200.ops import dense_conv as dc
    x = np.random.default_rng(scale * 100 + C).normal(0, 3, size=(B, C, h, w)).astype(np.float32)
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    H, W = h * scale, w * scale
    out = torch.full((B * H * W, 2 * out_C), 7.0, dtype=torch.float16, device=cuda)
    dc.upsample_bilinear_h16(xs, (B, h, w, C), scale, out_h16=out, out_channels=out_C, out_c0=c0)
    torch.cuda.synchronize()
    hi, lo = _pairs(xs, B, h, w, C)
    want = ob.upsample_bilinear_fp32(ob.merge_h16(hi, lo), scale)
    whi, wlo = (hi, lo) if scale == 1 else ob.split_h16(want)
    ghi, glo = _pairs(out, B, H, W, out_C)
    assert np.array_equal(ghi[..., c0:c0 + C].view(np.int16), whi.view(np.int16))
    assert np.array_equal(glo[..., c0:c0 + C].view(np.int16), wlo.view(np.int16))
    rest = np.ones(out_C, bool)
    rest[c0:c0 + C] = False
    assert (ghi[..., rest] == 7.0).all() and (glo[..., rest] == 7.0).all()
    # fp64 at Paddle's fp32 source coordinates: 1e-6 relative; at the exact coordinates the fp32 ratio moves a sample by
    # up to ~1e-5 of the largest value (4e-6 seen for 64 -> 128)
    x64 = ob.merge_h16(hi, lo).transpose(0, 3, 1, 2)
    got = ob.merge_h16(ghi[..., c0:c0 + C], glo[..., c0:c0 + C]).astype(np.float64)
    ref = ob.upsample_bilinear(x64, scale, src_fp32=True).transpose(0, 2, 3, 1)
    assert np.abs(got - ref).max() <= 1e-6 * np.abs(ref).max()
    exact = ob.upsample_bilinear(x64, scale).transpose(0, 2, 3, 1)
    assert np.abs(got - exact).max() <= 1e-5 * np.abs(exact).max()


def test_pool_into_pixel_rows(cuda):
    """Bytes equal to nchw_to_pixel_h16 of the planar pool zero-padded to the row width: empty cells and padding channels
    zero (the buffer is filled with garbage first); Z > 1 keeps channel z * C + c."""
    import torch
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import dense_conv as dc
    for seed, C, D, grid, b in ((5, 80, 118, (128, 128, 1), (-51.2, 51.2)), (6, 16, 30, (64, 64, 4), (-40.0, 40.0))):
        d = synth.bev_pool_inputs(seed, C=C, D=D, grid=grid, bounds=(b, b, (-5.0, 3.0)))
        prep = bp.voxel_pooling_prepare_v2(_t(cuda, d["coor"]), d["grid_lower_bound"], d["grid_interval"], d["grid_size"])
        depth, feat = _t(cuda, d["depth"]), _t(cuda, d["feat"])
        X, Y, Z = grid
        shape = (1, Z, Y, X, C)
        planar = bp.bev_pool_v2_dev(depth, feat, prep, shape, planar=True)
        oc = (Z * C + 31) // 32 * 32
        padded = torch.zeros((1, oc, Y, X), dtype=torch.float32, device=cuda)
        padded[:, :Z * C] = planar
        want = dc.nchw_to_pixel_h16(padded)
        out = torch.full((Y * X, 2 * oc), -3.0, dtype=torch.float16, device=cuda)
        got = bp.bev_pool_v2_dev_h16(depth, feat, prep, shape, out=out)
        torch.cuda.synchronize()
        assert got.data_ptr() == out.data_ptr()
        assert torch.equal(got.view(torch.int16), want.view(torch.int16))
        assert bool((planar == 0).any()) and bool(planar.any())
        if oc > Z * C:
            hi, lo = _pairs(got, 1, Y, X, oc)
            assert not hi[..., Z * C:].any() and not lo[..., Z * C:].any()


# ---------------------------------------------------------------------------------------------------- the frame
def _inputs(m, seed):
    vt = m.vt
    rng = np.random.default_rng(seed)
    logits = rng.normal(0, 2, (m.N, vt.D, vt.H, vt.W)).astype(np.float32)
    tran = rng.normal(0, 1, (m.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)
    return logits, tran


def _cams(rig):
    from paddle3d_b200.ops import bev_pool_v2 as bp
    return bp.unpack_cameras(bp.pack_cameras(*synth.lss_mats(rig)), 1, 6)


@pytest.fixture(scope="module")
def frame(cuda):
    """A seeded, calibrated BEVDet with its first frame's inputs and the CPU arm's result for them."""
    from oracle.bevdet import CpuBEVDet
    from paddle3d_b200.bevdet import BEVDet
    m = BEVDet(device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    rig = synth.camera_rig(31)
    logits, tran = _inputs(m, 7)
    m.calibrate_heatmap_bias(synth.lss_mats(rig), _t(cuda, logits), _t(cuda, tran))
    axes = tuple(a.numpy() for a in m.vt.axes_host)
    cpu = CpuBEVDet(m.export_numpy(), m.test_cfg, m.label_off).run(_cams(rig), axes, logits, tran, *m.vt.grid_args())
    return dict(m=m, rig=rig, logits=logits, tran=tran, cpu=cpu)


def _pair(got, cpu, tol=1e-3):
    """test_gpu_centerpoint_pillars._pair: the fraction of CPU boxes paired by centre with a GPU box of equal label whose
    values and score are within tol (relative, absolute below 1)."""
    gb, gs, gl = got
    used, n = set(), 0
    for i in range(len(cpu["boxes"])):
        if not len(gb):
            break
        j = int(np.argmin(np.abs(gb[:, :3] - cpu["boxes"][i, :3]).max(1)))
        eb = (np.abs(gb[j] - cpu["boxes"][i]) / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
        es = abs(gs[j] - cpu["scores"][i]) / max(1.0, abs(cpu["scores"][i]))
        if j not in used and eb <= tol and es <= tol and gl[j] == cpu["labels"][i]:
            used.add(j)
            n += 1
    return n / max(1, len(cpu["boxes"]))


def test_encoder_matches_cpu_arm(cuda, frame):
    """The pool image against the oracle's view transform (bev_pool tolerances, padding channels zero) and the encoder's
    output against CpuBEVDet's fp64 encoder."""
    from paddle3d_b200.ops import dense_conv as dc
    m, cpu = frame["m"], frame["cpu"]
    tl, tt = _t(cuda, frame["logits"]), _t(cuda, frame["tran"])
    img = m.image(synth.lss_mats(frame["rig"]), tl, tt)
    bev = dc.pixel_h16_to_nchw(img, m.image_shape).cpu().numpy()
    assert not bev[:, 80:].any()
    np.testing.assert_allclose(bev[:, :80], cpu["bev"], rtol=1e-4, atol=1e-5)
    y, shape = m.encode(img)
    assert shape == (1, 128, 128, 256)
    got = dc.pixel_h16_to_nchw(y, shape).cpu().numpy()
    e = rel_errors(got, cpu["feat"])
    assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e


def test_frame_matches_cpu_arm(cuda, oracle_mod, frame):
    """Captured frame: head planes on the parity bar of the CenterPoint-pillars frame, its postprocess equal to the
    oracle's on the frame's own planes, boxes paired with equal labels."""
    from paddle3d_b200.bevdet import BEVDetHotPath
    m, cpu = frame["m"], frame["cpu"]
    hot = BEVDetHotPath(m, device=cuda).capture(count_nodes=True)
    assert hot.graph_nodes["kernel"] > 0 and hot.graph_nodes["memcpy"] >= 6
    got = [t.clone().numpy() for t in hot.infer(synth.lss_mats(frame["rig"]), _t(cuda, frame["logits"]),
                                                 _t(cuda, frame["tran"]))]
    h = {k: [t.cpu().numpy() for t in v] for k, v in hot.out["head"].items()}
    assert sum(t.shape[1] for v in h.values() for t in v) == 70 and h["hm"][0].shape[2:] == (128, 128)
    # 5e-3, not the CenterPoint-pillars frame's 2e-3: FPN_LSS's 3x3 convs sum 7200 and 4608 terms, more than any layer of
    # that frame (test_gpu_dense.py widens its floor above 2304 terms for the same reason); 2.1e-3 seen on an H100
    for name in h:
        for t, (g, w) in enumerate(zip(h[name], cpu["head"][name])):
            e = rel_errors(g, w)
            assert e["max_rel"] <= 5e-3 and e["max_small_abs_over_scale"] <= 1e-4, (name, t, e)
    tc = m.test_cfg
    r = oracle_mod.centerpoint_postprocess(h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"],
                                           tc["point_cloud_range"], tc["post_center_limit_range"], m.label_off,
                                           tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
                                           tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
    assert len(got[0]) == len(r[0]) > 0
    np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
    assert np.array_equal(got[2], r[2])
    assert abs(len(got[0]) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    assert _pair(got, cpu) >= 0.95


def test_captured_eager_lanes_accelerate(cuda, frame):
    """Captured == eager bit for bit with a new calibration on every replay; four lanes sharing the model == one lane;
    accelerate=True == the full frame."""
    import torch
    from paddle3d_b200.bevdet import BEVDet, BEVDetHotPath
    m = frame["m"]
    rigs = [synth.camera_rig(40 + i) for i in range(4)]
    ins = [[_t(cuda, a) for a in _inputs(m, 50 + i)] for i in range(4)]
    hot = BEVDetHotPath(m, device=cuda).capture()
    want = []
    for r, (tl, tt) in zip(rigs, ins):
        boxes, scores, labels, counts = m.forward(synth.lss_mats(r), tl, tt)
        k = int(counts[-1])
        eager = [boxes[:k].cpu(), scores[:k].cpu(), labels[:k].cpu()]
        got = [t.clone() for t in hot.infer(synth.lss_mats(r), tl, tt)]
        assert k > 0 and all(torch.equal(g, e) for g, e in zip(got, eager))
        want.append(got)
    lanes = [BEVDetHotPath(m, device=cuda).capture() for _ in range(4)]
    for rep in range(2):
        for i, lane in enumerate(lanes):
            lane.launch(synth.lss_mats(rigs[i]), *ins[i])
        for i, lane in enumerate(lanes):
            assert all(torch.equal(g, w) for g, w in zip(lane.result(), want[i])), "lane %d" % i
    acc_model = BEVDet(accelerate=True, device=cuda)
    acc_model.encoder, acc_model.head = m.encoder, m.head
    acc = BEVDetHotPath(acc_model, device=cuda).capture()
    for i in (0, 0, 1, 0):
        got = acc.infer(synth.lss_mats(rigs[i]), *ins[i])
        assert all(torch.equal(g, w) for g, w in zip(got, want[i]))


def test_frustum_outside_the_grid_and_overflow(cuda, frame):
    """A rig whose frustum misses the grid: zero pool image, status 0, the same result for any such rig and equal to the
    eager frame.  Features scaled past fp16's range raise from check_status."""
    import torch
    from paddle3d_b200.bevdet import BEVDetHotPath
    from paddle3d_b200.ops import sparse_nn as sp
    m = frame["m"]
    tl, tt = _t(cuda, frame["logits"]), _t(cuda, frame["tran"])
    far = [synth.camera_rig(60 + i) for i in range(2)]
    for r in far:
        r["sensor2ego"][:, :, :3, 3] += np.float32(1000.0)
    hot = BEVDetHotPath(m, device=cuda).capture()
    res = []
    for r in far:
        res.append([t.clone() for t in hot.infer(synth.lss_mats(r), tl, tt)])
        assert not hot.image.any() and int(hot.h_status[0]) == 0
    assert all(torch.equal(a, b) for a, b in zip(*res))
    boxes, scores, labels, counts = m.forward(synth.lss_mats(far[0]), tl, tt)
    k = int(counts[-1])
    assert all(torch.equal(g, e.cpu()) for g, e in zip(res[0], (boxes[:k], scores[:k], labels[:k])))
    try:
        hot.launch(synth.lss_mats(frame["rig"]), tl, tt * 1e6)
        with pytest.raises(RuntimeError, match="fp16"):
            hot.result()
    finally:
        torch.cuda.synchronize()
        sp.status_tensor(cuda).zero_()  # the flag is sticky per device: clear it for the tests that follow
