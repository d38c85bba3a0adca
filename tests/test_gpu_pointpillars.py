"""GPU: PointPillars inference - the anchor-head postprocess kernel (csrc/anchor_postprocess.cu) against the numpy oracle,
the dense conv at the shapes only this model uses, the captured frame against eager execution and against the CPU arm,
and the shared SecondTrunk leaving CenterPoint's dense head unchanged."""
import numpy as np
import pytest
import torch

import oracle.pointpillars as opp
from parity import rel_check, rel_errors
from test_pointpillars_oracle import GRID, _frame

pytestmark = pytest.mark.gpu
BN_GAIN = 6.0 ** 0.5


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def model(cuda):
    from paddle3d_b200 import pointpillars as pp
    return pp.PointPillars().init_weight(seed=1, device=cuda)


@pytest.mark.parametrize("seed,cls_mean,occ,tie", [
    (0, -4.0, 0.3, False),    # a few hundred candidates
    (1, -2.0, 0.3, True),     # > 1000 candidates, exact score ties (quarter-step logits)
    (4, -1.0, 0.05, False),   # sparse pillars: most anchors masked, still > 1000 candidates
    (2, -30.0, 0.3, False),   # no candidate: empty output
    (3, 0.0, 0.0, False),     # no pillar: every anchor masked
])
def test_postprocess_vs_oracle(cuda, oracle_mod, model, seed, cls_mean, occ, tie):
    from paddle3d_b200.ops import nms_utils
    tc = model.mc["test"]
    head, coords = _frame(seed, cls_mean, occ, tie)
    cap = max(len(coords), 1)
    coords_dev = torch.zeros((cap + 7, 4), dtype=torch.int32, device=cuda)  # capacity rows beyond the count are ignored
    coords_dev[:len(coords)] = _t(cuda, coords)
    coords_dev[len(coords):, 2:] = 5
    num = torch.tensor([len(coords)], dtype=torch.int32, device=cuda)
    A = model.anchors.shape[0]
    mask = torch.empty((A,), dtype=torch.uint8, device=cuda)
    sb = torch.empty((tc["nms_pre_max_size"], 7), dtype=torch.float32, device=cuda)
    ss = torch.empty((tc["nms_pre_max_size"],), dtype=torch.float32, device=cuda)
    boxes, scores, labels, counts = model.postprocess(_t(cuda, head), coords_dev, num, anchor_mask=mask, sorted_out=(sb, ss))
    torch.cuda.synchronize()
    r = opp.anchor_head_postprocess(head, model.anchors_np, model.corners_np, coords, GRID,
                                    tc["post_center_limit_range"], tc["anchor_area_threshold"],
                                    tc["nms_score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"],
                                    tc["nms_post_max_size"])
    assert np.array_equal(mask.cpu().numpy().astype(bool), r["mask"])
    ncand, k = [int(v) for v in counts.cpu()]
    assert ncand == r["candidates"] and k == len(r["boxes"])
    n = min(ncand, tc["nms_pre_max_size"])
    np.testing.assert_allclose(sb[:n].cpu().numpy(), r["cand_boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(ss[:n].cpu().numpy(), r["cand_scores"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(boxes[:k].cpu().numpy(), r["boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(scores[:k].cpu().numpy(), r["scores"], rtol=1e-6, atol=0)
    assert np.array_equal(labels[:k].cpu().numpy(), r["labels"])
    # the NMS keep list equals rotate_nms_pcdet's on the kernel's own thresholded, decoded candidates
    if n:
        sel = nms_utils.rotate_nms_pcdet(sb[:n], ss[:n], tc["nms_iou_threshold"], tc["nms_pre_max_size"],
                                         tc["nms_post_max_size"])
        want = sb[sel]
        lo = torch.tensor(tc["post_center_limit_range"][:3], device=cuda)
        hi = torch.tensor(tc["post_center_limit_range"][3:], device=cuda)
        want = want[((want[:, :3] >= lo) & (want[:, :3] <= hi)).all(1)]
        got = boxes[:k]
        assert torch.equal(got[:, :6], want[:, :6])
        dth = (got[:, 6] - want[:, 6]).abs().cpu().numpy()  # the direction fix adds 0 or pi
        assert np.all((dth == 0) | (np.abs(dth - np.pi) < 1e-6))
    if tie:
        assert len(np.unique(r["cand_scores"])) < n
    if occ == 0.0:
        assert k == 0 and not mask.bool().any()


@pytest.mark.parametrize("cin,cout,k,stride,pad,up,h,w", [
    (64, 64, 3, 2, 1, 1, 496, 432),    # first backbone conv on the pillar image
    (256, 128, 4, 4, 0, 4, 62, 54),    # up-4 transposed conv of the last block: mostly partial tiles
    (64, 128, 1, 1, 0, 1, 248, 216),   # stride-1 Conv2DTranspose k = 1 (use_conv_for_no_stride off), transposed weight
])
def test_dense_conv_at_pointpillars_shapes(cuda, oracle_mod, cin, cout, k, stride, pad, up, h, w):
    from paddle3d_b200.dense_head import _Conv
    rng = np.random.default_rng(cin * 7 + cout)
    x = rng.normal(size=(1, cin, h, w)).astype(np.float32)
    transposed = up > 1 or k == 1
    conv = _Conv(cin, cout, k, stride, pad, bn_eps=1e-3, up=up, transposed=transposed).init(rng, cuda, randomize_bn=True)
    p = conv.np
    ref = (oracle_mod.deconv2d(x, p["weight"], None, max(up, 1)) if transposed else
           oracle_mod.conv2d(x, p["weight"], None, stride, pad))
    bn = p["bn"]
    ref = oracle_mod.bn2d_relu(ref, bn["gamma"], bn["beta"], bn["mean"], bn["var"], bn["eps"])
    from paddle3d_b200.ops import dense_conv as dc
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    _, o, _ = conv(xs, (1, h, w, cin), want_nchw=True)
    torch.cuda.synchronize()
    rel_check("pointpillars dense %d->%d k%d s%d up%d" % (cin, cout, k, stride, up), o.cpu().numpy(), ref)


def test_head_conv_384_to_20_fp32_planes(cuda, oracle_mod, model):
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(20)
    x = np.maximum(rng.normal(size=(1, 384, 248, 216)), 0).astype(np.float32)
    planes = model.head(dc.nchw_to_pixel_h16(_t(cuda, x)), (1, 248, 216, 384), want_nchw=True)[1]
    torch.cuda.synchronize()
    p = model.head.np
    rel_check("pointpillars head 384->20", planes.cpu().numpy(), oracle_mod.conv2d(x, p["weight"], p["bias"], 1, 0))


def test_trunk_refactor_keeps_centerpoint_dense_head(cuda):
    """DenseRPNHead on a seeded BEV equals the layer chain it ran before SecondTrunk was factored out, bit for bit."""
    from paddle3d_b200.dense_head import DenseRPNHead
    from paddle3d_b200.ops import dense_conv as dc
    net = DenseRPNHead(in_channels=64, out_channels=(32, 64), layer_nums=(1, 2), downsample_strides=(1, 2),
                       fpn_out_channels=(32, 32), upsample_strides=(1, 2), tasks=(1, 2), share_conv_channel=64)
    net.init_weight(seed=5, device=cuda, randomize_bn=True, bn_gain=BN_GAIN)
    bev = torch.from_numpy(np.random.default_rng(9).normal(size=(1, 64, 40, 36)).astype(np.float32)).to(cuda)
    s, shape = net._trunk(bev)
    x, sh = dc.nchw_to_pixel_h16(bev), (1, 40, 36, 64)
    feats = []
    for blk in net.blocks:
        for conv in blk:
            x, _, (b_, oh, ow) = conv(x, sh)
            sh = (b_, oh, ow, conv.cout)
        feats.append((x, sh))
    cat = torch.empty((40 * 36, 2 * net.fpn_channels), dtype=torch.float16, device=cuda)
    c0 = 0
    for (f, fs), de in zip(feats, net.deblocks):
        de(f, fs, out_split=cat, out_channels=net.fpn_channels, out_c0=c0)
        c0 += de.cout
    want, _, _ = net.shared(cat, (1, 40, 36, net.fpn_channels))
    torch.cuda.synchronize()
    assert shape == (1, 40, 36, 64) and torch.equal(s, want)


def _hot(cuda, n):
    from paddle3d_b200 import pointpillars as pp
    from paddle3d_b200 import synth
    hot = pp.PointPillarsHotPath(device=cuda, seed=1, num_points=n, bn_gain=BN_GAIN)
    pts = synth.lidar_cloud(synth.C2, 3, num_points=n)
    hot.calibrate_head(_t(cuda, pts))
    return hot, pts


def test_frame_graph_replay_equals_eager(cuda):
    hot, pts = _hot(cuda, 20000)
    host = torch.from_numpy(pts).pin_memory()
    eager = [t.clone() for t in hot.infer(host)]
    hot.capture()
    for _ in range(2):
        got = hot.infer(host)
        assert len(eager[0]) > 0
        for g, e in zip(got, eager):
            assert torch.equal(g, e)
    lanes = [r for r in hot.infer_many([host, host, host])]
    for r in lanes:
        for g, e in zip(r, eager):
            assert torch.equal(g, e)


@pytest.mark.parametrize("n", [3000, 20000])
def test_frame_matches_cpu_arm(cuda, oracle_mod, n):
    hot, pts = _hot(cuda, n)
    boxes, scores, labels = [t.clone().numpy() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    m = hot.model
    cpu = opp.CpuPointPillars(m.cfg, m.export_numpy(), m.anchors_np, m.corners_np, m.grid, m.mc["test"]).run(pts)
    nv = int(hot.out["num_voxels"][0])
    assert nv == cpu["num_voxels"]
    assert np.array_equal(hot.out["coors"][:nv].cpu().numpy(), cpu["coors"])
    planes = hot.out["planes"].cpu().numpy()
    e = rel_errors(planes, cpu["planes"])
    assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
    # the frame's postprocess equals the oracle's on the frame's own head planes
    tc = m.mc["test"]
    coors = hot.out["coors"][:nv].cpu().numpy()
    r = opp.anchor_head_postprocess(planes, m.anchors_np, m.corners_np, coors, GRID, tc["post_center_limit_range"],
                                    tc["anchor_area_threshold"], tc["nms_score_threshold"], tc["nms_iou_threshold"],
                                    tc["nms_pre_max_size"], tc["nms_post_max_size"])
    np.testing.assert_allclose(boxes, r["boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(scores, r["scores"], rtol=1e-6, atol=0)
    # against the CPU arm end to end: head planes differ at the 1e-4 level, so only anchors within that of the score
    # threshold or of an IoU / top-k boundary may differ
    assert abs(len(boxes) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    if len(cpu["boxes"]):
        d = np.abs(cpu["boxes"][:, None, :3] - boxes[None, :, :3]).max(-1) if len(boxes) else np.full((len(cpu["boxes"]), 1), np.inf)
        matched = d.min(1) < 1e-2
        assert matched.mean() >= 0.95, matched.mean()
