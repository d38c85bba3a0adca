"""GPU: the two-class PointPillars model (pointpillars.CONFIG_PED_CYCLIST on synth.C2_PED_CYCLIST) - the multi-class
anchor-head postprocess kernel against the numpy oracle (labels equal), the dense convs at the full-resolution
248 x 296 shapes only this model uses against the fp64 oracle, and the captured frame against eager execution and
against the CPU arm."""
import numpy as np
import pytest
import torch

import oracle.pointpillars_multiclass as opm
from parity import rel_check, rel_errors
from test_pointpillars_multiclass_oracle import C, GRID, MC_FRAMES, _mc_frame

pytestmark = pytest.mark.gpu
BN_GAIN = 6.0 ** 0.5


def _t(dev, a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


@pytest.fixture(scope="module")
def model(cuda):
    from paddle3d_b200 import pointpillars as pp
    from paddle3d_b200 import synth
    return pp.PointPillars(synth.C2_PED_CYCLIST, pp.CONFIG_PED_CYCLIST).init_weight(seed=1, device=cuda)


@pytest.mark.parametrize("seed,cls_mean,occ,tie", MC_FRAMES)
def test_multiclass_postprocess_vs_oracle(cuda, oracle_mod, model, seed, cls_mean, occ, tie):
    from paddle3d_b200.ops import nms_utils
    tc = model.mc["test"]
    head, coords = _mc_frame(seed, cls_mean, occ, tie)
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
    r = opm.anchor_head_postprocess(head, model.anchors_np, model.corners_np, coords, GRID,
                                    tc["post_center_limit_range"], tc["anchor_area_threshold"],
                                    tc["nms_score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"],
                                    tc["nms_post_max_size"], num_classes=C)
    assert np.array_equal(mask.cpu().numpy().astype(bool), r["mask"])
    ncand, k = [int(v) for v in counts.cpu()]
    assert ncand == r["candidates"] and k == len(r["boxes"])
    n = min(ncand, tc["nms_pre_max_size"])
    np.testing.assert_allclose(sb[:n].cpu().numpy(), r["cand_boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(ss[:n].cpu().numpy(), r["cand_scores"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(boxes[:k].cpu().numpy(), r["boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(scores[:k].cpu().numpy(), r["scores"], rtol=1e-6, atol=0)
    assert np.array_equal(labels[:k].cpu().numpy(), r["labels"])
    # NMS is class-agnostic: the keep list equals rotate_nms_pcdet's on the kernel's own thresholded, decoded candidates
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
    if k > 50:
        assert set(r["labels"].tolist()) == {0, 1}
    if tie:
        assert len(np.unique(r["cand_scores"])) < n
    if occ == 0.0:
        assert k == 0 and not mask.bool().any()


@pytest.mark.parametrize("cin,cout,k,stride,pad,up,h,w", [
    (64, 64, 3, 1, 1, 1, 248, 296),    # first block at stride 1: full-resolution 3x3
    (64, 128, 3, 2, 1, 1, 248, 296),   # second block's strided conv from the full-resolution map
    (256, 128, 4, 4, 0, 4, 62, 74),    # up-4 transposed conv of the last block
])
def test_dense_conv_at_ped_cyclist_shapes(cuda, oracle_mod, cin, cout, k, stride, pad, up, h, w):
    from paddle3d_b200.dense_head import _Conv
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(cin * 7 + cout + stride)
    x = rng.normal(size=(1, cin, h, w)).astype(np.float32)
    transposed = up > 1
    conv = _Conv(cin, cout, k, stride, pad, bn_eps=1e-3, up=up, transposed=transposed).init(rng, cuda, randomize_bn=True)
    p = conv.np
    ref = (oracle_mod.deconv2d(x, p["weight"], None, up) if transposed else
           oracle_mod.conv2d(x, p["weight"], None, stride, pad))
    bn = p["bn"]
    ref = oracle_mod.bn2d_relu(ref, bn["gamma"], bn["beta"], bn["mean"], bn["var"], bn["eps"])
    _, o, _ = conv(dc.nchw_to_pixel_h16(_t(cuda, x)), (1, h, w, cin), want_nchw=True)
    torch.cuda.synchronize()
    assert o.shape == ref.shape
    rel_check("ped/cyclist dense %d->%d k%d s%d up%d at %dx%d" % (cin, cout, k, stride, up, h, w), o.cpu().numpy(), ref)


def test_head_conv_384_to_44_fp32_planes(cuda, oracle_mod, model):
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(44)
    x = np.maximum(rng.normal(size=(1, 384, 248, 296)), 0).astype(np.float32)
    planes = model.head(dc.nchw_to_pixel_h16(_t(cuda, x)), (1, 248, 296, 384), want_nchw=True)[1]
    torch.cuda.synchronize()
    p = model.head.np
    assert tuple(planes.shape) == (1, 44, 248, 296)
    rel_check("ped/cyclist head 384->44", planes.cpu().numpy(), oracle_mod.conv2d(x, p["weight"], p["bias"], 1, 0))


def _hot(cuda, n):
    from paddle3d_b200 import pointpillars as pp
    from paddle3d_b200 import synth
    hot = pp.PointPillarsHotPath(synth.C2_PED_CYCLIST, device=cuda, seed=1, num_points=n, bn_gain=BN_GAIN,
                                 model_cfg=pp.CONFIG_PED_CYCLIST)
    pts = synth.lidar_cloud(synth.C2_PED_CYCLIST, 3, num_points=n)
    hot.calibrate_head(_t(cuda, pts))
    return hot, pts


def test_ped_cyclist_frame_graph_replay_equals_eager(cuda):
    hot, pts = _hot(cuda, 20000)
    host = torch.from_numpy(pts).pin_memory()
    eager = [t.clone() for t in hot.infer(host)]
    assert len(eager[0]) > 0 and set(eager[2].tolist()) == {0, 1}
    hot.capture()
    for _ in range(2):
        got = hot.infer(host)
        for g, e in zip(got, eager):
            assert torch.equal(g, e)
    for r in hot.infer_many([host, host, host]):
        for g, e in zip(r, eager):
            assert torch.equal(g, e)


def test_ped_cyclist_frame_matches_cpu_arm(cuda, oracle_mod):
    hot, pts = _hot(cuda, 20000)
    boxes, scores, labels = [t.clone().numpy() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    m = hot.model
    cpu = opm.CpuPointPillarsMulticlass(m.cfg, m.export_numpy(), m.anchors_np, m.corners_np, m.grid, m.mc["test"],
                                        m.num_classes).run(pts)
    nv = int(hot.out["num_voxels"][0])
    assert nv == cpu["num_voxels"]
    assert np.array_equal(hot.out["coors"][:nv].cpu().numpy(), cpu["coors"])
    planes = hot.out["planes"].cpu().numpy()
    assert planes.shape == (1, 44, 248, 296)
    e = rel_errors(planes, cpu["planes"])
    assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
    # the frame's postprocess equals the oracle's on the frame's own head planes
    tc = m.mc["test"]
    coors = hot.out["coors"][:nv].cpu().numpy()
    r = opm.anchor_head_postprocess(planes, m.anchors_np, m.corners_np, coors, GRID, tc["post_center_limit_range"],
                                    tc["anchor_area_threshold"], tc["nms_score_threshold"], tc["nms_iou_threshold"],
                                    tc["nms_pre_max_size"], tc["nms_post_max_size"], num_classes=m.num_classes)
    np.testing.assert_allclose(boxes, r["boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(scores, r["scores"], rtol=1e-6, atol=0)
    assert np.array_equal(labels, r["labels"])
    # against the CPU arm end to end: head planes differ at the 1e-4 level, so only anchors within that of the score
    # threshold, of an IoU / top-k boundary or of a class tie may differ
    assert set(cpu["labels"].tolist()) == {0, 1} and set(labels.tolist()) == {0, 1}
    assert abs(len(boxes) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    assert len(cpu["boxes"]) and len(boxes)
    d = np.abs(cpu["boxes"][:, None, :3] - boxes[None, :, :3]).max(-1)
    j = d.argmin(1)
    matched = d.min(1) < 1e-2
    assert matched.mean() >= 0.95, matched.mean()
    assert np.array_equal(cpu["labels"][matched], labels[j[matched]])
