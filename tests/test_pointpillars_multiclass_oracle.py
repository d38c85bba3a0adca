"""CPU: the two-class PointPillars model (pointpillars.CONFIG_PED_CYCLIST on synth.C2_PED_CYCLIST) and the multi-class
anchor-head oracle (oracle.pointpillars_multiclass: anchors_3d_stride_classes, anchor_head_postprocess), each against
an independent restatement: a direct meshgrid formula for the anchors, a torch restatement of VoxelNet.predict
(torch.sigmoid, torch.max over the classes, NMS through ops.nms_utils.rotate_nms_pcdet), and, with one class, the
single-class oracle (oracle.pointpillars)."""
import ctypes

import numpy as np
import torch

import oracle.pointpillars as opp
import oracle.pointpillars_multiclass as opm
from paddle3d_b200 import pointpillars as pp
from paddle3d_b200 import synth
from paddle3d_b200.ops import nms_utils
from test_pointpillars_oracle import GRID as CAR_GRID
from test_pointpillars_oracle import _frame as _car_frame
from test_pointpillars_oracle import _nms_fn

CFG = pp.CONFIG_PED_CYCLIST
PC = synth.C2_PED_CYCLIST
GRID = pp.grid_size(PC)
H, W, R, C = 248, 296, 4, 2


def _model():
    return pp.PointPillars(PC, CFG)


def test_multiclass_anchors_match_a_direct_meshgrid_formula(oracle_mod):
    f = np.float32
    assert GRID == (W, H)
    gens = CFG["anchors"]
    ys, xs, cs, rs = np.meshgrid(np.arange(H, dtype=f), np.arange(W, dtype=f), np.arange(C), np.arange(2), indexing="ij")
    size = np.asarray([g["sizes"] for g in gens], f)[cs]
    rot = np.asarray(gens[0]["rotations"], f)[rs]
    g = gens[0]
    want = np.stack([xs * f(g["strides"][0]) + f(g["offsets"][0]), ys * f(g["strides"][1]) + f(g["offsets"][1]),
                     np.full_like(xs, g["offsets"][2]), size[..., 0], size[..., 1], size[..., 2], rot], -1).reshape(-1, 7)
    assert want.shape == (H * W * 4, 7) == (293632, 7)
    model = _model()
    assert np.array_equal(opm.anchors_3d_stride_classes((1, H, W), gens), want)
    assert np.array_equal(model.anchors_np, want)
    # anchor (y * W + x) * 4 + 2 c + r: class c's size, rotation r
    for y, x, c, r in ((0, 0, 0, 0), (17, 5, 1, 1), (247, 295, 0, 1), (100, 200, 1, 0)):
        a = model.anchors_np[(y * W + x) * 4 + 2 * c + r]
        assert a[0] == f(x) * f(0.16) + f(0.08) and a[1] == f(y) * f(0.16) + f(-19.76) and a[2] == f(-1.465)
        assert tuple(a[3:6]) == tuple(np.asarray(gens[c]["sizes"], f)) and a[6] == f((0.0, 1.57)[r])
    assert np.array_equal(model.corners_np, opp.anchor_corners(want, PC["voxel_size"], PC["point_cloud_range"], GRID))
    assert model.head_channels == 44 and model.feat_hw == (H, W) and model.num_classes == 2


def test_flops_follow_the_stride_one_block():
    fl = _model().flops()
    hw = [H * W, H * W // 4, H * W // 16]
    mac = lambda n, cin, cout, k: 2.0 * n * cin * cout * k * k  # noqa: E731
    backbone = (mac(hw[0], 64, 64, 3) * 4 + mac(hw[1], 64, 128, 3) + mac(hw[1], 128, 128, 3) * 5 +
                mac(hw[2], 128, 256, 3) + mac(hw[2], 256, 256, 3) * 5)
    fpn = mac(hw[0], 64, 128, 1) + mac(hw[0], 128, 128, 1) + mac(hw[0], 256, 128, 1)  # every deblock writes 248 x 296
    assert fl == dict(backbone=backbone, fpn=fpn, head=mac(hw[0], 384, 44, 1))


def test_num_classes_below_one_is_invalid():
    """Rejected before any CUDA call (dummy 16-byte aligned pointers are never touched)."""
    from paddle3d_b200 import _lib
    L = _lib.lib()
    p = ctypes.c_void_p(256)
    pcr = _lib.host_floats(PC["point_cloud_range"])
    for nc in (0, -1):
        assert L.p3d_anchor_head_postprocess(p, H, W, R, nc, p, p, None, None, 0, W, H, 1, 0.05, 0.5, 1000, 300, pcr, p,
                                             p, p, p, None, None, None, p, 1 << 30, None) == -1


def _mc_frame(seed, cls_mean, occupancy=0.3, tie=False):
    """Random two-class head planes at 248 x 296 and random pillars.  tie=True: quarter-step logits (exact score ties
    across anchors) and identical logits in both class planes on every third row (ties across the classes of one anchor).
    Otherwise logits of the two classes of an anchor are kept at least 9e-4 apart, far more than the exp rounding
    difference between implementations, so the label does not depend on it."""
    rng = np.random.default_rng(seed)
    head = np.empty((1, R * (C + 9), H, W), np.float32)
    cls = rng.normal(cls_mean, 1.0, size=(R, C, H, W)).astype(np.float32)
    if tie:
        cls = np.round(cls * 4) / 4
        cls[:, 1, ::3] = cls[:, 0, ::3]
    else:
        close = np.abs(cls[:, 1] - cls[:, 0]) < 1e-4
        cls[:, 1][close] += np.float32(1e-3)
    head[0, :R * C] = cls.reshape(R * C, H, W)
    head[0, R * C:R * (C + 7)] = rng.normal(0, 0.3, size=(R * 7, H, W))
    head[0, R * (C + 7):] = rng.normal(0, 1, size=(R * 2, H, W))
    head[0, R * (C + 7), :5, :5] = head[0, R * (C + 7) + 1, :5, :5]  # dir ties
    cells = rng.choice(H * W, size=int(occupancy * H * W), replace=False)
    coords = np.stack([np.zeros_like(cells), np.zeros_like(cells), cells // W, cells % W], 1).astype(np.int32)
    return head, coords


MC_FRAMES = [
    (0, -4.0, 0.3, False),    # > 1000 candidates
    (1, -2.0, 0.3, True),     # > 1000 candidates, exact ties across anchors and across the classes of one anchor
    (4, -1.0, 0.05, False),   # sparse pillars: most anchors masked
    (2, -30.0, 0.3, False),   # no candidate: empty output
    (3, 0.0, 0.0, False),     # no pillar: every anchor masked
]


def _torch_predict(oracle_mod, head, anchors, corners, coords, tc, num_classes):
    """VoxelNet.predict restated in torch (fp32): integral-image mask, torch.sigmoid and torch.max over the classes (ties
    to the lowest class), stable descending argsort and NMS inside rotate_nms_pcdet, decode, direction fix, range
    filter.  Returns (boxes, scores, labels, candidates)."""
    nx, ny = GRID
    m = torch.zeros((ny, nx), dtype=torch.int64)
    c = torch.from_numpy(coords).long()
    m.index_put_((c[:, 2], c[:, 3]), torch.ones(len(c), dtype=torch.int64), accumulate=True)
    s = m.cumsum(0).cumsum(1)
    k = torch.from_numpy(corners).long()
    area = s[k[:, 3], k[:, 2]] - s[k[:, 3], k[:, 0]] - s[k[:, 1], k[:, 2]] + s[k[:, 1], k[:, 0]]
    h = torch.from_numpy(head)[0]
    nc = num_classes
    r = h.shape[0] // (nc + 9)
    cls = h[:r * nc].reshape(r, nc, *h.shape[1:]).permute(2, 3, 0, 1).reshape(-1, nc)
    box = h[r * nc:r * (nc + 7)].reshape(r, 7, *h.shape[1:]).permute(2, 3, 0, 1).reshape(-1, 7)
    dirs = h[r * (nc + 7):].reshape(r, 2, *h.shape[1:]).permute(2, 3, 0, 1).reshape(-1, 2)
    score, label = torch.max(torch.sigmoid(cls), dim=-1)
    a = torch.from_numpy(anchors)
    idx = torch.nonzero((area > tc["anchor_area_threshold"]) & (score >= tc["nms_score_threshold"])).reshape(-1)
    sc, lb, bt, an, dl = score[idx], label[idx], box[idx], a[idx], torch.argmax(dirs[idx], dim=1)
    za = an[:, 2] + an[:, 5] * 0.5
    diag = torch.sqrt(an[:, 4] * an[:, 4] + an[:, 3] * an[:, 3])
    hh = torch.exp(bt[:, 5]) * an[:, 5]
    dec = torch.stack([bt[:, 0] * diag + an[:, 0], bt[:, 1] * diag + an[:, 1], (bt[:, 2] * an[:, 5] + za) - hh * 0.5,
                       torch.exp(bt[:, 3]) * an[:, 3], torch.exp(bt[:, 4]) * an[:, 4], hh, bt[:, 6] + an[:, 6]], 1)
    sel = nms_utils.rotate_nms_pcdet(dec, sc, tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"],
                                     nms_fn=_nms_fn(oracle_mod))
    out, scores, labels, d = dec[sel].clone(), sc[sel], lb[sel], dl[sel]
    flip = (out[:, 6] > 0) ^ d.bool()
    out[flip, 6] = out[flip, 6] + np.float32(np.pi)
    lo, hi = torch.tensor(tc["post_center_limit_range"][:3]), torch.tensor(tc["post_center_limit_range"][3:])
    ok = ((out[:, :3] >= lo) & (out[:, :3] <= hi)).all(1)
    return out[ok].numpy(), scores[ok].numpy(), labels[ok].numpy(), len(idx)


def test_multiclass_postprocess_matches_a_torch_restatement(oracle_mod):
    model = _model()
    tc = CFG["test"]
    args = (model.anchors_np, model.corners_np)
    seen = dict(over_pre=False, anchor_ties=False, class_ties=False, both_labels=False, empty=False, no_pillar=False)
    for seed, cls_mean, occ, tie in MC_FRAMES:
        head, coords = _mc_frame(seed, cls_mean, occ, tie)
        r = opm.anchor_head_postprocess(head, *args, coords, GRID, tc["post_center_limit_range"],
                                        tc["anchor_area_threshold"], tc["nms_score_threshold"], tc["nms_iou_threshold"],
                                        tc["nms_pre_max_size"], tc["nms_post_max_size"], num_classes=C)
        wb, ws, wl, ncand = _torch_predict(oracle_mod, head, *args, coords, tc, C)
        assert r["candidates"] == ncand
        assert len(r["boxes"]) == len(wb)
        np.testing.assert_allclose(r["scores"], ws, rtol=1e-6)  # torch.sigmoid differs from 1 / (1 + exp(-x)) by an ulp
        np.testing.assert_allclose(r["boxes"], wb, rtol=1e-6, atol=1e-6)
        assert r["labels"].dtype == np.int64 and np.array_equal(r["labels"], wl)
        seen["over_pre"] |= ncand > tc["nms_pre_max_size"]
        seen["anchor_ties"] |= tie and len(np.unique(r["cand_scores"])) < len(r["cand_scores"])
        if tie:  # candidates whose two class logits are equal (label 0 in both restatements)
            cls = head[0, :R * C].reshape(R, C, H, W).transpose(2, 3, 0, 1).reshape(-1, C)
            cand = r["mask"] & (1.0 / (1.0 + np.exp(-cls.max(1).astype(np.float64))) >= tc["nms_score_threshold"])
            seen["class_ties"] |= int((cand & (cls[:, 0] == cls[:, 1])).sum()) > 100
        seen["both_labels"] |= set(r["labels"].tolist()) == {0, 1}
        seen["empty"] |= ncand == 0 and occ > 0
        if occ == 0.0:
            assert not r["mask"].any() and len(r["boxes"]) == 0
            seen["no_pillar"] = True
    assert all(seen.values()), seen


def test_one_class_equals_the_single_class_oracle(oracle_mod):
    """num_classes=1 (the default) gives oracle.pointpillars' results bit for bit on the car frames, labels all 0; and
    one generator through anchors_3d_stride_classes gives the car anchors."""
    model = pp.PointPillars()
    a = pp.CONFIG["anchor"]
    assert np.array_equal(opm.anchors_3d_stride_classes((1, 248, 216), [a]),
                          opp.anchors_3d_stride((1, 248, 216), a["sizes"], a["strides"], a["offsets"], a["rotations"]))
    tc = pp.CONFIG["test"]
    for seed, cls_mean, occ, tie in ((0, -4.0, 0.3, False), (1, -2.0, 0.3, True), (2, -9.0, 0.3, False),
                                     (3, 0.0, 0.0, False)):
        head, coords = _car_frame(seed, cls_mean, occ, tie)
        args = (head, model.anchors_np, model.corners_np, coords, CAR_GRID, tc["post_center_limit_range"],
                tc["anchor_area_threshold"], tc["nms_score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"],
                tc["nms_post_max_size"])
        want = opp.anchor_head_postprocess(*args)
        for got in (opm.anchor_head_postprocess(*args), opm.anchor_head_postprocess(*args, num_classes=1)):
            for key, v in want.items():
                g = got[key]
                assert type(g) is type(v) and np.array_equal(g, v), key
                if isinstance(v, np.ndarray):
                    assert g.dtype == v.dtype and g.shape == v.shape, key
            assert np.array_equal(got["cand_labels"], np.zeros(len(want["cand_scores"]), np.int64))
