"""CPU: the PointPillars anchor-head oracle (oracle.pointpillars: anchors_3d_stride / anchor_corners / anchor_areas /
anchor_head_postprocess) and the model's host-side anchor tables, each against an independent restatement: a direct
meshgrid formula, brute-force counting, and a torch restatement of VoxelNet.predict that runs the NMS through
ops.nms_utils.rotate_nms_pcdet."""
import numpy as np
import torch

import oracle.pointpillars as opp
from paddle3d_b200 import pointpillars as pp
from paddle3d_b200 import synth
from paddle3d_b200.ops import nms_utils

CFG = pp.CONFIG
GRID = pp.grid_size(synth.C2)


def _anchor_args():
    a = CFG["anchor"]
    return a["sizes"], a["strides"], a["offsets"], a["rotations"]


def test_anchors_match_a_direct_meshgrid_formula(oracle_mod):
    f = np.float32
    sizes, strides, offsets, rots = _anchor_args()
    H, W = 248, 216
    ys, xs, rs = np.meshgrid(np.arange(H, dtype=f), np.arange(W, dtype=f), np.asarray(rots, f), indexing="ij")
    want = np.stack([xs * f(strides[0]) + f(offsets[0]), ys * f(strides[1]) + f(offsets[1]),
                     np.full_like(xs, offsets[2]), np.full_like(xs, sizes[0]), np.full_like(xs, sizes[1]),
                     np.full_like(xs, sizes[2]), rs], -1).reshape(-1, 7)
    assert want.shape == (107136, 7)
    got_oracle = opp.anchors_3d_stride((1, H, W), sizes, strides, offsets, rots)
    model = pp.PointPillars()
    assert np.array_equal(got_oracle, want)
    assert np.array_equal(model.anchors_np, want)
    # anchor (y * W + x) * 2 + a sits at cell (y, x) with rotation a
    i = (17 * W + 5) * 2 + 1
    assert model.anchors_np[i, 0] == f(5) * f(0.32) + f(0.16) and model.anchors_np[i, 6] == f(1.57)
    assert np.array_equal(model.corners_np, opp.anchor_corners(want, synth.C2["voxel_size"],
                                                                      synth.C2["point_cloud_range"], GRID))


def test_anchor_area_matches_brute_force_counting(oracle_mod):
    rng = np.random.default_rng(3)
    nx, ny = GRID
    cells = rng.choice(nx * ny, size=12000, replace=False)
    coords = np.stack([np.zeros_like(cells), np.zeros_like(cells), cells // nx, cells % nx], 1).astype(np.int32)
    anchors = pp.PointPillars().anchors_np
    corners = opp.anchor_corners(anchors, synth.C2["voxel_size"], synth.C2["point_cloud_range"], GRID)
    # the corners reach both grid edges (clamped) and both rotations swap the near box
    assert corners[:, 0].min() == 0 and corners[:, 2].max() == nx - 1 and corners[:, 1].min() == 0
    assert corners[:, 3].max() == ny - 1
    assert not np.array_equal(corners[0::2, 2] - corners[0::2, 0], corners[1::2, 2] - corners[1::2, 0])
    areas = opp.anchor_areas(coords, corners, GRID)
    pick = np.concatenate([rng.choice(len(anchors), 3000, replace=False), np.arange(40), np.arange(len(anchors) - 40, len(anchors))])
    y, x = coords[:, 2], coords[:, 3]
    for i in pick:  # integral image counts y in (y_min, y_max], x in (x_min, x_max]
        c = corners[i]
        want = int(((x > c[0]) & (x <= c[2]) & (y > c[1]) & (y <= c[3])).sum())
        assert areas[i] == want, (i, areas[i], want)


def _nms_fn(oracle_mod):
    def fn(boxes, thresh):
        keep, n = oracle_mod.nms(boxes.numpy(), thresh)
        return torch.from_numpy(np.asarray(keep, np.int64)), torch.tensor([n], dtype=torch.int64)
    return fn


def _torch_predict(oracle_mod, head, anchors, corners, coords, tc):
    """VoxelNet.predict restated in torch (fp32): integral-image mask, sigmoid, stable descending argsort inside
    rotate_nms_pcdet, decode, direction fix, range filter."""
    nx, ny = GRID
    m = torch.zeros((ny, nx), dtype=torch.int64)
    c = torch.from_numpy(coords).long()
    m.index_put_((c[:, 2], c[:, 3]), torch.ones(len(c), dtype=torch.int64), accumulate=True)
    s = m.cumsum(0).cumsum(1)
    k = torch.from_numpy(corners).long()
    area = s[k[:, 3], k[:, 2]] - s[k[:, 3], k[:, 0]] - s[k[:, 1], k[:, 2]] + s[k[:, 1], k[:, 0]]
    h = torch.from_numpy(head)[0]
    R = h.shape[0] // 10
    cls = h[:R].permute(1, 2, 0).reshape(-1)
    box = h[R:8 * R].reshape(R, 7, *h.shape[1:]).permute(2, 3, 0, 1).reshape(-1, 7)
    dirs = h[8 * R:].reshape(R, 2, *h.shape[1:]).permute(2, 3, 0, 1).reshape(-1, 2)
    a = torch.from_numpy(anchors)
    keep = (area > tc["anchor_area_threshold"]) & (torch.sigmoid(cls) >= tc["nms_score_threshold"])
    idx = torch.nonzero(keep).reshape(-1)
    sc, bt, an, dl = torch.sigmoid(cls)[idx], box[idx], a[idx], torch.argmax(dirs[idx], dim=1)
    za = an[:, 2] + an[:, 5] * 0.5
    diag = torch.sqrt(an[:, 4] * an[:, 4] + an[:, 3] * an[:, 3])
    hh = torch.exp(bt[:, 5]) * an[:, 5]
    dec = torch.stack([bt[:, 0] * diag + an[:, 0], bt[:, 1] * diag + an[:, 1], (bt[:, 2] * an[:, 5] + za) - hh * 0.5,
                       torch.exp(bt[:, 3]) * an[:, 3], torch.exp(bt[:, 4]) * an[:, 4], hh, bt[:, 6] + an[:, 6]], 1)
    sel = nms_utils.rotate_nms_pcdet(dec, sc, tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"],
                                     nms_fn=_nms_fn(oracle_mod))
    out, scores, d = dec[sel].clone(), sc[sel], dl[sel]
    flip = (out[:, 6] > 0) ^ d.bool()
    out[flip, 6] = out[flip, 6] + np.float32(np.pi)
    lo, hi = torch.tensor(tc["post_center_limit_range"][:3]), torch.tensor(tc["post_center_limit_range"][3:])
    ok = ((out[:, :3] >= lo) & (out[:, :3] <= hi)).all(1)
    return out[ok].numpy(), scores[ok].numpy(), len(idx)


def _frame(seed, cls_mean, occupancy=0.3, tie=False):
    """Random head planes at 248 x 216 and random pillars; tie=True repeats a handful of cls values exactly."""
    rng = np.random.default_rng(seed)
    nx, ny = GRID
    head = np.empty((1, 20, 248, 216), np.float32)
    head[0, :2] = rng.normal(cls_mean, 1.0, size=(2, 248, 216))
    if tie:
        head[0, :2] = np.round(head[0, :2] * 4) / 4  # quarter steps: many exact ties in score
    head[0, 2:16] = rng.normal(0, 0.3, size=(14, 248, 216))
    head[0, 16:] = rng.normal(0, 1, size=(4, 248, 216))
    head[0, 16, :5, :5] = head[0, 17, :5, :5]  # dir ties
    cells = rng.choice(nx * ny, size=int(occupancy * nx * ny), replace=False)
    coords = np.stack([np.zeros_like(cells), np.zeros_like(cells), cells // nx, cells % nx], 1).astype(np.int32)
    return head, coords


def test_postprocess_matches_a_torch_restatement(oracle_mod):
    model = pp.PointPillars()
    tc = CFG["test"]
    args = (model.anchors_np, model.corners_np)
    seen = dict(over_pre=False, ties=False, empty=False)
    for seed, cls_mean, occ, tie in ((0, -4.0, 0.3, False), (1, -2.0, 0.3, True), (2, -9.0, 0.3, False),
                                     (3, 0.0, 0.0, False)):
        head, coords = _frame(seed, cls_mean, occ, tie)
        r = opp.anchor_head_postprocess(head, *args, coords, GRID, tc["post_center_limit_range"],
                                        tc["anchor_area_threshold"], tc["nms_score_threshold"],
                                        tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"])
        wb, ws, ncand = _torch_predict(oracle_mod, head, *args, coords, tc)
        assert r["candidates"] == ncand
        assert len(r["boxes"]) == len(wb)
        np.testing.assert_allclose(r["scores"], ws, rtol=1e-6)  # torch.sigmoid differs from 1 / (1 + exp(-x)) by an ulp
        np.testing.assert_allclose(r["boxes"], wb, rtol=1e-6, atol=1e-6)
        seen["over_pre"] |= ncand > tc["nms_pre_max_size"]
        seen["ties"] |= tie and len(np.unique(r["cand_scores"])) < len(r["cand_scores"])
        seen["empty"] |= ncand == 0
        if occ == 0.0:
            assert not r["mask"].any() and len(r["boxes"]) == 0
    assert all(seen.values()), seen
