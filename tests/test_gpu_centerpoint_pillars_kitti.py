"""GPU: CenterPoint-pillars KITTI (synth.CP_PILLARS_KITTI with centerpoint_pillars.CONFIG_KITTI: 100 points per pillar,
no velocity head, two tasks, the head at 248 x 216).

  * the wide two-layer pillar encoder (p3d_pillar_feature_net2_wide) against the fp64 oracle at M = 65, 100 and 128,
    with padding rows deciding maxima, far pillars and rows past the count untouched, and bit-equal to
    p3d_pillar_feature_net2 on the inputs both accept;
  * hard_voxelize at P = 100 bit for bit against the reference's CPU op (oracle/_ref when built) and the oracle port, on a
    culled KITTI scan and on clouds whose pillars hold more than 100 and more than 400 points;
  * the full-size frame stage by stage (the chain of tests/test_gpu_pillar_frames_full_size.py), eager, captured and the
    hot path bit-equal;
  * the frame against the CPU arm (tests/centerpoint_pillars_kitti_oracle.py), seeded and with random BatchNorm
    statistics;
  * raw scans through infer_kitti / infer_kitti_many on one frame and on CenterPointSweep lanes, a .pdparams checkpoint
    and tools/infer_kitti.py --config centerpoint;
  * the nuScenes frame unchanged.

Lines starting with "POST" (pytest -s) give the measured counts, "MEM" each test's peak device memory and wall time."""
import hashlib
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

import bench
from conftest import ROOT
from paddle3d_b200 import checkpoint, kitti, synth
from parity import rel_check
from test_gpu_centerpoint_full_size import RTOL, _clean_status_and_peak_memory  # noqa: F401 (autouse)
from test_gpu_dense_schedule import _bits_equal
from test_gpu_head_fused_schedule import PLANE_TERMS, tap_sum_f32, tap_sum_ref, w2_image
from test_gpu_dense_schedule import check_images, conv_ref, epilogue, from_pixel_h16
from test_gpu_kitti import _bits, _png_header, _reduced, _scans
from test_gpu_pillar_frames_full_size import (_hard_voxelize_into, _run_chains, check_convs, check_pfn,
                                              check_pixel_image, check_voxelize, cp_chain_convs, cp_pillars_chain)

pytestmark = pytest.mark.gpu

CFG = synth.CP_PILLARS_KITTI
N_POINTS = CFG["num_points"]


def _kw(cuda, **kw):
    from paddle3d_b200.centerpoint_pillars import CONFIG_KITTI
    return dict(dict(cfg=CFG, model_cfg=CONFIG_KITTI, device=cuda, seed=0, bn_gain=bench.BN_GAIN), **kw)


def _hot(cuda, **kw):
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    return CenterPointPillarsHotPath(**_kw(cuda, **kw))


def _culled(seed=1):
    """A synth.kitti_raw_cloud scan culled on the host, NaN-padded to the frame's rows: (points [N_POINTS, 4], kept)."""
    cloud, c, shape = synth.kitti_raw_cloud(seed)
    planes = kitti.frustum_planes(c, shape)
    kept = kitti.remove_camera_invisible(cloud, planes)
    pts = np.full((N_POINTS, 4), np.nan, np.float32)
    pts[:len(kept)] = kept
    return pts, len(kept)


# ---------------------------------------------------------------------------------------------- wide pillar encoder
def _pfn_case(M, seed, F=4, n=600):
    """Voxels [n, M, F] with counts 1, M - 1, M and random ones, pillars at the near and far ends of the KITTI grid (the
    decoration's centre offsets up to 69 m), the two layers' parameters with random BatchNorm statistics and a shift
    that makes ReLU(BN(0)) of the padding rows the maximum of some channels."""
    rng = np.random.default_rng(seed)
    vs, pcr = CFG["voxel_size"], CFG["point_cloud_range"]
    cnt = rng.integers(1, M + 1, n).astype(np.int32)
    cnt[:3 * 20] = np.repeat([1, M - 1, M], 20)
    xs = np.where(rng.uniform(size=n) < 0.5, rng.integers(0, 8, n), rng.integers(424, 432, n))
    ys = rng.integers(0, 496, n)
    coors = np.stack([np.zeros(n), np.zeros(n), ys, xs], 1).astype(np.int32)
    vox = np.zeros((n, M, F), np.float32)
    for i in range(n):
        cx, cy = pcr[0] + (xs[i] + 0.5) * vs[0], pcr[1] + (ys[i] + 0.5) * vs[1]
        k = cnt[i]
        vox[i, :k, 0] = cx + rng.uniform(-0.08, 0.08, k)
        vox[i, :k, 1] = cy + rng.uniform(-0.08, 0.08, k)
        vox[i, :k, 2] = rng.uniform(-3, 1, k)
        vox[i, :k, 3] = rng.uniform(0, 1, k)
    layers = []
    for (fi, fo) in ((F + 5, 32), (64, 64)):
        layers.append(dict(weight=synth.kaiming_uniform(rng, (fi, fo), fi), gamma=rng.uniform(0.5, 1.5, fo).astype(np.float32),
                           beta=rng.uniform(-0.5, 1.0, fo).astype(np.float32),
                           mean=rng.uniform(-0.2, 0.2, fo).astype(np.float32),
                           var=rng.uniform(0.5, 1.5, fo).astype(np.float32), eps=1e-3))
    return vox, cnt, coors, layers


def _launch(fn, vox, cnt, coors, layers, n_valid, fill=np.nan):
    """A two-layer entry on device copies, into an output prefilled with `fill`, num_voxels = n_valid."""
    import torch

    from paddle3d_b200._lib import check, host_floats
    from paddle3d_b200._mem import ptr, stream
    from paddle3d_b200.ops import pillar_encoder as pe
    dev = torch.device("cuda:0")
    t = [torch.from_numpy(np.ascontiguousarray(a)).to(dev) for a in (vox, cnt, coors)]
    w = [torch.from_numpy(l["weight"]).to(dev) for l in layers]
    (s1, t1), (s2, t2) = [pe.fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], dev) for l in layers]
    n, M, F = vox.shape
    out = torch.full((n, 64), fill, dtype=torch.float32, device=dev)
    nv = torch.tensor([n_valid], dtype=torch.int32, device=dev)
    check(fn(ptr(t[0]), ptr(t[1]), ptr(t[2]), ptr(nv), n, M, F, 32, ptr(w[0]), ptr(s1), ptr(t1), 64, ptr(w[1]), ptr(s2),
             ptr(t2), host_floats(CFG["voxel_size"]), host_floats(CFG["point_cloud_range"]), ptr(out), stream(dev)),
          "pfn2")
    torch.cuda.synchronize()
    return out.cpu().numpy()


@pytest.mark.parametrize("M", [65, 100, 128])
def test_wide_pfn_matches_fp64(cuda, M):
    from oracle.centerpoint_pillars import _decorate, _linear_bn_relu, pillar_feature_net2

    from paddle3d_b200._lib import lib
    vox, cnt, coors, layers = _pfn_case(M, M)
    n = len(vox)
    got = _launch(lib().p3d_pillar_feature_net2_wide, vox, cnt, coors, layers, n - 17)
    want = pillar_feature_net2(vox, cnt, coors, layers, CFG["voxel_size"], CFG["point_cloud_range"])
    rel_check("wide PFN M=%d" % M, got[:n - 17], want[:n - 17], rtol=1e-4)
    assert np.isnan(got[n - 17:]).all(), "rows past the count were written"
    # the padding rows decide maxima: the max over the real rows alone differs in some channels of the first layer
    x = _linear_bn_relu(_decorate(vox, cnt, coors, CFG["voxel_size"], CFG["point_cloud_range"]), layers[0])
    real = np.arange(M)[None, :, None] < cnt[:, None, None]
    partial = cnt < M
    decided = (x.max(1) > np.where(real, x, -np.inf).max(1))[partial]
    assert decided.any(), "no channel where a padding row decides the layer-1 max"
    # through the op: M > 64 selects the wide entry
    import torch

    from paddle3d_b200.ops import pillar_encoder as pe
    dl = [dict(l, weight=torch.from_numpy(l["weight"]).to(cuda)) for l in layers]
    via_op = pe.pillar_feature_net2(torch.from_numpy(vox).to(cuda), torch.from_numpy(cnt).to(cuda),
                                    torch.from_numpy(coors).to(cuda), dl, CFG["voxel_size"], CFG["point_cloud_range"])
    assert np.array_equal(via_op.cpu().numpy().view(np.uint32), _launch(lib().p3d_pillar_feature_net2_wide, vox, cnt,
                                                                         coors, layers, n).view(np.uint32))


def test_wide_pfn_bit_equal_to_narrow(cuda):
    from paddle3d_b200._lib import lib
    vox, cnt, coors, layers = _pfn_case(64, 5, n=900)
    a = _launch(lib().p3d_pillar_feature_net2, vox, cnt, coors, layers, 900)
    b = _launch(lib().p3d_pillar_feature_net2_wide, vox, cnt, coors, layers, 900)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    vox, cnt, coors, layers = _pfn_case(20, 6, n=900)
    a = _launch(lib().p3d_pillar_feature_net2, vox, cnt, coors, layers, 850)
    b = _launch(lib().p3d_pillar_feature_net2_wide, vox, cnt, coors, layers, 850)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))


# ------------------------------------------------------------------------------------------------ voxelizer at P = 100
def _dense_cloud(seed):
    """A culled scan plus three stacks of points in one pillar each: 150, 450 and 1200 points (past P = 100 and past
    the 4 P = 400 arrivals hard_voxelize records per pillar), interleaved with the scan."""
    rng = np.random.default_rng(seed)
    pts, kept = _culled(seed)
    scan = pts[:kept]
    stacks = []
    for k, (x, y) in zip((150, 450, 1200), ((10.05, 0.05), (30.01, -5.1), (50.1, 20.02))):
        s = np.stack([x + rng.uniform(0, 0.15, k), y + rng.uniform(0, 0.15, k), rng.uniform(-2.5, 0.5, k),
                      rng.uniform(0, 1, k)], 1)
        stacks.append(s)
    cloud = np.concatenate([scan] + stacks, 0).astype(np.float32)
    return cloud[rng.permutation(len(cloud))]


@pytest.mark.parametrize("case", ["culled_scan", "over_capacity_pillars"])
def test_voxelize_p100(cuda, oracle_mod, case):
    import torch

    from paddle3d_b200.ops import voxelize as vox
    pts = _culled(3)[0] if case == "culled_scan" else _dense_cloud(4)
    if case == "culled_scan":
        pts = pts[~np.isnan(pts[:, 0])]
    pd = torch.from_numpy(pts).to(cuda)
    v, co, npv, nv = vox.hard_voxelize(pd, CFG["voxel_size"], CFG["point_cloud_range"], 100, CFG["max_voxels"])
    torch.cuda.synchronize()
    r = dict(voxels=v, co=co, npv=npv, nv=nv)
    k, at_max, one, most = check_voxelize(case, oracle_mod, r, pts, CFG)
    if oracle_mod.ref_lib("cpu") is not None:
        ref = oracle_mod.ref_hard_voxelize_cpu(pts, CFG["voxel_size"], CFG["point_cloud_range"], 100, CFG["max_voxels"])
        for g, w in zip((v, co, npv, nv), ref):
            assert np.array_equal(g.cpu().numpy().view(np.uint32), np.asarray(w).view(np.uint32)), case
    else:
        print("POST voxelize %s: oracle/_ref not built, checked against the oracle port only" % case)
    again = _hard_voxelize_into(pd, CFG, 0xFF)
    torch.cuda.synchronize()
    assert torch.equal(again[0].view(torch.int32), v.view(torch.int32))
    print("POST voxelize %s: %d points, %d pillars, %d at 100 points, %d with one, most %d" % (
        case, len(pts), k, at_max, one, most))
    # measured: the culled scan's fullest pillar holds 35 points; the stacks fill three pillars to 100
    want = {"culled_scan": (13551, 4671, 0, 1564, 35), "over_capacity_pillars": (16362, 4581, 3, 1465, 100)}[case]
    assert (len(pts), k, at_max, one, most) == want


# ------------------------------------------------------------------------------------------------- full-size frame
def _bench_frame(cuda, **kw):
    import torch
    pts, kept = _culled(1)
    pts_d = torch.from_numpy(pts).to(cuda)
    hot = _hot(cuda, **kw)
    hot.calibrate_head(pts_d)
    hot.points.copy_(pts_d)
    return hot, pts, pts_d, kept


def _check_fused_head(name, d, r):
    """The fused head's 19 planes against the tap-sum reference of the float64 ConvModule output, and bit for bit the
    fp32 tap sum of the P buffer the fused conv wrote."""
    import torch
    bp = r["bp"]
    heads = [(n, a, f) for hs in d.heads for n, a, f in hs]
    b, H, W, cin = r["head_shape"]
    wbig = torch.cat([torch.from_numpy(a.np["weight"]) for _, a, _ in heads], 0).to(r["planes"].device).double()
    acc, _ = conv_ref(from_pixel_h16(r["shared"], b, H, W, cin), wbig, 3, 1, 1, 1)
    mid = epilogue(acc, bp["big"].dev["scale"], bp["big"].dev["shift"], True)
    del acc, wbig
    P = torch.stack([torch.einsum("bhwc,cn->bhwn", mid[..., 64 * g:64 * (g + 1)],
                                  w2_image(torch.from_numpy(f.np["weight"]).to(mid.device).double()))
                     for g, (_, _, f) in enumerate(heads)], 1)
    del mid
    p9, c9 = [int(v) for v in bp["plane0_9"]], [int(v) for v in bp["cnt9"]]
    want = tap_sum_ref(P, bp["bias9"], p9, c9, bp["planes"])
    del P
    assert want.shape[1] == 19
    check_images("%s fused head planes" % name, r["planes"], want, PLANE_TERMS)
    assert _bits_equal(r["planes"], tap_sum_f32(r["P"], bp["bias9"], p9, c9, bp["planes"])), name


def _check_post(name, oracle_mod, m, r):
    """oracle.centerpoint_postprocess (without velocity) of the actual planes.  Returns (passing cells, boxes) per task."""
    h = {k: [t.cpu().numpy() for t in v] for k, v in r["heads"].items()}
    assert "vel" not in h
    cfg, tc = m.cfg, m.test_cfg
    wb, ws, wl, wc = oracle_mod.centerpoint_postprocess(
        h["hm"], h["reg"], h["height"], h["dim"], h["reg"], h["rot"], cfg["voxel_size"][:2], cfg["point_cloud_range"],
        tc["post_center_limit_range"], m.label_off, tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
        tc["nms_pre_max_size"], tc["nms_post_max_size"], False)
    boxes, scores, labels, counts = (t.cpu().numpy() for t in r["post"])
    k = int(counts[-1])
    assert boxes.shape[1] == 7 and wb.shape[1] == 7
    assert np.array_equal(counts[:-1], wc) and k == len(wl), "%s: counts %s, oracle %s" % (name, counts, wc)
    assert np.array_equal(labels[:k], wl), "%s: labels / order" % name
    np.testing.assert_allclose(scores[:k], ws, rtol=RTOL)
    np.testing.assert_allclose(boxes[:k], wb, rtol=RTOL, atol=1e-5)
    passing = [int((1.0 / (1.0 + np.exp(-hm.astype(np.float64).max(1))) > tc["score_threshold"]).sum()) for hm in h["hm"]]
    return passing, [int(c) for c in wc]


def test_full_size_frame_stage_by_stage(cuda, oracle_mod):
    import torch
    from oracle.centerpoint_pillars import pillar_feature_net2
    hot, pts, pts_d, kept = _bench_frame(cuda)
    m = hot.model
    assert m.head.fused_heads(m.head._batched_params(cuda))  # 10 heads x 64 = 640 channels: the fused path
    hot.capture(count_nodes=True)
    want = [t.clone() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    assert want[0].shape[1] == 7 and hot.slot.shape[:2] == (166, 7)
    eager, captured, graph = _run_chains(cp_pillars_chain, hot, pts_d)
    for label, r in (("eager", eager), ("captured", captured)):
        assert not r["status"].any(), label
        assert _bits_equal(r["image"], eager["image"]), label
        for i, (a, b) in enumerate(zip(eager["convs"], r["convs"])):
            assert _bits_equal(a[3], b[3]), "%s chain: conv %d" % (label, i)
        for key, planes in hot.out["head"].items():
            for t, p in enumerate(planes):
                assert _bits_equal(r["heads"][key][t], p), "%s chain: %s task %d" % (label, key, t)
        boxes, scores, labels, counts = r["post"]
        k = int(counts[-1])
        assert k == len(want[2])
        assert _bits_equal(boxes[:k].cpu(), want[0]) and _bits_equal(scores[:k].cpu(), want[1])
        assert torch.equal(labels[:k].cpu(), want[2])
    del captured, graph
    torch.cuda.empty_cache()
    r = eager
    k, at_max, one, most = check_voxelize("kitti", oracle_mod, r, pts[~np.isnan(pts[:, 0])], CFG)
    w = pillar_feature_net2(r["voxels"][:k].cpu().numpy(), r["npv"][:k].cpu().numpy(), r["coors"][:k].cpu().numpy(),
                            m.pfn, CFG["voxel_size"], CFG["point_cloud_range"])
    check_pfn("kitti", r, w, True)
    occupied = check_pixel_image("kitti", m, r)
    assert [c for c, *_ in r["convs"]] == cp_chain_convs(m.head)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    check_convs("kitti", r, sms)
    _check_fused_head("kitti", m.head, r)
    passing, per_task = _check_post("kitti", oracle_mod, m, r)
    tc = m.test_cfg
    print("POST kitti frame: %d kept points, %d pillars (%d at 100 points, %d with one, most %d), %d occupied pixels; "
          "cells above the threshold per task %s (nms_pre %d cuts: %s); boxes per task %s (nms_post %d binds: %s); "
          "graph nodes %s" % (kept, k, at_max, one, most, occupied, passing, tc["nms_pre_max_size"],
                              max(passing) > tc["nms_pre_max_size"], per_task, tc["nms_post_max_size"],
                              max(per_task) == tc["nms_post_max_size"], hot.graph_nodes))
    # measured on an H100: scan 1 keeps 14 472 points in 3 904 pillars (none full); the calibration puts 751 of each
    # task's 53 568 cells above the threshold, so nms_pre (1000) never cuts and nms_post (83) binds in both tasks
    assert occupied == k and (kept, k, at_max, one, most) == (14472, 3904, 0, 1020, 49)
    assert passing == [751, 751] and max(passing) < tc["nms_pre_max_size"]
    assert per_task == [tc["nms_post_max_size"]] * 2 and sum(per_task) == len(want[2])
    assert hot.graph_nodes == {"kernel": 38, "memcpy": 1, "memset": 2, "other": 0}


# ------------------------------------------------------------------------------------------------ against the CPU arm
# the first 25.6 m of the KITTI range (a 160 x 160 grid): the CPU arm's dense part at full size takes minutes
SMALL = dict(CFG, point_cloud_range=[0.0, -12.8, -3.0, 25.6, 12.8, 1.0])


@pytest.mark.parametrize("bn", ["seeded", "random_bn"])
def test_frame_matches_cpu_arm(cuda, oracle_mod, bn):
    """The frame against the CPU arm as tests/test_gpu_centerpoint_pillars.py checks the nuScenes one: equal pillars, head
    planes on the parity bar, the frame's postprocess equal to the oracle's on its own planes, box counts within 2 %
    and 95 % of the CPU boxes paired with equal labels (the others sit at the score threshold or an NMS decision)."""
    import torch
    from centerpoint_pillars_kitti_oracle import CpuCenterPointPillarsHeads
    from parity import rel_errors
    from test_gpu_centerpoint_pillars import _pair
    pts, kept = _culled(2)
    hot = _hot(cuda, cfg=SMALL)
    if bn == "random_bn":
        rng = np.random.default_rng(11)
        sd = hot.state_dict()
        for key, v in sd.items():
            if key.endswith("._mean"):
                sd[key] = rng.uniform(-0.05, 0.05, v.shape).astype(np.float32)
            elif key.endswith("._variance"):
                sd[key] = rng.uniform(0.8, 1.2, v.shape).astype(np.float32)
        hot.load_state_dict(sd)
    else:
        hot.calibrate_head(torch.from_numpy(pts).to(cuda))
    m = hot.model
    got = [t.clone().numpy() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    cpu = CpuCenterPointPillarsHeads(SMALL, m.export_numpy(), m.test_cfg, m.label_off).run(pts[:kept])
    nv = int(hot.out["num_voxels"][0])
    assert nv == cpu["num_voxels"]
    assert np.array_equal(hot.out["coors"][:nv].cpu().numpy(), cpu["coors"])
    h = {k: [t.cpu().numpy() for t in v] for k, v in hot.out["head"].items()}
    assert sorted(h) == sorted(cpu["head"]) and "vel" not in h
    for name in h:
        for t, (g, w) in enumerate(zip(h[name], cpu["head"][name])):
            e = rel_errors(g, w)
            assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, (name, t, e)
    tc = m.test_cfg
    r = oracle_mod.centerpoint_postprocess(h["hm"], h["reg"], h["height"], h["dim"], h["reg"], h["rot"],
                                           SMALL["voxel_size"][:2], SMALL["point_cloud_range"],
                                           tc["post_center_limit_range"], m.label_off, tc["down_ratio"],
                                           tc["score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"],
                                           tc["nms_post_max_size"], False)
    assert got[0].shape[1] == cpu["boxes"].shape[1] == 7
    assert len(got[0]) == len(r[0]) > 0
    np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
    assert np.array_equal(got[2], r[2])
    assert abs(len(got[0]) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    frac = _pair(got, cpu)
    print("POST cpu arm %s: %d pillars, %d GPU / %d CPU boxes, %.3f of the CPU boxes paired" % (
        bn, nv, len(got[0]), len(cpu["boxes"]), frac))
    assert frac >= 0.95, frac


# ---------------------------------------------------------------------------------------------------------- raw scans
def test_raw_scans_lanes_and_checkpoint(cuda, tmp_path):
    import torch

    from paddle3d_b200 import frame
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    scans = _scans()
    ref = _hot(cuda)
    hot = _hot(cuda, sweep_input=frame.KITTI_INPUT)
    calib_pts = _reduced(scans[0][0], scans[0][3]).to(cuda)
    ref.calibrate_head(calib_pts)
    hot.share_model(ref)
    want = [tuple(t.clone() for t in ref.infer(_reduced(c, pl))) for c, _, _, pl in scans]
    assert sum(len(w[0]) for w in want) > 0 and all(w[0].shape[1] == 7 for w in want)
    assert _bits(hot.infer_kitti(scans[1][0], scans[1][3]), want[1])
    hot.capture(count_nodes=True)
    for j in range(len(scans)):  # one graph over six calibrations, image shapes and point counts
        assert _bits(hot.infer_kitti(scans[j][0], scans[j][3]), want[j]), j
    got = list(hot.infer_kitti_many((c, pl) for c, _, _, pl in scans))
    assert all(_bits(g, w) for g, w in zip(got, want))
    with pytest.raises(ValueError):  # larger than the raw capacity: refused before anything is enqueued
        hot.infer_kitti(np.zeros((frame.KITTI_INPUT["slot_cap"] + 1, 4), np.float32), scans[0][3])
    assert _bits(hot.infer_kitti(scans[2][0], scans[2][3]), want[2])
    lanes = CenterPointSweep(4, frame_cls=CenterPointPillarsHotPath, **_kw(cuda, sweep_input=frame.KITTI_INPUT))
    for p in lanes.lanes:
        p.share_model(ref)
        p.infer_kitti(scans[0][0], scans[0][3])
        p.capture()
    items = [(c, pl) for c, _, _, pl in scans] * 2
    got = list(lanes.infer_kitti_many(iter(items)))
    assert len(got) == len(items) and all(_bits(g, want[i % len(scans)]) for i, g in enumerate(got))
    del lanes
    # the calibrated model through a .pdparams file, into a model of another seed: same frame, head planes and graph
    path = tmp_path / "cp_kitti.pdparams"
    sd = dict(ref.state_dict())
    assert not [k for k in sd if ".vel." in k]
    sd[checkpoint.STRUCTURED_NAMES] = {k: "param_%d" % i for i, k in enumerate(ref.state_dict())}
    with open(path, "wb") as f:
        pickle.dump(sd, f, protocol=4)
    loaded = _hot(cuda, seed=7, weights=str(path), sweep_input=frame.KITTI_INPUT)
    loaded.infer_kitti(scans[0][0], scans[0][3])
    loaded.capture(count_nodes=True)
    assert loaded.graph_nodes == hot.graph_nodes
    for j in (0, 4):
        assert _bits(loaded.infer_kitti(scans[j][0], scans[j][3]), want[j]), j
        hot.infer_kitti(scans[j][0], scans[j][3])
        for key in hot.out["head"]:
            for a, b in zip(hot.out["head"][key], loaded.out["head"][key]):
                assert _bits_equal(a, b), key
    file_lanes = CenterPointSweep(2, frame_cls=CenterPointPillarsHotPath,
                                  **_kw(cuda, seed=5, weights=str(path), sweep_input=frame.KITTI_INPUT))
    for p in file_lanes.lanes:
        p.infer_kitti(scans[0][0], scans[0][3])
        p.capture()
    got = list(file_lanes.infer_kitti_many(iter(items)))
    assert all(_bits(g, want[i % len(scans)]) for i, g in enumerate(got))
    print("POST raw scans: boxes per scan %s, graph nodes %s" % ([len(w[0]) for w in want], hot.graph_nodes))
    del file_lanes, loaded
    torch.cuda.empty_cache()


def test_infer_kitti_cli_centerpoint(cuda, tmp_path):
    """tools/infer_kitti.py --config centerpoint writes the label files of to_kitti on the hot path's converted boxes."""
    from paddle3d_b200 import frame
    scans = _scans()[:3]
    root = tmp_path / "training"
    for d in ("velodyne", "calib", "image_2"):
        (root / d).mkdir(parents=True)
    ids = ["%06d" % i for i in range(len(scans))]
    calib_lines = synth.KITTI_CALIB.splitlines()
    for fid, (cloud, c, shape, _) in zip(ids, scans):
        cloud.tofile(root / "velodyne" / (fid + ".bin"))
        tr = " ".join("%.17g" % v for v in c["Tr_velo_to_cam"][:3].reshape(-1))
        (root / "calib" / (fid + ".txt")).write_text(
            "\n".join("Tr_velo_to_cam: " + tr if ln.startswith("Tr_velo_to_cam:") else ln for ln in calib_lines) + "\n")
        if shape != kitti.DEFAULT_IMAGE_SHAPE:
            _png_header(root / "image_2" / (fid + ".png"), *shape)
    hot = _hot(cuda, sweep_input=frame.KITTI_INPUT)
    hot.calibrate_head(_reduced(scans[0][0], scans[0][3]).to(cuda))
    path = tmp_path / "cp.pdparams"
    with open(path, "wb") as f:
        pickle.dump(dict(hot.state_dict()), f, protocol=4)
    out = tmp_path / "labels"
    r = subprocess.run([sys.executable, "tools/infer_kitti.py", "--model", str(path), "--config", "centerpoint", "--root",
                        str(root), "--out", str(out), "--lanes", "2"], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    n_lines = 0
    for fid, (cloud, _, shape, _) in zip(ids, scans):
        c = kitti.read_calib(root / "calib" / (fid + ".txt"))
        b, s, lab = hot.infer_kitti(cloud, kitti.frustum_planes(c, shape))
        want = kitti.format_label_lines(kitti.to_kitti(kitti.centerpoint_to_lidar_boxes(b.numpy()), s.numpy(),
                                                       lab.numpy(), c, shape, kitti.CLASS_NAMES["centerpoint"]))
        assert (out / (fid + ".txt")).read_text().splitlines() == want, fid
        n_lines += len(want)
    assert n_lines > 0
    assert sorted(os.listdir(out)) == sorted(i + ".txt" for i in ids)


# ---------------------------------------------------------------------------------------------------------- unchanged
# the nuScenes frame (seed 0, bench.BN_GAIN, head calibrated on bench.frame_pool(CP_PILLARS, 1)[0]) at the parent commit:
# its graph's node counts and a digest of its boxes, scores and labels on that cloud
NUSC_NODES = {"kernel": 38, "memcpy": 1, "memset": 2, "other": 0}
NUSC_DIGEST = "cbc5c0fb6799bafe84ea5368a43c02b17dbd33d8458ed1b4369483d4e7b65960"


def test_nuscenes_frame_unchanged(cuda):
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    pts = bench.frame_pool(synth.CP_PILLARS, 1)[0]
    hot = CenterPointPillarsHotPath(synth.CP_PILLARS, cuda, seed=0, bn_gain=bench.BN_GAIN)
    hot.calibrate_head(torch.from_numpy(pts).to(cuda))
    hot.capture(count_nodes=True)
    b, s, lab = hot.infer(torch.from_numpy(pts).pin_memory())
    h = hashlib.sha256()
    for t in (b, s, lab):
        h.update(t.numpy().tobytes())
    print("POST nuScenes frame: graph nodes %s, digest %s, boxes %d" % (hot.graph_nodes, h.hexdigest(), len(b)))
    assert b.shape[1] == 9
    assert hot.graph_nodes == NUSC_NODES
    assert h.hexdigest() == NUSC_DIGEST
