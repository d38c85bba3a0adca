#!/usr/bin/env python
"""Op-level roofline table for the HBM-bound ops of the hot path at their BASELINE.json configurations
(SURVEY.md §8d byte counts).  Each op call is captured into a CUDA graph and every replay is timed on its own with CUDA events on the
launching stream after an L2 flush (a 256 MB write), so neither cached inputs nor host launch gaps distort it.  Output: one JSON line per op.

    python tools/op_bench.py [--iters 30] [--only voxelize,scatter,bev_pool,nms,postprocess]
Under Nsight Compute, e.g.
    ncu --set full --clock-control none -k regex:'vox_write|scat_write|bev_fwd' -c 6 -o ops python tools/op_bench.py --iters 2
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from paddle3d_b200 import synth  # noqa: E402
from paddle3d_b200.ops import (bev_pool_v2, centerpoint_postprocess, iou3d_nms, pillar_encoder, pillar_scatter,  # noqa: E402
                               voxelize)


def timed(fn, iters, flush):
    """Device time of one call of `fn`: the call is captured into a CUDA graph (its launches then run back to back,
    without Python / ctypes gaps between them) and each replay is bracketed by events after an L2 flush."""
    st = torch.cuda.Stream()
    ts = []
    with torch.cuda.stream(st):
        for _ in range(3):
            fn()
        st.synchronize()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=st):
            fn()
        for _ in range(iters):
            # the flush is also what keeps the GPU busy while the host enqueues event + graph launch: with one 256 MB
            # write the replay could arrive after the start event had fired; three writes give the host slack
            for _ in range(3):
                flush.zero_()
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record(st)
            g.replay()
            e.record(st)
            e.synchronize()
            ts.append(s.elapsed_time(e) * 1e3)
    ts.sort()
    return ts[0], ts[len(ts) // 2]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--only", default="")
    ap.add_argument("--c3-only", action="store_true", help="voxelize: skip the KITTI config (for an ncu capture of the C3 launches)")
    args = ap.parse_args()
    only = set(x for x in args.only.split(",") if x)
    dev = torch.device("cuda:0")
    flush = torch.empty(256 * 2 ** 20, dtype=torch.uint8, device=dev)
    pk = os.path.join(ROOT, "MEASURED_PEAKS.json")
    peak = json.load(open(pk))["hbm_gbs"] if os.path.exists(pk) else 6650.0
    out = []

    def report(name, cfg, nbytes, fn, note=""):
        if only and name.split(":")[0] not in only:
            return
        mn, med = timed(fn, args.iters, flush)
        line = {"op": name, "config": cfg, "algorithmic_bytes": nbytes, "us_min": round(mn, 2), "us_median": round(med, 2),
                "achieved_gbs": round(nbytes / (med * 1e-6) / 1e9, 1), "peak_gbs": peak,
                "frac": round(nbytes / (med * 1e-6) / 1e9 / peak, 4), "note": note}
        out.append(line)
        print(json.dumps(line), flush=True)

    # hard_voxelize (whole op, 5 launches) — C2 and C3
    for cfg, gen in ((synth.C2, synth.lidar_cloud), (synth.C3, synth.lidar_cloud)):
        if args.c3_only and cfg is synth.C2:
            continue
        pts = torch.from_numpy(gen(cfg, 0)).to(dev)
        N, F, P, V = pts.shape[0], pts.shape[1], cfg["max_points"], cfg["max_voxels"]
        nbytes = 4 * N * F + 4 * V * P * F + 12 * V + 4 * V + 4
        report("voxelize:hard_voxelize", cfg["name"], nbytes,
               lambda: voxelize.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V),
               "whole op: vox_init+insert+rank+slots+write")
        report("voxelize:voxelize_mean", cfg["name"], 4 * N * F + 4 * V * F + 16 * V + 4 * V,
               lambda: voxelize.voxelize_mean(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V),
               "fused VoxelMean front end (no padded tensor)")
    # PillarScatter — C2: [nv, 64] -> [1, 64, 496, 432]
    cfg = synth.C2
    _, c_dev, _, nv_dev = voxelize.hard_voxelize(torch.from_numpy(synth.uniform_cloud(cfg, 1)).to(dev), cfg["voxel_size"],
                                                 cfg["point_cloud_range"], 4, 40000)
    k = int(nv_dev[0].item())
    coors = torch.cat([torch.zeros((k, 1), dtype=torch.int32, device=dev), c_dev[:k]], 1).contiguous()
    feats = torch.randn((k, 64), device=dev)
    report("scatter:pillar_scatter", "C2 nv=%d C=64 496x432" % k, 4 * k * 64 + 16 * k + 4 * 64 * 496 * 432,
           lambda: pillar_scatter.pillar_scatter(feats, coors, 1, 496, 432), "memset map + scat_map + scat_write")
    # to_dense_bev — C3 shape [n,128] -> [1,256,180,180]
    rng = np.random.default_rng(0)
    occ = np.argwhere(rng.random((1, 2, 180, 180)) < 0.09).astype(np.int32)
    f2 = torch.randn((len(occ), 128), device=dev)
    occ_dev = torch.from_numpy(occ).to(dev)
    report("scatter:sparse_to_dense_bev", "C3 n=%d C=128 2x180x180" % len(occ), 4 * len(occ) * 128 + 16 * len(occ) + 4 * 256 * 180 * 180,
           lambda: pillar_scatter.sparse_to_dense_bev(f2, occ_dev, 1, (2, 180, 180)))
    # bev_pool_v2 — C4 reference grid (128x128) and BASELINE grid (200x200)
    for grid, b in (((128, 128, 1), (-51.2, 51.2)), ((200, 200, 1), (-50.0, 50.0))):
        d = synth.bev_pool_inputs(5, grid=grid, bounds=(b, b, (-5.0, 3.0)))
        keys = ["depth", "feat", "ranks_depth", "ranks_feat", "ranks_bev", "interval_lengths", "interval_starts"]
        t = [torch.from_numpy(d[kk]).to(dev) for kk in keys]
        npts, nint = len(d["ranks_bev"]), len(d["interval_starts"])
        nbytes = 12 * npts + 4 * npts + 4 * d["feat"].size + 8 * nint + 4 * int(np.prod(d["bev_feat_shape"]))
        report("bev_pool:bev_pool_v2", "C4 grid %dx%d n_pts=%d n_int=%d C=80" % (grid[0], grid[1], npts, nint), nbytes,
               lambda: bev_pool_v2.bev_pool_v2(*t, d["bev_feat_shape"]), "memset + bev_fwd")
    # BASELINE.json config 4, camera branch: rank preparation (on the device, every frame) + bev_pool_v2 onto 200 x 200
    d = synth.bev_pool_inputs(5, grid=(200, 200, 1), bounds=((-50.0, 50.0), (-50.0, 50.0), (-5.0, 3.0)))
    coor_dev, depth_dev, feat_dev = [torch.from_numpy(d[kk]).to(dev) for kk in ("coor", "depth", "feat")]
    n_all = d["coor"].size // 3
    npts, nint = len(d["ranks_bev"]), len(d["interval_starts"])

    def camera_branch():
        rb, rd, rf, st_, ln, counts = bev_pool_v2.voxel_pooling_prepare_v2(coor_dev, d["grid_lower_bound"], d["grid_interval"],
                                                                            d["grid_size"])
        # capacity-sized arrays + the known interval count of this rig (a deployment reads counts once per calibration)
        return bev_pool_v2.bev_pool_v2(depth_dev, feat_dev, rd, rf, rb, ln[:nint], st_[:nint], d["bev_feat_shape"])
    report("c4:camera_branch prepare+bev_pool", "6 cams 16x44x118 -> 200x200x80, n_pts=%d kept=%d n_int=%d" % (n_all, npts, nint),
           12 * n_all + 20 * npts + 4 * npts + 4 * d["feat"].size + 8 * nint + 4 * int(np.prod(d["bev_feat_shape"])), camera_branch,
           "prep_rank + radix sort + gather + scan + starts + lengths + memset + bev_fwd_warp")
    report("c4:prepare only", "n_pts=%d" % n_all, 12 * n_all + 20 * npts,
           lambda: bev_pool_v2.voxel_pooling_prepare_v2(coor_dev, d["grid_lower_bound"], d["grid_interval"], d["grid_size"]))
    # configs 2 and 4 (LiDAR branch): hard_voxelize -> PillarFeatureNet -> PointPillarsScatter
    for cfg, hw, label in ((synth.C2, (496, 432), "c2:pointpillars voxelize+PFN+scatter"),
                           (synth.C4_LIDAR, (400, 400), "c4:lidar_branch voxelize+PFN+scatter")):
        pts = torch.from_numpy(synth.lidar_cloud(cfg, 0)).to(dev)
        N, F, P, V = pts.shape[0], pts.shape[1], cfg["max_points"], cfg["max_voxels"]
        rng = np.random.default_rng(1)
        w = torch.from_numpy((rng.normal(size=(F + 5, 64)) * 0.3).astype(np.float32)).to(dev)
        g_, b_, mu, var = np.ones(64), np.zeros(64), np.zeros(64), np.ones(64)
        folded = pillar_encoder.fold_bn(g_, b_, mu, var, 1e-3, dev)

        def chain():
            vox, co, npv, nv = voxelize.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
            coors4 = torch.cat([torch.zeros((V, 1), dtype=torch.int32, device=dev), co], 1)
            f = pillar_encoder.pillar_feature_net(vox, npv, coors4, w, g_, b_, mu, var, 1e-3, cfg["voxel_size"],
                                                  cfg["point_cloud_range"], num_voxels=nv, folded=folded)
            return pillar_scatter.pillar_scatter(f, coors4, 1, hw[0], hw[1], nv)
        nbytes = 4 * N * F + 2 * (4 * V * P * F + 16 * V) + 4 * V * 64 * 2 + 4 * 64 * hw[0] * hw[1]
        report(label, "%s: %d pts, V=%d P=%d -> [1,64,%d,%d]" % (cfg["name"], N, V, P, hw[0], hw[1]), nbytes, chain,
               "hard_voxelize (5 launches) + cat + PFN + memset + scat_map + scat_write")
    # NMS — 1000 boxes (latency/ALU bound: report pairs/s instead of an HBM fraction)
    boxes = torch.from_numpy(synth.random_boxes(1000, 3)).to(dev)
    report("nms:nms_gpu", "1000 boxes thr 0.2", 28 * 1000 + 8 * 1000 * 16,
           lambda: iou3d_nms.nms_gpu(boxes, 0.2, device_outputs=True), "ALU/latency bound; bytes = boxes + bit-matrix")
    # centerpoint_postprocess — 6 tasks 180x180
    h = synth.centerpoint_head_outputs(0)
    th = {kk: [torch.from_numpy(x).to(dev) for x in vv] for kk, vv in h.items()}
    tc = synth.CENTERPOINT_TEST_CFG
    nb = 4 * sum(x.size for vv in h.values() for x in vv)
    report("postprocess:centerpoint_postprocess", "6 tasks 180x180", nb,
           lambda: centerpoint_postprocess.centerpoint_postprocess_device(
               th["hm"], th["reg"], th["height"], th["dim"], th["vel"], th["rot"], [0.075, 0.075],
               synth.C3["point_cloud_range"], tc["post_center_limit_range"], synth.label_offsets(), tc["down_ratio"],
               tc["score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"], True),
           "5 launches, zero host syncs; latency bound")


if __name__ == "__main__":
    main()
