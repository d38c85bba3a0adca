#!/usr/bin/env python
"""tools/lss_bench.py — camera-to-BEV lifting (LSSViewTransformer after the depth net) on an H100.

  python tools/lss_bench.py [--steps K] [--warmup W] [--in-flight L] [--config4] [--no-cpu-baseline]

Six cameras, 16 x 44 feature maps (256 x 704 input, downsample 16), D = 118 depth bins, C = 80, on the BEVDet grid
(128 x 128 over +-51.2 m) and the config-4 grid (200 x 200 over +-50 m).  Per grid: frames/s of lss.LSSHotPath with
--in-flight lanes and one frame at a time, for the full frame and for accelerate=True (ranks kept while the calibration
is unchanged); graph-timed stages with algorithmic bytes and GB/s against the H100 SXM's 3.35 TB/s (data sheet, 700 W);
the frame graph's node counts; the numpy oracle frame on the host cores.  --config4 adds BASELINE config 4: the camera
frame and the C4_LIDAR front end (hard_voxelize -> PillarFeatureNet -> pillar scatter onto 400 x 400) captured into one
graph on two forked streams.  Prints one JSON line.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import graph_time_ms  # noqa: E402
from pointpillars_bench import gpu_identity  # noqa: E402

HBM_TBS = 3.35  # H100 SXM data sheet, 700 W
GRIDS = ("bevdet", "config4")


def _rate(launch, sync, n):
    """frames/s of n calls of launch(i), host clock around work that ends in a device synchronise."""
    sync()
    t0 = time.perf_counter()
    for i in range(n):
        launch(i)
    sync()
    return n / (time.perf_counter() - t0)


def stage(ms, nbytes, what):
    gbs = nbytes / (ms * 1e-3) / 1e9
    return {"ms": ms, "algorithmic_bytes": int(nbytes), "GB/s": gbs, "frac_of_hbm": gbs / (HBM_TBS * 1e3), "kernels": what}


def camera_grid(args, name, dev):
    import torch
    from paddle3d_b200 import synth
    from paddle3d_b200.lss import LSSHotPath, LSSViewTransformer
    from paddle3d_b200.ops import bev_pool_v2 as bp
    grid = synth.LSS_BEVDET if name == "bevdet" else synth.LSS_C4
    B, N, C = 1, 6, synth.LSS_CHANNELS
    mk = lambda acc: LSSViewTransformer(grid, synth.LSS_INPUT_SIZE, synth.LSS_DOWNSAMPLE, C, accelerate=acc, device=dev)  # noqa: E731
    vt = mk(False)
    rigs = [synth.camera_rig(s) for s in range(4)]
    mats = [synth.lss_mats(r) for r in rigs]
    rng = np.random.default_rng(0)
    logits = torch.from_numpy(rng.normal(0, 2, (B * N, vt.D, vt.H, vt.W)).astype(np.float32)).to(dev)
    tran = torch.from_numpy(rng.normal(0, 1, (B * N, C, vt.H, vt.W)).astype(np.float32)).to(dev)
    out = {"grid": "%dx%d" % tuple(vt.grid[:2]), "D": vt.D, "H": vt.H, "W": vt.W, "C": C, "cameras": N,
           "points": B * N * vt.D * vt.H * vt.W}
    lanes_n = max(1, args.in_flight)
    for acc in (False, True):
        v = mk(acc)
        lanes = [LSSHotPath(v, B, N, device=dev).capture(count_nodes=(i == 0)) for i in range(lanes_n)]
        for ln in lanes:  # write the inputs once: the timed frames replay on resident features
            ln.logits.copy_(logits)
            ln.tran_feat.copy_(tran)
        torch.cuda.synchronize()
        # a calibration per frame for the full frame (ranks recomputed every frame); accelerate: a fixed rig
        pick = (lambda i: mats[i % 4]) if not acc else (lambda i: mats[0])
        for i in range(args.warmup):
            lanes[i % lanes_n].launch(pick(i))
        key = "accelerate" if acc else "full"
        r = {"fps_in_flight": _rate(lambda i: lanes[i % lanes_n].launch(pick(i)), torch.cuda.synchronize, args.steps),
             "fps_one_at_a_time": _rate(lambda i: lanes[0].infer(pick(i)), torch.cuda.synchronize, args.steps),
             "lanes": lanes_n}
        if not acc:
            r["graph_nodes"] = lanes[0].graph_nodes
            _, counts = lanes[0].infer(mats[0])
            out["n_kept"], out["n_intervals"] = counts
        out[key] = r
    # graph-timed stages on one stream
    st = torch.cuda.Stream(dev)
    n = out["points"]
    with torch.cuda.stream(st):
        desc = vt.descriptor(*mats[0])
        prepared = vt._prepare(desc, B, N, with_coor=True)
        coor = prepared[6].clone()
        depth, feat = bp.lss_depth_feat(logits, tran)
        st.synchronize()
    k, m = out["n_kept"], out["n_intervals"]
    X, Y, Z = vt.grid
    # prepare: keys + indices written and read once by the sort (16 n) and the five int32 outputs (20 n); the op path
    # also reads the uploaded coor (12 n)
    out["stages"] = {
        "fused_geometry_ranks (p3d_lss_prepare)": stage(graph_time_ms(lambda: vt._prepare(desc, B, N), st, 10), 36 * n,
                                                        "lss_rank + radix sort + gather + scan + starts + lengths"),
        "op_path_ranks (p3d_bev_pool_prepare on uploaded coor)": stage(
            graph_time_ms(lambda: bp.voxel_pooling_prepare_v2(coor, *vt.grid_args()), st, 10), 48 * n,
            "prep_rank + radix sort + gather + scan + starts + lengths"),
        "softmax_permute (p3d_lss_depth_feat)": stage(graph_time_ms(lambda: bp.lss_depth_feat(logits, tran, depth, feat), st, 20),
                                                      8 * B * N * (vt.D + C) * vt.H * vt.W, "lss_depth_feat"),
        "pool (p3d_bev_pool_v2_dev, planar)": stage(
            graph_time_ms(lambda: bp.bev_pool_v2_dev(depth, feat, prepared, vt.bev_feat_shape(B), planar=True), st, 20),
            16 * k + 4 * feat.numel() + 8 * m + 4 * B * Z * Y * X * C, "memset + bev_fwd_warp<DEV, PLANAR>"),
    }
    if not args.no_cpu_baseline:
        import oracle
        from oracle import lss
        cams = bp.unpack_cameras(bp.pack_cameras(*mats[0]), B, N)
        ln, tn = logits.cpu().numpy(), tran.cpu().numpy()
        axes = tuple(a.numpy() for a in vt.axes_host)
        t0 = time.perf_counter()
        lss.view_transform(cams, axes, ln, tn, *vt.grid_args())
        s = time.perf_counter() - t0
        out["cpu_oracle_frame"] = {"fps": 1.0 / s, "s": s, "omp_threads": oracle.num_threads(), "host_cores": os.cpu_count(),
                                   "kind": "numpy + OpenMP oracle (oracle/lss.py), not a tuned CPU implementation"}
    return out, (vt, mats, logits, tran)


def config4_graph(args, dev, cam):
    import torch
    from paddle3d_b200 import synth
    from paddle3d_b200.lss import LSSHotPath
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import pillar_encoder, pillar_scatter, voxelize
    from paddle3d_b200.frame import count_graph_nodes
    vt, mats, logits, tran = cam
    frame = LSSHotPath(vt, 1, 6, device=dev)
    frame.logits.copy_(logits)
    frame.tran_feat.copy_(tran)
    frame.h_desc.copy_(torch.from_numpy(bp.pack_cameras(*mats[0])))
    cfg = synth.C4_LIDAR
    pts = torch.from_numpy(synth.lidar_cloud(cfg, 0)).to(dev)
    F, P, V = pts.shape[1], cfg["max_points"], cfg["max_voxels"]
    rng = np.random.default_rng(1)
    w = torch.from_numpy((rng.normal(size=(F + 5, 64)) * 0.3).astype(np.float32)).to(dev)
    g_, b_, mu, var = np.ones(64), np.zeros(64), np.zeros(64), np.ones(64)
    folded = pillar_encoder.fold_bn(g_, b_, mu, var, 1e-3, dev)
    zcol = torch.zeros((V, 1), dtype=torch.int32, device=dev)

    def lidar():
        vox, co, npv, nv = voxelize.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
        coors4 = torch.cat([zcol, co], 1)
        f = pillar_encoder.pillar_feature_net(vox, npv, coors4, w, g_, b_, mu, var, 1e-3, cfg["voxel_size"],
                                              cfg["point_cloud_range"], num_voxels=nv, folded=folded)
        return pillar_scatter.pillar_scatter(f, coors4, 1, 400, 400, nv)

    main, side = torch.cuda.Stream(dev), torch.cuda.Stream(dev)

    def both():
        side.wait_stream(main)
        with torch.cuda.stream(side):
            lid = lidar()
        frame._full()
        main.wait_stream(side)
        return lid

    with torch.cuda.stream(main):
        for _ in range(2):
            both()
        main.synchronize()
        g = torch.cuda.CUDAGraph(keep_graph=True)
        with torch.cuda.graph(g, stream=main):
            both()
        nodes = count_graph_nodes(g)
        for _ in range(args.warmup):
            g.replay()
        main.synchronize()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        s.record(main)
        for _ in range(args.steps):
            g.replay()
        e.record(main)
    e.synchronize()
    ms = s.elapsed_time(e) / args.steps
    return {"definition": "BASELINE config 4: 6-cam 256x704 features -> 200x200 BEV (LSSHotPath) + LiDAR branch "
                          "(C4_LIDAR: hard_voxelize -> PFN -> scatter 400x400), one graph, two forked streams",
            "ms_per_frame": ms, "fps": 1e3 / ms, "graph_nodes": nodes, "frames_in_flight": 1,
            "lidar_points": int(pts.shape[0])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--in-flight", type=int, default=4)
    ap.add_argument("--config4", action="store_true", help="also time BASELINE config 4 (camera frame + LiDAR front end)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("lss_bench.py needs a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    line = {"metric": "LSS view transform frames/s (6 cams, 16x44x118, C=80) after the depth net", "unit": "frames/s",
            "gpu": gpu_identity(0), "steps": args.steps, "warmup": args.warmup}
    cams = {}
    for name in GRIDS:
        line[name], cams[name] = camera_grid(args, name, dev)
    if args.config4:
        line["config4_frame"] = config4_graph(args, dev, cams["config4"])
    print(json.dumps(line))


if __name__ == "__main__":
    main()
