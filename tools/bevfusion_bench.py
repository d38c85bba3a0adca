#!/usr/bin/env python
"""tools/bevfusion_bench.py — BEVFusion (bevf_pp) frames/s on an H100: bevfusion.BEVFusionHotPath from six cameras'
depth-net output (synth camera rig, seeded logits / features) and a 300k-point synth.lidar_cloud to boxes.

  python tools/bevfusion_bench.py [--steps K] [--warmup W] [--cpu-baseline]

Prints one JSON line: frames/s with one lane and with three lanes in flight (one frame each, all launched, then all
read back), stage times of the eager frame from CUDA events (camera pool, camera encoder, LiDAR branch, fusion + SE,
head + decode), dense TFLOP/s from BEVFusion.flops(), the card's name and power limit read in the same run, and with
--cpu-baseline the CPU arm's (tests/bevfusion_oracle.CpuBEVFusion) time for one frame.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from tools.pointpillars_bench import gpu_identity  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=60)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--cpu-baseline", action="store_true")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bevfusion_bench: no CUDA device (nothing is measured without one)")
    from paddle3d_b200 import bevfusion as bf
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import bev_pool_v2 as bp
    dev = torch.device("cuda:0")
    m = bf.BEVFusion(device=dev).init_weight(seed=0)
    vt = m.vt
    rng = np.random.default_rng(0)
    frames = []
    for s in range(3):
        pts = synth.lidar_cloud(dict(synth.C4_LIDAR), s).astype(np.float32)
        mats = synth.lss_mats(synth.camera_rig(s, bda=False))
        lg = torch.from_numpy(rng.normal(0, 2, (m.N, vt.D, vt.H, vt.W)).astype(np.float32)).to(dev)
        tr = torch.from_numpy(rng.normal(0, 1, (m.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)).to(dev)
        frames.append((torch.from_numpy(pts).pin_memory(), mats, lg, tr))
    m.calibrate_cls_bias(frames[0][0].to(dev), *frames[0][1:])
    n_pts = synth.C4_LIDAR["num_points"]
    lanes = [bf.BEVFusionHotPath(m, num_points=n_pts, device=dev)]
    lanes[0].capture()
    lanes += [bf.BEVFusionHotPath(m, num_points=n_pts, device=dev).share_model(lanes[0]).capture() for _ in range(2)]
    res = {}
    for name, L in (("lanes_1", 1), ("lanes_3", 3)):
        for i in range(args.warmup):
            lanes[0].infer(*frames[i % 3])
        t0 = time.perf_counter()
        done = 0
        while done < args.steps:
            k = min(L, args.steps - done)
            for j in range(k):
                lanes[j].launch(*frames[(done + j) % 3])
            for j in range(k):
                lanes[j].result()
            done += k
        res[name + "_frames_per_s"] = args.steps / (time.perf_counter() - t0)
    # stage times of the eager frame
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
    pts, mats, lg, tr = frames[0]
    ptsd = pts.to(dev)
    stages = dict(camera_pool=0.0, camera_encoder=0.0, lidar_branch=0.0, fusion_se=0.0, head_decode=0.0)
    reps = 10
    for _ in range(reps + 1):
        fused = m.fused_image()
        torch.cuda.synchronize()
        ev[0].record()
        prepared = m.vt.ranks(mats, 1, m.N)
        depth, feat = bp.lss_depth_feat(lg, tr)
        img = m.pool(depth, feat, prepared)
        ev[1].record()
        m.camera(img, fused)
        ev[2].record()
        m.lidar(ptsd, fused)
        ev[3].record()
        Y, X = m.bev_hw
        x, _, _ = m.reduc(fused, (1, Y, X, m.fuse_C))
        from paddle3d_b200.ops.se_gate import se_gate_h16
        se_gate_h16(x, (1, Y, X, m.cfg["fusion_channels"]), m.se_dev["weight"], m.se_dev["bias"])
        ev[4].record()
        _, planes, _ = m.head(x, (1, Y, X, m.cfg["fusion_channels"]), want_nchw=True)
        m.postprocess(planes)
        ev[5].record()
        torch.cuda.synchronize()
        if _ == 0:
            continue
        for k, name in enumerate(stages):
            stages[name] += ev[k].elapsed_time(ev[k + 1]) / reps
    res["stage_ms_eager"] = {k: round(v, 4) for k, v in stages.items()}
    fl = m.flops()
    res["dense_gflop_per_frame"] = {k: round(v / 1e9, 1) for k, v in fl.items()}
    res["camera_encoder_tflops"] = round(fl["camera_encoder"] / (stages["camera_encoder"] * 1e9), 1)
    res["frame_dense_tflops"] = round(fl["total"] * res["lanes_1_frames_per_s"] / 1e12, 1)
    res["rows_frame0"] = int(lanes[0].h_counts[-1])
    if args.cpu_baseline:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import bevfusion_oracle as bo
        cams = bp.unpack_cameras(bp.pack_cameras(*mats), 1, m.N)
        axes = tuple(a.numpy() for a in m.vt.axes_host)
        t0 = time.perf_counter()
        bo.CpuBEVFusion(m.export_numpy(), m.cfg, m.anchors_np).run(pts.numpy(), cams, axes, lg.cpu().numpy(),
                                                                    tr.cpu().numpy(), *m.vt.grid_args())
        res["cpu_arm_s_per_frame"] = round(time.perf_counter() - t0, 2)
    else:
        res["cpu_arm_s_per_frame"] = "not measured (--cpu-baseline)"
    res = {k: (round(v, 2) if isinstance(v, float) else v) for k, v in res.items()}
    print(json.dumps(dict(res, steps=args.steps, gpu=gpu_identity())))


if __name__ == "__main__":
    main()
