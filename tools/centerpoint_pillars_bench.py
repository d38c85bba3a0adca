#!/usr/bin/env python
"""tools/centerpoint_pillars_bench.py — CenterPoint-pillars nuScenes or KITTI frames/s on an H100.

  python tools/centerpoint_pillars_bench.py [--steps K] [--warmup W] [--in-flight L] [--no-cpu-baseline] [--stream]
                                            [--dump-outputs DIR]
  python tools/centerpoint_pillars_bench.py --config kitti [--kitti-raw] [--steps K] [--warmup W] [--in-flight L]
                                            [--no-cpu-baseline]

A step = one 300k x 5-point synth.lidar_cloud frame (synth.CP_PILLARS) through
centerpoint_pillars.CenterPointPillarsHotPath: hard_voxelize (0.2 m pillars, 20 points) -> two-layer PillarFeatureNet ->
pixel fp16-pair image 512 x 512 x 64 -> SecondBackbone + SecondFPN + CenterHead (127.2 GFLOP) -> centerpoint postprocess
-> boxes.  Prints one JSON line.  The timing harness (CenterPointSweep lanes, e2e through infer_many / infer,
graph-timed stages) is bench.py's, imported from it, so every model is measured the same way.  --stream adds frames/s
through CenterPointSweep.infer_stream over a 70-sweep synth.sweep_sequence (10 sweeps per frame, merged on the device),
measured as tools/sweep_bench.py measures the voxel model.

--config kitti runs centerpoint_pillars_016voxel_kitti (synth.CP_PILLARS_KITTI, CONFIG_KITTI: 100 points per pillar,
432 x 496 grid, two velocity-free tasks, the head at 248 x 216) on synth.kitti_raw_cloud scans: culled to the camera
frustum on the host and NaN-padded to the frame's 40000 rows (infer_many), or with --kitti-raw the raw scans culled inside
the captured frame (frame.KITTI_INPUT, infer_kitti_many).  See run_kitti.
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import numpy as np  # noqa: E402

from bench import BN_GAIN, POOL, UNIT, frame_pool, graph_time_ms, measure, rel_errors  # noqa: E402
from pointpillars_bench import gpu_identity  # noqa: E402

METRIC = ("CenterPoint-pillars nuScenes frames/sec @300k pts, 0.2 m pillars, 512x512 BEV "
          "(centerpoint_pillars_02voxel_nuscenes_10sweep)")


def frame_check(got, cpu, gpu_rows_per_task, tc, tol=1e-3):
    """GPU frame vs CPU arm on the same points.  Boxes are paired by centre; a pair matches when every box value and the
    score agree within `tol` (relative, absolute below 1) and the labels are equal.  Every CPU box without a match is
    listed with its score and the likely cause, so a difference is explained rather than hidden by a wider tolerance."""
    gb, gs, gl = got[0].numpy(), got[1].numpy(), got[2].numpy()
    cb, cs, cl = cpu["boxes"], cpu["scores"], cpu["labels"]
    chk = {"pillars_gpu": None, "pillars_cpu": int(cpu["num_voxels"]), "boxes_gpu": int(len(gb)),
           "boxes_cpu": int(len(cb)), "boxes_per_task_gpu": gpu_rows_per_task, "tolerance": tol}
    used, worst_box, worst_score, unmatched = set(), 0.0, 0.0, []
    for i in range(len(cb)):
        j = int(np.argmin(np.abs(gb[:, :3] - cb[i, :3]).max(1))) if len(gb) else -1
        if j >= 0 and j not in used:
            eb = float((np.abs(gb[j] - cb[i]) / np.maximum(1.0, np.abs(cb[i]))).max())
            es = float(abs(gs[j] - cs[i]) / max(1.0, abs(cs[i])))
            if eb <= tol and es <= tol and gl[j] == cl[i]:
                used.add(j)
                worst_box, worst_score = max(worst_box, eb), max(worst_score, es)
                continue
        thr = tc["score_threshold"]
        cause = ("label differs (GPU %d, CPU %d)" % (gl[j], cl[i]) if j >= 0 and j not in used and gl[j] != cl[i] else
                 "score within %g of the threshold" % tol if abs(cs[i] - thr) <= tol else
                 "last rows of a task: nms_pre_max_size / nms_post_max_size boundary" if i >= len(cb) - 5 else
                 "NMS decision of a box pair at the IoU threshold (or a neighbour of one)")
        unmatched.append({"cpu_row": i, "score": float(cs[i]), "box": [float(v) for v in cb[i]], "cause": cause})
    chk.update({"matched": len(used), "max_rel_box_err": worst_box, "max_rel_score_err": worst_score,
                "unmatched_cpu": unmatched, "unmatched_gpu_rows": [j for j in range(len(gb)) if j not in used]})
    return chk


def stream_rate(args, dev):
    """frames/s of CenterPointSweep.infer_stream: one frame per pushed sweep of a 70-sweep stream, K = 10 sweeps per
    frame merged on the device, --in-flight lanes sharing one ring (the first frames merge fewer sweeps)."""
    from paddle3d_b200 import synth
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    K, L = 10, max(1, args.in_flight)
    seq = synth.sweep_sequence(70, 7)
    si = dict(max_sweeps=K, slot_cap=-(-max(len(c) for c, _, _ in seq) // 4) * 4)
    sweep = CenterPointSweep(L, frame_cls=CenterPointPillarsHotPath, device=dev, seed=0, bn_gain=BN_GAIN, sweep_input=si)
    from sweep_bench import frame_inputs
    lane0 = sweep.lanes[0]
    lane0.infer_sweeps(*frame_inputs(seq, K - 1, K))
    lane0.calibrate_head(lane0.points.clone())  # on the first full 10-sweep frame; the lanes share the model
    for p in sweep.lanes:
        p.infer_sweeps(*frame_inputs(seq, K - 1, K))
        p.capture()

    def timed(items):
        t0 = time.perf_counter()
        n = sum(1 for _ in sweep.infer_stream(iter(items)))
        return n, time.perf_counter() - t0
    timed(seq[:K + 2 * L])  # warm-up
    n, secs = timed(seq)
    return {"value": n / secs, "unit": UNIT, "frames": n, "lanes": L, "sweeps_per_frame": K,
            "api": "CenterPointSweep(frame_cls=CenterPointPillarsHotPath, sweep_input=...).infer_stream",
            "note": "one frame per sweep of synth.sweep_sequence(70, 7); the first K - 1 frames merge fewer sweeps"}


def run(args):
    import torch
    from paddle3d_b200 import synth
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox
    from paddle3d_b200.pipeline import CenterPointSweep
    if not torch.cuda.is_available():
        raise SystemExit("centerpoint_pillars_bench.py needs a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = synth.CP_PILLARS
    lanes = max(1, args.in_flight)
    sweep = CenterPointSweep(lanes, frame_cls=CenterPointPillarsHotPath, cfg=cfg, device=dev, seed=0, bn_gain=BN_GAIN)
    pipe = sweep.lanes[0]
    m = pipe.model
    frames = frame_pool(cfg, POOL)
    dev_frames = [torch.from_numpy(f).to(dev) for f in frames]
    host_frames = [torch.from_numpy(f).pin_memory() for f in frames]
    sweep.calibrate_head(dev_frames[0])  # ~1.4 % of the cells above the score threshold
    pipe.points.copy_(dev_frames[0])
    pipe.capture(count_nodes=True)
    for p in sweep.lanes[1:]:
        p.points.copy_(dev_frames[0])
        p.capture()
    ident = gpu_identity(0)
    res = measure(sweep, dev_frames, host_frames, args, 1, None, True, 0, dump_dir=args.dump_outputs)
    st = pipe.stream
    # eager per-stage device times (first pass warms the allocator, the second is timed with the GPU parked first)
    P, V = cfg["max_points"], cfg["max_voxels"]
    nx, ny = m.grid
    for rep in range(2):
        with torch.cuda.stream(st):
            pipe.points.copy_(dev_frames[0])
            if rep == 1:
                torch.cuda._sleep(int(2e7))
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(6)]
            ev[0].record(st)
            voxels, co, npv, nv = vox.hard_voxelize(pipe.points, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
            coors = torch.nn.functional.pad(co, (1, 0))
            ev[1].record(st)
            feats = pe.pillar_feature_net2(voxels, npv, coors, m.pfn_dev, cfg["voxel_size"], cfg["point_cloud_range"],
                                           num_voxels=nv, folded=m.pfn_folded)
            ev[2].record(st)
            image, shape = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, m.C], num=nv).to_pixel_h16()
            ev[3].record(st)
            h = m.dense(image, shape)
            ev[4].record(st)
            m.postprocess(h)
            ev[5].record(st)
        ev[5].synchronize()
    names = ["hard_voxelize", "pillar_feature_net2", "pixel_image (rows_convert_h16 + sparse_rows_to_pixel_h16)",
             "dense (backbone + FPN + CenterHead)", "centerpoint_postprocess"]
    stage = {names[k]: ev[k].elapsed_time(ev[k + 1]) for k in range(5)}
    n_pillars = int(nv.item())
    fl = m.flops()
    parts = {k: fl[k] for k in ("backbone", "fpn", "head")}
    ms_dense = graph_time_ms(lambda: m.dense(image, shape), st, 5)
    ach = sum(parts.values()) / (ms_dense * 1e-3) / 1e12
    dense = {"ms": ms_dense, "algorithmic_flops": sum(parts.values()), "achieved": ach, "unit": "TFLOP/s",
             "gflop": {k: round(v / 1e9, 2) for k, v in fl.items()},
             "note": "algorithmic flops (2 x MACs); the kernels execute 3 fp16 MMAs per product (fp16-pair operands)"}
    ms_enc = graph_time_ms(lambda: pe.pillar_feature_net2(voxels, npv, coors, m.pfn_dev, cfg["voxel_size"],
                                                          cfg["point_cloud_range"], num_voxels=nv, folded=m.pfn_folded),
                           st, 20)
    M, F = P, m.F
    (c1, c2), D = m.pfn_channels, F + 5
    pts_in = int(npv[:n_pillars].sum().item())
    pad_rows = int((npv[:n_pillars] < M).sum().item())  # one evaluated padding row per pillar with count < M
    rows = pts_in + pad_rows
    enc_flops = 2.0 * (rows * D * c1 + rows * c1 * c2 + n_pillars * c1 * c2)
    enc_bytes = 4.0 * n_pillars * (M * F + 1 + 4 + c2)
    encoder = {"ms": ms_enc, "pillars": n_pillars, "points_in_pillars": pts_in, "algorithmic_flops": enc_flops,
               "algorithmic_bytes": enc_bytes, "GFLOP_per_s": enc_flops / (ms_enc * 1e-3) / 1e9,
               "GB_per_s": enc_bytes / (ms_enc * 1e-3) / 1e9,
               "note": "flops: 2 x MACs of layer 1 on the real rows and one padding row per non-full pillar, layer 2's "
                       "per-row half (32 x 64) on the same rows, its x_max half once per pillar; bytes: voxels [n, M, F], "
                       "counts, coors, features out"}
    ms_post = graph_time_ms(lambda: m.postprocess(h), st, 20)
    line = {"metric": METRIC, "model": "centerpoint_pillars", "value": res["value"], "unit": UNIT, "n_gpus": 1,
            "steps": args.steps, "warmup": args.warmup, "ms_per_step": res["ms_per_step"], "higher_is_better": True,
            "frames_in_flight": lanes, "data": "synthetic (synth.lidar_cloud, config CP_PILLARS)",
            "dtype": "f16x3 (fp16 hi/lo' pairs, f32 accumulation) dense; fp32 encoder and postprocess",
            "gpu": ident, "clocks": res["clocks"],
            "e2e": {"value": res["e2e_value"], "unit": UNIT,
                    "api": "CenterPointSweep(frame_cls=CenterPointPillarsHotPath).infer_many, %d lanes" % lanes},
            "sync_value": res["e2e_sync_value"], "sync_note": "CenterPointPillarsHotPath.infer, one frame at a time",
            "gpu_launches_per_step": pipe.graph_nodes["kernel"] if pipe.graph_nodes else None,
            "stage_ms_eager": stage, "dense": dense, "encoder": encoder, "postprocess_ms": ms_post,
            "num_pillars_frame0": n_pillars}
    if not args.no_cpu_baseline:
        import oracle
        from oracle.centerpoint_pillars import CpuCenterPointPillars
        cpu = CpuCenterPointPillars(cfg, m.export_numpy(), m.test_cfg, m.label_off)
        t0 = time.perf_counter()
        r = cpu.run(frames[0])
        cpu_s = time.perf_counter() - t0
        line["cpu_baseline"] = {"value": 1.0 / cpu_s, "unit": UNIT, "cores": oracle.num_threads(), "kind": "port",
                                "sample": "1 full frame; voxelize = %s; other stages = oracle port (OpenMP / numpy)" %
                                          ("reference hard_voxelize_cpu (oracle/_ref)" if cpu.use_ref else "oracle port"),
                                "stage_s": r["times"]}
        got = pipe.infer(host_frames[0])
        chk = frame_check(got, r, [int(v) for v in pipe.h_counts[:-1]], m.test_cfg)
        chk["pillars_gpu"] = int(pipe.out["num_voxels"][0].item())
        chk["head_planes"] = {name: [rel_errors(g.cpu().numpy(), w) for g, w in zip(pipe.out["head"][name],
                                                                                   r["head"][name])]
                              for name in r["head"]}
        line["frame0_check"] = chk
    if args.stream:
        line["stream"] = stream_rate(args, dev)
    print(json.dumps(line))


KITTI_SCANS = 8  # distinct synth.kitti_raw_cloud scans cycled through


def run_kitti(args):
    """CenterPoint-pillars KITTI: frames/s with 1 and --in-flight frames in flight (host arrays in, host boxes out), next
    to the card's name and power limit; frame 0 against the CPU arm (tests/centerpoint_pillars_kitti_oracle.py); the
    stages graph-timed on frame 0 (hard_voxelize at P = 100, the wide pillar encoder, the pixel image, the dense part, the
    postprocess), with the bytes of the [40000, 100, 4] padded-voxel tensor hard_voxelize zero-fills per frame."""
    import torch
    from paddle3d_b200 import frame, kitti, synth
    from paddle3d_b200.centerpoint_pillars import CONFIG_KITTI, CenterPointPillarsHotPath
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox
    from paddle3d_b200.pipeline import CenterPointSweep
    if not torch.cuda.is_available():
        raise SystemExit("centerpoint_pillars_bench.py needs a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    cfg = synth.CP_PILLARS_KITTI
    n = cfg["num_points"]
    scans = [synth.kitti_raw_cloud(s) for s in range(KITTI_SCANS)]
    items = [(c, kitti.frustum_planes(cal, shape)) for c, cal, shape in scans]
    kept = [kitti.remove_camera_invisible(*it) for it in items]

    def padded(k):
        full = np.full((n, 4), np.nan, np.float32)
        full[:len(k)] = k
        return full
    frames = [padded(k) for k in kept]
    host_frames = [torch.from_numpy(f).pin_memory() for f in frames]
    calib_pts = torch.from_numpy(frames[0]).to(dev)
    ident = gpu_identity(0)
    kw = dict(cfg=cfg, model_cfg=CONFIG_KITTI, device=dev, seed=0, bn_gain=BN_GAIN)
    if args.kitti_raw:
        kw["sweep_input"] = frame.KITTI_INPUT
    rates, first = {}, None
    for lanes in sorted({1, max(1, args.in_flight)}):
        sweep = CenterPointSweep(lanes, frame_cls=CenterPointPillarsHotPath, **kw)
        sweep.calibrate_head(calib_pts)
        for p in sweep.lanes:
            if args.kitti_raw:
                p.infer_kitti(*items[0])
            else:
                p.points.copy_(calib_pts)
            p.capture(count_nodes=p is sweep.lanes[0])
        if args.kitti_raw:
            def run_items(seq):
                return sweep.infer_kitti_many(iter(seq))
            src = items
        else:
            def run_items(seq):
                return sweep.infer_many(iter(seq))
            src = host_frames
        list(run_items([src[i % len(src)] for i in range(args.warmup)]))
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        k = sum(1 for _ in run_items([src[i % len(src)] for i in range(args.steps)]))
        rates["frames_per_s_%d_in_flight" % lanes] = k / (time.perf_counter() - t0)
        if first is None:
            first = sweep
        else:
            del sweep
    pipe = first.lanes[0]
    m = pipe.model
    got = [t.clone() for t in (pipe.infer_kitti(*items[0]) if args.kitti_raw else pipe.infer(host_frames[0]))]
    line = {"metric": "CenterPoint-pillars KITTI frames/sec (centerpoint_pillars_016voxel_kitti), %s" % (
                "raw scans, camera cull inside the frame" if args.kitti_raw else "host-culled scans"),
            "model": "centerpoint_pillars_kitti", "unit": UNIT, "steps": args.steps, "warmup": args.warmup,
            "data": "synthetic scans (synth.kitti_raw_cloud, %d seeds; %.0f of %.0f points in the camera's view), "
                    "num_points %d" % (len(items), np.mean([len(k) for k in kept]), np.mean([len(c) for c, _ in items]), n),
            "dtype": "f16x3 (fp16 hi/lo' pairs, f32 accumulation) dense; fp32 encoder and postprocess",
            "gpu": ident, **rates, "gpu_launches_per_step": pipe.graph_nodes["kernel"] if pipe.graph_nodes else None,
            "boxes_frame0": int(len(got[0])), "boxes_per_task_frame0": [int(v) for v in pipe.h_counts[:-1]],
            "reference_figure": "Paddle3D's docs/models/centerpoint/README.md gives 43.96 FPS (fp32) and 74.21 FPS (fp16) "
                                "for this config on a V100 with TensorRT: the reference's own figure on other hardware, "
                                "not a like-for-like comparison"}
    # stages on frame 0, each graph-timed on the frame's stream
    st = pipe.stream
    P, V = cfg["max_points"], cfg["max_voxels"]
    nx, ny = m.grid
    pts = torch.from_numpy(frames[0]).to(dev)
    with torch.cuda.stream(st):
        voxels, co, npv, nv = vox.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], P, V)
        coors = torch.nn.functional.pad(co, (1, 0))
        feats = pe.pillar_feature_net2(voxels, npv, coors, m.pfn_dev, cfg["voxel_size"], cfg["point_cloud_range"],
                                       num_voxels=nv, folded=m.pfn_folded)
        image, shape = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, m.C], num=nv).to_pixel_h16()
        h = m.dense(image, shape)
    st.synchronize()
    n_pillars = int(nv.item())
    stage = {
        "hard_voxelize (P = 100)": graph_time_ms(lambda: vox.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"],
                                                                          P, V), st, 20),
        "pillar_feature_net2 (p3d_pillar_feature_net2_wide)": graph_time_ms(
            lambda: pe.pillar_feature_net2(voxels, npv, coors, m.pfn_dev, cfg["voxel_size"], cfg["point_cloud_range"],
                                           num_voxels=nv, folded=m.pfn_folded), st, 20),
        "pixel_image": graph_time_ms(lambda: sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, m.C],
                                                                  num=nv).to_pixel_h16(), st, 20),
        "dense (backbone + FPN + CenterHead)": graph_time_ms(lambda: m.dense(image, shape), st, 5),
        "centerpoint_postprocess": graph_time_ms(lambda: m.postprocess(h), st, 20),
    }
    fl = m.flops()
    dense_flops = fl["backbone"] + fl["fpn"] + fl["head"]
    pts_in = int(npv[:n_pillars].sum().item())
    line.update(stage_ms_graph=stage, num_pillars_frame0=n_pillars, points_in_pillars_frame0=pts_in,
                dense={"gflop": {k: round(v / 1e9, 2) for k, v in fl.items()}, "algorithmic_flops": dense_flops,
                       "achieved_TFLOP_per_s": dense_flops / (stage["dense (backbone + FPN + CenterHead)"] * 1e-3) / 1e12},
                voxelize={"padded_voxel_bytes": V * P * cfg["point_dim"] * 4,
                          "note": "hard_voxelize writes the whole [max_voxels, max_points, 4] fp32 tensor, zero rows "
                                  "included, every frame; the pillar encoder reads the pillars' rows of it"})
    if not args.no_cpu_baseline:
        sys.path.insert(0, os.path.join(ROOT, "tests"))
        import oracle
        from centerpoint_pillars_kitti_oracle import CpuCenterPointPillarsHeads
        cpu = CpuCenterPointPillarsHeads(cfg, m.export_numpy(), m.test_cfg, m.label_off)
        t0 = time.perf_counter()
        r = cpu.run(kept[0])
        cpu_s = time.perf_counter() - t0
        line["cpu_baseline"] = {"value": 1.0 / cpu_s, "unit": UNIT, "cores": oracle.num_threads(), "stage_s": r["times"]}
        chk = frame_check(got, r, [int(v) for v in pipe.h_counts[:-1]], m.test_cfg)
        chk["pillars_gpu"] = n_pillars
        line["frame0_check"] = chk
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=("nuscenes", "kitti"), default="nuscenes",
                    help="nuscenes: centerpoint_pillars_02voxel_nuscenes_10sweep; kitti: centerpoint_pillars_016voxel_kitti")
    ap.add_argument("--kitti-raw", action="store_true",
                    help="with --config kitti: raw scans, the camera frustum cull inside the captured frame")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--in-flight", type=int, default=4, help="frames computing concurrently (CenterPointSweep lanes)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--stream", action="store_true", help="add frames/s through infer_stream over a 70-sweep stream")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the boxes / scores / labels of the last timed frame to DIR/*.npy")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)
    if args.kitti_raw and args.config != "kitti":
        ap.error("--kitti-raw needs --config kitti")
    (run_kitti if args.config == "kitti" else run)(args)


if __name__ == "__main__":
    main()
