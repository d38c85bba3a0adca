#!/usr/bin/env python
"""tools/pointpillars_bench.py — PointPillars KITTI frames/s on an H100 (BASELINE config 2).

  python tools/pointpillars_bench.py [--config car|ped_cyclist] [--steps K] [--warmup W] [--in-flight L]
                                     [--no-cpu-baseline] [--dump-outputs DIR] [--kitti-raw]

A step = one 20k x 4-point synth.lidar_cloud frame through pointpillars.PointPillarsHotPath: hard_voxelize ->
PillarFeatureNet -> pixel fp16-pair image -> SecondBackbone + SecondFPN + SSD head conv -> anchor_head_postprocess ->
boxes.  --config car (default): synth.C2 with pointpillars.CONFIG, a 496 x 432 image, 66.2 GFLOP dense; ped_cyclist:
synth.C2_PED_CYCLIST with pointpillars.CONFIG_PED_CYCLIST (two classes), a 248 x 296 image with a stride-1 first block.
--kitti-raw times raw KITTI scans instead (run_kitti_raw).  Prints one JSON line.  The timing harness (CenterPointSweep lanes, e2e through
infer_many / infer, graph-timed stages) is bench.py's, imported from it, so both models are measured the same way.
"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from bench import BN_GAIN, POOL, UNIT, frame_pool, graph_time_ms, measure, rel_errors  # noqa: E402

PP_METRIC = "PointPillars KITTI frames/sec @20k pts, 0.16 m pillars, 496x432 BEV (pointpillars_xyres16_kitti_car)"
PP_PED_CYCLIST_METRIC = ("PointPillars KITTI frames/sec @20k pts, 0.16 m pillars, 248x296 BEV "
                         "(pointpillars_xyres16_kitti_cyclist_pedestrian)")
CLASS_NAMES = {"car": ("car",), "ped_cyclist": ("cyclist", "pedestrian")}


def gpu_identity(index=0):
    """Card name, power limit and max SM clock, read with nvidia-smi in the same run as the measurement."""
    try:
        out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm",
                              "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
        name, power, clk = [x.strip() for x in out.split(",")]
        return {"name": name, "power_limit": power, "sm_max_clock": clk}
    except Exception as e:  # noqa: BLE001
        return {"error": repr(e)}


def pp_frame_check(got, cpu, gpu_candidates, tc, tol=1e-3):
    """GPU frame vs CPU arm on the same points.  Boxes are paired by centre; a pair matches when every box value and the
    score agree within `tol` (relative, absolute below 1) and the labels are equal.  Every CPU box without a match is
    listed with its score and the likely cause, so a difference is explained rather than hidden by a wider tolerance."""
    gb, gs, gl = got[0].numpy(), got[1].numpy(), got[2].numpy()
    cb, cs, cl = cpu["boxes"], cpu["scores"], cpu["labels"]
    chk = {"pillars_gpu": None, "pillars_cpu": int(cpu["num_voxels"]), "boxes_gpu": int(len(gb)), "boxes_cpu": int(len(cb)),
           "candidates_gpu": int(gpu_candidates), "candidates_cpu": int(cpu["candidates"]), "tolerance": tol}
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
        thr = tc["nms_score_threshold"]
        cause = ("label differs (GPU %d, CPU %d)" % (gl[j], cl[i]) if j >= 0 and j not in used and gl[j] != cl[i] else
                 "score within %g of the threshold" % tol if abs(cs[i] - thr) <= tol else
                 "candidate count over nms_pre_max_size: top-k boundary" if cpu["candidates"] > tc["nms_pre_max_size"]
                 and i >= len(cb) - 5 else "NMS decision of a box pair at the IoU threshold (or a neighbour of one)")
        unmatched.append({"cpu_row": i, "score": float(cs[i]), "box": [float(v) for v in cb[i]], "cause": cause})
    chk.update({"matched": len(used), "max_rel_box_err": worst_box, "max_rel_score_err": worst_score,
                "unmatched_cpu": unmatched, "unmatched_gpu_rows": [j for j in range(len(gb)) if j not in used]})
    return chk


def run(args):
    """PointPillars KITTI-shape inference (BASELINE config 2): synth.C2 (or synth.C2_PED_CYCLIST) frames (20k x 4 points)
    through pointpillars.PointPillarsHotPath.  `value` = frames/s with --in-flight frames resident in HBM (CUDA-graph replay);
    e2e = pinned host points in, host boxes out (pipelined and one frame at a time); eager per-stage device times; the
    graph-timed dense stage (backbone + FPN + head) with its algorithmic TFLOP/s; the anchor postprocess alone; the CPU
    arm; a check of the GPU frame against the CPU arm on frame 0."""
    import torch
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox
    from paddle3d_b200.pipeline import CenterPointSweep
    from paddle3d_b200.pointpillars import CONFIG, CONFIG_PED_CYCLIST, PointPillarsHotPath
    if not torch.cuda.is_available():
        raise SystemExit("pointpillars_bench.py needs a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    car = args.config == "car"
    cfg, model_cfg = (synth.C2, CONFIG) if car else (synth.C2_PED_CYCLIST, CONFIG_PED_CYCLIST)
    lanes = max(1, args.in_flight)
    sweep = CenterPointSweep(lanes, frame_cls=PointPillarsHotPath, cfg=cfg, device=dev, seed=0, bn_gain=BN_GAIN,
                             model_cfg=model_cfg)
    pipe = sweep.lanes[0]
    m = pipe.model
    frames = frame_pool(cfg, POOL)
    dev_frames = [torch.from_numpy(f).to(dev) for f in frames]
    host_frames = [torch.from_numpy(f).pin_memory() for f in frames]
    sweep.calibrate_head(dev_frames[0])  # ~2 % of the anchors above the score threshold (PointPillars.calibrate_cls_bias)
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
    pf = m.pfn
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
            feats = pe.pillar_feature_net(voxels, npv, coors, m.pfn_weight, pf["gamma"], pf["beta"], pf["mean"], pf["var"],
                                          pf["eps"], cfg["voxel_size"], cfg["point_cloud_range"], num_voxels=nv,
                                          folded=m.pfn_folded)
            ev[2].record(st)
            image, shape = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, m.C], num=nv).to_pixel_h16()
            ev[3].record(st)
            planes = m.dense(image, shape)
            ev[4].record(st)
            m.postprocess(planes, coors, nv)
            ev[5].record(st)
        ev[5].synchronize()
    names = ["hard_voxelize", "pillar_feature_net", "pixel_image (rows_convert_h16 + sparse_rows_to_pixel_h16)",
             "dense (backbone + FPN + head conv)", "anchor_postprocess"]
    stage = {names[k]: ev[k].elapsed_time(ev[k + 1]) for k in range(5)}
    fl = m.flops()
    ms_dense = graph_time_ms(lambda: m.dense(image, shape), st, 5)
    ms_post = graph_time_ms(lambda: m.postprocess(planes, coors, nv), st, 20)
    pk = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
    bf16_peak = pk.get("bf16_tflops", 989.0)
    ach = sum(fl.values()) / (ms_dense * 1e-3) / 1e12
    dense_roof = {"bound": "tensor", "kernel": "dcf::dense_conv_f16_kernel (13 backbone + 3 FPN + 1 head launches)",
                  "ms": ms_dense, "algorithmic_flops": sum(fl.values()),
                  "gflop": {k: round(v / 1e9, 2) for k, v in fl.items()}, "achieved": ach, "unit": "TFLOP/s",
                  "peak": bf16_peak, "frac": ach / bf16_peak,
                  "peak_source": "MEASURED_PEAKS.json bf16_tflops" if pk else
                  "H100 SXM data sheet 989 TFLOP/s dense fp16/bf16 at 700 W (not measured)",
                  "note": "algorithmic flops (2 x MACs); the kernel executes 3 fp16 MMAs per product (fp16-pair operands)"}
    line = {"metric": PP_METRIC if car else PP_PED_CYCLIST_METRIC, "model": "pointpillars", "value": res["value"],
            "unit": UNIT, "n_gpus": 1, "steps": args.steps, "warmup": args.warmup, "ms_per_step": res["ms_per_step"],
            "higher_is_better": True, "frames_in_flight": lanes,
            "data": "synthetic (synth.lidar_cloud, config %s)" % ("C2" if car else "C2_PED_CYCLIST"),
            "dtype": "f16x3 (fp16 hi/lo' pairs, f32 accumulation) dense; fp32 encoder and postprocess",
            "gpu": ident, "clocks": res["clocks"],
            "e2e": {"value": res["e2e_value"], "sync_value": res["e2e_sync_value"], "unit": UNIT,
                    "api": "CenterPointSweep(frame_cls=PointPillarsHotPath).infer_many, %d lanes" % lanes,
                    "sync_note": "sync_value = PointPillarsHotPath.infer, one frame at a time"},
            "gpu_launches_per_step": pipe.graph_nodes["kernel"] if pipe.graph_nodes else None,
            "stage_ms_eager": stage, "dense": dense_roof, "anchor_postprocess_ms": ms_post,
            "num_pillars_frame0": int(nv.item())}
    names = CLASS_NAMES[args.config]
    if len(names) > 1:
        labels0 = pipe.infer(host_frames[0])[2].numpy()
        line["boxes_per_class_frame0"] = {n: int((labels0 == c).sum()) for c, n in enumerate(names)}
    if not args.no_cpu_baseline:
        import oracle
        from oracle.pointpillars import CpuPointPillars
        from oracle.pointpillars_multiclass import CpuPointPillarsMulticlass
        cpu = (CpuPointPillars(cfg, m.export_numpy(), m.anchors_np, m.corners_np, m.grid, m.mc["test"]) if car else
               CpuPointPillarsMulticlass(cfg, m.export_numpy(), m.anchors_np, m.corners_np, m.grid, m.mc["test"],
                                         m.num_classes))
        t0 = time.perf_counter()
        r = cpu.run(frames[0])
        cpu_s = time.perf_counter() - t0
        line["cpu_baseline"] = {"value": 1.0 / cpu_s, "unit": UNIT, "cores": oracle.num_threads(), "kind": "port",
                                "sample": "1 full frame; voxelize = %s; other stages = oracle port (OpenMP / numpy)" %
                                          ("reference hard_voxelize_cpu (oracle/_ref)" if cpu.use_ref else "oracle port"),
                                "stage_s": r["times"]}
        got = pipe.infer(host_frames[0])
        chk = pp_frame_check(got, r, int(pipe.h_counts[0]), m.mc["test"])
        chk["pillars_gpu"] = int(pipe.out["num_voxels"][0].item())
        chk["head_planes"] = rel_errors(pipe.out["planes"].cpu().numpy(), r["planes"])
        if len(names) > 1:
            chk["boxes_per_class_cpu"] = {n: int((r["labels"] == c).sum()) for c, n in enumerate(names)}
        line["frame0_check"] = chk
    print(json.dumps(line))


KITTI_RAW_POINTS = 40000  # rows a frame takes after the camera cull (tools/infer_kitti.py's default)


def run_kitti_raw(args):
    """Raw KITTI scans (synth.kitti_raw_cloud: ~115k points over 360 degrees, ~14.5k in the camera's view) end to end,
    host arrays in, host boxes out, at 1 and --in-flight frames in flight:
      device  the raw scan uploaded, culled to the camera frustum inside the captured frame (frame.KITTI_INPUT,
              infer_kitti_many);
      host    the same scan culled on the host by kitti.remove_camera_invisible, padded to the frame's rows and uploaded
              reduced (infer_many), the cull inside the timed loop.
    Also: the cull kernel alone (CUDA events over 200 launches on a full-size scan), the H2D bytes per frame of each
    path, and that frame 0's boxes, scores and labels are bit-equal between the two."""
    import torch
    from paddle3d_b200 import frame, kitti, synth
    from paddle3d_b200.ops import sweep_merge as sm
    from paddle3d_b200.pipeline import CenterPointSweep
    from paddle3d_b200.pointpillars import CONFIG, CONFIG_PED_CYCLIST, PointPillarsHotPath
    if not torch.cuda.is_available():
        raise SystemExit("pointpillars_bench.py needs a CUDA device (no CPU fallback exists)")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    car = args.config == "car"
    cfg, model_cfg = (synth.C2, CONFIG) if car else (synth.C2_PED_CYCLIST, CONFIG_PED_CYCLIST)
    n = KITTI_RAW_POINTS
    scans = [synth.kitti_raw_cloud(s) for s in range(POOL)]
    items = [(c, kitti.frustum_planes(cal, shape)) for c, cal, shape in scans]

    def reduced(item):
        kept = kitti.remove_camera_invisible(*item)
        full = np.full((n, 4), np.nan, np.float32)
        full[:len(kept)] = kept
        return torch.from_numpy(full)

    ident = gpu_identity(0)
    kw = dict(cfg=cfg, model_cfg=model_cfg, device=dev, seed=0, bn_gain=BN_GAIN, num_points=n)
    calib_pts = reduced(items[0]).to(dev)
    out = {}
    for lanes in sorted({1, max(1, args.in_flight)}):
        raw = CenterPointSweep(lanes, frame_cls=PointPillarsHotPath, sweep_input=frame.KITTI_INPUT, **kw)
        host = CenterPointSweep(lanes, frame_cls=PointPillarsHotPath, **kw)
        raw.calibrate_head(calib_pts)
        host.calibrate_head(calib_pts)
        for p in raw.lanes:
            p.infer_kitti(*items[0])
            p.capture()
        host.capture(calib_pts)
        if lanes == 1:
            got_raw = [t.clone() for t in raw.lanes[0].infer_kitti(*items[0])]
            got_host = host.lanes[0].infer(reduced(items[0]).pin_memory())
            out["frame0_bit_equal"] = all(torch.equal(a, b) for a, b in zip(got_raw, got_host))
            out["frame0_boxes"] = int(len(got_raw[0]))
        seq = [items[i % len(items)] for i in range(args.steps)]
        warm = [items[i % len(items)] for i in range(args.warmup)]
        row = {}
        for name, run_items in (("device_cull", lambda it: raw.infer_kitti_many(iter(it))),
                                ("host_cull", lambda it: host.infer_many(reduced(x) for x in it))):
            list(run_items(warm))
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            k = sum(1 for _ in run_items(seq))
            row[name] = k / (time.perf_counter() - t0)
        out["frames_per_s_%d_in_flight" % lanes] = row
        if lanes == 1:
            p = raw.lanes[0]
            st = p.stream
            big = max(range(len(items)), key=lambda i: len(items[i][0]))
            p.infer_kitti(*items[big])
            ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
            with torch.cuda.stream(st):
                for _ in range(20):
                    p._merge_sweeps()
                ev[0].record(st)
                for _ in range(200):
                    p._merge_sweeps()
                ev[1].record(st)
            ev[1].synchronize()
            out["cull_kernel_us"] = {"mean": 1e3 * ev[0].elapsed_time(ev[1]) / 200, "raw_points": int(len(items[big][0])),
                                     "what": "p3d_merge_sweeps_frustum: workspace memset + merge_sweeps_kernel<true> + "
                                             "merge_tail_kernel, eager launches"}
        del raw, host
        torch.cuda.empty_cache()
    mean_raw = float(np.mean([len(c) for c, _ in items]))
    mean_kept = float(np.mean([len(kitti.remove_camera_invisible(*it)) for it in items]))
    out["h2d_bytes_per_frame"] = {"device_cull": mean_raw * 16 + sm.DESC_DTYPE.itemsize + 6 * 4 * 8,
                                  "host_cull": n * 4 * 4, "mean_raw_points": mean_raw, "mean_kept_points": mean_kept}
    line = {"metric": "PointPillars KITTI frames/sec on raw scans, camera cull on the device vs on the host",
            "model": "pointpillars_%s" % args.config, "unit": UNIT, "steps": args.steps, "warmup": args.warmup,
            "data": "synthetic raw scans (synth.kitti_raw_cloud, %d seeds), num_points %d" % (len(items), n),
            "gpu": ident, **out}
    print(json.dumps(line))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", choices=sorted(CLASS_NAMES), default="car",
                    help="car: pointpillars_xyres16_kitti_car; ped_cyclist: the two-class cyclist / pedestrian model")
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--in-flight", type=int, default=4, help="frames computing concurrently (CenterPointSweep lanes)")
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="after the timed steps, write the boxes / scores / labels of the last timed frame to DIR/*.npy")
    ap.add_argument("--kitti-raw", action="store_true",
                    help="raw KITTI scans: camera frustum cull inside the frame vs on the host (run_kitti_raw)")
    args = ap.parse_args()
    args.warmup = max(args.warmup, 3)
    (run_kitti_raw if args.kitti_raw else run)(args)


if __name__ == "__main__":
    main()
