#!/usr/bin/env python
"""Deploy-style CLI (mirrors deploy/centerpoint/python/infer.py:54-201): one `.bin` sweep in, detections out.

    python tools/infer.py --model model.pdparams --lidar_file sweep.bin --num_point_dim 5 [--use_timelag 1]
                          [--out results.txt] [--sweeps sweeps.json]

--model: the trained CenterPoint-voxel parameters, a `.pdparams` file as paddle.save writes a Paddle3D model's
state_dict (paddle3d_b200/checkpoint.py maps its names; the reference's own --model_file / --params_file take the
exported inference model instead).  Without it the model runs with the seeded weights of the benchmark (same
architecture), whose boxes are noise.
--sweeps: the earlier sweeps of a multi-sweep frame, [{"path": ..., "ref_from_curr": 4x4 or null, "time_lag": s}, ...];
the frame then merges them with the key sweep on the GPU (as the reference's LoadPointCloud does on the host)."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from paddle3d_b200 import deploy  # noqa: E402
from paddle3d_b200 import io as p3d_io  # noqa: E402


def run_sweeps(args):
    """Key sweep + the sweeps of the JSON list, merged on the GPU as LoadPointCloud merges them (x, y, z, intensity and
    the time lag, close points of earlier sweeps within 1 m removed)."""
    import numpy as np
    with open(args.sweeps) as f:
        entries = json.load(f)
    key = p3d_io.read_bin(args.lidar_file, args.num_point_dim)
    sweeps = [(p3d_io.read_bin(e["path"], args.num_point_dim),
               None if e.get("ref_from_curr") is None else np.asarray(e["ref_from_curr"], np.float64),
               float(e.get("time_lag", 0.0))) for e in entries]
    rows = [len(key)] + [len(c) for c, _, _ in sweeps]
    si = dict(max_sweeps=len(rows), raw_dim=args.num_point_dim, use_dim=4, use_time_lag=bool(args.use_timelag),
              slot_cap=max(4, -(-max(rows) // 4) * 4))
    pred = deploy.Predictor(device="cuda:%d" % args.gpu_id, max_points=max(args.max_points, sum(rows)),
                            with_head=not args.no_head, sweep_input=si, weights=args.model)
    return pred.run_sweeps(key, sweeps)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", default=None, help="trained CenterPoint-voxel parameters (.pdparams); default: seeded weights")
    ap.add_argument("--lidar_file", required=True, help="path of a float32 .bin point file")
    ap.add_argument("--num_point_dim", type=int, default=5, help="values per point in the file (infer.py:61-65)")
    ap.add_argument("--use_timelag", type=int, default=1, help="append the time-lag column (infer.py:66-70)")
    ap.add_argument("--gpu_id", type=int, default=0)
    ap.add_argument("--max_points", type=int, default=300000)
    ap.add_argument("--no_head", action="store_true")
    ap.add_argument("--out", default=None, help="also write the detections to this text file")
    ap.add_argument("--sweeps", default=None,
                    help="JSON list of earlier sweeps {path, ref_from_curr (4x4 or null), time_lag} merged with the key "
                         "sweep (--lidar_file) on the GPU, in the listed order")
    args = ap.parse_args()
    if args.model and args.no_head:
        ap.error("--model loads the whole CenterPoint, dense head included: drop --no_head")
    if args.sweeps:
        box3d_lidar, label_preds, scores = run_sweeps(args)
    else:
        points = deploy.preprocess(args.lidar_file, args.num_point_dim, bool(args.use_timelag))
        pred = deploy.Predictor(device="cuda:%d" % args.gpu_id, max_points=max(args.max_points, len(points)),
                                with_head=not args.no_head, weights=args.model)
        box3d_lidar, label_preds, scores = pred.run(points)
    deploy.parse_result(box3d_lidar, label_preds, scores)
    if args.out:
        deploy.write_results(args.out, box3d_lidar, label_preds, scores)


if __name__ == "__main__":
    main()
