#!/usr/bin/env python
"""tools/infer_kitti.py — PointPillars or CenterPoint-pillars on a KITTI object split, raw scans in, KITTI label files out.

  python tools/infer_kitti.py --model X.pdparams --config car|ped_cyclist|centerpoint --root <split dir> [--ids list.txt]
                              --out DIR [--lanes L] [--num-points N] [--device cuda:0]

<split dir> is a KITTI object split (e.g. training/ or testing/) with velodyne/<id>.bin (raw HDL-64E scans, x y z
reflectance fp32), calib/<id>.txt and image_2/<id>.png (only the PNG header is read, for the image size; without the
image the reference's 375 x 1242 is used).  --ids: a file of frame ids, one per line (default: every velodyne/*.bin).
Each scan is culled to the left colour camera's view frustum inside the captured frame (frame.KITTI_INPUT), L frames
run in flight (pipeline.CenterPointSweep), and DIR/<id>.txt gets one KITTI result line per box (kitti.to_kitti; the
CenterPoint boxes through kitti.centerpoint_to_lidar_boxes first), the format the KITTI devkit's evaluate_object reads.
--config centerpoint is centerpoint_pillars_016voxel_kitti (centerpoint_pillars.CONFIG_KITTI).
"""
import argparse
import collections
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from paddle3d_b200 import kitti  # noqa: E402


def frame_ids(root, ids_file):
    if ids_file:
        with open(ids_file) as f:
            return [line.strip() for line in f if line.strip()]
    return sorted(f[:-4] for f in os.listdir(os.path.join(root, "velodyne")) if f.endswith(".bin"))


def load_frame(root, fid):
    """(raw scan [n, 4] fp32, calib, image shape) of one frame id."""
    cloud = np.fromfile(os.path.join(root, "velodyne", fid + ".bin"), dtype=np.float32)
    if cloud.size % 4:
        raise ValueError("velodyne/%s.bin: %d floats is not a whole number of 4-value points" % (fid, cloud.size))
    calib = kitti.read_calib(os.path.join(root, "calib", fid + ".txt"))
    png = os.path.join(root, "image_2", fid + ".png")
    return cloud.reshape(-1, 4), calib, kitti.image_shape(png if os.path.exists(png) else None)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--model", required=True,
                    help="a Paddle3D checkpoint (.pdparams) of --config: PointPillars (car, ped_cyclist) or "
                         "CenterPoint-pillars (centerpoint)")
    ap.add_argument("--config", choices=sorted(kitti.CLASS_NAMES), default="car",
                    help="car: pointpillars_xyres16_kitti_car; ped_cyclist: the cyclist / pedestrian model; "
                         "centerpoint: centerpoint_pillars_016voxel_kitti")
    ap.add_argument("--root", required=True, help="KITTI object split directory (velodyne/, calib/, image_2/)")
    ap.add_argument("--ids", default=None, help="file of frame ids, one per line")
    ap.add_argument("--out", required=True, help="directory for the <id>.txt label files")
    ap.add_argument("--lanes", type=int, default=2, help="frames computing concurrently")
    ap.add_argument("--num-points", type=int, default=40000,
                    help="rows the frame takes after the camera cull (more raise, nothing is dropped silently)")
    ap.add_argument("--device", default="cuda:0")
    args = ap.parse_args()

    import torch
    from paddle3d_b200 import frame, synth
    from paddle3d_b200.centerpoint_pillars import CONFIG_KITTI, CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    from paddle3d_b200.pointpillars import CONFIG, CONFIG_PED_CYCLIST, PointPillarsHotPath
    if not torch.cuda.is_available():
        raise SystemExit("infer_kitti.py needs a CUDA device (no CPU fallback exists)")
    frame_cls, cfg, model_cfg = {"car": (PointPillarsHotPath, synth.C2, CONFIG),
                                 "ped_cyclist": (PointPillarsHotPath, synth.C2_PED_CYCLIST, CONFIG_PED_CYCLIST),
                                 "centerpoint": (CenterPointPillarsHotPath, synth.CP_PILLARS_KITTI, CONFIG_KITTI)}[args.config]
    centerpoint = frame_cls is CenterPointPillarsHotPath
    names = kitti.CLASS_NAMES[args.config]
    ids = frame_ids(args.root, args.ids)
    os.makedirs(args.out, exist_ok=True)
    sweep = CenterPointSweep(max(1, args.lanes), frame_cls=frame_cls, cfg=cfg, model_cfg=model_cfg,
                             device=torch.device(args.device), num_points=args.num_points, weights=args.model,
                             sweep_input=frame.KITTI_INPUT)
    if not ids:
        return
    frames = [load_frame(args.root, fid) for fid in ids[:1]]
    for p in sweep.lanes:  # warm up on the first scan (sizes the workspaces), then capture
        p.infer_kitti(frames[0][0], kitti.frustum_planes(frames[0][1], frames[0][2]))
        p.capture()
    meta = collections.deque()  # (id, calib, image shape) of the scans submitted and not yet written

    def items():
        for fid in ids:
            cloud, calib, shape = load_frame(args.root, fid)
            meta.append((fid, calib, shape))
            yield cloud, kitti.frustum_planes(calib, shape)

    for boxes, scores, labels in sweep.infer_kitti_many(items()):
        fid, calib, shape = meta.popleft()
        boxes = kitti.centerpoint_to_lidar_boxes(boxes.numpy()) if centerpoint else boxes.numpy()
        annos = kitti.to_kitti(boxes, scores.numpy(), labels.numpy(), calib, shape, names)
        kitti.write_label_file(os.path.join(args.out, fid + ".txt"), annos)
    print("wrote %d label files to %s" % (len(ids), args.out))


if __name__ == "__main__":
    main()
