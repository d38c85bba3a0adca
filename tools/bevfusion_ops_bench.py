#!/usr/bin/env python
"""tools/bevfusion_ops_bench.py — device time of BEVFusion's (bevf_pp) new entry points at the model's sizes on an H100.

  python tools/bevfusion_ops_bench.py [--iters N]

  hard_vfe              40 000 pillars x 64 points x 4 features, feat_channels [64, 64] (synth.C4_LIDAR's capacity)
  se_gate_h16           the 384-channel 200 x 200 fused BEV image, in place
  anchor3d_postprocess  the 294-plane head on 200 x 200 (560 000 anchors, 10 classes), with class logits where about
                        2 % of the (anchor, class) scores pass score_thr 0.05, so the nms_pre cut and max_num cut run
Times are CUDA events around N back-to-back calls after a warm-up, per call, into preallocated outputs.  Prints one JSON line with the card's name
and power limit read in the same run.  Inputs are seeded; no file is read or written.
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402

from tools.pointpillars_bench import gpu_identity  # noqa: E402


def event_ms(fn, iters):
    import torch
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("bevfusion_ops_bench: no CUDA device (nothing is measured without one)")
    from paddle3d_b200 import bevfusion as bf
    from paddle3d_b200.ops.anchor3d_postprocess import anchor3d_postprocess_device
    from paddle3d_b200.ops.pillar_encoder import fold_bn, hard_vfe
    from paddle3d_b200.ops.se_gate import se_gate_h16
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(0)
    cfg = bf.CONFIG
    res = {}

    # HardVFE
    n, M, Fd = cfg["max_voxels"], cfg["max_points"], cfg["vfe"]["in_channels"]
    npv = rng.integers(1, M + 1, n).astype(np.int32)
    coors = np.zeros((n, 4), np.int32)
    coors[:, 2:] = rng.integers(0, 400, (n, 2))
    vox = (rng.normal(0, 1, (n, M, Fd)) * (np.arange(M)[None, :, None] < npv[:, None, None])).astype(np.float32)
    mid, out = cfg["vfe"]["feat_channels"]
    layers = [dict(weight=torch.from_numpy(rng.normal(0, 0.3, (ci, co)).astype(np.float32)).to(dev), gamma=np.ones(co),
                   beta=np.zeros(co), mean=np.zeros(co), var=np.ones(co), eps=1e-3)
              for ci, co in ((Fd + 6, mid), (2 * mid, out))]
    folded = [fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], dev) for l in layers]
    t = [torch.from_numpy(a).to(dev) for a in (vox, npv, coors)]
    feats = torch.empty((n, out), dtype=torch.float32, device=dev)
    res["hard_vfe_ms"] = event_ms(lambda: hard_vfe(t[0], t[1], t[2], layers, cfg["voxel_size"], cfg["point_cloud_range"],
                                                   folded=folded, out=feats), args.iters)

    # SE gate on the fused image
    C, (H, W) = cfg["fusion_channels"], cfg["feat_size"]
    img = torch.from_numpy(rng.normal(0, 1, (H * W, 2 * C)).astype(np.float16)).to(dev)
    wt = torch.from_numpy((rng.normal(0, 1, (C, C)) / np.sqrt(C)).astype(np.float32)).to(dev)
    bias = torch.zeros(C, dtype=torch.float32, device=dev)
    gate = torch.empty((1, C), dtype=torch.float32, device=dev)
    res["se_gate_h16_ms"] = event_ms(lambda: se_gate_h16(img, (1, H, W, C), wt, bias, gate=gate), args.iters)
    res["se_gate_h16_gbps"] = 2 * H * W * C * 4 / (res["se_gate_h16_ms"] * 1e6)  # the image read twice, written once

    # Anchor3DHead decode
    nc, R = len(bf.CLASSES), bf.anchors_per_loc()
    q = rng.integers(-60, -12, (R * nc, H, W))
    hot = rng.random(q.shape) < 0.02
    q[hot] = rng.integers(-11, 12, int(hot.sum()))
    head = np.zeros((1, R * (nc + 11), H, W), np.float32)
    head[0, :R * nc] = q / 4.0
    head[0, R * nc:] = rng.normal(0, 0.3, (R * 11, H, W))
    hd = torch.from_numpy(head).to(dev)
    anchors = torch.from_numpy(bf.make_anchors()).to(dev)
    tc = cfg["test"]
    outs = anchor3d_postprocess_device(hd, anchors, nc, R, tc["nms_pre"], tc["score_thr"], tc["nms_thr"], tc["max_num"],
                                       tc["dir_offset"], tc["dir_limit_offset"])
    res["anchor3d_postprocess_ms"] = event_ms(
        lambda: anchor3d_postprocess_device(hd, anchors, nc, R, tc["nms_pre"], tc["score_thr"], tc["nms_thr"],
                                            tc["max_num"], tc["dir_offset"], tc["dir_limit_offset"], out=outs), args.iters)
    res["anchor3d_rows"] = int(outs[3].item())
    res = {k: (round(v, 4) if isinstance(v, float) else v) for k, v in res.items()}
    print(json.dumps(dict(res, iters=args.iters, gpu=gpu_identity())))


if __name__ == "__main__":
    main()
