#!/usr/bin/env python
"""Run the narrow-layer warp-MMA kernel twice on the level-0 / level-1 index sets of a C3 frame and compare bit for bit
(stream-K fix-up order), and against the wgmma kernel (same arithmetic, different summation order)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from paddle3d_b200 import synth  # noqa: E402
from paddle3d_b200.ops import sparse_nn as sp  # noqa: E402
from paddle3d_b200.ops import voxelize  # noqa: E402


def main():
    dev = torch.device("cuda:0")
    cfg = synth.C3
    pts = torch.from_numpy(synth.lidar_cloud(cfg, 0)).to(dev)
    mean, coors, npv, nv = voxelize.voxelize_mean(pts, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"], cfg["max_voxels"], 0)
    n = int(nv.item())
    rng = np.random.default_rng(0)
    grid = [41, 1440, 1440]
    for cin, cout, subm in ((16, 16, True), (32, 32, True), (16, 32, False)):
        feats = torch.from_numpy(rng.normal(size=(cfg["max_voxels"], cin)).astype(np.float32)).to(dev)
        cls = sp.SubmConv3D if subm else sp.Conv3D
        conv = cls(cin, cout, 3, 1 if subm else 2, padding=1, bias_attr=True).init_parameters(rng, dev)
        conv.precision = sp.F16X3
        outs = []
        for rep, wm in ((0, True), (1, True), (2, True), (3, False)):
            sp.NARROW_WM[0] = wm
            x = sp.sparse_coo_tensor(coors[:, :4].t(), feats, [1] + grid + [cin])
            x.index.num = nv
            y = sp.ReLU()(conv(x))
            v = y.get(sp.ROWS_H16)
            torch.cuda.synchronize()
            m = int(y.index.num[0].item())
            outs.append(v[:m].clone())
        sp.NARROW_WM[0] = True
        same01 = torch.equal(outs[0], outs[1]) and torch.equal(outs[1], outs[2])
        nd = (outs[0] != outs[1]).sum().item() + (outs[1] != outs[2]).sum().item()
        d = (outs[0].float() - outs[3].float()).abs().max().item()
        print("%d->%d rows %d: wm run-to-run bit-identical %s (%d halfs differ); wm vs wgmma max |diff| of the half words %.3g"
              % (cin, cout, outs[0].shape[0], same01, nd, d), flush=True)


if __name__ == "__main__":
    main()
