"""TEST INFRASTRUCTURE ONLY — the CPU arm of a CenterPoint-pillars frame whose CenterHead has no velocity head (the KITTI
model, centerpoint_pillars.CONFIG_KITTI), for tests/ and tools/centerpoint_pillars_bench.py --config kitti.

oracle.centerpoint_pillars.CpuCenterPointPillars.run postprocesses with velocity; this arm runs the same stages and takes
velocity from the head: with_velocity is whether the exported weights carry a "vel" head, and the boxes have 7 columns
(x, y, z, d0, d1, d2, rot) without one."""
import time

import numpy as np

from oracle import centerpoint_postprocess, hard_voxelize, pillar_scatter, ref_hard_voxelize_cpu
from oracle.centerpoint_pillars import CpuCenterPointPillars, pillar_feature_net2


class CpuCenterPointPillarsHeads(CpuCenterPointPillars):
    """CpuCenterPointPillars with the velocity of the postprocess taken from the head."""

    def run(self, points):
        cfg, tc = self.cfg, self.tc
        t = {}
        t0 = time.perf_counter()
        vox = ref_hard_voxelize_cpu if self.use_ref else hard_voxelize
        v, c, n, nv = vox(points, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"], cfg["max_voxels"])
        k = int(nv[0])
        coors = np.concatenate([np.zeros((k, 1), np.int32), c[:k]], 1)
        t["voxelize"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        feats = pillar_feature_net2(v[:k], n[:k], coors, self.w["pfn"], cfg["voxel_size"], cfg["point_cloud_range"])
        t["pfn"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        nx, ny = self.grid
        bev = pillar_scatter(feats, coors, 1, ny, nx)
        t["scatter"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        h = self.dense.run(bev)
        t["dense"] = time.perf_counter() - t0
        t0 = time.perf_counter()
        with_vel = "vel" in h
        boxes, scores, labels, _ = centerpoint_postprocess(
            h["hm"], h["reg"], h["height"], h["dim"], h["vel"] if with_vel else h["reg"], h["rot"], cfg["voxel_size"][:2],
            cfg["point_cloud_range"], tc["post_center_limit_range"], self.off, tc["down_ratio"], tc["score_threshold"],
            tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"], with_vel)
        t["postprocess"] = time.perf_counter() - t0
        return dict(boxes=boxes, scores=scores, labels=labels, head=h, feats=feats, num_voxels=k, coors=coors, times=t)
