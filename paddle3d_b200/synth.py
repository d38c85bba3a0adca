"""Seeded synthetic inputs for the hot path (numpy only; no datasets exist offline).

Shapes follow SURVEY.md §8 / BASELINE.json configs:
  C1 1k pts (C2 geometry)   C2 PointPillars KITTI 20k x 4   C3 CenterPoint-voxel nuScenes 300k x 5
  C4 bev_pool_v2 (6 cams, 16x44 feature maps, D=118, C=80, 128x128 / 200x200 BEV grid)
Config values cite the reference YAMLs they come from.
"""
import math

import numpy as np

# configs/pointpillars/pointpillars_xyres16_kitti_car.yml:87-108
C2 = dict(name="pointpillars_kitti", num_points=20000, point_dim=4, voxel_size=[0.16, 0.16, 4.0],
          point_cloud_range=[0.0, -39.68, -3.0, 69.12, 39.68, 1.0], max_points=32, max_voxels=40000)
# configs/centerpoint/centerpoint_voxels_0075voxel_nuscenes_10sweep.yml:111-172
C3 = dict(name="centerpoint_voxel_0075", num_points=300000, point_dim=5, voxel_size=[0.075, 0.075, 0.2],
          point_cloud_range=[-54.0, -54.0, -5.0, 54.0, 54.0, 3.0], max_points=10, max_voxels=160000)
# 0.1 m variant named by BASELINE.json.metric: same 1440x1440x40 grid over a 144 m square
C3_01 = dict(name="centerpoint_voxel_01", num_points=300000, point_dim=5, voxel_size=[0.1, 0.1, 0.2],
             point_cloud_range=[-72.0, -72.0, -5.0, 72.0, 72.0, 3.0], max_points=10, max_voxels=160000)
# SECOND v1.5 ped_cycle/xyres_16, which configs/pointpillars/pointpillars_xyres16_kitti_cyclist_pedestrian.yml descends
# from (PARITY UNPINNED: not checked against the yml): 0.16 m pillars over 47.36 x 39.68 m -> 296 x 248.  SECOND keeps
# 100 points per pillar; the fused PFN kernel takes at most 64, so this uses C2's 32.
C2_PED_CYCLIST = dict(name="pointpillars_kitti_ped_cyclist", num_points=20000, point_dim=4, voxel_size=[0.16, 0.16, 3.0],
                      point_cloud_range=[0.0, -19.84, -2.5, 47.36, 19.84, 0.5], max_points=32, max_voxels=40000)
C1 = dict(C2, name="c1_cpu", num_points=1000)
# LiDAR branch of BEVFusion (configs/bevfusion/bevf_pp_2x8_1x_nusc.yaml:87-105): 0.25 m pillars on a 400 x 400 grid
C4_LIDAR = dict(name="bevfusion_lidar_pillars", num_points=300000, point_dim=4, voxel_size=[0.25, 0.25, 8.0],
                point_cloud_range=[-50.0, -50.0, -5.0, 50.0, 50.0, 3.0], max_points=64, max_voxels=40000)
# CenterPoint-pillars, configs/centerpoint/centerpoint_pillars_02voxel_nuscenes_10sweep.yml and det3d's
# nusc_centerpoint_pp_02voxel_two_pfn_10sweep it descends from (PARITY UNPINNED: recalled, not checked against the yml):
# 0.2 m pillars over +-51.2 m -> 512 x 512, 20 points per pillar, max_num_voxels 60000 (the test-time value)
CP_PILLARS = dict(name="centerpoint_pillars_02", num_points=300000, point_dim=5, voxel_size=[0.2, 0.2, 8.0],
                  point_cloud_range=[-51.2, -51.2, -5.0, 51.2, 51.2, 3.0], max_points=20, max_voxels=60000)

CENTERPOINT_TASKS = [1, 2, 2, 1, 2, 2]  # classes per task (yml:139-151)
CENTERPOINT_TEST_CFG = dict(  # yml:163-172
    post_center_limit_range=[-61.2, -61.2, -10.0, 61.2, 61.2, 10.0], nms_pre_max_size=1000, nms_post_max_size=83,
    nms_iou_threshold=0.2, score_threshold=0.1, down_ratio=8)
# the same test config for CenterPoint-pillars, whose head runs at a quarter of the 512 x 512 grid (PARITY UNPINNED)
CENTERPOINT_PILLARS_TEST_CFG = dict(CENTERPOINT_TEST_CFG, down_ratio=4)

# CenterPoint-pillars KITTI, configs/centerpoint/centerpoint_pillars_016voxel_kitti.yml (PARITY UNPINNED: recalled from the
# yml and its deploy command line `--max_points_in_voxel 100`, not checked against either): 0.16 m pillars over the KITTI
# camera range -> 432 x 496, 100 points per pillar, 40000 pillars at test time (the yml's test max_num_voxels).
# num_points: the rows a frame takes after the camera cull (tools/infer_kitti.py's default).
CP_PILLARS_KITTI = dict(name="centerpoint_pillars_016_kitti", num_points=40000, point_dim=4, voxel_size=[0.16, 0.16, 4.0],
                        point_cloud_range=[0.0, -39.68, -3.0, 69.12, 39.68, 1.0], max_points=100, max_voxels=40000)
CP_PILLARS_KITTI_TASKS = [1, 2]  # [Car], [Pedestrian, Cyclist] (yml tasks; the order is recalled)
# the yml's test_cfg (PARITY UNPINNED): the head runs at half the 432 x 496 grid
CP_PILLARS_KITTI_TEST_CFG = dict(
    post_center_limit_range=[-10.0, -50.0, -10.0, 80.0, 50.0, 10.0], nms_pre_max_size=1000, nms_post_max_size=83,
    nms_iou_threshold=0.1, score_threshold=0.1, down_ratio=2)


def uniform_cloud(cfg, seed, num_points=None, margin=0.02):
    """Worst case for hashing: x,y,z ~ U(range, slightly overshooting so some points fall outside)."""
    rng = np.random.default_rng(seed)
    n = cfg["num_points"] if num_points is None else num_points
    lo = np.asarray(cfg["point_cloud_range"][:3], np.float64)
    hi = np.asarray(cfg["point_cloud_range"][3:], np.float64)
    span = hi - lo
    xyz = rng.uniform(lo - margin * span, hi + margin * span, size=(n, 3))
    extra = rng.uniform(0.0, 1.0, size=(n, cfg["point_dim"] - 3))
    return np.concatenate([xyz, extra], 1).astype(np.float32)


def lidar_cloud(cfg, seed, num_points=None, sweeps=10, beams=32):
    """LiDAR-like occupancy (SURVEY.md §8d): `sweeps` x `beams` rings hitting the ground plane
    z=-1.8 m or one of 64 seeded boxes; sigma = 2 cm noise; intensity U(0,1); time lag = sweep*0.05."""
    rng = np.random.default_rng(seed)
    n = cfg["num_points"] if num_points is None else num_points
    pcr = cfg["point_cloud_range"]
    rmax = min(pcr[3], pcr[4])
    az_steps = int(math.ceil(n / (sweeps * beams))) + 8
    elev = np.deg2rad(np.linspace(-30.67, 10.67, beams))
    # boxes: centre (x,y), half sizes, height
    nb = 64
    bc = rng.uniform(-0.8 * rmax, 0.8 * rmax, size=(nb, 2))
    bs = rng.uniform(0.75, 5.0, size=(nb, 2))
    bh = rng.uniform(1.0, 3.5, size=(nb,))
    pts = []
    for s in range(sweeps):
        az = rng.uniform(0, 2 * np.pi) + np.linspace(0, 2 * np.pi, az_steps, endpoint=False)
        a, e = np.meshgrid(az, elev, indexing="ij")
        dx, dy, dz = np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)
        # ground hit
        with np.errstate(divide="ignore", invalid="ignore"):
            tg = np.where(dz < -1e-3, -1.8 / dz, np.inf)
        t = np.minimum(tg, rmax * 1.2)
        # box hits (slab test in xy, then height check)
        for k in range(nb):
            with np.errstate(divide="ignore", invalid="ignore"):
                tx1, tx2 = (bc[k, 0] - bs[k, 0]) / dx, (bc[k, 0] + bs[k, 0]) / dx
                ty1, ty2 = (bc[k, 1] - bs[k, 1]) / dy, (bc[k, 1] + bs[k, 1]) / dy
            tn = np.maximum(np.minimum(tx1, tx2), np.minimum(ty1, ty2))
            tf = np.minimum(np.maximum(tx1, tx2), np.maximum(ty1, ty2))
            hit = (tn > 0.5) & (tn < tf)
            zh = -1.8 + bh[k]
            zz = tn * dz
            hit &= (zz < zh - 1.8 + 1.8) & (zz > -1.8)
            t = np.where(hit & (tn < t), tn, t)
        ok = np.isfinite(t) & (t < rmax * 1.1)
        x, y, z = (t * dx)[ok], (t * dy)[ok], (t * dz)[ok]
        p = np.stack([x, y, z], 1) + rng.normal(0, 0.02, size=(ok.sum(), 3))
        cols = [p]
        if cfg["point_dim"] >= 4:
            cols.append(rng.uniform(0, 1, size=(len(p), 1)))
        if cfg["point_dim"] >= 5:
            cols.append(np.full((len(p), 1), s * 0.05))
        pts.append(np.concatenate(cols, 1))
    pts = np.concatenate(pts, 0)
    rng.shuffle(pts, axis=0)
    if len(pts) < n:  # pad by jittered repeats
        rep = pts[rng.integers(0, len(pts), size=n - len(pts))].copy()
        rep[:, :3] += rng.normal(0, 0.05, size=(len(rep), 3))
        pts = np.concatenate([pts, rep], 0)
    return pts[:n].astype(np.float32)


def sweep_sequence(n_sweeps, seed, points_per_sweep=29500, speed=10.0, yaw_rate=0.3, period=0.05):
    """A raw multi-sweep LiDAR stream: [(cloud [n_i, 5] fp32 (x, y, z, intensity, ring) in the sensor frame,
    global_from_lidar [4, 4] float64, timestamp [s])], one sweep every `period` (20 Hz) from an ego vehicle driving at
    `speed` m/s while turning at `yaw_rate` rad/s.  Each sweep is one ring sweep of lidar_cloud (its scene drawn per
    sweep); n_i = points_per_sweep +- 500, so ten merged sweeps stay within C3's 300k points."""
    rng = np.random.default_rng(seed)
    out = []
    for s in range(n_sweeps):
        n = int(points_per_sweep + rng.integers(-500, 501))
        pts = lidar_cloud(dict(C3, point_dim=4), seed * 1000 + s, num_points=n, sweeps=1)
        elev = np.degrees(np.arctan2(pts[:, 2], np.hypot(pts[:, 0], pts[:, 1])))
        ring = np.clip(np.rint((elev + 30.67) / (41.34 / 31)), 0, 31).astype(np.float32)
        t = 1000.0 + s * period
        yaw = yaw_rate * s * period
        x, y = speed * s * period * np.cos(yaw / 2), speed * s * period * np.sin(yaw / 2)
        pose = np.array([[np.cos(yaw), -np.sin(yaw), 0.0, x], [np.sin(yaw), np.cos(yaw), 0.0, y], [0.0, 0.0, 1.0, 1.84],
                         [0.0, 0.0, 0.0, 1.0]])
        out.append((np.concatenate([pts, ring[:, None]], 1).astype(np.float32), pose, t))
    return out


# A KITTI object-split calib file (the 2011_09_26 drive's camera and LiDAR calibration, as in training/calib/000000.txt)
KITTI_CALIB = """P0: 7.215377e+02 0.000000e+00 6.095593e+02 0.000000e+00 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P1: 7.215377e+02 0.000000e+00 6.095593e+02 -3.875744e+02 0.000000e+00 7.215377e+02 1.728540e+02 0.000000e+00 0.000000e+00 0.000000e+00 1.000000e+00 0.000000e+00
P2: 7.215377e+02 0.000000e+00 6.095593e+02 4.485728e+01 0.000000e+00 7.215377e+02 1.728540e+02 2.163791e-01 0.000000e+00 0.000000e+00 1.000000e+00 2.745884e-03
P3: 7.215377e+02 0.000000e+00 6.095593e+02 -3.395242e+02 0.000000e+00 7.215377e+02 1.728540e+02 2.199936e+00 0.000000e+00 0.000000e+00 1.000000e+00 2.729905e-03
R0_rect: 9.999239e-01 9.837760e-03 -7.445048e-03 -9.869795e-03 9.999421e-01 -4.278459e-03 7.402527e-03 4.351614e-03 9.999631e-01
Tr_velo_to_cam: 7.533745e-03 -9.999714e-01 -6.166020e-04 -4.069766e-03 1.480249e-02 7.280733e-04 -9.998902e-01 -7.631618e-02 9.998621e-01 7.523790e-03 1.480755e-02 -2.717806e-01
Tr_imu_to_velo: 9.999976e-01 7.553071e-04 -2.035826e-03 -8.086759e-01 -7.854027e-04 9.998898e-01 -1.482298e-02 3.195559e-01 2.024406e-03 1.482454e-02 9.998881e-01 -7.997231e-01
"""


def kitti_raw_cloud(seed, beams=64, max_range=80.0, height=1.73):
    """A raw KITTI `velodyne/*.bin`-like scan: (cloud [n, 4] fp32 (x, y, z, reflectance), ~120k points over 360 degrees
    from an HDL-64E-like sensor (64 beams from +2 to -24.8 degrees, ~1900 azimuth steps, ~3 % dropped returns) over a
    ground plane `height` m below it and 96 seeded boxes, in azimuth order; the calib dict of KITTI_CALIB
    (kitti.parse_calib); the image shape (H, W) of the reference's default).  About a quarter of the points lie in the
    camera's view."""
    from . import kitti
    rng = np.random.default_rng(seed)
    az_steps = 1850 + int(rng.integers(0, 100))
    az = rng.uniform(0, 2 * np.pi) + np.linspace(0, 2 * np.pi, az_steps, endpoint=False)
    elev = np.deg2rad(np.linspace(2.0, -24.8, beams))
    a, e = np.meshgrid(az, elev, indexing="ij")  # azimuth-major: one column of 64 beams after another
    dx, dy, dz = np.cos(e) * np.cos(a), np.cos(e) * np.sin(a), np.sin(e)
    with np.errstate(divide="ignore", invalid="ignore"):
        t = np.where(dz < -1e-3, -height / dz, np.inf)
    nb = 96
    bc = rng.uniform(-60.0, 60.0, size=(nb, 2))
    bs = rng.uniform(0.5, 3.0, size=(nb, 2))
    bh = rng.uniform(1.0, 3.5, size=(nb,))
    for k in range(nb):
        with np.errstate(divide="ignore", invalid="ignore"):
            tx1, tx2 = (bc[k, 0] - bs[k, 0]) / dx, (bc[k, 0] + bs[k, 0]) / dx
            ty1, ty2 = (bc[k, 1] - bs[k, 1]) / dy, (bc[k, 1] + bs[k, 1]) / dy
        tn = np.maximum(np.minimum(tx1, tx2), np.minimum(ty1, ty2))
        tf = np.minimum(np.maximum(tx1, tx2), np.maximum(ty1, ty2))
        zz = tn * dz
        hit = (tn > 1.0) & (tn < tf) & (zz > -height) & (zz < bh[k] - height)
        t = np.where(hit & (tn < t), tn, t)
    ok = (t < max_range) & (rng.uniform(size=t.shape) > 0.03)
    p = np.stack([(t * dx)[ok], (t * dy)[ok], (t * dz)[ok]], 1) + rng.normal(0, 0.02, size=(int(ok.sum()), 3))
    cloud = np.concatenate([p, rng.uniform(0, 1, size=(len(p), 1))], 1).astype(np.float32)
    return cloud, kitti.parse_calib(KITTI_CALIB, "synth.KITTI_CALIB"), kitti.DEFAULT_IMAGE_SHAPE


def random_boxes(n, seed, extent=40.0, clustered=True):
    """[x,y,z,dx,dy,dz,heading] boxes; clustered centres so that rotated overlaps are common."""
    rng = np.random.default_rng(seed)
    if clustered:
        centres = rng.uniform(-extent, extent, size=(max(n // 8, 1), 2))
        xy = centres[rng.integers(0, len(centres), size=n)] + rng.normal(0, 1.2, size=(n, 2))
    else:
        xy = rng.uniform(-extent, extent, size=(n, 2))
    z = rng.normal(-1.0, 0.5, size=(n, 1))
    dims = np.abs(rng.normal([4.2, 1.9, 1.6], [1.0, 0.4, 0.3], size=(n, 3))) + 0.2
    heading = rng.uniform(-np.pi, np.pi, size=(n, 1))
    return np.concatenate([xy, z, dims, heading], 1).astype(np.float32)


def centerpoint_head_outputs(seed, tasks=CENTERPOINT_TASKS, H=180, W=180, hm_mean=-5.5, hm_std=1.5,
                             with_velocity=True):
    """Per-task head tensors (NCHW, batch 1) with the statistics of SURVEY.md §8d."""
    rng = np.random.default_rng(seed)
    out = dict(hm=[], reg=[], height=[], dim=[], vel=[], rot=[])
    for c in tasks:
        out["hm"].append(rng.normal(hm_mean, hm_std, size=(1, c, H, W)).astype(np.float32))
        out["reg"].append(rng.uniform(0, 1, size=(1, 2, H, W)).astype(np.float32))
        out["height"].append(rng.normal(-1, 1, size=(1, 1, H, W)).astype(np.float32))
        out["dim"].append(rng.normal(0.5, 0.4, size=(1, 3, H, W)).astype(np.float32))
        out["rot"].append(rng.normal(0, 1, size=(1, 2, H, W)).astype(np.float32))
        out["vel"].append(rng.normal(0, 1, size=(1, 2, H, W)).astype(np.float32) if with_velocity else out["reg"][-1])
    return out


def label_offsets(tasks=CENTERPOINT_TASKS):
    """num_classes attr as built by CenterHead.predict_by_custom_op (center_head.py:306-309):
    prefix sums; only the first T entries are used by the op."""
    off, flag = [], 0
    for c in tasks:
        off.append(flag)
        flag += c
    return off


def bev_pool_inputs(seed, n_cams=6, D=118, H=16, W=44, C=80, grid=(128, 128, 1), bounds=((-51.2, 51.2), (-51.2, 51.2), (-5.0, 3.0)),
                    depth_range=(1.0, 60.0)):
    """Restatement of LSSViewTransformer.voxel_pooling_prepare_v2
    (paddle3d/models/transformers/bevdet_transformer.py:230-274) on a synthetic 6-camera rig:
    pinhole cameras at 60-degree yaw steps, frustum points -> ego frame -> voxel ranks, argsort, run lengths."""
    rng = np.random.default_rng(seed)
    B, N = 1, n_cams
    gx, gy, gz = grid
    lower = np.array([b[0] for b in bounds], np.float32)
    interval = np.array([(bounds[0][1] - bounds[0][0]) / gx, (bounds[1][1] - bounds[1][0]) / gy,
                         (bounds[2][1] - bounds[2][0]) / gz], np.float32)
    fx = 1266.0 * (704.0 / 1600.0) / 16.0  # focal in feature-map pixels
    cx, cy = W / 2.0, H / 2.0
    d = np.linspace(depth_range[0], depth_range[1], D, dtype=np.float32)
    u = (np.arange(W, dtype=np.float32) + 0.5)
    v = (np.arange(H, dtype=np.float32) + 0.5)
    dd, vv, uu = np.meshgrid(d, v, u, indexing="ij")  # D,H,W
    xc = (uu - cx) / fx * dd
    yc = (vv - cy) / fx * dd
    zc = dd
    coor = np.zeros((B, N, D, H, W, 3), np.float32)
    for n in range(N):
        yaw = n * (2 * np.pi / N)
        # camera: z forward, x right, y down  ->  ego: x forward, y left, z up
        fwd = np.array([np.cos(yaw), np.sin(yaw), 0.0], np.float32)
        right = np.array([np.sin(yaw), -np.cos(yaw), 0.0], np.float32)
        up = np.array([0.0, 0.0, 1.0], np.float32)
        p = zc[..., None] * fwd + xc[..., None] * right - yc[..., None] * up
        p[..., 2] += 1.5
        coor[0, n] = p
    num_points = B * N * D * H * W
    ranks_depth = np.arange(num_points, dtype=np.int64)
    ranks_feat = np.arange(num_points // D, dtype=np.int64).reshape(B, N, 1, H, W)
    ranks_feat = np.broadcast_to(ranks_feat, (B, N, D, H, W)).reshape(-1)
    c = ((coor - lower) / interval).astype(np.int64).reshape(num_points, 3)  # trunc toward 0 (:241-243)
    batch_idx = np.repeat(np.arange(B), num_points // B)
    kept = (c[:, 0] >= 0) & (c[:, 0] < gx) & (c[:, 1] >= 0) & (c[:, 1] < gy) & (c[:, 2] >= 0) & (c[:, 2] < gz)
    c, ranks_depth, ranks_feat, batch_idx = c[kept], ranks_depth[kept], ranks_feat[kept], batch_idx[kept]
    ranks_bev = batch_idx * (gz * gy * gx) + c[:, 2] * (gy * gx) + c[:, 1] * gx + c[:, 0]
    order = np.argsort(ranks_bev, kind="stable")
    ranks_bev, ranks_depth, ranks_feat = ranks_bev[order], ranks_depth[order], ranks_feat[order]
    first = np.ones(len(ranks_bev), bool)
    first[1:] = ranks_bev[1:] != ranks_bev[:-1]
    interval_starts = np.nonzero(first)[0].astype(np.int32)
    interval_lengths = np.zeros_like(interval_starts)
    interval_lengths[:-1] = interval_starts[1:] - interval_starts[:-1]
    interval_lengths[-1] = len(ranks_bev) - interval_starts[-1]
    logits = rng.normal(0, 1, size=(B * N, D, H, W)).astype(np.float32)
    e = np.exp(logits - logits.max(1, keepdims=True))
    depth = (e / e.sum(1, keepdims=True)).astype(np.float32)
    feat = rng.normal(0, 1, size=(B * N, H, W, C)).astype(np.float32)
    return dict(depth=depth, feat=feat, ranks_depth=ranks_depth.astype(np.int32), ranks_feat=ranks_feat.astype(np.int32),
                ranks_bev=ranks_bev.astype(np.int32), interval_starts=interval_starts,
                interval_lengths=interval_lengths.astype(np.int32), bev_feat_shape=(B, gy, gx, C),
                coor=coor, grid_lower_bound=lower, grid_interval=interval, grid_size=(gx, gy, gz))


def kaiming_uniform(rng, shape, fan_in):
    bound = math.sqrt(6.0 / fan_in) / math.sqrt(1 + 5.0)  # a = sqrt(5), as reset_parameters does
    return rng.uniform(-bound, bound, size=shape).astype(np.float32)


# LSSViewTransformer grids (BEVDet-R50's 0.8 m grid and BASELINE config 4's 0.5 m grid; D = 118 depth bins of 0.5 m)
LSS_BEVDET = dict(x=[-51.2, 51.2, 0.8], y=[-51.2, 51.2, 0.8], z=[-5.0, 3.0, 8.0], depth=[1.0, 60.0, 0.5])
LSS_C4 = dict(LSS_BEVDET, x=[-50.0, 50.0, 0.5], y=[-50.0, 50.0, 0.5])
LSS_INPUT_SIZE, LSS_DOWNSAMPLE, LSS_CHANNELS = (256, 704), 16, 80


def _rot(axis, a):
    c, s = np.cos(a), np.sin(a)
    i, j = [(1, 2), (2, 0), (0, 1)][axis]
    m = np.eye(3)
    m[i, i], m[i, j], m[j, i], m[j, j] = c, -s, s, c
    return m


def camera_rig(seed, B=1, n_cams=6, bda=True):
    """Camera matrices of a nuScenes-like rig in the form BEVDet's LSSViewTransformer.get_lidar_coor takes them, float32:
    sensor2ego / ego2global [B, N, 4, 4], cam2imgs / post_rots [B, N, 3, 3], post_trans [B, N, 3], bda [B, 3, 3].
    Pinhole intrinsics at the 1600 x 900 scale (fx = fy = 1266, seeded principal point near the centre); cameras at
    60-degree yaw steps (z forward, x right, y down) with a seeded pitch / roll of up to 2 degrees and seeded mounting
    offsets; image augmentation = resize by 0.44 to 704 x 396 and a crop of the bottom 256 rows; bda = a seeded flip +
    rotation of up to 22.5 degrees (bda=True) or the identity."""
    rng = np.random.default_rng(seed)
    N = n_cams
    s2e = np.zeros((B, N, 4, 4))
    e2g = np.zeros((B, N, 4, 4))
    k = np.zeros((B, N, 3, 3))
    prot = np.zeros((B, N, 3, 3))
    ptr = np.zeros((B, N, 3))
    bd = np.zeros((B, 3, 3))
    # camera axes in the ego frame (x forward, y left, z up): x_cam = right, y_cam = down, z_cam = forward
    base = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])
    for b in range(B):
        for n in range(N):
            yaw = n * np.pi / 3 + rng.uniform(-0.02, 0.02)
            r = _rot(2, yaw) @ _rot(1, rng.uniform(-0.035, 0.035)) @ _rot(0, rng.uniform(-0.035, 0.035)) @ base
            s2e[b, n, :3, :3] = r
            s2e[b, n, :3, 3] = [1.0 * np.cos(yaw) + rng.uniform(-0.1, 0.1), 0.5 * np.sin(yaw) + rng.uniform(-0.1, 0.1),
                                1.5 + rng.uniform(-0.05, 0.05)]
            s2e[b, n, 3, 3] = 1.0
            e2g[b, n] = np.eye(4)
            e2g[b, n, :3, :3] = _rot(2, 0.3 * b + 0.1)
            e2g[b, n, :3, 3] = [600.0 + b, 1600.0, 0.0]
            k[b, n] = [[1266.0, 0.0, 800.0 + rng.uniform(-20, 20)], [0.0, 1266.0, 450.0 + rng.uniform(-10, 10)], [0, 0, 1]]
            prot[b, n] = np.diag([0.44, 0.44, 1.0])
            ptr[b, n] = [0.0, -(900 * 0.44 - 256), 0.0]
        if bda:
            flip = np.diag([-1.0 if rng.uniform() < 0.5 else 1.0, -1.0 if rng.uniform() < 0.5 else 1.0, 1.0])
            bd[b] = flip @ _rot(2, rng.uniform(-np.pi / 8, np.pi / 8))
        else:
            bd[b] = np.eye(3)
    f = np.float32
    return dict(sensor2ego=s2e.astype(f), ego2global=e2g.astype(f), cam2imgs=k.astype(f), post_rots=prot.astype(f),
                post_trans=ptr.astype(f), bda=bd.astype(f))


def ego_poses(n_frames, speed=10.0, yaw_rate=0.3, period=0.5, origin=(600.0, 1600.0)):
    """global_from_ego [n_frames, 4, 4] float64 of an ego vehicle driving at `speed` m/s while turning at `yaw_rate` rad/s,
    one pose every `period` s (sweep_sequence's motion; 0.5 s = nuScenes' 2 Hz key frames), starting at `origin`."""
    out = np.zeros((n_frames, 4, 4))
    for s in range(n_frames):
        yaw = yaw_rate * s * period
        x, y = speed * s * period * np.cos(yaw / 2), speed * s * period * np.sin(yaw / 2)
        out[s] = [[np.cos(yaw), -np.sin(yaw), 0.0, origin[0] + x], [np.sin(yaw), np.cos(yaw), 0.0, origin[1] + y],
                  [0.0, 0.0, 1.0, 0.0], [0.0, 0.0, 0.0, 1.0]]
    return out


def camera_images(seed, n_cams=6, H=256, W=704, cell=16):
    """Seeded normalised camera images [n_cams, 3, H, W] float32, what BEVDet's data pipeline hands the image backbone
    (img_inputs[0] after mean / std normalisation): spatially smooth (white noise on a grid of `cell`-pixel cells,
    interpolated bilinearly, plus 10 % pixel noise), each channel scaled to zero mean and unit variance, so that the convs
    see image-like structure rather than white noise."""
    rng = np.random.default_rng([seed, 11])
    gh, gw = H // cell + 2, W // cell + 2
    coarse = rng.normal(size=(n_cams, 3, gh, gw))

    def axis(n, g):
        src = (np.arange(n) + 0.5) / cell
        i = np.minimum(np.floor(src).astype(np.int64), g - 2)
        return i, (src - i)[:, None] if n == H else (src - i)[None, :]
    yi, ly = axis(H, gh)
    xi, lx = axis(W, gw)
    a = coarse[:, :, yi][:, :, :, xi]
    b = coarse[:, :, yi][:, :, :, xi + 1]
    c = coarse[:, :, yi + 1][:, :, :, xi]
    d = coarse[:, :, yi + 1][:, :, :, xi + 1]
    img = (a * (1 - lx) + b * lx) * (1 - ly) + (c * (1 - lx) + d * lx) * ly
    img = img + 0.1 * rng.normal(size=img.shape)
    img = (img - img.mean(axis=(2, 3), keepdims=True)) / img.std(axis=(2, 3), keepdims=True)
    return img.astype(np.float32)


def camera_frames(seed, n_cams=6, H=900, W=1600):
    """Seeded decoded camera frames [n_cams, H, W, 3] uint8 (HWC RGB, what np.array(Image.open(path)) gives for a nuScenes
    image): smooth structure (noise on a 48-pixel grid, interpolated bilinearly), a dozen hard-edged rectangles, pixel
    noise, and a contrast that saturates part of every frame at 0 and at 255, so that resampling meets edges and both
    clamps."""
    rng = np.random.default_rng([seed, 13])
    cell = 48
    gh, gw = H // cell + 2, W // cell + 2
    coarse = rng.normal(size=(n_cams, gh, gw, 3)).astype(np.float32)
    ys, xs = (np.arange(H, dtype=np.float32) + 0.5) / cell, (np.arange(W, dtype=np.float32) + 0.5) / cell
    yi, xi = np.minimum(ys.astype(np.int64), gh - 2), np.minimum(xs.astype(np.int64), gw - 2)
    ly, lx = (ys - yi)[None, :, None, None], (xs - xi)[None, None, :, None]
    top = coarse[:, yi][:, :, xi] * (1 - lx) + coarse[:, yi][:, :, xi + 1] * lx
    bot = coarse[:, yi + 1][:, :, xi] * (1 - lx) + coarse[:, yi + 1][:, :, xi + 1] * lx
    img = 128.0 + 110.0 * (top * (1 - ly) + bot * ly)
    for n in range(n_cams):
        for _ in range(12):
            h, w = int(rng.integers(8, H // 3)), int(rng.integers(8, W // 3))
            y, x = int(rng.integers(0, H - h)), int(rng.integers(0, W - w))
            img[n, y:y + h, x:x + w] = rng.uniform(-40, 300, 3).astype(np.float32)
    img += rng.normal(0, 6, img.shape).astype(np.float32)
    return np.ascontiguousarray(np.clip(np.rint(img), 0, 255).astype(np.uint8))


def camera_jpegs(seed, n_cams=6, H=900, W=1600, **pillow_save_kwargs):
    """camera_frames(seed, n_cams, H, W) encoded by Pillow as JPEG files: a list of n_cams bytes objects.
    pillow_save_kwargs go to Image.save (quality, subsampling, optimize, restart_marker_blocks, ...).  Pillow is
    imported here: the package itself does not depend on it."""
    import io

    from PIL import Image

    out = []
    for frame in camera_frames(seed, n_cams, H, W):
        buf = io.BytesIO()
        Image.fromarray(frame).save(buf, "JPEG", **pillow_save_kwargs)
        out.append(buf.getvalue())
    return out


def lss_mats(rig):
    """(sensor2ego, cam2imgs, post_rots, post_trans, bda) of a camera_rig, the order LSSHotPath takes them in."""
    return rig["sensor2ego"], rig["cam2imgs"], rig["post_rots"], rig["post_trans"], rig["bda"]
