"""GPU: the camera frustum cull inside the sweep merge kernel (p3d_merge_sweeps_frustum) against its host oracle
kitti.remove_camera_invisible, and PointPillars on raw KITTI scans (frame.KITTI_INPUT: infer_kitti, a captured graph,
infer_kitti_many over lanes, a .pdparams checkpoint, tools/infer_kitti.py) against the same frame fed the host-culled
clouds through infer()."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from conftest import ROOT
from paddle3d_b200 import checkpoint, kitti, synth

pytestmark = pytest.mark.gpu

QNAN = 0x7fc00000
BN_GAIN = 6.0 ** 0.5
N_POINTS = 40000  # rows after the cull: the turned calibrations keep up to ~24k of a scan


def _check_cull(name, out, n_out, status, want, expect_status=0):
    """Kept rows, their order and count bit-equal to the oracle; NaN tail."""
    got = out.cpu().numpy()
    n = int(n_out.item())
    assert int(status.item()) == expect_status, name
    assert n == len(want), (name, n, len(want))
    assert np.array_equal(got[:n].view(np.uint32), np.ascontiguousarray(want, np.float32).view(np.uint32)), name
    assert (got[n:].view(np.uint32) == QNAN).all(), name


def _scan(seed=1):
    cloud, c, shape = synth.kitti_raw_cloud(seed)
    return cloud, c, shape, kitti.frustum_planes(c, shape)


def _cases():
    cloud, _, _, planes = _scan()
    rng = np.random.default_rng(3)
    ahead = np.stack([rng.uniform(5, 50, 3000), rng.uniform(-1, 1, 3000), rng.uniform(-1, 1, 3000),
                      rng.uniform(0, 1, 3000)], 1).astype(np.float32)
    behind = ahead * np.array([-1, 1, 1, 1], np.float32)
    on = np.zeros((6, 4))
    on[:, 3] = -1.0
    on[2] = (1.0, 0.0, 0.0, -3.0)  # the plane x = 3 among planes every point is inside
    on_rows = np.array([[3.0, 0, 0, 1], [2.9999998, 0, 0, 2], [3.0000002, 0, 0, 3], [3.0, 5, -5, 4]] * 300, np.float32)
    special = cloud[:5000].copy()
    special[::7, 0] = np.nan
    special[1::7, 1] = np.nan
    special[2::7, 2] = np.inf
    special[3::7, 0] = -np.inf
    special[4::7, 2] = np.nan
    cap = synth.kitti_raw_cloud(0)[0]
    full = np.concatenate([cap] * 2, 0)[:196608]
    return {
        "scan": (cloud, planes),
        "all_kept": (ahead, planes),
        "none_kept": (behind, planes),
        "on_planes": (on_rows, on),
        "nan_inf_rows": (special, planes),
        "empty": (np.zeros((0, 4), np.float32), planes),
        "n_1000": (cloud[:1000], planes),
        "n_5003": (cloud[:5003], planes),
        "raw_capacity": (full, planes),
    }


@pytest.mark.parametrize("case", ["scan", "all_kept", "none_kept", "on_planes", "nan_inf_rows", "empty", "n_1000",
                                  "n_5003", "raw_capacity"])
def test_cull_matches_host(cuda, case):
    from paddle3d_b200.ops import sweep_merge as sm
    cloud, planes = _cases()[case]
    want = kitti.remove_camera_invisible(cloud, planes)
    out, n, st = sm.frustum_cull_device(cloud, planes, cap=len(cloud) + 9, device=cuda)
    _check_cull(case, out, n, st, want)
    if case == "all_kept":
        assert len(want) == len(cloud)
    if case in ("none_kept", "empty"):
        assert len(want) == 0
    if case == "on_planes":
        assert 0 < len(want) < len(cloud)
    if case == "nan_inf_rows":
        assert np.isnan(want[:, :3]).any()


def test_cull_overflow_bad_entry_and_refusals(cuda):
    import torch

    from paddle3d_b200._lib import P3DError
    from paddle3d_b200.ops import sweep_merge as sm
    cloud, _, _, planes = _scan()
    want = kitti.remove_camera_invisible(cloud, planes)
    cap = len(want) - 123
    out, n, st = sm.frustum_cull_device(cloud, planes, cap=cap, device=cuda)
    _check_cull("overflow", out, n, st, want[:cap], expect_status=sm.OVERFLOW)
    # a descriptor naming more rows than the slot holds: read as empty, flagged
    raw = torch.zeros((1, 1024, 4), dtype=torch.float32, device=cuda)
    out = torch.empty((64, 4), dtype=torch.float32, device=cuda)
    n_out = torch.empty((1,), dtype=torch.int32, device=cuda)
    status = torch.empty((1,), dtype=torch.int32, device=cuda)
    pl = torch.from_numpy(planes).to(cuda)
    desc = np.zeros(2, sm.DESC_DTYPE)
    sm.set_entry(desc[0], 0, 1025)
    sm.set_entry(desc[1], 0, 10)
    desc_dev = torch.from_numpy(desc.view(np.uint8)).to(cuda)
    sm.merge_frustum_into(raw, desc_dev, pl, [0, 1, 2, 3], out, n_out, status)
    _check_cull("bad entry", out, n_out, status, np.zeros((0, 4), np.float32), expect_status=sm.BAD_ENTRY)
    with pytest.raises(P3DError, match="merge_sweeps_frustum"):
        sm.merge_frustum_into(raw, desc_dev, pl, [0, 1, 2, 3], out, n_out, status, num_entries=2)
    with pytest.raises(ValueError):
        sm.merge_frustum_into(raw, desc_dev, pl.float(), [0, 1, 2, 3], out, n_out, status)


CONFIGS = ["car", "ped_cyclist"]


def _kw(config, cuda, **kw):
    from paddle3d_b200 import pointpillars as pp
    cfg, mc = (synth.C2, pp.CONFIG) if config == "car" else (synth.C2_PED_CYCLIST, pp.CONFIG_PED_CYCLIST)
    return dict(dict(cfg=cfg, model_cfg=mc, device=cuda, seed=0, bn_gain=BN_GAIN, num_points=N_POINTS), **kw)


def _reduced(cloud, planes, n=N_POINTS):
    import torch
    kept = kitti.remove_camera_invisible(cloud, planes)
    full = np.full((n, 4), np.nan, np.float32)
    full[:len(kept)] = kept
    return torch.from_numpy(full).pin_memory()


def _rotz(a):
    return np.array([[np.cos(a), -np.sin(a), 0, 0], [np.sin(a), np.cos(a), 0, 0], [0, 0, 1, 0], [0, 0, 0, 1.0]])


def _scans():
    """Raw scans of different point counts, calibrations (the LiDAR turned by a few degrees) and image shapes."""
    out = []
    for s, (yaw, shape) in enumerate([(0.0, (375, 1242)), (0.05, (370, 1224)), (-0.08, (376, 1241)), (0.02, (512, 1392)),
                                      (0.0, (374, 1238)), (-0.03, (375, 1242))]):
        cloud, c, _ = synth.kitti_raw_cloud(10 + s)
        c = dict(c, Tr_velo_to_cam=c["Tr_velo_to_cam"] @ _rotz(yaw))
        out.append((cloud, c, shape, kitti.frustum_planes(c, shape)))
    return out


def _bits(a, b):
    import torch
    return all(x.dtype == y.dtype and x.shape == y.shape and torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("config", CONFIGS)
def test_frame_on_raw_scans_matches_host_cull(cuda, config, tmp_path):
    import torch

    from paddle3d_b200 import frame
    from paddle3d_b200.pipeline import CenterPointSweep
    from paddle3d_b200.pointpillars import PointPillarsHotPath
    scans = _scans()
    assert len({len(s[0]) for s in scans}) == len(scans)
    ref = PointPillarsHotPath(**_kw(config, cuda))
    hot = PointPillarsHotPath(**_kw(config, cuda, sweep_input=frame.KITTI_INPUT))
    assert hot.h_status.numel() == ref.h_status.numel() + 1
    calib_pts = _reduced(scans[0][0], scans[0][3]).to(cuda)
    ref.calibrate_head(calib_pts)
    hot.calibrate_head(calib_pts)
    want = [tuple(t.clone() for t in ref.infer(_reduced(c, pl))) for c, _, _, pl in scans]
    assert sum(len(w[0]) for w in want) > 0
    eager = hot.infer_kitti(scans[1][0], scans[1][3])
    assert hot.merged_rows() == len(kitti.remove_camera_invisible(scans[1][0], scans[1][3]))
    assert _bits(eager, want[1])
    hot.capture()
    for j in (1, 0, 3):  # one graph over every calibration, image shape and point count
        assert _bits(hot.infer_kitti(scans[j][0], scans[j][3]), want[j]), j
    got = list(hot.infer_kitti_many((c, pl) for c, _, _, pl in scans))
    assert len(got) == len(scans) and all(_bits(g, w) for g, w in zip(got, want))
    with pytest.raises(ValueError):  # larger than the raw capacity: refused before anything is enqueued
        hot.infer_kitti(np.zeros((frame.KITTI_INPUT["slot_cap"] + 1, 4), np.float32), scans[0][3])
    with pytest.raises(ValueError):
        hot.infer_kitti(scans[0][0], scans[0][3][:5])
    assert _bits(hot.infer_kitti(scans[2][0], scans[2][3]), want[2])
    # 4 lanes sharing one ring = one lane
    lanes = CenterPointSweep(4, frame_cls=PointPillarsHotPath, **_kw(config, cuda, sweep_input=frame.KITTI_INPUT))
    assert all(p.ring is lanes.lanes[0].ring for p in lanes.lanes) and lanes.lanes[0].ring.slots == 5
    lanes.calibrate_head(calib_pts)
    for p in lanes.lanes:
        p.infer_kitti(scans[0][0], scans[0][3])
        p.capture()
    items = [(c, pl) for c, _, _, pl in scans] * 2
    got = list(lanes.infer_kitti_many(iter(items)))
    assert len(got) == len(items) and all(_bits(g, want[i % len(scans)]) for i, g in enumerate(got))
    # the seeded, calibrated model through a .pdparams file gives the same bits
    path = tmp_path / "model.pdparams"
    sd = dict(hot.state_dict())
    sd[checkpoint.STRUCTURED_NAMES] = {k: "param_%d" % i for i, k in enumerate(hot.state_dict())}
    with open(path, "wb") as f:
        pickle.dump(sd, f, protocol=4)
    loaded = PointPillarsHotPath(**_kw(config, cuda, seed=7, weights=str(path), sweep_input=frame.KITTI_INPUT))
    loaded.infer_kitti(scans[0][0], scans[0][3])
    loaded.capture()
    got = list(loaded.infer_kitti_many((c, pl) for c, _, _, pl in scans))
    assert all(_bits(g, w) for g, w in zip(got, want))
    del lanes, loaded
    torch.cuda.empty_cache()


def test_frame_raises_when_the_cull_overflows(cuda):
    from paddle3d_b200 import frame
    from paddle3d_b200.pointpillars import PointPillarsHotPath
    cloud, _, _, planes = _scan()
    kept = len(kitti.remove_camera_invisible(cloud, planes))
    hot = PointPillarsHotPath(**_kw("car", cuda, num_points=kept - 100, sweep_input=frame.KITTI_INPUT))
    with pytest.raises(RuntimeError, match="capacity"):
        hot.infer_kitti(cloud, planes)
    hot.infer_kitti(cloud[:len(cloud) // 2], planes)  # fits
    with pytest.raises(ValueError, match="one sweep"):
        PointPillarsHotPath(**_kw("car", cuda, sweep_input=dict(frame.KITTI_INPUT, max_sweeps=2)))


def test_default_graph_is_unchanged(cuda):
    """Without sweep input the PointPillars graph is the one it was (48 kernels, 12 memsets, the status copy); KITTI
    input adds the cull's two kernels and memset, and stacks the two status words with a kernel instead of the copy."""
    import torch

    from paddle3d_b200 import frame
    from paddle3d_b200.pointpillars import PointPillarsHotPath
    cloud, _, _, planes = _scan()
    counts = []
    for si in (None, frame.KITTI_INPUT):
        p = PointPillarsHotPath(**_kw("car", cuda, sweep_input=si))
        p.points.copy_(_reduced(cloud, planes).to(cuda))
        if si is not None:
            p.infer_kitti(cloud, planes)
        p.capture(count_nodes=True)
        counts.append(p.graph_nodes)
        del p
        torch.cuda.empty_cache()
    print("graph nodes: default %s, KITTI input %s" % tuple(counts))
    assert counts[0] == {"kernel": 48, "memcpy": 1, "memset": 12, "other": 0}
    assert counts[1] == {"kernel": 51, "memcpy": 0, "memset": 13, "other": 0}


def _png_header(path, h, w):
    import struct
    import zlib
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 2, 0, 0, 0)
    path.write_bytes(b"\x89PNG\r\n\x1a\n" + struct.pack(">I", 13) + b"IHDR" + ihdr +
                     struct.pack(">I", zlib.crc32(b"IHDR" + ihdr)) + bytes(12))


def test_infer_kitti_cli(cuda, tmp_path):
    """tools/infer_kitti.py on a KITTI-layout directory writes the label files of to_kitti on the hot path's boxes."""
    from paddle3d_b200 import frame
    from paddle3d_b200.pointpillars import PointPillarsHotPath
    scans = _scans()[:4]
    root = tmp_path / "training"
    for d in ("velodyne", "calib", "image_2"):
        (root / d).mkdir(parents=True)
    ids = ["%06d" % i for i in range(len(scans))]
    calib_lines = synth.KITTI_CALIB.splitlines()
    for fid, (cloud, c, shape, _) in zip(ids, scans):
        cloud.tofile(root / "velodyne" / (fid + ".bin"))
        tr = " ".join("%.17g" % v for v in c["Tr_velo_to_cam"][:3].reshape(-1))
        (root / "calib" / (fid + ".txt")).write_text(
            "\n".join("Tr_velo_to_cam: " + tr if ln.startswith("Tr_velo_to_cam:") else ln for ln in calib_lines) + "\n")
        if shape != kitti.DEFAULT_IMAGE_SHAPE:
            _png_header(root / "image_2" / (fid + ".png"), *shape)
    (tmp_path / "ids.txt").write_text("\n".join(ids[::-1]) + "\n")
    hot = PointPillarsHotPath(**_kw("car", cuda, num_points=40000, sweep_input=frame.KITTI_INPUT))
    hot.calibrate_head(_reduced(scans[0][0], scans[0][3], 40000).to(cuda))
    path = tmp_path / "car.pdparams"
    sd = dict(hot.state_dict())
    sd[checkpoint.STRUCTURED_NAMES] = {k: "param_%d" % i for i, k in enumerate(hot.state_dict())}
    with open(path, "wb") as f:
        pickle.dump(sd, f, protocol=4)
    out = tmp_path / "labels"
    r = subprocess.run([sys.executable, "tools/infer_kitti.py", "--model", str(path), "--config", "car", "--root",
                        str(root), "--ids", str(tmp_path / "ids.txt"), "--out", str(out), "--lanes", "2"],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    n_lines = 0
    for fid, (cloud, _, shape, _) in zip(ids, scans):
        c = kitti.read_calib(root / "calib" / (fid + ".txt"))
        planes = kitti.frustum_planes(c, shape)
        b, s, lab = hot.infer_kitti(cloud, planes)
        want = kitti.format_label_lines(kitti.to_kitti(b.numpy(), s.numpy(), lab.numpy(), c, shape, ("Car",)))
        assert (out / (fid + ".txt")).read_text().splitlines() == want, fid
        n_lines += len(want)
    assert n_lines > 0
    assert sorted(os.listdir(out)) == sorted(i + ".txt" for i in ids)
