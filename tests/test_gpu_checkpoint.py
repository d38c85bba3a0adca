"""GPU: the four LiDAR frames on parameters loaded from a `.pdparams` file (checkpoint.py).

- Round trip: a seeded frame's state_dict through a file into a frame of another seed gives the same captured frame
  (boxes, scores, labels, head planes) bit for bit, with the same graph, and the same state_dict; CenterPointSweep built
  with weights= gives what one lane gives.
- Non-trivial statistics: random BatchNorm statistics and conv biases, loaded, against the CPU arm fed the model's
  export_numpy / export_weights_numpy, at the bars of the frames' own tests; captured equals eager; calibration refuses.
- CenterPoint-voxel's deploy.Predictor(weights=) and tools/infer.py --model print what the hot path gives."""
import os
import pickle
import subprocess
import sys

import numpy as np
import pytest

from paddle3d_b200 import checkpoint, synth
from parity import rel_check, rel_errors

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BN_GAIN = 6.0 ** 0.5
CP_SMALL = dict(synth.CP_PILLARS, point_cloud_range=[-25.6, -25.6, -5.0, 25.6, 25.6, 3.0], num_points=60000)
N_VOXEL = 40000
MODELS = ["centerpoint_voxel", "centerpoint_pillars", "pointpillars_car", "pointpillars_cyclist_pedestrian"]


def _frame(name, cuda, lanes=None, **kw):
    """The model's hot-path frame (or, with lanes, a CenterPointSweep of them) at a test size; kw: seed / weights."""
    from paddle3d_b200 import pointpillars as pp
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointHotPath, CenterPointSweep
    cls, args = {
        "centerpoint_voxel": (CenterPointHotPath, dict(cfg=synth.C3, precision=sp.F16X3, num_points=N_VOXEL,
                                                       with_head=True, keep_bev=False)),
        "centerpoint_pillars": (CenterPointPillarsHotPath, dict(cfg=CP_SMALL)),
        "pointpillars_car": (pp.PointPillarsHotPath, dict(cfg=synth.C2, num_points=20000)),
        "pointpillars_cyclist_pedestrian": (pp.PointPillarsHotPath, dict(cfg=synth.C2_PED_CYCLIST, num_points=20000,
                                                                         model_cfg=pp.CONFIG_PED_CYCLIST)),
    }[name]
    args = dict(args, device=cuda, bn_gain=BN_GAIN, **kw)
    if lanes:
        return CenterPointSweep(lanes, frame_cls=cls, **args)
    return cls(**args)


def _points(name, n, seed=3):
    cfg = {"centerpoint_voxel": synth.C3, "centerpoint_pillars": CP_SMALL, "pointpillars_car": synth.C2,
           "pointpillars_cyclist_pedestrian": synth.C2_PED_CYCLIST}[name]
    return synth.lidar_cloud(cfg, seed, num_points=n)


def _planes(hot):
    """The head planes of the frame's last result, as one list of tensors."""
    if "planes" in hot.out:
        return [hot.out["planes"]]
    return [t for k in sorted(hot.out["head"]) for t in hot.out["head"][k]]


def _bits(a, b):
    import torch
    return a.dtype == b.dtype and a.shape == b.shape and (torch.equal(a.view(torch.int32), b.view(torch.int32))
                                                          if a.dtype == torch.float32 else torch.equal(a, b))


def _save(path, sd):
    obj = dict(sd)
    obj[checkpoint.STRUCTURED_NAMES] = {k: "param_%d" % i for i, k in enumerate(sd)}
    with open(path, "wb") as f:
        pickle.dump(obj, f, protocol=4)


_SEEDED = {}


def _seeded(name, cuda, tmp_path_factory):
    """Model A: seeded (seed 2), calibrated, captured with its node counts; its state_dict saved as a .pdparams file."""
    if name not in _SEEDED:
        import torch
        _SEEDED.clear()  # one model's frames alive at a time
        torch.cuda.empty_cache()
        a = _frame(name, cuda, seed=2)
        pts = _points(name, a.n)
        a.calibrate_head(torch.from_numpy(pts).to(cuda))
        a.points.copy_(torch.from_numpy(pts).to(cuda))
        a.capture(count_nodes=True)
        path = str(tmp_path_factory.mktemp(name) / "model.pdparams")
        _save(path, a.state_dict())
        _SEEDED[name] = (a, pts, path)
    return _SEEDED[name]


@pytest.mark.parametrize("name", MODELS)
def test_round_trip_is_bit_exact(cuda, tmp_path_factory, name):
    import torch
    a, pts, path = _seeded(name, cuda, tmp_path_factory)
    sd = checkpoint.read_pdparams(path)
    b = _frame(name, cuda, seed=7)
    b.load_state_dict(sd)
    b.points.copy_(torch.from_numpy(pts).to(cuda))
    b.capture(count_nodes=True)
    assert a.graph_nodes is not None and b.graph_nodes == a.graph_nodes
    frames = [torch.from_numpy(_points(name, a.n, s)).pin_memory() for s in (3, 4)]
    want = []
    for f in frames:
        ra = [t.clone() for t in a.infer(f)]
        pa = [t.clone() for t in _planes(a)]
        rb = b.infer(f)
        assert len(ra[0]) > 0
        assert all(_bits(x, y) for x, y in zip(rb, ra))
        assert all(_bits(x, y) for x, y in zip(_planes(b), pa))
        want.append(ra)
    got = b.state_dict()
    assert list(got) == list(sd) and all(got[k].dtype == np.float32 and np.array_equal(got[k].view(np.uint32),
                                                                                       sd[k].view(np.uint32)) for k in sd)
    # two lanes built from the file: one model, read once on lane 0, and the single lane's results
    sweep = _frame(name, cuda, lanes=2, seed=9, weights=path)
    l0, l1 = sweep.lanes
    assert (l1.net is l0.net and l1.dense is l0.dense) if hasattr(l0, "net") else l1.model is l0.model
    sweep.capture(torch.from_numpy(pts).to(cuda))
    got = list(sweep.infer_many(frames[i % 2] for i in range(4)))
    for i, g in enumerate(got):
        assert all(_bits(x, y) for x, y in zip(g, want[i % 2])), i
    del sweep, b
    torch.cuda.empty_cache()


def _perturbed(sd, seed):
    """Random BatchNorm statistics (gamma around the frames' bn_gain) and conv biases moved by up to 0.1, all O(1); the
    heat-map / cls biases keep their calibrated values so the frame still detects."""
    rng = np.random.default_rng(seed)
    out = {}
    for k, v in sd.items():
        n = v.shape[0]
        is_bn = k[:k.rfind(".") + 1] + "_mean" in sd
        if is_bn and k.endswith(".weight"):
            v = rng.uniform(0.5, 1.5, n) * BN_GAIN
        elif is_bn and k.endswith(".bias"):
            v = rng.uniform(-0.2, 0.2, n)
        elif k.endswith("._mean"):
            v = rng.uniform(-0.1, 0.1, n)
        elif k.endswith("._variance"):
            v = rng.uniform(0.5, 1.5, n)
        elif k.endswith(".bias") and ".hm." not in k and "cls_head" not in k:
            v = v + rng.uniform(-0.1, 0.1, n)
        out[k] = np.asarray(v, np.float32)
    return out


def _matched(cpu_boxes, boxes):
    if not len(cpu_boxes):
        return 1.0
    if not len(boxes):
        return 0.0
    return float((np.abs(cpu_boxes[:, None, :3] - boxes[None, :, :3]).max(-1).min(1) < 1e-2).mean())


@pytest.mark.parametrize("name", MODELS)
def test_loaded_statistics_match_cpu_arm(cuda, oracle_mod, tmp_path_factory, name):
    import torch
    a, pts, _ = _seeded(name, cuda, tmp_path_factory)
    sd = _perturbed(a.state_dict(), 5)
    hot = _frame(name, cuda, weights=sd)  # built from the state dict: never seeded
    assert all(np.array_equal(v, sd[k]) for k, v in hot.state_dict().items())
    host = torch.from_numpy(pts).pin_memory()
    boxes, scores, labels = [t.clone() for t in hot.infer(host)]
    planes = [t.clone() for t in _planes(hot)]
    nv = int(hot.out["num_voxels"][0])
    if name == "centerpoint_voxel":
        from oracle.cpu_reference import CpuDenseHead, CpuFrame
        bev = hot.bev_nchw()
        ref = CpuFrame(synth.C3, hot.export_weights_numpy(), hot.head_host, hot.test_cfg, hot.label_off).run(pts)
        assert nv == ref["num_voxels"]
        rel_check("loaded voxel bev", bev.cpu().numpy(), ref["bev"])
        want = CpuDenseHead(hot.dense.export_numpy()).run(bev.cpu().numpy())
        for k in want:  # the head reads the (z, c)-ordered pixel rows through the permuted image of the loaded first conv
            for g, w in zip(hot.out["head"][k], want[k]):
                assert np.abs(g.cpu().numpy() - w).max() <= 1e-4 * max(1.0, np.abs(w).max()), k
    elif name == "centerpoint_pillars":
        from oracle.centerpoint_pillars import CpuCenterPointPillars
        from test_gpu_centerpoint_pillars import _pair
        m = hot.model
        cpu = CpuCenterPointPillars(m.cfg, m.export_numpy(), m.test_cfg, m.label_off).run(pts)
        assert nv == cpu["num_voxels"]
        for k in cpu["head"]:
            for g, w in zip(hot.out["head"][k], cpu["head"][k]):
                e = rel_errors(g.cpu().numpy(), w)
                assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, (k, e)
        assert abs(len(boxes) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
        if len(cpu["boxes"]):
            assert _pair((boxes.numpy(), scores.numpy(), labels.numpy()), cpu) >= 0.95
    else:
        import oracle.pointpillars as opp
        import oracle.pointpillars_multiclass as opm
        m = hot.model
        if m.num_classes == 1:
            cpu = opp.CpuPointPillars(m.cfg, m.export_numpy(), m.anchors_np, m.corners_np, m.grid, m.mc["test"]).run(pts)
        else:
            cpu = opm.CpuPointPillarsMulticlass(m.cfg, m.export_numpy(), m.anchors_np, m.corners_np, m.grid,
                                                m.mc["test"], m.num_classes).run(pts)
        assert nv == cpu["num_voxels"]
        e = rel_errors(planes[0].cpu().numpy(), cpu["planes"])  # the loaded cls | box | dir convs as one head conv
        assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
        assert abs(len(boxes) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
        assert _matched(cpu["boxes"], boxes.numpy()) >= 0.95
    print("loaded %s: %d voxels, %d boxes" % (name, nv, len(boxes)))
    assert int(hot.h_status.max()) == 0
    # captured equals eager on loaded weights, with the seeded frame's graph
    with pytest.raises(RuntimeError, match="loaded from a checkpoint"):
        hot.calibrate_head(torch.from_numpy(pts).to(cuda))
    hot.points.copy_(torch.from_numpy(pts).to(cuda))
    hot.capture(count_nodes=True)
    assert hot.graph_nodes == a.graph_nodes
    got = hot.infer(host)
    assert all(_bits(x, y) for x, y in zip(got, (boxes, scores, labels)))
    assert all(_bits(x, y) for x, y in zip(_planes(hot), planes))
    with pytest.raises(RuntimeError, match="after capture"):
        hot.load_state_dict(sd)
    del hot
    torch.cuda.empty_cache()


def test_predictor_and_cli_load_the_checkpoint(cuda, tmp_path_factory, tmp_path):
    """deploy.Predictor(weights=path).run equals the hot path built with the same weights; tools/infer.py --model on a
    .bin file prints the predictor's lines."""
    import torch
    from paddle3d_b200 import deploy
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointHotPath
    _, _, path = _seeded("centerpoint_voxel", cuda, tmp_path_factory)
    cloud = tmp_path / "cloud.bin"
    synth.lidar_cloud(synth.C3, 21, num_points=30000).tofile(cloud)
    pts = deploy.preprocess(str(cloud), 5, True)
    pred = deploy.Predictor(synth.C3, cuda, max_points=N_VOXEL, weights=path)
    assert pred.pipe.dense.loaded
    b, l, s = pred.run(pts)
    lines = deploy.format_result(b, l, s)
    assert len(lines) > 0
    ref = CenterPointHotPath(synth.C3, cuda, precision=sp.F16X3, num_points=N_VOXEL, with_head=True, weights=path)
    full = np.full((N_VOXEL, 5), np.nan, np.float32)
    full[:len(pts)] = pts
    rb, rs, rl = ref.infer(torch.from_numpy(full).pin_memory())
    assert np.array_equal(b, rb.numpy()) and np.array_equal(l, rl.numpy()) and np.array_equal(s, rs.numpy())
    del pred, ref
    torch.cuda.empty_cache()
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "infer.py"), "--model", path, "--lidar_file",
                        str(cloud), "--num_point_dim", "5", "--use_timelag", "1", "--max_points", str(N_VOXEL),
                        "--gpu_id", str(cuda.index or 0)], capture_output=True, text=True, timeout=200)
    assert r.returncode == 0, r.stderr[-2000:]
    assert r.stdout.splitlines() == lines
