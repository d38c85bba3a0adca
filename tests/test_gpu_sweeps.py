"""GPU: the device sweep merge (ops.sweep_merge, csrc/sweep_merge.cu) against its host oracle io.merge_sweeps, and the
CenterPoint frame on raw sweeps (infer_sweeps, a captured graph, infer_stream, CenterPointSweep lanes sharing one ring)
against the same frame fed the host merge through infer()."""
import numpy as np
import pytest

from conftest import golden
from paddle3d_b200 import io as p3d_io
from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu

QNAN = 0x7fc00000


def _check_merge(name, got, n_out, status, want, expect_status=0):
    """Row count and order equal, non-xyz columns and the lag bit-identical, xyz within 1 fp32 ulp, NaN tail exact."""
    got = got.cpu().numpy()
    n = int(n_out.item())
    assert int(status.item()) == expect_status, name
    assert n == len(want) and got.shape[1] == want.shape[1], (name, n, len(want))
    g = got[:n]
    assert np.array_equal(g[:, 3:].view(np.uint32), want[:, 3:].view(np.uint32)), name
    gi, wi = g[:, :3].view(np.int32).astype(np.int64), want[:, :3].view(np.int32).astype(np.int64)
    diff = np.abs(gi - wi)
    rows = int((diff.max(1) > 0).sum()) if n else 0
    print("%s: %d rows, %d differ in xyz (max %d ulp)" % (name, n, rows, int(diff.max()) if n else 0))
    assert n == 0 or diff.max() <= 1, name  # more than 1 ulp is a bug, not a tolerance to widen
    assert (got[n:].view(np.uint32) == QNAN).all(), name
    return rows


def _golden_sweeps(g):
    return [(g["cloud1"], g["mat0"], float(g["lags"][0])), (g["cloud2"], None, float(g["lags"][1])),
            (g["cloud3"], g["mat2"], float(g["lags"][2]))]


def test_merge_matches_host_on_golden(cuda):
    from paddle3d_b200.ops import sweep_merge as sm
    g = golden("sweeps.npz")
    kw = dict(use_dim=[0, 1, 2, 4], use_time_lag=True, sweep_remove_radius=1, order=g["order"])
    want = p3d_io.merge_sweeps(g["cloud0"], _golden_sweeps(g), **kw)
    assert np.array_equal(want, g["merged"])
    out, n, st = sm.merge_sweeps_device(g["cloud0"], _golden_sweeps(g), cap=len(want) + 37, device=cuda, **kw)
    _check_merge("golden", out, n, st, want)


def _edge_cases(g):
    c0, c1, c3 = g["cloud0"], g["cloud1"], g["cloud3"]
    m0 = g["mat0"]
    empty = np.zeros((0, 5), np.float32)
    near = (c1 * np.float32(1e-3)).astype(np.float32)  # every point inside the 1 m removal square
    return {
        "no_sweeps": (c0, [], dict(use_dim=[0, 1, 2, 3], use_time_lag=True)),
        "empty_sweep": (c0, [(empty, m0, 0.05), (c3, m0, 0.1)], dict(use_dim=[0, 1, 2, 3], use_time_lag=True)),
        "all_removed": (c0, [(near, m0, 0.05), (c3, None, 0.1)], dict(use_dim=[0, 1, 2, 3], use_time_lag=True)),
        "none_transform": (c0, [(c1, None, 0.05)], dict(use_dim=3, use_time_lag=False)),
        "falsy_use_dim": (c0, [(c1, m0, 0.05), (c3, m0, 0.1)], dict(use_dim=None, use_time_lag=True)),
        "fp32_3x4_matrix": (c0, [(c1, m0[:3].astype(np.float32), 0.05)], dict(use_dim=[0, 1, 2, 4], use_time_lag=True)),
        "empty_key": (empty, [(c1, m0, 0.05)], dict(use_dim=[0, 1, 2, 3], use_time_lag=True, sweep_remove_radius=2.5)),
        "all_empty": (empty, [(empty, m0, 0.05)], dict(use_dim=[0, 1, 2, 3], use_time_lag=True)),
    }


@pytest.mark.parametrize("case", ["no_sweeps", "empty_sweep", "all_removed", "none_transform", "falsy_use_dim",
                                  "fp32_3x4_matrix", "empty_key", "all_empty"])
def test_merge_edge_cases(cuda, case):
    from paddle3d_b200.ops import sweep_merge as sm
    key, sweeps, kw = _edge_cases(golden("sweeps.npz"))[case]
    want = p3d_io.merge_sweeps(key, sweeps, **kw)
    out, n, st = sm.merge_sweeps_device(key, sweeps, cap=len(want) + 5, device=cuda, **kw)
    _check_merge(case, out, n, st, want)
    if case == "all_removed":
        assert len(want) == len(key) + len(sweeps[1][0]) - int((np.abs(sweeps[1][0][:, :2]) < 1).all(1).sum())


def test_merge_overflow_sets_the_flag(cuda):
    from paddle3d_b200.ops import sweep_merge as sm
    g = golden("sweeps.npz")
    kw = dict(use_dim=[0, 1, 2, 4], use_time_lag=True, order=g["order"])
    want = p3d_io.merge_sweeps(g["cloud0"], _golden_sweeps(g), **kw)
    cap = len(want) - 301
    out, n, st = sm.merge_sweeps_device(g["cloud0"], _golden_sweeps(g), cap=cap, device=cuda, **kw)
    _check_merge("overflow", out, n, st, want[:cap], expect_status=sm.OVERFLOW)
    with pytest.raises(ValueError):
        sm.merge_sweeps_device(g["cloud0"], _golden_sweeps(g), use_dim=[], device=cuda)


def _frame_inputs(seq, j, K, first=0):
    from paddle3d_b200 import sweep_ring
    ids = sweep_ring.frame_sweeps(j, K, first)
    key, pk, tk = seq[ids[0]]
    sweeps = [(seq[s][0], sweep_ring.ref_from_curr(pk, seq[s][1]), tk - seq[s][2]) for s in ids[1:]]
    return key, sweeps


def test_merge_full_size_stream(cuda):
    """Ten synthetic sweeps (~300k merged points, the C3 frame's size), the ego moving and turning between them."""
    from paddle3d_b200.ops import sweep_merge as sm
    seq = synth.sweep_sequence(10, 1)
    key, sweeps = _frame_inputs(seq, 9, 10)
    kw = dict(use_dim=4, use_time_lag=True, sweep_remove_radius=1.0)
    want = p3d_io.merge_sweeps(key, sweeps, **kw)
    assert 280000 < len(want) <= synth.C3["num_points"]
    out, n, st = sm.merge_sweeps_device(key, sweeps, cap=synth.C3["num_points"], device=cuda, **kw)
    _check_merge("full-size stream", out, n, st, want)


N_POINTS = 40000
SWEEP = dict(slot_cap=8000)


def _pipe(cuda, sweep_input=None):
    from paddle3d_b200.pipeline import CenterPointHotPath
    return CenterPointHotPath(synth.C3, cuda, precision=2, seed=3, num_points=N_POINTS, sweep_input=sweep_input)


def _host_frame(key, sweeps):
    import torch
    merged = p3d_io.merge_sweeps(key, sweeps, use_dim=4, use_time_lag=True, sweep_remove_radius=1.0)
    full = np.full((N_POINTS, 5), np.nan, np.float32)
    full[:len(merged)] = merged
    return merged, torch.from_numpy(full).pin_memory()


def _equal(a, b):
    import torch
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_frame_on_raw_sweeps_matches_host_merge(cuda):
    """infer_sweeps eager and captured, and infer_stream (one frame per pushed sweep, ring slots reused), against the
    pipeline fed io.merge_sweeps' cloud: equal boxes, scores and labels wherever the merged clouds are bit-equal."""
    import torch
    seq = synth.sweep_sequence(13, 2, points_per_sweep=3800)
    ref = _pipe(cuda)
    pipe = _pipe(cuda, SWEEP)
    assert pipe.h_status.numel() == ref.h_status.numel() + 1
    want = []
    for j in range(len(seq)):
        key, sweeps = _frame_inputs(seq, j, 10)
        merged, host = _host_frame(key, sweeps)
        want.append((merged, tuple(t.clone() for t in ref.infer(host))))
    j = 9
    key, sweeps = _frame_inputs(seq, j, 10)
    eager = pipe.infer_sweeps(key, sweeps)
    assert pipe.merged_rows() == len(want[j][0])
    rows = _check_merge("frame merge", pipe.points, pipe._n_merged, pipe._merge_status, want[j][0])
    if rows == 0:
        assert _equal(eager, want[j][1])
    pipe.capture()
    assert _equal(pipe.infer_sweeps(key, sweeps), eager)
    got = list(pipe.infer_stream(iter(seq)))
    assert len(got) == len(seq)
    equal_frames = 0
    for j, (g, (merged, w)) in enumerate(zip(got, want)):
        assert len(g[2]) == len(w[2]), j
        if _equal(g, w):
            equal_frames += 1
    print("infer_stream: %d of %d frames bit-equal to the host-merge pipeline" % (equal_frames, len(seq)))
    assert equal_frames >= len(seq) - 1
    assert list(pipe.infer_stream(iter([]))) == []


def test_frame_raises_when_the_merge_overflows(cuda):
    from paddle3d_b200.pipeline import CenterPointHotPath
    seq = synth.sweep_sequence(3, 4, points_per_sweep=1500)
    pipe = CenterPointHotPath(synth.C3, cuda, precision=2, seed=3, num_points=2000, sweep_input=dict(slot_cap=2048))
    key, sweeps = _frame_inputs(seq, 2, 10)
    with pytest.raises(RuntimeError, match="capacity"):
        pipe.infer_sweeps(key, sweeps)
    pipe.infer_sweeps(key, [])  # one sweep fits


def test_lanes_stream_matches_single_lane(cuda):
    """CenterPointSweep.infer_stream: 2 lanes sharing one ring of K + 2 slots over 2 * lanes + K sweeps return, in order,
    the single-lane stream's results."""
    from paddle3d_b200.pipeline import CenterPointSweep
    lanes, K = 2, 10
    seq = synth.sweep_sequence(2 * lanes + K + 1, 5, points_per_sweep=3800)
    single = _pipe(cuda, SWEEP)
    single.infer_sweeps(*_frame_inputs(seq, 0, K))
    single.capture()
    want = list(single.infer_stream(iter(seq)))
    sweep = CenterPointSweep(lanes, cfg=synth.C3, device=cuda, precision=2, seed=3, num_points=N_POINTS, sweep_input=SWEEP)
    assert sweep.lanes[1].ring is sweep.lanes[0].ring and sweep.lanes[0].ring.slots == K + lanes
    for p in sweep.lanes:
        p.infer_sweeps(*_frame_inputs(seq, 0, K))
        p.capture()
    got = list(sweep.infer_stream(iter(seq)))
    assert len(got) == len(want) == len(seq)
    for j, (g, w) in enumerate(zip(got, want)):
        assert _equal(g, w), j


def test_deploy_runner_with_sweeps(cuda, tmp_path):
    """tools/infer.py --sweeps: the key .bin + a JSON list of earlier sweeps, merged on the GPU, gives the detections of
    the predictor fed io.merge_sweeps' cloud."""
    import json
    import subprocess
    import sys

    from conftest import ROOT
    from paddle3d_b200 import deploy
    seq = synth.sweep_sequence(3, 6, points_per_sweep=3000)
    key, sweeps = _frame_inputs(seq, 2, 10)
    entries = []
    for i, (c, m, lag) in enumerate(sweeps):
        c.tofile(tmp_path / ("s%d.bin" % i))
        entries.append({"path": str(tmp_path / ("s%d.bin" % i)), "ref_from_curr": m.tolist(), "time_lag": lag})
    key.tofile(tmp_path / "key.bin")
    (tmp_path / "sweeps.json").write_text(json.dumps(entries))
    si = dict(max_sweeps=3, slot_cap=4096)
    b, l, s = deploy.Predictor(synth.C3, cuda, max_points=12000, seed=0, precision=2, with_head=False,
                               sweep_input=si).run_sweeps(key, sweeps)
    merged = p3d_io.merge_sweeps(key, sweeps, use_dim=4, use_time_lag=True)
    rb, rl, rs = deploy.Predictor(synth.C3, cuda, max_points=12000, seed=0, precision=2, with_head=False).run(merged)
    assert np.array_equal(b, rb) and np.array_equal(l, rl) and np.array_equal(s, rs)
    out = tmp_path / "det.txt"
    r = subprocess.run([sys.executable, "tools/infer.py", "--lidar_file", str(tmp_path / "key.bin"), "--sweeps",
                        str(tmp_path / "sweeps.json"), "--no_head", "--max_points", "12000", "--out", str(out)],
                       cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert len(out.read_text().splitlines()) >= 1


def test_default_frame_graph_is_unchanged(cuda):
    """Without sweep input the bench frame captures the same 61 kernel nodes as before; with it, the merge adds its two
    kernels and one memset."""
    import torch

    import bench
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointHotPath
    pts = torch.from_numpy(synth.lidar_cloud(synth.C3, 0)).to(cuda)
    counts = []
    for si in (None, dict()):
        p = CenterPointHotPath(synth.C3, cuda, precision=sp.F16X3, seed=0, with_head=True, keep_bev=False,
                               bn_gain=bench.BN_GAIN, sweep_input=si)
        p.points.copy_(pts)
        if si is not None:
            seq = synth.sweep_sequence(2, 0)
            p.infer_sweeps(*_frame_inputs(seq, 1, 10))
        p.capture(count_nodes=True)
        counts.append(p.graph_nodes)
        del p
    print("graph nodes: default %s, sweep input %s" % tuple(counts))
    assert counts[0]["kernel"] == 61
    assert counts[1]["kernel"] == counts[0]["kernel"] + 2 and counts[1]["memset"] == counts[0]["memset"] + 1
