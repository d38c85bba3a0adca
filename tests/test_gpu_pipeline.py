"""GPU parity of the whole hot-path frame (CenterPointHotPath: hard_voxelize + VoxelMean + SparseResNet3D + dense BEV +
centerpoint_postprocess) against the CPU oracle frame, and of the three ways of running it (eager, CUDA graph,
pipelined sweep).  Voxel counts and box labels exact, BEV features / boxes within 1e-4 relative (BASELINE.json)."""
import numpy as np
import pytest

from paddle3d_b200 import synth
from parity import rel_check

pytestmark = pytest.mark.gpu

N_POINTS = 40000  # same 1440x1440x40 geometry as C3, fewer points so that the CPU oracle frame takes seconds


def _pipe(cuda, precision, **kw):
    from paddle3d_b200.pipeline import CenterPointHotPath
    return CenterPointHotPath(synth.C3, cuda, precision=precision, seed=3, num_points=N_POINTS, **kw)


def _frames(n):
    return [synth.lidar_cloud(synth.C3, 10 + i, num_points=N_POINTS) for i in range(n)]


@pytest.mark.parametrize("precision", [0, 1, 2, 4])
def test_frame_matches_cpu_oracle_frame(cuda, oracle_mod, precision):
    import torch
    from oracle.cpu_reference import CpuFrame
    pipe = _pipe(cuda, precision)
    pts = _frames(1)[0]
    pipe.points.copy_(torch.from_numpy(pts).to(cuda))
    with torch.cuda.stream(pipe.stream):
        out = pipe.forward_device()
    pipe.stream.synchronize()
    ref = CpuFrame(synth.C3, pipe.export_weights_numpy(), pipe.head_host, pipe.test_cfg, pipe.label_off).run(pts)
    assert int(out["num_voxels"][0].item()) == ref["num_voxels"]
    bev = out["bev"].cpu().numpy()
    assert bev.shape == ref["bev"].shape
    rel_check("frame bev p%d" % precision, bev, ref["bev"])
    k = int(out["counts"][-1].item())
    assert k == len(ref["labels"])
    np.testing.assert_array_equal(out["labels"][:k].cpu().numpy(), ref["labels"])
    np.testing.assert_allclose(out["scores"][:k].cpu().numpy(), ref["scores"], rtol=1e-5, atol=1e-6)
    np.testing.assert_allclose(out["boxes"][:k].cpu().numpy(), ref["boxes"], rtol=1e-4, atol=1e-4)


def test_graph_sweep_and_side_stream_agree_with_eager(cuda):
    import torch
    frames = _frames(4)
    pinned = [torch.from_numpy(f).pin_memory() for f in frames]
    eager = _pipe(cuda, 2)
    want = []
    for f in pinned:
        b, s, l = eager.infer(f)
        want.append((b.clone(), s.clone(), l.clone(), eager.out["bev"].clone()))

    graph = _pipe(cuda, 2)
    graph.points.copy_(pinned[0])
    graph.capture()
    for f, w in zip(pinned, want):  # one frame at a time through the captured graph: bit-identical
        b, s, l = graph.infer(f)
        assert torch.equal(b, w[0]) and torch.equal(s, w[1]) and torch.equal(l, w[2])
        assert torch.equal(graph.out["bev"], w[3])
    got = list(graph.infer_many(iter(pinned)))  # pipelined sweep: same results, same order
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert torch.equal(g[0], w[0]) and torch.equal(g[1], w[1]) and torch.equal(g[2], w[2])
    assert len(list(graph.infer_many(iter(pinned[:1])))) == 1 and list(graph.infer_many(iter([]))) == []

    side = _pipe(cuda, 2)  # rulebooks built on a side stream (optional mode): same bits
    side.net.side_stream_rulebooks = True
    for f, w in zip(pinned[:2], want):
        b, s, l = side.infer(f)
        assert torch.equal(b, w[0]) and torch.equal(side.out["bev"], w[3])
    side.points.copy_(pinned[0])
    side.capture()
    b, s, l = side.infer(pinned[1])
    assert torch.equal(b, want[1][0]) and torch.equal(side.out["bev"], want[1][3])


def test_frame_with_dense_head(cuda, oracle_mod):
    """with_head=True: BEV -> DenseRPNHead -> postprocess.  The head tensors must match the CPU reference run on the
    GPU's own BEV tensor (the per-layer and small-network parity is in test_gpu_dense.py); boxes are not compared bit
    for bit because candidates within 1e-4 of the score threshold may flip."""
    import torch
    from oracle.cpu_reference import CpuDenseHead
    pipe = _pipe(cuda, 4, with_head=True)
    pipe.points.copy_(torch.from_numpy(_frames(1)[0]).to(cuda))
    with torch.cuda.stream(pipe.stream):
        out = pipe.forward_device()
        heads = pipe.dense(out["bev"])
    pipe.stream.synchronize()
    want = CpuDenseHead(pipe.dense.export_numpy()).run(out["bev"].cpu().numpy())
    for name in want:
        for g, w in zip(heads[name], want[name]):
            assert np.abs(g.cpu().numpy() - w).max() <= 1e-4 * max(1.0, np.abs(w).max()), name
    assert int(out["status"].max().item()) == 0
    assert int(out["counts"][-1].item()) >= len(pipe.label_off)  # at least the one row per task the op always emits


def test_deploy_predictor_matches_pipeline(cuda, tmp_path):
    """deploy.Predictor (SURVEY §8f-4): a .bin sweep with fewer points than the capacity gives the same detections as the
    pipeline fed the same points (NaN padding rows are dropped by the voxelizer), and the result file has one line per
    real detection."""
    import torch
    from paddle3d_b200 import deploy
    pts = synth.lidar_cloud(synth.C3, 21, num_points=30000)
    f = tmp_path / "sweep.bin"
    pts.tofile(f)
    p = deploy.preprocess(str(f), 5, False)
    p = np.hstack([p, pts[:, 4:5]])  # keep the file's own lag column for this check
    pred = deploy.Predictor(synth.C3, cuda, max_points=N_POINTS, seed=3, with_head=False)
    b, l, s = pred.run(p)
    ref = _pipe(cuda, 4)
    full = np.full((N_POINTS, 5), np.nan, np.float32)
    full[:len(p)] = p
    rb, rs, rl = ref.infer(torch.from_numpy(full).pin_memory())
    assert np.array_equal(b, rb.numpy()) and np.array_equal(l, rl.numpy()) and np.array_equal(s, rs.numpy())
    out = tmp_path / "det.txt"
    deploy.write_results(str(out), b, l, s)
    assert len(out.read_text().splitlines()) == int((s >= 0).sum())


def test_fused_pixel_h16_bev_matches_nchw_path(cuda):
    """keep_bev=False (the bench frame): sparse rows -> pixel fp16-pair image -> dense head, no fp32 NCHW BEV in between.
    The rebuilt BEV tensor equals the NCHW one to the pair format's 2^-22, the detections agree."""
    import torch
    pts = torch.from_numpy(_frames(1)[0]).pin_memory()
    a = _pipe(cuda, 4, with_head=True, keep_bev=True)
    b = _pipe(cuda, 4, with_head=True, keep_bev=False)
    ra = a.infer(pts)
    rb = b.infer(pts)
    bev_a, bev_b = a.bev_nchw().cpu().numpy(), b.bev_nchw().cpu().numpy()
    assert b.out["bev"] is None and bev_a.shape == bev_b.shape
    # Two sources of difference, both far inside the parity bar: the pair format of the last rows (2^-22 relative) and the
    # fp32 summation order of the stream-K pieces of the narrow layers, which follows the row order - and the strided
    # levels number their output sites with atomics, so two frames of the same cloud order their rows differently.
    # The bound is the parity bar.
    rel_check('fused pixel BEV vs NCHW BEV', bev_b, bev_a)
    # the dense head reads the pixel rows in (z, c) channel order through the permuted image of its first conv
    ha, hb = a.dense(a.bev_nchw()), b.dense.forward_h16(*b.out["bev_h16"])
    torch.cuda.synchronize()
    for name in ha:
        for x, y in zip(ha[name], hb[name]):
            assert np.abs(x.cpu().numpy() - y.cpu().numpy()).max() <= 1e-5 * max(1.0, float(x.abs().max())), name
    assert len(ra[2]) == len(rb[2])
    same = (ra[2].numpy() == rb[2].numpy()).mean()
    assert same > 0.98  # candidates within 1e-6 of each other may swap ranks
    b.points.copy_(pts.to(cuda))
    b.capture()
    rc = b.infer(pts)
    # graph replay vs eager run of the same frame: bit-identical only when every layer's result is independent of the row
    # order (P3D_SPARSE_WM=0); with the stream-K warp-MMA layers the last bits of the BEV follow the (atomics-numbered) row
    # order of that run, so detections agree to the parity tolerance instead
    assert len(rc[2]) == len(rb[2])
    keep = rc[2].numpy() == rb[2].numpy()
    assert keep.mean() > 0.98
    assert np.abs(rc[0].numpy()[keep] - rb[0].numpy()[keep]).max() <= 1e-4 * max(1.0, float(rb[0].abs().max()))


def test_sweep_lanes_match_single_lane(cuda):
    """CenterPointSweep (two frames in flight: two lanes sharing one model, frames dealt round-robin) returns, in order,
    what the single-lane pipeline returns for each frame of a sweep of distinct frames."""
    import torch
    from paddle3d_b200.pipeline import CenterPointSweep
    frames = [torch.from_numpy(f).pin_memory() for f in _frames(5)]
    single = _pipe(cuda, 4, with_head=True, keep_bev=False)
    single.calibrate_head(frames[0].to(cuda))
    single.points.copy_(frames[0].to(cuda))
    single.capture()
    want = list(single.infer_many(iter(frames)))
    sweep = CenterPointSweep(2, cfg=synth.C3, device=cuda, precision=4, seed=3, num_points=N_POINTS, with_head=True, keep_bev=False)
    assert sweep.lanes[1].net is sweep.lanes[0].net and sweep.lanes[1].dense is sweep.lanes[0].dense
    sweep.calibrate_head(frames[0].to(cuda))
    sweep.capture(frames[0].to(cuda))
    got = list(sweep.infer_many(iter(frames)))
    assert len(got) == len(want) == 5
    counts = [len(w[2]) for w in want]
    assert len(set(counts)) > 1 or counts[0] > 6  # the frames really differ / detect something
    for g, w in zip(got, want):
        assert len(g[2]) == len(w[2])
        same = (g[2].numpy() == w[2].numpy())
        assert same.mean() > 0.98
        assert np.abs(g[0].numpy()[same] - w[0].numpy()[same]).max() <= 1e-4 * max(1.0, float(w[0].abs().max()))
    assert list(sweep.infer_many(iter([]))) == [] and len(list(sweep.infer_many(iter(frames[:1])))) == 1
    assert len(list(sweep.infer_many(iter(frames[:3])))) == 3
