"""GPU: the strided levels number their rows in first-appearance order (test_strided_site_order restates it), so the
CenterPoint-voxel frame gives the same bits for the same cloud in its default mode, the one bench.py times, with the
warp-MMA kernel and the wgmma kernel's stream-K on: captured or eager, on one lane or four, from merged points or from
raw sweeps, and through deploy.Predictor.

Lines starting with "REGIME" (pytest -s) name each sparse conv's work decomposition at its real row count."""
import numpy as np
import pytest

import bench
import lidar_front_end_oracle as lfo
from paddle3d_b200 import synth
from test_gpu_centerpoint_full_size import (GEOMS, UNIFORM_LEVELS, WIDE_CAPS, _bench_frame, frame_chain, sparse_frame,
                                            sparse_steps)
from test_gpu_dense_schedule import _bits_equal
from test_gpu_sparse_schedule import f16_sched, wm_ranges
from test_strided_site_order import first_appearance_sites

pytestmark = pytest.mark.gpu


def _strided(net, r):
    """(step, conv, input index, output index, neighbour map) of each strided level of a sparse_frame result."""
    out = []
    for i, (conv, _, _) in enumerate(sparse_steps(net)):
        if not conv.subm:
            out.append((i, conv, r["outs"][i].index, r["outs"][i + 1].index, r["pend"][i].nbr))
    return out


def _same(a, b):
    """(boxes, scores, labels) bit for bit."""
    import torch
    return all(_bits_equal(x, y) if x.is_floating_point() else torch.equal(x, y) for x, y in zip(a, b))


def _check_level(label, src_coords, batch, spatial, conv, out_coords, counters, nbr, out_cap, use_lfo=True):
    """out_coords / nbr / counters of one strided level against the first-appearance restatement: the first out_cap
    sites in order, the overflow flag iff they do not all fit, the raw count exact."""
    want, want_nbr, _ = first_appearance_sites(src_coords, batch, spatial, conv.kernel_size, conv.stride, conv.padding)
    cnt = counters.cpu().numpy()
    m = min(len(want), out_cap)
    assert list(cnt[:4]) == [m, int(len(want) > out_cap), len(want), 0], "%s: counters %s, %d sites" % (label, cnt, len(want))
    got = out_coords[:m].cpu().numpy()
    assert np.array_equal(got, want[:m]), "%s: rows not in first-appearance order" % label
    nb = nbr[:m].cpu().numpy()
    assert np.array_equal(nb, want_nbr[:m]), "%s: strided map" % label
    if use_lfo:
        assert np.array_equal(nb, lfo.nbr_map(src_coords, got, spatial, conv.kernel_size, conv.stride, conv.padding))
    return len(want)


def _rulebook_conv(cuda, coords, num, n_cap, batch, spatial, conv, out_cap):
    """p3d_sparse_rulebook_conv (the workspace entry point): (out_coords, counters, nbr)."""
    import torch
    from paddle3d_b200._lib import check, host_ints, lib
    from paddle3d_b200._mem import ptr, stream
    L = lib()
    K = int(np.prod(conv.kernel_size))
    out_coords = torch.empty((out_cap, 4), dtype=torch.int32, device=cuda)
    n_out = torch.full((4,), -7, dtype=torch.int32, device=cuda)
    nbr = torch.empty((out_cap, K), dtype=torch.int32, device=cuda)
    ws = torch.empty((L.p3d_sparse_rulebook_workspace_bytes(n_cap, out_cap),), dtype=torch.uint8, device=cuda)
    check(L.p3d_sparse_rulebook_conv(ptr(coords), ptr(num) if num is not None else None, n_cap, batch,
                                     host_ints(spatial), host_ints(conv.kernel_size), host_ints(conv.stride),
                                     host_ints(conv.padding), ptr(out_coords), ptr(n_out), out_cap, ptr(nbr), ptr(ws),
                                     ws.numel(), stream(cuda)), "rulebook_conv")
    torch.cuda.synchronize()
    return out_coords, n_out, nbr


def _check_frame_levels(cuda, name, hot, r, both_entry_points=True):
    counts = []
    for i, conv, src, ix, nbr in _strided(hot.net, r):
        label = "%s step %d" % (name, i)
        pc = src.coords[:int(src.num[0])].cpu().numpy()
        counts.append(_check_level(label, pc, src.batch, src.spatial, conv, ix.coords, ix.counters, nbr, ix.cap))
        if both_entry_points:
            oc, cnt, nb = _rulebook_conv(cuda, src.coords, src.num, src.cap, src.batch, src.spatial, conv, ix.cap)
            _check_level(label + " (workspace entry point)", pc, src.batch, src.spatial, conv, oc, cnt, nb, ix.cap,
                         use_lfo=False)
    return counts


@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_bench_cloud_levels_in_first_appearance_order(cuda, geom):
    """The bench cloud's four strided levels, through p3d_sparse_rulebook_level_t (the frame's path) and
    p3d_sparse_rulebook_conv on the same input rows."""
    import torch
    name, cfg, _, n_levels = geom
    hot = _bench_frame(cuda, cfg, with_head=False)
    r = sparse_frame(hot, torch.from_numpy(synth.lidar_cloud(cfg, 0)).to(cuda))
    torch.cuda.synchronize()
    assert _check_frame_levels(cuda, name, hot, r) == n_levels


def test_uniform_cloud_wide_caps_levels_in_first_appearance_order(cuda):
    """The uniform cloud with caps [4V, 4V, 2V, V]: 635 490 rows at level 2, thousands of look-back tiles."""
    import torch
    hot = _bench_frame(cuda, synth.C3, with_head=False)
    hot.net.set_level_caps(WIDE_CAPS)
    r = sparse_frame(hot, torch.from_numpy(synth.uniform_cloud(synth.C3, 0)).to(cuda))
    torch.cuda.synchronize()
    assert _check_frame_levels(cuda, "uniform", hot, r, both_entry_points=False) == UNIFORM_LEVELS


def _sites(rng, b, d, h, w, p):
    return np.argwhere(rng.random((b, d, h, w)) < p).astype(np.int32)


@pytest.mark.parametrize("case", ["overflow", "duplicates", "outside_grid"])
def test_level_edge_cases(cuda, case):
    """Both entry points on random batch-2 sites (rows shuffled): an out_cap below the site count keeps the first
    out_cap sites of the order with the flag set; repeated coordinates (the later row stands for the coordinate);
    rows outside the grid (no sites, in no map)."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(11)
    spatial = [9, 33, 31]
    coords = _sites(rng, 2, *spatial, 0.12)
    coords = coords[rng.permutation(len(coords))]
    if case == "duplicates":
        dup = coords[rng.choice(len(coords), len(coords) // 5, replace=False)]
        coords = np.concatenate([coords, dup])[rng.permutation(len(coords) + len(dup))]
    elif case == "outside_grid":
        bad = coords[rng.choice(len(coords), 300, replace=False)].copy()
        which = rng.integers(0, 4, len(bad))
        bad[np.arange(len(bad)), which] = np.where(rng.random(len(bad)) < 0.5, -1 - rng.integers(0, 3, len(bad)),
                                                   np.asarray([2] + spatial)[which] + rng.integers(0, 3, len(bad)))
        coords = np.concatenate([coords, bad])[rng.permutation(len(coords) + len(bad))]
    n = len(coords)
    tc = torch.from_numpy(coords).to(cuda)
    x = sp.sparse_coo_tensor(tc.t(), torch.zeros((n, 16), dtype=torch.float32, device=cuda), [2] + spatial + [16])
    convs = []  # kept alive: an index set caches its strided outputs by the conv's id
    for ks, st, pd in ((3, 2, 1), ((3, 1, 1), (2, 1, 1), 0), (3, 2, (0, 1, 1))):
        conv = sp.Conv3D(16, 16, ks, st, padding=pd, bias_attr=False)
        convs.append(conv)
        want, _, _ = first_appearance_sites(coords, 2, spatial, conv.kernel_size, conv.stride, conv.padding)
        out_cap = len(want) // 2 + 3 if case == "overflow" else 4 * n
        conv.out_cap = out_cap
        index, nbr = conv.build_index(x.index)
        torch.cuda.synchronize()
        label = "%s %s" % (case, (ks, st, pd))
        use_lfo = case == "overflow"  # lfo.nbr_map takes the first of repeated rows and has no notion of the grid
        _check_level(label, coords, 2, spatial, conv, index.coords, index.counters, nbr, out_cap, use_lfo)
        oc, cnt, nb = _rulebook_conv(cuda, tc, None, n, 2, spatial, conv, out_cap)
        _check_level(label + " (workspace entry point)", coords, 2, spatial, conv, oc, cnt, nb, out_cap, use_lfo)


def _print_regimes(name, r):
    import torch
    from paddle3d_b200._lib import lib
    from paddle3d_b200.ops import sparse_nn as sp
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    stream_k = 0
    for i, q in enumerate(r["pend"]):
        n = int(q.num[0])
        if q.precision != sp.F16X3:
            regime = "fp32 FMA"
        elif q.wm:
            grid, Wp, U, tiles = wm_ranges(sms, n, q.cap, q.K)
            regime = "warp MMA, %d warps over %d tiles, %.1f units per warp" % (Wp, tiles, U / Wp if Wp else 0.0)
            stream_k += 1
        else:
            ws = lib().p3d_sparse_conv_f16_workspace_bytes(q.cap, q.cout, sp.F16_MAX_SPLITS)
            regime = "wgmma, " + f16_sched(sms, n, q.cap, q.K, q.cout, sp.F16_MAX_SPLITS, ws).label()
            stream_k += "stream" in regime.lower()
        print("REGIME %s conv %d %d->%d rows %d of %d: %s" % (name, i, q.cin, q.cout, n, q.cap, regime))
    return stream_k


def test_default_frame_is_bit_reproducible(cuda):
    """The bench frame in its default mode, captured, run three times on one cloud with two other clouds in between:
    boxes, scores, labels and the BEV pixel image bit-equal every time; the eager chain (frame_chain) equal to it."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    assert sp.NARROW_WM[0] and sp.F16_MAX_SPLITS == 4
    cfg = synth.C3
    frames = bench.frame_pool(cfg, 3)
    pinned = [torch.from_numpy(f).pin_memory() for f in frames]
    dev0 = torch.from_numpy(frames[0]).to(cuda)
    hot = _bench_frame(cuda, cfg)
    hot.calibrate_head(dev0)
    hot.points.copy_(dev0)
    hot.capture()
    runs = []
    for rnd in range(3):
        out = [t.clone() for t in hot.infer(pinned[0])]
        assert not hot.h_status.any()
        runs.append((out, hot.out["bev_h16"][0].clone()))
        for f in pinned[1:]:
            hot.infer(f)
    (b0, s0, l0), bev0 = runs[0]
    assert len(l0) > 0
    for rnd, ((b, s, l), bev) in enumerate(runs[1:], 1):
        assert _bits_equal(bev, bev0), "run %d: BEV pixel image differs" % rnd
        assert len(l) == len(l0) and torch.equal(l, l0), "run %d: labels" % rnd
        assert _bits_equal(b, b0) and _bits_equal(s, s0), "run %d: boxes / scores" % rnd
    eager = frame_chain(hot, dev0)
    torch.cuda.synchronize()
    assert not eager["status"].any()
    assert _bits_equal(eager["bev"], bev0), "eager chain: BEV pixel image"
    boxes, scores, labels, counts = eager["post"]
    k = int(counts[-1])
    assert k == len(l0) and torch.equal(labels[:k].cpu(), l0)
    assert _bits_equal(boxes[:k].cpu(), b0) and _bits_equal(scores[:k].cpu(), s0)
    assert _print_regimes("C3", eager) > 0  # the row-order dependent decompositions ran


def test_sweep_lanes_default_mode(cuda):
    """CenterPointSweep with bench.py's four lanes in the default mode, six clouds of bench.frame_pool twice: every
    frame bit-equal to the single-lane captured frame on the same cloud."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointSweep
    cfg = synth.C3
    frames = bench.frame_pool(cfg, 6)
    pinned = [torch.from_numpy(f).pin_memory() for f in frames]
    dev0 = torch.from_numpy(frames[0]).to(cuda)
    sweep = CenterPointSweep(4, cfg=cfg, device=cuda, precision=sp.F16X3, seed=0, with_head=True, keep_bev=False,
                             bn_gain=bench.BN_GAIN)
    sweep.calibrate_head(dev0)
    sweep.capture(dev0)
    single = _bench_frame(cuda, cfg)
    single.share_model(sweep.lanes[0])
    single.points.copy_(dev0)
    single.capture()
    want = [[t.clone() for t in single.infer(f)] for f in pinned]
    for rnd in range(2):
        got = list(sweep.infer_many(iter(pinned)))
        assert len(got) == len(want)
        for i, (g, w) in enumerate(zip(got, want)):
            assert len(g[2]) == len(w[2]), "round %d frame %d: box count" % (rnd, i)
            assert _bits_equal(g[0], w[0]) and _bits_equal(g[1], w[1]) and torch.equal(g[2], w[2]), \
                "round %d frame %d differs from the single-lane frame" % (rnd, i)


def test_sweep_input_modes_agree_at_f16x3(cuda):
    """At F16X3: infer_stream equal to infer_sweeps on every frame (both merge on the device), and infer on the host
    merge equal to infer_sweeps wherever the two merged clouds are bit-equal."""
    import torch
    from paddle3d_b200 import io as p3d_io
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointHotPath
    from test_gpu_sweeps import _frame_inputs
    N = 40000
    seq = synth.sweep_sequence(12, 2, points_per_sweep=3800)
    kw = dict(precision=sp.F16X3, seed=3, num_points=N)
    ref = CenterPointHotPath(synth.C3, cuda, **kw)
    pipe = CenterPointHotPath(synth.C3, cuda, sweep_input=dict(slot_cap=8000), **kw)
    pipe.infer_sweeps(*_frame_inputs(seq, 0, 10))
    pipe.capture()
    per_frame, same_cloud = [], 0
    for j in range(len(seq)):
        key, sweeps = _frame_inputs(seq, j, 10)
        got = tuple(t.clone() for t in pipe.infer_sweeps(key, sweeps))
        per_frame.append(got)
        merged = p3d_io.merge_sweeps(key, sweeps, use_dim=4, use_time_lag=True, sweep_remove_radius=1.0)
        n = pipe.merged_rows()
        if n == len(merged) and np.array_equal(pipe.points[:n].cpu().numpy().view(np.uint32), merged.view(np.uint32)):
            full = np.full((N, 5), np.nan, np.float32)
            full[:n] = merged
            host = tuple(t.clone() for t in ref.infer(torch.from_numpy(full).pin_memory()))
            assert _same(host, got), "frame %d: infer != infer_sweeps" % j
            same_cloud += 1
    assert same_cloud >= len(seq) // 2
    stream = list(pipe.infer_stream(iter(seq)))
    assert len(stream) == len(seq)
    for j, (g, w) in enumerate(zip(stream, per_frame)):
        assert _same(g, w), "frame %d: infer_stream != infer_sweeps" % j
    print("SWEEP MODES %d frames, %d with bit-equal host and device merges" % (len(seq), same_cloud))


def test_predictor_writes_the_same_lines(cuda, tmp_path):
    """deploy.Predictor.run on one .bin file, twice on one predictor (another cloud in between) and once on a second
    predictor: the same format_result lines."""
    from paddle3d_b200 import deploy
    path = tmp_path / "cloud.bin"
    synth.lidar_cloud(synth.C3, 0).tofile(path)

    def load(f):  # the reference's loader: x, y, z, intensity of a 5-value .bin, time lag 0
        return deploy.insert_time_to_points(deploy.read_point(str(f), 5))
    a = deploy.Predictor(synth.C3, cuda, seed=0)
    first = deploy.format_result(*a.run(load(path)))
    other = tmp_path / "other.bin"
    synth.lidar_cloud(synth.C3, 1).tofile(other)
    a.run(load(other))
    again = deploy.format_result(*a.run(load(path)))
    del a
    fresh = deploy.format_result(*deploy.Predictor(synth.C3, cuda, seed=0).run(load(path)))
    assert len(first) > 0 and first == again == fresh
