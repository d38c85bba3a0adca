"""GPU: CenterPoint-pillars — the two-layer pillar encoder (p3d_pillar_feature_net2) against the fp64 oracle, the dense
fp16-pair convs at the model's shapes in every work decomposition the frame runs (float64 reference, the bar of
test_gpu_dense_schedule.py), SecondTrunk with upsample strides (0.5, 1, 2) against the CPU trunk, and the frame: eager
against the CPU arm (oracle/centerpoint_pillars.py), captured against eager, lanes against one lane, raw sweeps against
the host merge."""
import numpy as np
import pytest

from paddle3d_b200 import io as p3d_io
from paddle3d_b200 import synth
from parity import rel_check, rel_errors
from test_gpu_dense_schedule import DenseCase, _n_tile, _sms, run_dense, run_out9

pytestmark = pytest.mark.gpu

BN_GAIN = 6.0 ** 0.5
SMALL = dict(synth.CP_PILLARS, point_cloud_range=[-25.6, -25.6, -5.0, 25.6, 25.6, 3.0], num_points=60000)  # 256 x 256


# ------------------------------------------------------------------------------------------------- encoder
def _layers(rng, f, mid=32, out=64):
    ls = []
    for cin, c in ((f + 5, mid), (2 * mid, out)):
        ls.append(dict(weight=(rng.normal(size=(cin, c)) * 0.4).astype(np.float32), gamma=rng.uniform(0.5, 1.5, c),
                       beta=rng.normal(size=c) * 0.3, mean=rng.normal(size=c) * 0.1, var=rng.uniform(0.5, 1.5, c),
                       eps=1e-3))
    return ls


def _voxelized(cuda, cloud, f, m):
    import torch
    from paddle3d_b200.ops import voxelize
    cfg = dict(synth.CP_PILLARS, point_dim=f, point_cloud_range=[-12.8, -12.8, -5.0, 12.8, 12.8, 3.0])
    if cloud == "lidar":
        pts = synth.lidar_cloud(cfg, 5, num_points=40000)
    else:
        pts = synth.uniform_cloud(cfg, 6, num_points=60000)
    V = 20000
    vox, co, npv, nv = voxelize.hard_voxelize(torch.from_numpy(pts).to(cuda), cfg["voxel_size"],
                                              cfg["point_cloud_range"], m, V)
    coors = torch.cat([torch.zeros((V, 1), dtype=torch.int32, device=cuda), co], 1).contiguous()
    return cfg, vox, npv, coors, nv


def _crafted(cuda, f, m):
    """Pillars with 1 and with M points and random counts in between, at random cells; 50 capacity rows beyond num."""
    import torch
    rng = np.random.default_rng(f * 100 + m)
    cfg = dict(synth.CP_PILLARS, point_dim=f)
    n, cap = 300, 350
    npv = np.zeros(cap, np.int32)
    npv[:n] = np.concatenate([[1] * 20, [m] * 20, rng.integers(1, m + 1, n - 40)])
    cells = rng.choice(512 * 512, cap, replace=False)
    coors = np.stack([np.zeros(cap), np.zeros(cap), cells // 512, cells % 512], 1).astype(np.int32)
    vox = np.zeros((cap, m, f), np.float32)
    for i in range(n):
        x0 = coors[i, 3] * 0.2 - 51.2 + rng.uniform(0, 0.2, npv[i])
        y0 = coors[i, 2] * 0.2 - 51.2 + rng.uniform(0, 0.2, npv[i])
        vox[i, :npv[i]] = np.concatenate([np.stack([x0, y0, rng.uniform(-3, 1, npv[i])], 1),
                                          rng.uniform(0, 1, (npv[i], f - 3))], 1)
    t = lambda a: torch.from_numpy(a).to(cuda)  # noqa: E731
    return cfg, t(vox), t(npv), t(coors), torch.tensor([n], dtype=torch.int32, device=cuda)


@pytest.mark.parametrize("cloud,f,m", [("lidar", 5, 20), ("uniform", 5, 20), ("uniform", 4, 32), ("crafted", 5, 20),
                                       ("crafted", 4, 32)])
def test_pillar_feature_net2_vs_oracle(cuda, cloud, f, m):
    """p3d_pillar_feature_net2 against oracle.centerpoint_pillars.pillar_feature_net2: true relative 1e-4; rows beyond
    num_voxels untouched (they keep a sentinel)."""
    import torch
    from oracle.centerpoint_pillars import pillar_feature_net2 as oracle_pfn2
    from paddle3d_b200.ops import pillar_encoder as pe
    cfg, vox, npv, coors, nv = _crafted(cuda, f, m) if cloud == "crafted" else _voxelized(cuda, cloud, f, m)
    k = int(nv[0].item())
    counts = npv.cpu().numpy()[:k]
    if cloud == "crafted":
        assert (counts == 1).any() and (counts == m).any()
    rng = np.random.default_rng(3 + f)
    layers = _layers(rng, f)
    dev_layers = [dict(l, weight=torch.from_numpy(l["weight"]).to(cuda)) for l in layers]
    got = pe.pillar_feature_net2(vox, npv, coors, dev_layers, cfg["voxel_size"], cfg["point_cloud_range"], num_voxels=nv)
    want = oracle_pfn2(vox.cpu().numpy()[:k], counts, coors.cpu().numpy()[:k], layers, cfg["voxel_size"],
                       cfg["point_cloud_range"])
    rel_check("pfn2 %s F%d M%d" % (cloud, f, m), got.cpu().numpy()[:k], want, rtol=1e-4)
    assert (got.cpu().numpy()[k:] == 0).all()
    # capacity rows beyond num_voxels are not written: a pre-filled output keeps its sentinel
    from paddle3d_b200._lib import check, host_floats, lib
    from paddle3d_b200._mem import ptr, stream
    out = torch.full((vox.shape[0], 64), 7.0, device=cuda)
    (s1, t1), (s2, t2) = [pe.fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], cuda) for l in layers]
    check(lib().p3d_pillar_feature_net2(ptr(vox), ptr(npv), ptr(coors), ptr(nv), vox.shape[0], m, f, 32,
                                        ptr(dev_layers[0]["weight"]), ptr(s1), ptr(t1), 64, ptr(dev_layers[1]["weight"]),
                                        ptr(s2), ptr(t2), host_floats(cfg["voxel_size"]),
                                        host_floats(cfg["point_cloud_range"]), ptr(out), stream(cuda)), "pfn2")
    torch.cuda.synchronize()
    assert bool((out[k:] == 7.0).all())
    assert torch.equal(out[:k], got[:k])


# ------------------------------------------------------------------------------------------------- dense shapes
# (name, H, W, cin, cout, k, stride, pad, up): the layers of the frame whose shapes no other test runs
CP_PILLARS_LAYERS = [
    ("block1 64->64 s2 from 512", 512, 512, 64, 64, 3, 2, 1, 1),
    ("deblock0 2x2 s2 64->128 from 256", 256, 256, 64, 128, 2, 2, 0, 1),
    ("deblock1 1x1 128->128 at 128", 128, 128, 128, 128, 1, 1, 0, 1),
    ("deblock2 deconv 256->128 from 64", 64, 64, 256, 128, 2, 2, 0, 2),
    ("shared 384->64 at 128", 128, 128, 384, 64, 3, 1, 1, 1),
    ("heads 64->2304 at 128", 128, 128, 64, 2304, 3, 1, 1, 1),
]


@pytest.mark.parametrize("layer", CP_PILLARS_LAYERS, ids=lambda l: l[0].replace(" ", "_").replace(">", ""))
def test_dense_layer_every_decomposition(cuda, layer):
    """Each layer at full size: the frame's N tile with the MT rule's choice and (N = 64) the other M tiling, the other N
    tile where the layer has at least 128 channels, and for the 3x3 stride-1 layers the forced per-tap loads."""
    import torch
    name, H, W, cin, cout, k, stride, pad, up = layer
    case = DenseCase(cuda, 1, H, W, cin, cout, k, stride if up == 1 else up, pad, up, seed=cin * 7 + cout + H)
    tiles = [_n_tile(cout)] + ([64] if cout >= 128 else [])
    for nt in tiles:
        p, _, _ = run_dense("%s N%d" % (name, nt), case, nt, guards=nt == tiles[0])
        print("REGIME cp_pillars %s N%d: %s" % (name, nt, p.describe()))
        if nt == 64:
            other = 3 - p.inst[1]
            po, _, _ = run_dense("%s N64 MT%d" % (name, other), case, nt, m_tiles=other, guards=False)
            assert po.inst[1] == other
        if k == 3 and stride == 1:
            pt, _, _ = run_dense("%s N%d per-tap" % (name, nt), case, nt, mode=1, guards=False)
            assert not pt.halo
    del case
    torch.cuda.empty_cache()


def test_head_output_convs_at_128(cuda):
    """The 36 output convs of the six tasks (1..3 planes each, 70 planes) over the 2304-channel image at 128 x 128."""
    from paddle3d_b200.dense_head import COMMON_HEADS
    groups, p0 = [], 0
    for ncls in synth.CENTERPOINT_TASKS:
        for _, c in list(COMMON_HEADS) + [("hm", ncls)]:
            groups.append((c, p0, len(groups) * 64))
            p0 += c
    assert p0 == 70
    run_out9(cuda, "cp_pillars output convs 128x128", 1, 128, 128, 64, groups, 2304, True, seed=70)


def test_trunk_with_strided_deblock_vs_cpu(cuda):
    """SecondTrunk with upsample strides (0.5, 1, 2) (a 2x2 stride-2 conv, a 1x1 conv, a 2x2 transposed conv) on a small
    image against CpuDenseHead's convs, through the concat image."""
    import torch
    from oracle.cpu_reference import CpuDenseHead
    from paddle3d_b200.dense_head import SecondTrunk
    from paddle3d_b200.ops import dense_conv as dc
    trunk = SecondTrunk(64, (64, 128, 256), (1, 2, 2), (2, 2, 2), (128, 128, 128), (0.5, 1, 2))
    rng = np.random.default_rng(5)
    for c in trunk.convs():
        c.init(rng, cuda, randomize_bn=True, bn_gain=BN_GAIN)
    bev = np.random.default_rng(6).normal(size=(1, 64, 72, 88)).astype(np.float32)
    cat, shape = trunk(dc.nchw_to_pixel_h16(torch.from_numpy(bev).to(cuda)), (1, 72, 88, 64))
    assert shape == (1, 18, 22, 384)
    got = dc.pixel_h16_to_nchw(cat, shape).cpu().numpy()
    cpu = CpuDenseHead(trunk.export_numpy())
    x, feats = bev, []
    for blk in trunk.export_numpy()["blocks"]:
        for l in blk:
            x = cpu._conv(l, x)
        feats.append(x)
    want = np.concatenate([cpu._conv(l, f) for l, f in zip(trunk.export_numpy()["deblocks"], feats)], 1)
    rel_check("trunk (0.5, 1, 2) concat", got, want, rtol=2e-3, small_atol=1e-4)


# ------------------------------------------------------------------------------------------------- the frame
def _hot(cuda, cfg=SMALL, n=None, **kw):
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    hot = CenterPointPillarsHotPath(cfg, cuda, seed=2, num_points=n, bn_gain=BN_GAIN, **kw)
    pts = synth.lidar_cloud(cfg, 3, num_points=hot.n)
    hot.calibrate_head(torch.from_numpy(pts).to(cuda))
    return hot, pts


def _pair(got, cpu, tol=1e-3):
    """CPU boxes paired with GPU boxes by centre: every value and the score within tol (relative, absolute below 1) and
    equal labels.  Returns the fraction of CPU boxes paired."""
    gb, gs, gl = got
    used, n = set(), 0
    for i in range(len(cpu["boxes"])):
        if not len(gb):
            break
        j = int(np.argmin(np.abs(gb[:, :3] - cpu["boxes"][i, :3]).max(1)))
        eb = (np.abs(gb[j] - cpu["boxes"][i]) / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
        es = abs(gs[j] - cpu["scores"][i]) / max(1.0, abs(cpu["scores"][i]))
        if j not in used and eb <= tol and es <= tol and gl[j] == cpu["labels"][i]:
            used.add(j)
            n += 1
    return n / max(1, len(cpu["boxes"]))


def test_frame_matches_cpu_arm(cuda, oracle_mod):
    """The eager frame at a 256 x 256 grid against CpuCenterPointPillars: equal pillars, head planes on the parity bar,
    the frame's postprocess equal to the oracle's on the frame's own head planes, boxes paired with equal labels."""
    import torch
    from oracle.centerpoint_pillars import CpuCenterPointPillars
    hot, pts = _hot(cuda)
    got = [t.clone().numpy() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    m = hot.model
    cpu = CpuCenterPointPillars(m.cfg, m.export_numpy(), m.test_cfg, m.label_off).run(pts)
    nv = int(hot.out["num_voxels"][0])
    assert nv == cpu["num_voxels"]
    assert np.array_equal(hot.out["coors"][:nv].cpu().numpy(), cpu["coors"])
    h = {k: [t.cpu().numpy() for t in v] for k, v in hot.out["head"].items()}
    assert sum(t.shape[1] for v in h.values() for t in v) == 70 and h["hm"][0].shape[2:] == (64, 64)
    for name in h:
        for t, (g, w) in enumerate(zip(h[name], cpu["head"][name])):
            e = rel_errors(g, w)
            assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, (name, t, e)
    tc = m.test_cfg
    r = oracle_mod.centerpoint_postprocess(h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"],
                                           m.cfg["voxel_size"][:2], m.cfg["point_cloud_range"],
                                           tc["post_center_limit_range"], m.label_off, tc["down_ratio"],
                                           tc["score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"],
                                           tc["nms_post_max_size"], True)
    assert len(got[0]) == len(r[0]) > 0
    np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
    assert np.array_equal(got[2], r[2])
    assert abs(len(got[0]) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    frac = _pair(got, cpu)
    assert frac >= 0.95, frac


def test_graph_and_lanes_equal_eager(cuda):
    """Captured against eager, and four lanes (infer_many) against one: bit-equal boxes, scores and labels."""
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    hot, pts = _hot(cuda)
    frames = [torch.from_numpy(synth.lidar_cloud(SMALL, s, num_points=hot.n)).pin_memory() for s in (3, 4, 5)]
    eager = [[t.clone() for t in hot.infer(f)] for f in frames]
    assert all(len(e[0]) > 0 for e in eager)
    hot.capture(count_nodes=True)
    for f, e in zip(frames, eager):
        assert all(torch.equal(g, w) for g, w in zip(hot.infer(f), e))
    sweep = CenterPointSweep(4, frame_cls=CenterPointPillarsHotPath, cfg=SMALL, device=cuda, seed=2, bn_gain=BN_GAIN)
    for p in sweep.lanes:
        p.share_model(hot)
    sweep.capture(torch.from_numpy(pts).to(cuda))
    got = list(sweep.infer_many(frames[i % 3] for i in range(9)))
    for i, g in enumerate(got):
        assert all(torch.equal(a, b) for a, b in zip(g, eager[i % 3])), i


# ------------------------------------------------------------------------------------------------- sweep input
N_POINTS = 40000
SWEEP = dict(slot_cap=8000)


def _frame_inputs(seq, j, K):
    from paddle3d_b200 import sweep_ring
    ids = sweep_ring.frame_sweeps(j, K)
    key, pk, tk = seq[ids[0]]
    return key, [(seq[s][0], sweep_ring.ref_from_curr(pk, seq[s][1]), tk - seq[s][2]) for s in ids[1:]]


def _equal(a, b):
    import torch
    return all(torch.equal(x, y) for x, y in zip(a, b))


def test_sweeps_match_host_merge_and_lanes(cuda):
    """infer_sweeps (eager and captured) against infer on io.merge_sweeps' cloud of the same sweeps, and infer_stream
    over two lanes sharing one ring against the single-lane stream."""
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    K = 10
    seq = synth.sweep_sequence(K + 5, 2, points_per_sweep=3800)
    ref, _ = _hot(cuda, SMALL, N_POINTS)
    pipe = CenterPointPillarsHotPath(SMALL, cuda, seed=2, num_points=N_POINTS, bn_gain=BN_GAIN, sweep_input=SWEEP)
    pipe.share_model(ref)
    assert pipe.h_status.numel() == ref.h_status.numel() + 1 == 2
    key, sweeps = _frame_inputs(seq, K - 1, K)
    merged = p3d_io.merge_sweeps(key, sweeps, use_dim=4, use_time_lag=True, sweep_remove_radius=1.0)
    full = np.full((N_POINTS, 5), np.nan, np.float32)
    full[:len(merged)] = merged
    want = [t.clone() for t in ref.infer(torch.from_numpy(full).pin_memory())]
    eager = [t.clone() for t in pipe.infer_sweeps(key, sweeps)]
    assert pipe.merged_rows() == len(merged) and len(eager[0]) > 0
    if np.array_equal(pipe.points.cpu().numpy()[:len(merged)].view(np.uint32), merged.view(np.uint32)):
        assert _equal(eager, want)
    pipe.capture()
    assert _equal(pipe.infer_sweeps(key, sweeps), eager)
    single = list(pipe.infer_stream(iter(seq)))
    lanes = CenterPointSweep(2, frame_cls=CenterPointPillarsHotPath, cfg=SMALL, device=cuda, seed=2,
                             num_points=N_POINTS, bn_gain=BN_GAIN, sweep_input=SWEEP)
    assert lanes.lanes[1].ring is lanes.lanes[0].ring
    for p in lanes.lanes:
        p.share_model(ref)
        p.infer_sweeps(*_frame_inputs(seq, 0, K))
        p.capture()
    got = list(lanes.infer_stream(iter(seq)))
    assert len(got) == len(single) == len(seq)
    for j, (g, w) in enumerate(zip(got, single)):
        assert _equal(g, w), j
