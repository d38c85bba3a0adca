"""GPU suite for BEVFusion's new entry points against tests/bevfusion_oracle.py: p3d_hard_vfe (fp64 HardVFE, rows past
the device count untouched), p3d_se_gate_h16 (the gate against fp64, the scale bit for bit against its fp32 restatement,
reproducibility, the overflow bit) and p3d_anchor3d_postprocess (order, labels and counts bit-exact against the decode
restatement at full size and on small grids, above max_num, with NaN logits, with a reused workspace).

Class logits are quarter-integers: different logits give scores many ulps apart and equal logits give equal scores, so
the order never hangs on the last bit of expf and the tie rules are exercised."""
import ctypes

import numpy as np
import pytest

import bevfusion_oracle as bo

pytestmark = pytest.mark.gpu
F = np.float32


# ------------------------------------------------------------------------------------------------------------ HardVFE
def _vfe_case(rng, n, M, Fd, mid, out, shift_big=False, nz=1):
    """nz > 1: voxels of 8 / nz m in z, so coors' z column takes nz values and the decoration's z centre differs per
    pillar (with nz = 1 every pillar has z index 0)."""
    vs, pcr = (0.25, 0.25, 8.0 / nz), (-50.0, -50.0, -5.0, 50.0, 50.0, 3.0)
    coors = np.zeros((n, 4), np.int32)
    coors[:, 1] = rng.integers(0, nz, n)
    coors[:, 2] = rng.integers(0, 400, n)
    coors[:, 3] = rng.integers(0, 400, n)
    coors[:2, 2:] = [[0, 0], [399, 399]]                    # the grid's far corners
    npv = rng.integers(1, M + 1, n).astype(np.int32)
    npv[0] = M
    vox = np.zeros((n, M, Fd), F)
    for i in range(n):
        k = npv[i]
        vox[i, :k, 0] = pcr[0] + (coors[i, 3] + rng.random(k)) * vs[0]
        vox[i, :k, 1] = pcr[1] + (coors[i, 2] + rng.random(k)) * vs[1]
        vox[i, :k, 2] = pcr[2] + (coors[i, 1] + rng.random(k)) * vs[2]
        vox[i, :k, 3:] = rng.random((k, Fd - 3))
    vox[2, :npv[2], 2] = pcr[2] + coors[2, 1] * vs[2]          # points on the z edges of their voxel
    vox[3, :npv[3], 2] = pcr[2] + (coors[3, 1] + 1) * vs[2]
    layers = []
    for k, (cin, cout) in enumerate(((Fd + 6, mid), (2 * mid, out))):
        l = dict(weight=rng.normal(0, 0.3, (cin, cout)).astype(F), gamma=rng.uniform(0.5, 1.5, cout).astype(F),
                 beta=rng.normal(0, 0.5, cout).astype(F), mean=rng.normal(0, 0.1, cout).astype(F),
                 var=rng.uniform(0.5, 1.5, cout).astype(F), eps=1e-3)
        if shift_big:  # padding rows (zero inputs) give ReLU(shift): large shifts make them decide the max
            l["beta"] = (l["beta"] + 5.0).astype(F)
        layers.append(l)
    return vox, npv, coors, layers, vs, pcr


@pytest.mark.parametrize("Fd,M,mid,out,big,nz", [(3, 1, 64, 64, False, 1), (4, 64, 64, 64, False, 1),
                                                 (4, 32, 64, 64, True, 1), (5, 7, 16, 100, False, 1),
                                                 (8, 64, 33, 130, True, 1), (6, 20, 64, 64, False, 1),
                                                 (4, 16, 64, 64, False, 8), (5, 9, 32, 64, True, 5)])
def test_hard_vfe_matches_fp64(cuda, Fd, M, mid, out, big, nz):
    import torch
    from paddle3d_b200 import _lib
    from paddle3d_b200._mem import ptr
    from paddle3d_b200.ops.pillar_encoder import fold_bn
    rng = np.random.default_rng(Fd * 100 + M)
    n = 300
    vox, npv, coors, layers, vs, pcr = _vfe_case(rng, n, M, Fd, mid, out, big, nz)
    if nz > 1:
        assert len(np.unique(coors[:, 1])) == nz
    want = bo.hard_vfe_ref(vox, npv, coors, layers, vs, pcr)
    dv = [torch.from_numpy(a).to(cuda) for a in (vox, npv, coors)]
    w = [torch.from_numpy(l["weight"]).to(cuda) for l in layers]
    folded = [fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], cuda) for l in layers]
    nv = n - 17
    num = torch.tensor([nv], dtype=torch.int32, device=cuda)
    got = torch.full((n, out), float("nan"), dtype=torch.float32, device=cuda)
    L = _lib.lib()
    rc = L.p3d_hard_vfe(ptr(dv[0]), ptr(dv[1]), ptr(dv[2]), ptr(num), n, M, Fd, mid, ptr(w[0]), ptr(folded[0][0]),
                        ptr(folded[0][1]), out, ptr(w[1]), ptr(folded[1][0]), ptr(folded[1][1]), _lib.host_floats(vs),
                        _lib.host_floats(pcr), ptr(got), ctypes.c_void_p(torch.cuda.current_stream().cuda_stream))
    assert rc == 0
    g = got.cpu().numpy()
    assert np.isnan(g[nv:]).all()                            # rows past the device count untouched
    np.testing.assert_allclose(g[:nv], want[:nv], rtol=1e-4, atol=1e-4)
    # the op wrapper: every row, into a caller's buffer
    from paddle3d_b200.ops.pillar_encoder import hard_vfe
    lay = [dict(l, weight=w[k]) for k, l in enumerate(layers)]
    buf = torch.empty((n, out), dtype=torch.float32, device=cuda)
    res = hard_vfe(dv[0], dv[1], dv[2], lay, vs, pcr, out=buf)
    assert res.data_ptr() == buf.data_ptr()
    np.testing.assert_allclose(res.cpu().numpy(), want, rtol=1e-4, atol=1e-4)


# ------------------------------------------------------------------------------------------------------------ SE gate
def _se_case(cuda, rng, B, H, W, C, scale=1.0):
    import torch
    x = (rng.normal(0, scale, (B * H * W, C)) + rng.normal(0, 1, C)).astype(F)
    hi, lo, _ = bo.split_h16(x)
    rows = torch.from_numpy(bo.hilo_to_pair(hi, lo)).to(cuda)
    wt = (rng.normal(0, 1, (C, C)) / np.sqrt(C)).astype(F)
    bias = rng.normal(0, 0.5, C).astype(F)
    return rows, torch.from_numpy(wt).to(cuda), torch.from_numpy(bias).to(cuda)


@pytest.mark.parametrize("B,H,W,C", [(1, 200, 200, 384), (2, 7, 37, 64), (1, 1, 1, 32), (3, 16, 8, 1024)])
def test_se_gate(cuda, B, H, W, C):
    import torch
    from paddle3d_b200.ops.se_gate import se_gate_h16
    rng = np.random.default_rng(B * 1000 + C)
    rows, wt, bias = _se_case(cuda, rng, B, H, W, C)
    before = rows.cpu().numpy()
    status = torch.zeros(1, dtype=torch.int32, device=cuda)
    r1 = rows.clone()
    gate = se_gate_h16(r1, (B, H, W, C), wt, bias, status=status).cpu().numpy()
    hi, lo = bo.pair_to_hilo(before, C)
    x = bo.merge_h16(hi, lo).reshape(B, H, W, C)
    want = bo.se_gate_ref(x, wt.cpu().numpy(), bias.cpu().numpy())
    np.testing.assert_allclose(gate, want, rtol=0, atol=1e-5)
    want_rows, ovf = bo.se_scale_ref(before, C, np.repeat(gate, H * W, 0))
    np.testing.assert_array_equal(r1.cpu().numpy().view(np.uint16), want_rows.view(np.uint16))
    assert not ovf and int(status.item()) == 0
    r2 = rows.clone()
    gate2 = se_gate_h16(r2, (B, H, W, C), wt, bias, status=status).cpu().numpy()
    np.testing.assert_array_equal(gate2.view(np.uint32), gate.view(np.uint32))        # bit-reproducible
    np.testing.assert_array_equal(r2.cpu().numpy().view(np.uint16), r1.cpu().numpy().view(np.uint16))


def test_se_gate_overflow_bit(cuda):
    """A pair whose value exceeds 65504 (hi 65504, lo' > 0) scaled by a gate of exactly 1 leaves fp16's range: the value
    is saturated and status bit 0 set."""
    import torch
    from paddle3d_b200.ops.se_gate import se_gate_h16
    B, H, W, C = 1, 3, 5, 32
    hi = np.zeros((H * W, C), np.float16)
    lo = np.zeros((H * W, C), np.float16)
    hi[4, 7], lo[4, 7] = 65504.0, 1024.0
    rows = torch.from_numpy(bo.hilo_to_pair(hi, lo)).to(cuda)
    wt = torch.zeros((C, C), dtype=torch.float32, device=cuda)
    bias = torch.full((C,), 100.0, dtype=torch.float32, device=cuda)      # sigmoid(100) = 1 in fp32
    status = torch.zeros(1, dtype=torch.int32, device=cuda)
    gate = se_gate_h16(rows, (B, H, W, C), wt, bias, status=status)
    assert (gate == 1.0).all()
    assert int(status.item()) & 1
    h2, l2 = bo.pair_to_hilo(rows.cpu().numpy(), C)
    assert float(h2[4, 7]) == 65504.0 and float(l2[4, 7]) == 0.0
    status.zero_()
    hi[4, 7], lo[4, 7] = 65504.0, 0.0
    rows = torch.from_numpy(bo.hilo_to_pair(hi, lo)).to(cuda)
    se_gate_h16(rows, (B, H, W, C), wt, bias, status=status)
    assert int(status.item()) == 0


# ------------------------------------------------------------------------------------------------- anchor3d postprocess
TEST = dict(nms_pre=1000, score_thr=0.05, nms_thr=0.2, max_num=500, dir_offset=0.7854, dir_limit_offset=0.0)


def _head(rng, H, W, C, R, frac=0.02, nan=0):
    """Quarter-integer class logits, about `frac` of (anchor, class) values above logit(0.05) = -2.94; small deltas."""
    A = H * W * R
    q = rng.integers(-60, -12, (R * C, H, W))
    hot = rng.random((R * C, H, W)) < frac
    q[hot] = rng.integers(-11, 12, int(hot.sum()))
    head = np.zeros((R * (C + 11), H, W), F)
    head[:R * C] = q / 4.0
    head[R * C:R * (C + 9)] = rng.normal(0, 0.3, (R * 9, H, W))
    head[R * (C + 9):] = rng.integers(-2, 3, (R * 2, H, W)) / 2.0        # dir logits with ties
    if nan:
        idx = rng.choice(R * C * H * W, nan, replace=False)
        head[:R * C].reshape(-1)[idx] = np.nan
    assert A == H * W * R
    return head


def _anchors(rng, H, W, R):
    from paddle3d_b200 import bevfusion as bf
    if (H, W, R) == (200, 200, 14):
        return bf.make_anchors()
    a = np.zeros((H * W * R, 9), F)
    a[:, 0] = rng.uniform(-6, 6, len(a))          # crowded: boxes overlap
    a[:, 1] = rng.uniform(-6, 6, len(a))
    a[:, 2] = -1.8
    a[:, 3:6] = rng.uniform(0.5, 4.0, (len(a), 3))
    a[:, 6] = rng.choice([0.0, 1.57], len(a))
    return a


def _run(cuda, head, anchors, C, R, cfg, out=None):
    import torch
    from paddle3d_b200.ops.anchor3d_postprocess import anchor3d_postprocess_device
    res = anchor3d_postprocess_device(torch.from_numpy(head[None]).to(cuda), torch.from_numpy(anchors).to(cuda), C, R,
                                      cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"], cfg["max_num"], cfg["dir_offset"],
                                      cfg["dir_limit_offset"], out=out)
    k = int(res[3].item())
    return res, (res[0][:k].cpu().numpy(), res[1][:k].cpu().numpy(), res[2][:k].cpu().numpy())


def _compare(got, want):
    gb, gs, gl = got
    wb, ws, wl = want
    assert len(gb) == len(wb), (len(gb), len(wb))
    np.testing.assert_array_equal(gl, wl)
    np.testing.assert_allclose(gs, ws, rtol=1e-6, atol=0)
    np.testing.assert_allclose(gb, wb, rtol=1e-6, atol=1e-6)


@pytest.mark.parametrize("H,W,C,R,cfg,frac", [
    (200, 200, 10, 14, TEST, 0.02),                                   # the bevf_pp head at full size, cut at max_num
    (200, 200, 10, 14, TEST, 0.00005),                                # full size, class-major below max_num
    (200, 200, 10, 14, dict(TEST, max_num=40), 0.02),                  # far more survivors than max_num
    (6, 5, 3, 2, dict(TEST, nms_pre=1000, max_num=500), 0.5),         # A <= nms_pre: every anchor in anchor order
    (9, 7, 4, 6, dict(TEST, nms_pre=50, max_num=30), 0.4),             # the cut and max_num on a small grid
    (16, 16, 1, 2, dict(TEST, nms_pre=200, max_num=500, nms_thr=0.5), 0.3),
    (4, 4, 2, 2, dict(TEST, score_thr=0.999), 0.0),                    # every class empty: 0 rows
])
def test_anchor3d_postprocess_matches_restatement(cuda, oracle_mod, H, W, C, R, cfg, frac):
    rng = np.random.default_rng(H * 31 + C * 7 + cfg["max_num"])
    head = _head(rng, H, W, C, R, frac)
    anchors = _anchors(rng, H, W, R)
    _, got = _run(cuda, head, anchors, C, R, cfg)
    want = bo.anchor3d_decode_ref(head, anchors, C, R, cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"],
                                  cfg["max_num"], cfg["dir_offset"], cfg["dir_limit_offset"])
    _compare(got, want)
    if frac == 0.02:
        assert len(want[0]) == cfg["max_num"]                           # more survivors than max_num
    if frac == 0.00005:
        assert 0 < len(want[0]) < cfg["max_num"] and len(set(want[2].tolist())) == C


def test_anchor3d_postprocess_nan_logits_and_workspace_reuse(cuda, oracle_mod):
    """NaN class logits take kept slots at the cut (torch.topk's order) and never pass the threshold themselves; a second
    call on new planes with the same output buffers and workspace gives the restatement's rows for the new planes."""
    H, W, C, R = 40, 30, 10, 14
    rng = np.random.default_rng(5)
    anchors = _anchors(rng, H, W, R)
    cfg = dict(TEST, nms_pre=300, max_num=100)
    head = _head(rng, H, W, C, R, 0.05, nan=200)
    out, got = _run(cuda, head, anchors, C, R, cfg)
    want = bo.anchor3d_decode_ref(head, anchors, C, R, cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"], cfg["max_num"],
                                  cfg["dir_offset"], cfg["dir_limit_offset"], details=True)
    _compare(got, want[:3])
    head2 = _head(rng, H, W, C, R, 0.01)
    _, got2 = _run(cuda, head2, anchors, C, R, cfg, out=out)
    want2 = bo.anchor3d_decode_ref(head2, anchors, C, R, cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"],
                                   cfg["max_num"], cfg["dir_offset"], cfg["dir_limit_offset"])
    _compare(got2, want2)


# ---------------------------------------------------------------------------------------------------- the frame
def _frame_inputs(m, seed, n=20000):
    from paddle3d_b200 import synth
    c = m.cfg
    cloud_cfg = dict(num_points=n, point_dim=4, point_cloud_range=list(c["point_cloud_range"]))
    pts = synth.lidar_cloud(cloud_cfg, seed, n).astype(np.float32)
    rig = synth.camera_rig(seed, bda=False)
    vt = m.vt
    rng = np.random.default_rng(seed)
    logits = rng.normal(0, 2, (m.N, vt.D, vt.H, vt.W)).astype(np.float32)
    tran = rng.normal(0, 1, (m.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)
    return pts, synth.lss_mats(rig), logits, tran


def _cpu_run(m, pts, mats, logits, tran):
    from paddle3d_b200.ops import bev_pool_v2 as bp
    cams = bp.unpack_cameras(bp.pack_cameras(*mats), 1, m.N)
    axes = tuple(a.numpy() for a in m.vt.axes_host)
    return bo.CpuBEVFusion(m.export_numpy(), m.cfg, m.anchors_np).run(pts, cams, axes, logits, tran, *m.vt.grid_args())


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


@pytest.fixture(scope="module")
def fusion(cuda):
    """A seeded, calibrated BEVFusion at test size with one frame's inputs and the CPU arm's result for them."""
    from paddle3d_b200 import bevfusion as bf
    m = bf.BEVFusion(bf.small_config(), device=cuda).init_weight(seed=0)
    pts, mats, logits, tran = _frame_inputs(m, 3)
    m.calibrate_cls_bias(_t(cuda, pts), mats, _t(cuda, logits), _t(cuda, tran))
    cpu = _cpu_run(m, pts, mats, logits, tran)
    return dict(m=m, pts=pts, mats=mats, logits=logits, tran=tran, cpu=cpu)


def _pair(got, cpu, tol=1e-3):
    """Fraction of the CPU arm's boxes paired by centre with a GPU box of equal label whose values and score are within tol
    (relative, absolute below 1); the heading compared modulo 2 pi."""
    gb, gs, gl = [np.asarray(v) for v in got]
    used, n = set(), 0
    for i in range(len(cpu["boxes"])):
        if not len(gb):
            break
        j = int(np.argmin(np.abs(gb[:, :3] - cpu["boxes"][i, :3]).max(1)))
        d = np.abs(gb[j] - cpu["boxes"][i])
        d[6] = abs((gb[j, 6] - cpu["boxes"][i, 6] + np.pi) % (2 * np.pi) - np.pi)
        eb = (d / np.maximum(1.0, np.abs(cpu["boxes"][i]))).max()
        es = abs(gs[j] - cpu["scores"][i]) / max(1.0, abs(cpu["scores"][i]))
        if j not in used and eb <= tol and es <= tol and gl[j] == cpu["labels"][i]:
            used.add(j)
            n += 1
    return n / max(1, len(cpu["boxes"]))


def test_frame_matches_cpu_arm(cuda, oracle_mod, fusion):
    """The captured frame: fused BEV and head planes within the fp16-pair parity bar of the CPU arm, its decode equal to
    the restatement's on the frame's own planes, boxes paired with equal labels, every class in the output."""
    from paddle3d_b200.bevfusion import BEVFusionHotPath
    from paddle3d_b200.ops import dense_conv as dc
    from parity import rel_errors
    m, cpu = fusion["m"], fusion["cpu"]
    hot = BEVFusionHotPath(m, num_points=30000, device=cuda).capture(count_nodes=True)
    assert hot.graph_nodes["kernel"] > 0
    got = [t.clone().numpy() for t in hot.infer(fusion["pts"], fusion["mats"], _t(cuda, fusion["logits"]),
                                                 _t(cuda, fusion["tran"]))]
    Y, X = m.bev_hw
    fused = dc.pixel_h16_to_nchw(hot.fused, (1, Y, X, m.fuse_C)).cpu().numpy()
    e = rel_errors(fused, cpu["fused"])
    assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
    planes = hot.out["planes"].cpu().numpy()
    e = rel_errors(planes, cpu["planes"])
    assert e["max_rel"] <= 5e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
    want = bo.anchor3d_decode_ref(planes, m.anchors_np, m.num_classes, m.R, **m.cfg["test"])
    _compare(got, want)
    assert len(cpu["boxes"]) > 0 and len(set(cpu["labels"].tolist())) == m.num_classes
    assert _pair(got, cpu) >= 0.95


def test_captured_eager_lanes_accelerate(cuda, oracle_mod, fusion):
    """Captured = eager bit for bit; three lanes sharing the model, each on its own frame, = one lane; accelerate = full."""
    from paddle3d_b200 import bevfusion as bf
    from paddle3d_b200.bevfusion import BEVFusionHotPath
    m = fusion["m"]
    items = [(p, mt, _t(cuda, lg), _t(cuda, tr)) for p, mt, lg, tr in (_frame_inputs(m, s) for s in (3, 4, 5))]
    eager = []
    for p, mt, lg, tr in items:
        o = m.forward(_t(cuda, p), mt, lg, tr)
        k = int(o["counts"].item())
        eager.append([o["boxes"][:k].cpu(), o["scores"][:k].cpu(), o["labels"][:k].cpu()])
    one = BEVFusionHotPath(m, num_points=30000, device=cuda).capture()
    ref = one.infer_many(items)
    for r, e in zip(ref, eager):
        for a, b in zip(r, e):
            assert torch_equal(a, b)
    lanes = [BEVFusionHotPath(m, num_points=30000, device=cuda).share_model(one).capture() for _ in range(3)]
    for lane, it in zip(lanes, items):
        lane.launch(*it)
    for lane, r in zip(lanes, ref):
        for a, b in zip(lane.result(), r):
            assert torch_equal(a, b)
    acc_m = bf.BEVFusion(m.cfg, accelerate=True, device=cuda)
    acc_m.__dict__.update({k: v for k, v in m.__dict__.items() if k != "vt"})
    acc = BEVFusionHotPath(acc_m, num_points=30000, device=cuda).capture()
    for it, r in zip(items + items[:1], ref + ref[:1]):
        for a, b in zip(acc.infer(*it), r):
            assert torch_equal(a, b)


def torch_equal(a, b):
    import torch
    return a.shape == b.shape and bool(torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                                                   b.view(torch.int32) if b.dtype == torch.float32 else b))


def test_empty_cloud_empty_frustum_and_capacity(cuda, oracle_mod, fusion):
    """No points: the LiDAR half of the fused image is the trunk of an empty pillar image and the frame is valid; a camera
    rig that looks away from the grid: the camera half is the encoder of a zero pool; more points than the lane holds:
    ValueError before anything is enqueued."""
    from paddle3d_b200.bevfusion import BEVFusionHotPath
    from paddle3d_b200.ops import dense_conv as dc
    from parity import rel_errors
    m = fusion["m"]
    hot = BEVFusionHotPath(m, num_points=30000, device=cuda).capture()
    pts, mats, logits, tran = _frame_inputs(m, 6)
    empty = np.zeros((0, 4), np.float32)
    got = [t.clone().numpy() for t in hot.infer(empty, mats, _t(cuda, logits), _t(cuda, tran))]
    cpu = _cpu_run(m, empty, mats, logits, tran)
    assert cpu["num_voxels"] == 0
    Y, X = m.bev_hw
    fused = dc.pixel_h16_to_nchw(hot.fused, (1, Y, X, m.fuse_C)).cpu().numpy()
    e = rel_errors(fused, cpu["fused"])
    assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
    want = bo.anchor3d_decode_ref(hot.out["planes"].cpu().numpy(), m.anchors_np, m.num_classes, m.R, **m.cfg["test"])
    _compare(got, want)
    s2e = np.array(mats[0], copy=True)
    s2e[..., 2, 3] += 1000.0                                         # every camera 1 km above the grid
    far = (s2e,) + tuple(mats[1:])
    got = [t.clone().numpy() for t in hot.infer(pts, far, _t(cuda, logits), _t(cuda, tran))]
    cpu = _cpu_run(m, pts, far, logits, tran)
    fused = dc.pixel_h16_to_nchw(hot.fused, (1, Y, X, m.fuse_C)).cpu().numpy()
    e = rel_errors(fused, cpu["fused"])
    assert e["max_rel"] <= 2e-3 and e["max_small_abs_over_scale"] <= 1e-4, e
    want = bo.anchor3d_decode_ref(hot.out["planes"].cpu().numpy(), m.anchors_np, m.num_classes, m.R, **m.cfg["test"])
    _compare(got, want)
    with pytest.raises(ValueError):
        hot.launch(np.zeros((30001, 4), np.float32), mats, _t(cuda, logits), _t(cuda, tran))
