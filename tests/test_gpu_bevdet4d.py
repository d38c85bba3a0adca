"""GPU tests of BEVDet4D: p3d_bev_shift_h16 bit for bit against its numpy fp32 restatement and within fp32 coordinate
rounding of the fp64 shift_feature, and drives of the sequential frame (captured, eager, restart, lanes, accelerate)
against the CPU arm (bevdet4d_oracle.CpuBEVDet4D)."""
import numpy as np
import pytest

from bevdet4d_oracle import CpuBEVDet4D, shift_feature, shift_h16_fp32
from oracle import bevdet as ob
from parity import rel_errors
from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu
BN_GAIN = 6.0 ** 0.5
FRAMES = 3


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _pairs(img, B, H, W, C):
    """pixel H16 rows [B*H*W, 2*C] float16 -> (hi, lo') numpy [B, H, W, C] float16"""
    a = img.cpu().numpy().reshape(B, H, W, C // 32, 2, 32)
    return a[:, :, :, :, 0].reshape(B, H, W, C), a[:, :, :, :, 1].reshape(B, H, W, C)


def _tf6(kind, h, w):
    """fp32 [6] transforms of the kernel tests, in BEV pixels."""
    if kind == "identity":
        return np.array([1, 0, 0, 0, 1, 0], np.float32)
    if kind == "fraction":
        return np.array([1, 0, 0.37, 0, 1, -0.61], np.float32)
    if kind == "yaw":  # 5 degrees about the centre and 2 m of 0.8 m cells
        a = np.radians(5.0)
        c, s = np.cos(a), np.sin(a)
        cx, cy = (w - 1) / 2, (h - 1) / 2
        return np.array([c, -s, cx - c * cx + s * cy + 2.5, s, c, cy - s * cx - c * cy], np.float32)
    if kind == "half":
        return np.array([1, 0, w / 2 + 0.3, 0, 1, 0.2], np.float32)
    if kind == "huge":
        return np.array([1, 0, 3e38, 0, 1, -1e30], np.float32)
    return np.array([1, 0, np.nan, 0, 1, 0], np.float32)


KINDS = ["identity", "fraction", "yaw", "half", "huge", "nan"]


@pytest.mark.parametrize("B,h,w,in_C,C,out_C,c0,same", [
    (2, 9, 13, 32, 16, 64, 16, False),
    (2, 12, 10, 64, 48, 96, 48, False),
    (1, 16, 20, 96, 80, 160, 80, False),    # BEVDet4D's history -> concat
    (1, 16, 20, 160, 80, 160, 80, True),    # the start frame: the concat's own bev_feat, in place
    (1, 128, 128, 96, 80, 160, 80, False),  # full size
])
def test_shift_bit_exact(cuda, B, h, w, in_C, C, out_C, c0, same):
    """Bit-equal to shift_h16_fp32 for every transform (huge / NaN: zeros, status 0), channels outside [c0, c0 + C) of the
    output rows unchanged, and within the fp32 coordinate rounding of the fp64 shift_feature."""
    import torch
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import dense_conv as dc
    from paddle3d_b200.ops import sparse_nn as sp
    rng = np.random.default_rng(h * w + C)
    for i in range(0, len(KINDS), B):
        kinds = [KINDS[(i + b) % len(KINDS)] for b in range(B)]
        tf6 = np.stack([_tf6(k, h, w) for k in kinds])
        x = rng.normal(0, 3, size=(B, in_C, h, w)).astype(np.float32)
        xs = dc.nchw_to_pixel_h16(_t(cuda, x))
        if same:
            out = xs
            before = xs.clone()
        else:
            out = torch.full((B * h * w, 2 * out_C), 7.0, dtype=torch.float16, device=cuda)
            before = out.clone()
        torch.cuda.synchronize()
        hi, lo = _pairs(xs, B, h, w, in_C)
        xin = ob.merge_h16(hi[..., :C], lo[..., :C])
        sp.status_tensor(cuda).zero_()
        bp.bev_shift_h16(xs, (B, h, w, in_C), _t(cuda, tf6), C, out_h16=out, out_channels=out_C, out_c0=c0)
        torch.cuda.synchronize()
        assert int(sp.status_tensor(cuda)[0]) == 0
        want = shift_h16_fp32(xin, tf6)
        whi, wlo = ob.split_h16(want)
        ghi, glo = _pairs(out, B, h, w, out_C)
        assert np.array_equal(ghi[..., c0:c0 + C].view(np.int16), whi.view(np.int16)), kinds
        assert np.array_equal(glo[..., c0:c0 + C].view(np.int16), wlo.view(np.int16)), kinds
        bhi, blo = _pairs(before, B, h, w, out_C)
        rest = np.ones(out_C, bool)
        rest[c0:c0 + C] = False
        assert np.array_equal(ghi[..., rest].view(np.int16), bhi[..., rest].view(np.int16))
        assert np.array_equal(glo[..., rest].view(np.int16), blo[..., rest].view(np.int16))
        got = ob.merge_h16(ghi[..., c0:c0 + C], glo[..., c0:c0 + C]).astype(np.float64)
        for b, k in enumerate(kinds):
            if k in ("huge", "nan"):
                assert not got[b].any()
                continue
            tf = np.vstack([tf6[b].reshape(2, 3).astype(np.float64), [0.0, 0.0, 1.0]])
            ref = shift_feature(xin[b:b + 1].transpose(0, 3, 1, 2), None, None, None, None, None, tf=tf[None])
            ref = ref[0].transpose(1, 2, 0)
            # about ten fp32 roundings on coordinates of magnitude <= 2 max(h, w) pixels; a sample that moves by e pixels
            # changes by at most 2 e max |x|; plus the fp32 sum and the pair split
            e_px = 16 * 2.0 ** -24 * 2 * max(h, w)
            bound = (2 * e_px + 2.0 ** -20) * np.abs(xin[b]).max()
            assert np.abs(got[b] - ref).max() <= bound, (k, np.abs(got[b] - ref).max(), bound)
            if k == "half":
                assert not got[b][:, w // 2 + 1:].any() and got[b][:, :w // 2 - 1].all()


# ---------------------------------------------------------------------------------------------------- the frame
def _drive(m, rig_seed, seed, speed=10.0, yaw_rate=0.3):
    """FRAMES frames of one camera rig on a moving ego (synth.ego_poses, 0.5 s apart): per frame the matrices, the previous
    frame's cameras in this frame's ego (None for the first), the depth net's output and the fp64 matrices of the CPU
    arm."""
    from paddle3d_b200.ops import bev_pool_v2 as bp
    vt = m.vt
    rig = synth.camera_rig(rig_seed)
    poses = synth.ego_poses(FRAMES, speed=speed, yaw_rate=yaw_rate)
    e2g = [np.broadcast_to(p, (1, m.N, 4, 4)) for p in poses]
    rng = np.random.default_rng(seed)
    out = []
    for k in range(FRAMES):
        prev = None if k == 0 else bp.sensor2keyegos(rig["sensor2ego"], e2g[k - 1], e2g[k])
        out.append(dict(mats=synth.lss_mats(rig), prev=prev, s2ke=rig["sensor2ego"].astype(np.float64),
                        bda=rig["bda"].astype(np.float64),
                        logits=rng.normal(0, 2, (m.N, vt.D, vt.H, vt.W)).astype(np.float32),
                        tran=rng.normal(0, 1, (m.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)))
    return out


def _cams(mats):
    from paddle3d_b200.ops import bev_pool_v2 as bp
    return bp.unpack_cameras(bp.pack_cameras(*mats), 1, 6)


def _run(hot, cuda, frames):
    """The drive on one lane: per frame the boxes / scores / labels (host copies)."""
    res = []
    for k, f in enumerate(frames):
        got = hot.infer(f["mats"], f["prev"], _t(cuda, f["logits"]), _t(cuda, f["tran"]), new_sequence=k == 0)
        res.append([t.clone() for t in got])
    return res


@pytest.fixture(scope="module")
def drive(cuda):
    """A seeded BEVDet4D calibrated on its first frame, a 3-frame drive and the CPU arm's result for every frame."""
    from paddle3d_b200.bevdet import BEVDet4D
    m = BEVDet4D(device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    frames = _drive(m, 31, 7)
    f0 = frames[0]
    m.calibrate_heatmap_bias(f0["mats"], _t(cuda, f0["logits"]), _t(cuda, f0["tran"]))
    axes = tuple(a.numpy() for a in m.vt.axes_host)
    arm = CpuBEVDet4D(m.export_numpy(), m.test_cfg, m.label_off)
    cpu = [arm.run(_cams(f["mats"]), axes, f["logits"], f["tran"], *m.vt.grid_args(), f["s2ke"], f["bda"],
                   s2ke_prev=f["prev"], new_sequence=k == 0) for k, f in enumerate(frames)]
    return dict(m=m, frames=frames, cpu=cpu)


def _pair(got, cpu, tol=1e-3):
    """test_gpu_bevdet._pair: the fraction of CPU boxes paired by centre with a GPU box of equal label whose values and
    score are within tol (relative, absolute below 1)."""
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


def test_drive_matches_cpu_arm(cuda, oracle_mod, drive):
    """Every frame of the captured drive: the concat (pre_process + shift) against the CPU arm's, head planes on
    test_gpu_bevdet's bar, the postprocess equal to the oracle's on the frame's own planes, boxes paired with equal
    labels; the moving frames' shifted channels differ from the unshifted history."""
    from paddle3d_b200.bevdet import BEVDet4DHotPath
    from paddle3d_b200.ops import dense_conv as dc
    m, frames, cpu = drive["m"], drive["frames"], drive["cpu"]
    hot = BEVDet4DHotPath(m, device=cuda).capture(count_nodes=True)
    assert hot.graph_nodes["kernel"] > 0 and hot.graph_nodes["memcpy"] >= 2 * 8
    tc = m.test_cfg
    prev_hist = None
    for k, (f, c) in enumerate(zip(frames, cpu)):
        got = [t.clone().numpy() for t in hot.infer(f["mats"], f["prev"], _t(cuda, f["logits"]), _t(cuda, f["tran"]),
                                                     new_sequence=k == 0)]
        cat = dc.pixel_h16_to_nchw(hot.concat, m.enc_shape).cpu().numpy()
        e = rel_errors(cat, np.concatenate([c["bev_feat"], c["shifted"]], 1))
        # 5e-3: the kernel samples at fp32 coordinates, the arm at fp64 ones (~1e-5 pixel apart at 128 pixels)
        assert e["max_rel"] <= 5e-3 and e["max_small_abs_over_scale"] <= 1e-4, (k, e)
        if k:  # not blind to the shift: the shifted history is far from the unshifted one
            unshifted = prev_hist[:, :80]
            assert np.linalg.norm(cat[:, 80:] - unshifted) > 0.2 * np.linalg.norm(unshifted), k
        prev_hist = dc.pixel_h16_to_nchw(hot.history, (1, 128, 128, 96)).cpu().numpy()
        h = {n: [t.cpu().numpy() for t in v] for n, v in hot.out["head"].items()}
        for name in h:
            for t, (g, w) in enumerate(zip(h[name], c["head"][name])):
                e = rel_errors(g, w)
                assert e["max_rel"] <= 5e-3 and e["max_small_abs_over_scale"] <= 1e-4, (k, name, t, e)
        r = oracle_mod.centerpoint_postprocess(h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"],
                                               tc["voxel_size"], tc["point_cloud_range"], tc["post_center_limit_range"],
                                               m.label_off, tc["down_ratio"], tc["score_threshold"],
                                               tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"],
                                               True)
        assert len(got[0]) == len(r[0]) > 0, k
        np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
        assert np.array_equal(got[2], r[2])
        assert _pair(got, c) >= 0.95, k


def test_captured_eager_restart_padding(cuda, drive):
    """Captured == eager bit for bit over the drive, the history equal to the eager bev_feat of the frame before;
    restarting the sequence reproduces frame 0; pre_process's padding channels stay zero; a lane's first frame without
    new_sequence raises."""
    import torch
    from paddle3d_b200.bevdet import BEVDet4DHotPath
    m, frames = drive["m"], drive["frames"]
    hot = BEVDet4DHotPath(m, device=cuda).capture()
    with pytest.raises(ValueError, match="new_sequence"):
        hot.launch(frames[1]["mats"], frames[1]["prev"], _t(cuda, frames[1]["logits"]), _t(cuda, frames[1]["tran"]))
    feat_prev, first = None, None
    for k, f in enumerate(frames):
        tl, tt = _t(cuda, f["logits"]), _t(cuda, f["tran"])
        (boxes, scores, labels, counts), bev_feat = m.forward(f["mats"], f["prev"], tl, tt, feat_prev)
        n = int(counts[-1])
        eager = [boxes[:n].cpu(), scores[:n].cpu(), labels[:n].cpu()]
        if feat_prev is not None:
            assert torch.equal(hot.history.view(torch.int16), feat_prev.view(torch.int16)), k
        got = [t.clone() for t in hot.infer(f["mats"], f["prev"], tl, tt, new_sequence=k == 0)]
        assert n > 0 and all(torch.equal(g, e) for g, e in zip(got, eager)), k
        assert torch.equal(hot.history.view(torch.int16), bev_feat.view(torch.int16)), k
        first = first or got
        feat_prev = bev_feat
    f = frames[0]
    again = hot.infer(f["mats"], None, _t(cuda, f["logits"]), _t(cuda, f["tran"]), new_sequence=True)
    assert all(torch.equal(g, w) for g, w in zip(again, first))
    for stage in hot.pre_bufs:
        for blk in stage:
            for buf in blk.values():
                hi, lo = _pairs(buf, 1, 128, 128, 96)
                assert not hi[..., 80:].any() and not lo[..., 80:].any()


def test_lanes_and_accelerate(cuda, drive):
    """Four lanes sharing the model on four drives, launched together frame by frame, == each drive alone on one lane;
    accelerate=True (the rank graph replayed once per drive) == the full frames."""
    import torch
    from paddle3d_b200.bevdet import BEVDet4D, BEVDet4DHotPath
    m = drive["m"]
    drives = [_drive(m, 40 + i, 50 + i, speed=6.0 + 3 * i, yaw_rate=0.1 * i) for i in range(4)]
    one = BEVDet4DHotPath(m, device=cuda).capture()
    want = [_run(one, cuda, d) for d in drives]
    lanes = [BEVDet4DHotPath(m, device=cuda).capture() for _ in range(4)]
    for k in range(FRAMES):
        for lane, d in zip(lanes, drives):
            f = d[k]
            lane.launch(f["mats"], f["prev"], _t(cuda, f["logits"]), _t(cuda, f["tran"]), new_sequence=k == 0)
        for i, lane in enumerate(lanes):
            assert all(torch.equal(g, w) for g, w in zip(lane.result(), want[i][k])), (i, k)
    acc_model = BEVDet4D(accelerate=True, device=cuda)
    acc_model.encoder, acc_model.head, acc_model.pre_process = m.encoder, m.head, m.pre_process
    acc = BEVDet4DHotPath(acc_model, device=cuda).capture()
    for i in (0, 1, 0):
        got = _run(acc, cuda, drives[i])
        for k in range(FRAMES):
            assert all(torch.equal(g, w) for g, w in zip(got[k], want[i][k])), (i, k)
