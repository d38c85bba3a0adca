"""GPU tests of BEVDet's box decode (p3d_bevdet_postprocess) against the numpy oracle (tests/bevdet_postprocess_oracle.py),
and of the BEVDet / BEVDet4D frames that end in it against their CPU arms.

Exact comparisons need the two sides to order the scores alike, and the device's expf and numpy's exp may differ in the
last bit of a sigmoid.  The synthetic heat maps are therefore rounded to multiples of 1/64 (the statistics of SURVEY §8d
otherwise): equal logits give equal scores on both sides and order by the defined tie rule, which every case below then
exercises, and different logits give scores many ulps apart.  What is compared bit for bit is what either side computes
without a transcendental: x, y (which name the cell), the gravity-centre inputs, velocities, labels, counts and order."""
import numpy as np
import pytest

from bevdet_postprocess_oracle import CpuBEVDet4DNMS, CpuBEVDetNMS, bevdet_postprocess_ref
from paddle3d_b200 import synth
from test_gpu_bevdet import BN_GAIN, _cams, _inputs, _pair, _t
from test_gpu_bevdet4d import _cams as _cams4d
from test_gpu_bevdet4d import _drive, _run as _run_drive

pytestmark = pytest.mark.gpu
TASKS = list(synth.CENTERPOINT_TASKS)
OFF = synth.label_offsets(TASKS)
STAGES = {"bdp_candidates_kernel", "bdp_select_kernel", "bdp_decode_kernel", "bdp_mask_kernel", "bdp_greedy_kernel",
          "bdp_emit_kernel"}


def _cfg(**over):
    from paddle3d_b200.bevdet import TEST_CFG_BEVDET
    return dict(TEST_CFG_BEVDET, **over)


def _heads(seed, tasks=TASKS, H=128, W=128, hm_mean=-5.5):
    h = synth.centerpoint_head_outputs(seed, tasks, H, W, hm_mean=hm_mean)
    h["hm"] = [(np.round(a * 64.0) / 64.0).astype(np.float32) for a in h["hm"]]
    return h


def _device(cuda, h, cfg, off=OFF):
    """The op's outputs as numpy: (boxes [K, 9], scores, labels, counts [T + 1]); the worst-case shapes are checked."""
    import torch
    from paddle3d_b200.ops import bevdet_postprocess as bdp
    ht = {k: [_t(cuda, a) for a in v] for k, v in h.items()}
    boxes, scores, labels, counts = bdp.bevdet_postprocess_heads(ht, cfg, off)
    torch.cuda.synchronize()
    c = counts.cpu().numpy()
    k = int(c[-1])
    assert c[:-1].sum() == k and boxes.shape == (len(h["hm"]) * cfg["post_max_size"], 9)
    return boxes[:k].cpu().numpy(), scores[:k].cpu().numpy(), labels[:k].cpu().numpy(), c


def _same(got, want, exact_dims=False):
    """Device rows against the oracle's: order, labels, counts and the transcendental-free columns bit for bit; scores,
    dims (the oracle's went through the multiply / divide round trip) and rot within a few ulp; z within ulps of dz."""
    gb, gs, gl, gc = got
    wb, ws, wl, wc = want
    assert np.array_equal(gc[:-1], wc), (gc, wc)
    assert np.array_equal(gl, wl)
    assert np.array_equal(gb[:, [0, 1, 7, 8]].view(np.int32), wb[:, [0, 1, 7, 8]].view(np.int32))
    np.testing.assert_allclose(gs, ws, rtol=1e-6)
    np.testing.assert_allclose(gb[:, 3:7], wb[:, 3:7], rtol=0 if exact_dims else 1e-6)
    np.testing.assert_allclose(gb[:, 2], wb[:, 2], rtol=1e-6, atol=1e-6 * float(max(1.0, np.abs(wb[:, 5]).max(initial=0))))


NO_NMS = dict(nms_type="rotate", nms_thr=2.0, nms_rescale_factor=1.0)   # an IoU never exceeds 2: rows = the selection


@pytest.mark.parametrize("hm_mean", [-5.5, -4.0])
@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_selection_and_kept_lists(cuda, oracle_mod, seed, hm_mean):
    """128 x 128 at the two heat-map statistics (the stress one pushes every task past max_num): the selected (class,
    cell) lists in order (the decode with suppression switched off), then the kept lists of the full config."""
    h = _heads(seed, hm_mean=hm_mean)
    sel = _cfg(**NO_NMS)
    got, want = _device(cuda, h, sel), bevdet_postprocess_ref(h, sel, OFF)
    n_cand = [int((a > np.log(0.1 / 0.9)).sum()) for a in h["hm"]]
    assert all(n > 500 for n in n_cand) if hm_mean == -4.0 else all(0 < n < 500 for n in n_cand), n_cand
    _same(got, want)
    assert got[3][-1] > 500
    got, want = _device(cuda, h, _cfg()), bevdet_postprocess_ref(h, _cfg(), OFF)
    _same(got, want)
    assert 0 < got[3][-1] < sum(min(n, 500) for n in n_cand)   # something was suppressed


def test_ties_at_the_cut(cuda, oracle_mod):
    """Three logit values only: thousands of equal scores straddle the top-K cut of every task."""
    rng = np.random.default_rng(5)
    h = _heads(9)
    h["hm"] = [rng.choice(np.asarray([-6.0, 0.5, 2.0], np.float32), size=a.shape, p=[0.9, 0.08, 0.02]) for a in h["hm"]]
    for cfg in (_cfg(**NO_NMS), _cfg(max_num=137, **NO_NMS), _cfg()):
        _same(_device(cuda, h, cfg), bevdet_postprocess_ref(h, cfg, OFF))


@pytest.mark.parametrize("n", [0, 1, 500, 501])
def test_candidate_counts_around_max_num(cuda, oracle_mod, n):
    """Exactly n candidates in every task (distinct logits at random (class, cell) pairs): none, one, max_num and one
    more, whose worst is cut."""
    h = _heads(11)
    rng = np.random.default_rng(n)
    for a in h["hm"]:
        a[...] = -20.0
        a.reshape(-1)[rng.choice(a.size, n, replace=False)] = (np.arange(n, dtype=np.float32) - 64.0) / 64.0
    cfg = _cfg(**NO_NMS)
    got = _device(cuda, h, cfg)
    assert got[3].tolist() == [min(n, 500)] * 6 + [6 * min(n, 500)]
    _same(got, bevdet_postprocess_ref(h, cfg, OFF))
    if n == 501:
        assert got[1].min() > 1 / (1 + np.exp(1.0)) * (1 + 1e-6)   # the logit -1 candidate is the one cut


def test_range_post_max_and_shapes(cuda, oracle_mod):
    """A task whose survivors all fail the range test gives no row; post_max_size below the kept count cuts the list;
    tasks of 1, 2 and 4 classes on a 100 x 88 map (no multiple of a block)."""
    h = _heads(2, hm_mean=-4.0)
    h["height"][2][...] = 10.5            # above the range's top
    h["reg"][4][0, 0] += 2000.0           # decoded x far outside
    got = _device(cuda, h, _cfg())
    assert got[3][2] == 0 and got[3][4] == 0 and got[3][0] > 0
    _same(got, bevdet_postprocess_ref(h, _cfg(), OFF))
    cfg = _cfg(post_max_size=5)
    got = _device(cuda, h, cfg)
    assert got[3].tolist() == [5, 5, 0, 5, 0, 5, 20]
    _same(got, bevdet_postprocess_ref(h, cfg, OFF))
    cfg = _cfg(pre_max_size=70)   # suppression among the first 70 survivors only
    _same(_device(cuda, h, cfg), bevdet_postprocess_ref(h, cfg, OFF))
    tasks, off = [1, 2, 4], [0, 1, 3]
    h = _heads(3, tasks, 100, 88, hm_mean=-4.0)
    for extra in (dict(NO_NMS, min_radius=1.0), dict(nms_type=["rotate", "circle", "rotate"], nms_thr=[0.2, 0.2, 0.3], min_radius=[1, 2.5, 1],
                               nms_rescale_factor=[1.0, [0.7, 1.3], [0.4, 0.55, 1.0, 4.5]])):
        cfg = _cfg(**extra)
        _same(_device(cuda, h, cfg, off), bevdet_postprocess_ref(h, cfg, off))


def test_factor_forms_and_plain_nms(cuda, oracle_mod):
    """A per-class list that repeats the scalar gives the same bytes; factor 1 and rotate everywhere keeps what p3d_nms
    keeps of the oracle's sorted boxes, with dims equal to the oracle's bit for bit (x 1 / 1 is exact)."""
    import torch
    from bevdet_postprocess_oracle import task_selection
    from paddle3d_b200.ops import iou3d_nms
    h = _heads(1, hm_mean=-4.0)
    a = _device(cuda, h, _cfg(nms_type="rotate", nms_rescale_factor=0.7))
    b = _device(cuda, h, _cfg(nms_type="rotate", nms_rescale_factor=[[0.7] * c for c in TASKS]))
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    cfg = _cfg(nms_type="rotate", nms_rescale_factor=1.0)
    got = _device(cuda, h, cfg)
    _same(got, bevdet_postprocess_ref(h, cfg, OFF))
    row = 0
    for t in range(len(TASKS)):
        boxes, _, cls, _ = task_selection(h["hm"][t], h["reg"][t], h["height"][t], h["dim"][t], h["vel"][t], h["rot"][t], cfg)
        keep, num = iou3d_nms.nms_gpu(_t(cuda, boxes[:, :7]), cfg["nms_thr"][t], device_outputs=True)
        torch.cuda.synchronize()
        keep = keep[:int(num)].cpu().numpy()[:cfg["post_max_size"]]
        assert got[3][t] == len(keep)
        rows = got[0][row:row + len(keep)]
        assert np.array_equal(rows[:, :2].view(np.int32), boxes[keep][:, :2].view(np.int32))
        assert np.array_equal(got[2][row:row + len(keep)], cls[keep] + OFF[t])
        row += len(keep)


def test_non_finite_inputs_are_data(cuda):
    """NaN and infinite logits and regressions: a NaN logit is no candidate, +inf scores 1.0, a NaN or infinite centre
    fails the range test and a box with any other non-finite value is dropped, so every row is finite with its centre
    inside the range."""
    h = _heads(4, hm_mean=-4.0)
    rng = np.random.default_rng(0)
    bad = np.asarray([np.nan, np.inf, -np.inf], np.float32)
    for name in ("hm", "reg", "height", "dim", "rot", "vel"):
        for a in h[name]:
            idx = rng.choice(a.size, a.size // 50, replace=False)
            a.reshape(-1)[idx] = rng.choice(bad, len(idx))
    for cfg in (_cfg(), _cfg(**NO_NMS)):
        boxes, scores, labels, counts = _device(cuda, h, cfg)
        assert counts[-1] > 0 and np.isfinite(scores).all() and (scores > 0.1).all() and (scores <= 1.0).all()
        assert np.isfinite(boxes).all() and (np.abs(boxes[:, :2]) <= np.float32(61.2)).all()
        assert labels.min() >= 0 and labels.max() <= 9
    assert (scores == 1.0).any()


_PROFILE = """
import json, sys
import numpy as np, torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, sys.argv[1])
from paddle3d_b200 import synth
from paddle3d_b200.bevdet import TEST_CFG_BEVDET
from paddle3d_b200.ops import bevdet_postprocess as bdp
h = synth.centerpoint_head_outputs(0, H=128, W=128, hm_mean=-4.0)
ht = {k: [torch.from_numpy(a).cuda() for a in v] for k, v in h.items()}
off = synth.label_offsets()
bdp.bevdet_postprocess_heads(ht, TEST_CFG_BEVDET, off)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    bdp.bevdet_postprocess_heads(ht, TEST_CFG_BEVDET, off)
    torch.cuda.synchronize()
print("KERNELS " + json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_every_stage_runs(cuda):
    """One call under torch.profiler: the six stages are seen by name (the stress map, so the radix select runs too).  In
    a process of its own: a profiler session here would precede the one test_gpu_camera_pool.py opens in this process."""
    import json
    import subprocess
    import sys
    from conftest import ROOT
    r = subprocess.run([sys.executable, "-c", _PROFILE, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][8:])
    if not names:
        pytest.skip("torch.profiler reported no CUDA kernels on this device")
    seen = {s for s in STAGES for n in names if s in n}
    assert seen == STAGES, (sorted(STAGES - seen), sorted(set(names)))


# ---------------------------------------------------------------------------------------------------- the frames
def _host_heads(hot):
    return {k: [t.cpu().numpy() for t in v] for k, v in hot.out["head"].items()}


@pytest.fixture(scope="module")
def frame(cuda):
    """test_gpu_bevdet's frame with BEVDet's own decode, and the same weights under CONFIG."""
    from paddle3d_b200.bevdet import CONFIG_BEVDET_NMS, BEVDet
    m = BEVDet(CONFIG_BEVDET_NMS, device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    rig = synth.camera_rig(31)
    logits, tran = _inputs(m, 7)
    m.calibrate_heatmap_bias(synth.lss_mats(rig), _t(cuda, logits), _t(cuda, tran))
    axes = tuple(a.numpy() for a in m.vt.axes_host)
    cpu = CpuBEVDetNMS(m.export_numpy(), m.test_cfg, m.label_off).run(_cams(rig), axes, logits, tran, *m.vt.grid_args())
    base = BEVDet(device=cuda)
    base.encoder, base.head = m.encoder, m.head
    return dict(m=m, base=base, rig=rig, logits=logits, tran=tran, cpu=cpu)


def test_frame_matches_cpu_arm(cuda, oracle_mod, frame):
    """The captured frame's rows equal the oracle's decode of the frame's own head planes (order and labels exactly) and
    pair with the CPU arm's boxes; the result slot holds 6 x 500 rows and is still copied once."""
    from paddle3d_b200.bevdet import BEVDetHotPath
    m, cpu = frame["m"], frame["cpu"]
    hot = BEVDetHotPath(m, device=cuda).capture(count_nodes=True)
    assert hot.slot.shape == (3000, 9, 7, 1) and hot.graph_nodes["memcpy"] >= 6
    got = [t.clone().numpy() for t in hot.infer(synth.lss_mats(frame["rig"]), _t(cuda, frame["logits"]),
                                                 _t(cuda, frame["tran"]))]
    r = bevdet_postprocess_ref(_host_heads(hot), m.test_cfg, m.label_off)
    assert len(got[0]) == len(r[0]) > 0 and np.array_equal(got[2], r[2])
    np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
    np.testing.assert_allclose(got[1], r[1], rtol=1e-6)
    assert abs(len(got[0]) - len(cpu["boxes"])) <= max(3, len(cpu["boxes"]) // 50)
    assert _pair(got, cpu) >= 0.95
    # the same node count as the frame with the Paddle op's decode, one kernel more (six stages against five)
    other = BEVDetHotPath(frame["base"], device=cuda).capture(count_nodes=True)
    assert hot.graph_nodes["kernel"] == other.graph_nodes["kernel"] + 1
    assert hot.graph_nodes["memcpy"] == other.graph_nodes["memcpy"]


def test_captured_eager_and_lanes(cuda, frame):
    """Captured == eager bit for bit on new calibrations; three lanes sharing the model == one lane."""
    import torch
    from paddle3d_b200.bevdet import BEVDetHotPath
    m = frame["m"]
    rigs = [synth.camera_rig(40 + i) for i in range(3)]
    ins = [[_t(cuda, a) for a in _inputs(m, 50 + i)] for i in range(3)]
    hot = BEVDetHotPath(m, device=cuda).capture()
    want = []
    for r, (tl, tt) in zip(rigs, ins):
        boxes, scores, labels, counts = m.forward(synth.lss_mats(r), tl, tt)
        k = int(counts[-1])
        got = [t.clone() for t in hot.infer(synth.lss_mats(r), tl, tt)]
        assert k > 0 and all(torch.equal(g, e.cpu()) for g, e in zip(got, (boxes[:k], scores[:k], labels[:k])))
        want.append(got)
    lanes = [BEVDetHotPath(m, device=cuda).capture() for _ in range(3)]
    for rep in range(2):
        for i, lane in enumerate(lanes):
            lane.launch(synth.lss_mats(rigs[i]), *ins[i])
        for i, lane in enumerate(lanes):
            assert all(torch.equal(g, w) for g, w in zip(lane.result(), want[i])), "lane %d" % i


def test_default_config_is_untouched(cuda, oracle_mod, frame):
    """With CONFIG the frame still ends in centerpoint_postprocess: its rows are the existing op's, called directly on the
    frame's head planes, bit for bit, in a 6 x 83-row slot; the two decodes differ on the same planes."""
    import torch
    from paddle3d_b200.bevdet import BEVDetHotPath
    from paddle3d_b200.ops import centerpoint_postprocess as cpp
    base = frame["base"]
    tc = base.test_cfg
    assert "nms_type" not in tc
    hot = BEVDetHotPath(base, device=cuda).capture()
    assert hot.slot.shape == (498, 9, 7, 1)
    got = [t.clone() for t in hot.infer(synth.lss_mats(frame["rig"]), _t(cuda, frame["logits"]), _t(cuda, frame["tran"]))]
    h = hot.out["head"]
    b, s, l = cpp.centerpoint_postprocess(h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], tc["voxel_size"],
                                          tc["point_cloud_range"], tc["post_center_limit_range"], base.label_off,
                                          tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
                                          tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
    assert len(b) > 0 and all(torch.equal(g, w.cpu()) for g, w in zip(got, (b, s, l)))
    hn = {k: [t.cpu().numpy() for t in v] for k, v in h.items()}
    r = oracle_mod.centerpoint_postprocess(hn["hm"], hn["reg"], hn["height"], hn["dim"], hn["vel"], hn["rot"],
                                           tc["voxel_size"], tc["point_cloud_range"], tc["post_center_limit_range"],
                                           base.label_off, tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
                                           tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
    assert np.array_equal(got[2].numpy(), r[2])
    np.testing.assert_allclose(got[0].numpy(), r[0], rtol=1e-5, atol=1e-5)


def test_bevdet4d_drive(cuda, oracle_mod):
    """A 3-frame BEVDet4D drive with BEVDet's own decode: every captured frame equals the oracle's decode of its own head
    planes and pairs with the CPU arm; captured == eager; three lanes on three drives == each drive alone."""
    import torch
    from paddle3d_b200.bevdet import CONFIG_4D_BEVDET_NMS, BEVDet4D, BEVDet4DHotPath
    m = BEVDet4D(CONFIG_4D_BEVDET_NMS, device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    frames = _drive(m, 31, 7)
    f0 = frames[0]
    m.calibrate_heatmap_bias(f0["mats"], _t(cuda, f0["logits"]), _t(cuda, f0["tran"]))
    axes = tuple(a.numpy() for a in m.vt.axes_host)
    arm = CpuBEVDet4DNMS(m.export_numpy(), m.test_cfg, m.label_off)
    hot = BEVDet4DHotPath(m, device=cuda).capture()
    assert hot.slot.shape == (3000, 9, 7, 1)
    feat_prev = None
    for k, f in enumerate(frames):
        tl, tt = _t(cuda, f["logits"]), _t(cuda, f["tran"])
        (boxes, scores, labels, counts), bev_feat = m.forward(f["mats"], f["prev"], tl, tt, feat_prev)
        n = int(counts[-1])
        got = [t.clone() for t in hot.infer(f["mats"], f["prev"], tl, tt, new_sequence=k == 0)]
        assert n > 0 and all(torch.equal(g, e.cpu()) for g, e in zip(got, (boxes[:n], scores[:n], labels[:n]))), k
        feat_prev = bev_feat
        got = [g.numpy() for g in got]
        r = bevdet_postprocess_ref(_host_heads(hot), m.test_cfg, m.label_off)
        assert len(got[0]) == len(r[0]) and np.array_equal(got[2], r[2]), k
        np.testing.assert_allclose(got[0], r[0], rtol=1e-5, atol=1e-5)
        c = arm.run(_cams4d(f["mats"]), axes, f["logits"], f["tran"], *m.vt.grid_args(), f["s2ke"], f["bda"],
                    s2ke_prev=f["prev"], new_sequence=k == 0)
        assert _pair(got, c) >= 0.95, k
    drives = [_drive(m, 40 + i, 50 + i, speed=6.0 + 3 * i, yaw_rate=0.1 * i) for i in range(3)]
    want = [_run_drive(hot, cuda, d) for d in drives]
    lanes = [BEVDet4DHotPath(m, device=cuda).capture() for _ in range(3)]
    for k in range(len(frames)):
        for lane, d in zip(lanes, drives):
            f = d[k]
            lane.launch(f["mats"], f["prev"], _t(cuda, f["logits"]), _t(cuda, f["tran"]), new_sequence=k == 0)
        for i, lane in enumerate(lanes):
            assert all(torch.equal(g, w) for g, w in zip(lane.result(), want[i][k])), (i, k)
