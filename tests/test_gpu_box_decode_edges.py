"""GPU: the LiDAR box decodes at their edges against the oracles.  p3d_centerpoint_postprocess against
oracle.centerpoint_postprocess, p3d_anchor_head_postprocess against oracle.pointpillars_multiclass, and p3d_nms (the
greedy pass nms_greedy_cta they share) against the known answers of tests/nms_chains.py.

Heat-map and class logits are multiples of 1/64 with |logit| <= 8: equal logits give equal scores on both sides and
order by the defined tie rule (ascending cell or anchor), different logits give scores many ulps apart, so the order
does not hang on the last bit of expf.  Compared bit for bit: counts, labels, order, the anchor mask, and every column
computed without a transcendental (cpp: x, y, z and vel; anchor head: x, y and the direction-fixed angle).  The cpp
centre is matched through the cell it decodes (_same_centres): the device, like the reference kernel under nvcc, fuses
the last multiply-add of (offset + cell) * down_ratio * voxel + range_min, and the oracle rounds the product first.
Scores and exp'd dims: rtol 1e-6."""
import numpy as np
import pytest

import nms_chains
import oracle.pointpillars_multiclass as ppm
from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu

F = np.float32
PCR = synth.C3["point_cloud_range"]
CPP_RANGE = synth.CENTERPOINT_TEST_CFG["post_center_limit_range"]
KEYS = ("hm", "reg", "height", "dim", "vel", "rot")
BG = -20.0                                   # a logit no threshold below lets through


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _q(a):
    """Logits on the 1/64 grid, |logit| <= 8 (non-finite values pass through)."""
    a = np.asarray(a, np.float64)
    with np.errstate(invalid="ignore"):
        return np.where(np.isfinite(a), np.clip(np.round(a * 64.0) / 64.0, -8.0, 8.0), a).astype(F)


# --------------------------------------------------------------------------- centerpoint_postprocess
def _heads(seed, tasks, H, W, p=0.02, with_vel=True):
    """Head outputs with a fraction p of cells scoring above 0.1 (logits in [-2.1, 8]) and the rest below it."""
    rng = np.random.default_rng(seed)
    h = {k: [] for k in KEYS}
    for c in tasks:
        shape = (1, c, H, W)
        h["hm"].append(_q(np.where(rng.random(shape) < p, rng.uniform(-2.1, 8, shape), rng.uniform(-8, -2.3, shape))))
        h["reg"].append(rng.uniform(0, 1, (1, 2, H, W)).astype(F))
        h["height"].append(rng.normal(-1, 1, (1, 1, H, W)).astype(F))
        h["dim"].append(rng.normal(0.5, 0.4, (1, 3, H, W)).astype(F))
        h["rot"].append(rng.normal(0, 1, (1, 2, H, W)).astype(F))
        h["vel"].append(rng.normal(0, 1, (1, 2, H, W)).astype(F) if with_vel else h["reg"][-1])
    return h


def _attrs(tasks, **over):
    cfg = synth.CENTERPOINT_TEST_CFG
    a = dict(voxel_size=[0.075, 0.075], point_cloud_range=PCR, post_center_range=CPP_RANGE,
             num_classes=synth.label_offsets(tasks), down_ratio=cfg["down_ratio"], score_threshold=cfg["score_threshold"],
             nms_iou_threshold=cfg["nms_iou_threshold"], nms_pre_max_size=cfg["nms_pre_max_size"],
             nms_post_max_size=cfg["nms_post_max_size"], with_velocity=True)
    a.update(over)
    return a


def _cpp_device(cuda, h, at):
    """(boxes [K, dims], scores, labels, rows per task) from the device; the worst-case output shapes are checked."""
    import torch
    from paddle3d_b200.ops import centerpoint_postprocess as cpp
    b, s, l, c = cpp.centerpoint_postprocess_device(*[[_t(cuda, a) for a in h[k]] for k in KEYS], **at)
    torch.cuda.synchronize()
    c = c.cpu().numpy()
    k = int(c[-1])
    T = len(h["hm"])
    assert c[:-1].sum() == k and b.shape == (T * max(at["nms_post_max_size"], 1), 9 if at["with_velocity"] else 7)
    return b[:k].cpu().numpy(), s[:k].cpu().numpy(), l[:k].cpu().numpy(), c[:-1]


def _same_cpp(got, want):
    gb, gs, gl, gc = got
    wb, ws, wl, wc = want
    assert np.array_equal(gc, wc), (gc, wc)
    assert np.array_equal(gl, wl)
    exact = [2, 6, 7] if gb.shape[1] == 9 else [2]
    assert np.array_equal(gb[:, exact].view(np.int32), wb[:, exact].view(np.int32))
    np.testing.assert_allclose(gs, ws, rtol=1e-6)
    np.testing.assert_allclose(gb[:, 3:6], wb[:, 3:6], rtol=1e-6)
    np.testing.assert_allclose(gb[:, -1], wb[:, -1], rtol=1e-6, atol=1e-6)


def _same_centres(h, at, got, want):
    """x, y bit for bit: each device row holds the fused decode fma((offset + cell) * down_ratio, voxel, range_min) of
    some cell of its task, and the oracle's row in the same place holds the plain decode of that same cell.  (The fused
    and plain results differ by an ulp of the product, which after the subtraction of the range can be hundreds of ulps
    of the centre.)  Fake rows (score -1) are zeros on both sides."""
    gb, gc, wb, ws = got[0], got[3], want[0], want[1]
    off = np.concatenate([[0], np.cumsum(gc)])
    for t in range(len(gc)):
        rows = np.arange(off[t], off[t + 1])
        rows = rows[ws[rows] != -1]
        reg = h["reg"][t][0]
        H, W = reg.shape[1:]
        cell = np.arange(H * W)
        fused, plain = [], []
        for k, idx in enumerate((cell % W, cell // W)):
            vs, pc = F(at["voxel_size"][k]), F(at["point_cloud_range"][k])
            with np.errstate(all="ignore"):
                b = (reg[k].reshape(-1) + idx.astype(F)) * F(at["down_ratio"])
                fused.append((b.astype(np.float64) * np.float64(vs) + np.float64(pc)).astype(F))  # exact sum, one rounding
                plain.append(b * vs + pc)
        key = lambda x, y: (x.view(np.uint32).astype(np.uint64) << np.uint64(32)) | y.view(np.uint32).astype(np.uint64)
        where = {int(k): c for c, k in enumerate(key(*fused))}
        cells = np.asarray([where.get(int(k), -1) for k in key(gb[rows, 0].copy(), gb[rows, 1].copy())], np.int64)
        assert (cells >= 0).all(), "task %d: a device centre is no cell's decode" % t
        for k in range(2):
            assert np.array_equal(plain[k][cells].view(np.int32), wb[rows, k].view(np.int32)), (t, k)


def _cpp_check(cuda, oracle_mod, h, **over):
    at = _attrs([a.shape[1] for a in h["hm"]], **over)
    got = _cpp_device(cuda, h, at)
    want = oracle_mod.centerpoint_postprocess(*[h[k] for k in KEYS], **at)
    _same_cpp(got, want)
    _same_centres(h, at, got, want)
    return got


def _place(h, t, n, seed, lo=8.0):
    """Exactly n candidates in task t: distinct logits lo, lo - 1/64, ... at n random cells, each in a random channel."""
    hm = h["hm"][t]
    C = hm.shape[1]
    hm[...] = BG
    rng = np.random.default_rng(seed)
    cells = rng.choice(hm.size // C, n, replace=False)
    hm.reshape(C, -1)[rng.integers(0, C, n), cells] = lo - np.arange(n, dtype=F) / 64.0


@pytest.mark.parametrize("pre,n", [(1000, 1), (1000, 63), (1000, 64), (1000, 65), (1000, 999), (1000, 1000),
                                   (1000, 1001), (64, 63), (64, 64), (64, 65), (65, 64), (65, 65), (65, 66),
                                   (100, 99), (100, 100), (100, 101)])
def test_cpp_candidate_counts(cuda, oracle_mod, pre, n):
    """Exactly n candidates per task around pre_max (the rank cut, 64-box words and 256-thread blocks)."""
    h = _heads(n, [1, 2], 180, 180)
    for t in range(2):
        _place(h, t, n, 10 * n + t)
    _cpp_check(cuda, oracle_mod, h, score_threshold=1e-4, nms_pre_max_size=pre)


def test_cpp_score_ties_at_the_cut(cuda, oracle_mod):
    """Three logit values only: thousands of equal scores straddle the pre_max cut (ascending cell wins), and the
    two-class tasks have cells whose channels tie."""
    rng = np.random.default_rng(5)
    h = _heads(9, synth.CENTERPOINT_TASKS, 180, 180)
    h["hm"] = [rng.choice(np.asarray([-6.0, 0.5, 2.0], F), size=a.shape, p=[0.9, 0.08, 0.02]) for a in h["hm"]]
    _cpp_check(cuda, oracle_mod, h)
    for pre in (1000, 137):
        assert (_cpp_check(cuda, oracle_mod, h, nms_pre_max_size=pre, nms_iou_threshold=2.0)[3] == 83).all()


def test_cpp_channel_ties(cuda, oracle_mod):
    """Equal logits in both channels of a cell: the first channel is the label.  Cells where channel 1 is larger keep
    label 1."""
    h = _heads(3, [2, 3], 32, 32)
    rng = np.random.default_rng(3)
    for t, hm in enumerate(h["hm"]):
        hm[...] = BG
        cells = rng.choice(32 * 32, 60, replace=False)
        v = 6.0 - np.arange(60, dtype=F) / 64.0
        hm[0, 0].reshape(-1)[cells] = v
        hm[0, 1].reshape(-1)[cells] = np.where(np.arange(60) % 3 == 0, v + 1 / 64.0, v)   # every third: channel 1 wins
        if t == 1:
            hm[0, 2].reshape(-1)[cells[::2]] = v[::2]                                      # three-way ties
    got = _cpp_check(cuda, oracle_mod, h, nms_iou_threshold=2.0)
    assert (got[3] == 60).all()
    lab = got[2] - np.repeat([0, 2], 60)
    assert (lab == 0).sum() == 80 and (lab == 1).sum() == 40


def test_cpp_empty_tasks_between(cuda, oracle_mod):
    """Tasks 0, 2 and 5 empty: one fake row each (zeros, score -1, label 0) at the right offsets."""
    h = _heads(4, synth.CENTERPOINT_TASKS, 128, 128, p=0.03)
    for t in (0, 2, 5):
        h["hm"][t][...] = BG
    for with_vel in (True, False):
        hv = dict(h, vel=h["vel"] if with_vel else h["reg"])
        b, s, l, c = _cpp_check(cuda, oracle_mod, hv, with_velocity=with_vel)
        assert c[0] == c[2] == c[5] == 1 and (c[[1, 3, 4]] > 1).all()
        off = np.concatenate([[0], np.cumsum(c)])
        for t in (0, 2, 5):
            r = off[t]
            assert s[r] == -1 and l[r] == 0 and not b[r].any()


@pytest.mark.parametrize("post", [0, 1, 64, 65, 83])
def test_cpp_post_max(cuda, oracle_mod, post):
    """post_max cuts, and the greedy pass's early exit: tasks 1 and 2 hold 128 and 129 boxes too small to overlap, so
    every box is kept and the kept count reaches 64 exactly at the end of the first tile."""
    h = _heads(6, [1, 2, 2], 64, 64, p=0.1)
    for t, n in ((1, 128), (2, 129)):
        _place(h, t, n, t)
        h["dim"][t][...] = -3.0                  # 5 cm boxes on cells 60 cm apart
        h["reg"][t][...] = 0.5
    got = _cpp_check(cuda, oracle_mod, h, nms_post_max_size=post)
    assert got[3][1] == got[3][2] == min(post, 128)


def _pair_heads(pairs, s=0.8):
    """A one-task head holding pairs of square boxes (side s) in the NMS frame: pair k is (row y_k, centre distance
    d_k along x, NMS heading th_k); the first box of a pair scores higher."""
    H, W = 3 * len(pairs) + 1, 4
    h = {k: [np.zeros((1, c, H, W), F)] for k, c in zip(KEYS, (1, 2, 1, 3, 2, 2))}
    h["hm"][0][...] = BG
    h["height"][0][...] = -1.0
    h["dim"][0][...] = np.log(F(s))
    for k, (d, th) in enumerate(pairs):
        ys = 3 * k + 1
        ang = -th - np.pi / 2                     # the NMS box is laid out with -rot - pi / 2
        for j, (xs, X) in enumerate(((0, 0.0), (3, d))):
            h["hm"][0][0, 0, ys, xs] = 4.0 - (2 * k + j) / 64.0
            h["reg"][0][0, 0, ys, xs] = X / 0.6 + 1.0 - xs           # centre x = (reg + xs) * 0.6 - 54
            h["reg"][0][0, 1, ys, xs] = 0.5
            h["rot"][0][0, :, ys, xs] = (np.sin(ang), np.cos(ang))
    return h


def test_cpp_iou_threshold_edges(cuda, oracle_mod):
    """IoU threshold 0 (any overlap suppresses) on pairs just inside and just outside touching distance, edge to edge
    and corner to corner, and at the distance where the tile's cheap reject starts; then thresholds 1 and 2, which
    keep every box.  The reject must be exact: the device equals the oracle's full polygon test."""
    s = 0.8
    diag = s * np.sqrt(2.0)
    reject = (diag + 0.1) * np.sqrt(1.001)
    pairs = [(s + g, 0.0) for g in (-0.05, -0.005, 0.005, 0.05)]
    pairs += [(diag + g, np.pi / 4) for g in (-0.05, -0.005, 0.005, 0.05)]
    pairs += [(reject * f, th) for f in (1 - 1e-4, 1 + 1e-4) for th in (0.0, np.pi / 4)]
    h = _pair_heads(pairs, s)
    got = _cpp_check(cuda, oracle_mod, h, nms_iou_threshold=0.0)
    assert len(pairs) + 2 <= got[3][0] <= 2 * len(pairs) - 4       # the overlapping pairs lose their second box
    for thr in (1.0, 2.0):
        assert _cpp_check(cuda, oracle_mod, h, nms_iou_threshold=thr)[3][0] == 2 * len(pairs)


def test_cpp_raw_offset_bounds(cuda, oracle_mod):
    """The range test on the raw offsets is inclusive: a value exactly on a bound passes, one ulp outside fails."""
    h = _heads(8, [1], 16, 16, p=0.0)
    hm, reg, z = h["hm"][0], h["reg"][0], h["height"][0]
    cell = 0
    for ch, plane, lo, hi in ((0, reg, CPP_RANGE[0], CPP_RANGE[3]), (1, reg, CPP_RANGE[1], CPP_RANGE[4]),
                              (0, z, CPP_RANGE[2], CPP_RANGE[5])):
        for v in (F(lo), F(hi), np.nextafter(F(lo), F(-np.inf)), np.nextafter(F(hi), F(np.inf))):
            hm.reshape(-1)[cell] = 5.0 - cell / 64.0
            plane[0, ch].reshape(-1)[cell] = v
            cell += 1
    assert _cpp_check(cuda, oracle_mod, h, nms_iou_threshold=2.0)[3][0] == 6


@pytest.mark.parametrize("with_vel", [True, False])
@pytest.mark.parametrize("H,W", [(1, 1), (7, 9), (17, 300), (128, 128), (180, 180)])
def test_cpp_shapes(cuda, oracle_mod, H, W, with_vel):
    """Map sizes below, across and at the 256-thread blocks; one task, and sixteen tasks of 1 to 4 channels."""
    for tasks in ([2], [1, 2, 3, 4] * 4):
        h = _heads(H * W + len(tasks), tasks, H, W, p=min(0.5, 150.0 / (H * W)), with_vel=with_vel)
        _cpp_check(cuda, oracle_mod, h, with_velocity=with_vel)


def test_cpp_non_finite_inputs(cuda, oracle_mod):
    """NaN and +-inf in the heat map (channel 0 and channel 1), the offsets, the height, the velocity and the angle;
    NaN in the dims.  A NaN in channel 0 gives a NaN score (no candidate); a NaN in a later channel is skipped by the
    first-channel-then-greater rule, as in the oracle."""
    h = _heads(12, [2, 2, 1], 64, 64, p=0.05)
    rng = np.random.default_rng(12)
    cand = [np.nonzero(a.max(1).reshape(-1) > -2.2)[0] for a in h["hm"]]
    for t, bad in ((0, np.nan), (1, np.inf), (2, -np.inf)):
        hw = 64 * 64
        c = rng.permutation(cand[t])
        h["hm"][t].reshape(-1)[c[:5]] = bad                          # channel 0 (or the only one)
        if h["hm"][t].shape[1] > 1:
            h["hm"][t].reshape(-1)[hw + c[5:10]] = bad               # channel 1
        for i, (k, off) in enumerate((("reg", 0), ("reg", hw), ("height", 0), ("vel", 0), ("vel", hw), ("rot", 0),
                                      ("rot", hw), ("dim", 0), ("dim", hw))):
            if k == "dim" and not np.isnan(bad):
                continue
            h[k][t].reshape(-1)[off + c[10 + 3 * i:13 + 3 * i]] = bad
    _cpp_check(cuda, oracle_mod, h)


def test_cpp_infinite_dims(cuda, oracle_mod):
    """+inf dims from exp overflow (dim logits of 100), near and among finite boxes: the IoU of an infinite box must be
    the same on both sides."""
    import torch
    from paddle3d_b200.ops import iou3d_nms
    h = _heads(13, [1, 2], 32, 32, p=0.3)
    rng = np.random.default_rng(13)
    for t in range(2):
        d = h["dim"][t].reshape(3, -1)
        d[rng.integers(0, 2, 40), rng.choice(32 * 32, 40, replace=False)] = 100.0
    b, s, l, c = _cpp_device(cuda, h, _attrs([1, 2]))
    assert np.isinf(b[:, 3:5]).any()
    nb = np.stack([b[:, 0], b[:, 1], b[:, 2], b[:, 4], b[:, 3], b[:, 5],
                   (-b[:, -1].astype(np.float64) - np.pi / 2).astype(F)], 1)
    dev = iou3d_nms.boxes_iou_bev_gpu(_t(cuda, nb), _t(cuda, nb)).cpu().numpy()
    torch.cuda.synchronize()
    want = oracle_mod.boxes_iou_bev(nb, nb)
    assert np.array_equal(dev > 0.2, want > 0.2), np.argwhere((dev > 0.2) != (want > 0.2))[:5]
    _cpp_check(cuda, oracle_mod, h)


def test_cpp_workspace_reuse(cuda, oracle_mod):
    """Back-to-back calls on one stream: calls made after a large one (about 3.7k candidates per task) equal the
    same calls made first, on a workspace filled with 0xff, so no stale workspace contents are read."""
    import torch
    from paddle3d_b200 import _lib, _mem
    small = [(_heads(20, [1, 2], 7, 9, p=0.4), dict(nms_pre_max_size=64)),
             (_heads(21, synth.CENTERPOINT_TASKS, 128, 128, p=0.02), dict()),
             (_heads(22, [2, 2, 1], 64, 64, p=0.1), dict(nms_pre_max_size=100, nms_post_max_size=65))]
    big = synth.centerpoint_head_outputs(1, hm_mean=-4.0)
    big["hm"] = [_q(a) for a in big["hm"]]
    L = _lib.lib()
    need = max(L.p3d_centerpoint_postprocess_workspace_bytes(len(h["hm"]), h["hm"][0].shape[2], h["hm"][0].shape[3],
                                                             o.get("nms_pre_max_size", 1000), 83) for h, o in small)
    st = torch.cuda.Stream(cuda)
    with torch.cuda.stream(st):
        _mem.workspace(need, cuda, "cpp").fill_(0xff)
        first = [_cpp_check(cuda, oracle_mod, h, **o) for h, o in small]
        _cpp_check(cuda, oracle_mod, big)
        again = [_cpp_device(cuda, h, _attrs([a.shape[1] for a in h["hm"]], **o)) for h, o in small]
    for a, b in zip(first, again):
        for x, y in zip(a, b):
            assert np.array_equal(x.view(np.uint8), y.view(np.uint8))


# --------------------------------------------------------------------------- anchor_head_postprocess
AHP_RANGE = [-100.0, -100.0, -10.0, 100.0, 100.0, 10.0]


def _ahp_case(seed, H=8, W=8, R=2, C=1, nx=32, ny=32, pillars=0.3, extent=40.0):
    """A hand-built head: anchors at random positions, random clamped corners on an nx x ny pillar grid, pillar coords
    covering a fraction of it (with duplicates)."""
    rng = np.random.default_rng(seed)
    A = H * W * R
    head = np.zeros((1, R * (C + 9), H, W), F)
    head[0, :R * C] = _q(rng.uniform(-8, 8, (R * C, H, W)))
    head[0, R * C:R * (C + 7)] = rng.normal(0, 0.3, (7 * R, H, W))
    head[0, R * (C + 7):] = _q(rng.normal(0, 1, (2 * R, H, W)))
    anchors = np.zeros((A, 7), F)
    anchors[:, :2] = rng.uniform(-extent, extent, (A, 2))
    anchors[:, 2:6] = (-1.78, 1.6, 3.9, 1.56)
    anchors[:, 6] = np.tile(np.asarray([0.0, np.pi / 2], F), A // 2 + 1)[:A]
    x = np.sort(rng.integers(0, nx, (A, 2)), 1)
    y = np.sort(rng.integers(0, ny, (A, 2)), 1)
    corners = np.stack([x[:, 0], y[:, 0], x[:, 1], y[:, 1]], 1).astype(np.int32)
    n = int(pillars * nx * ny)
    coords = np.zeros((n, 4), np.int32)
    coords[:, 2] = rng.integers(0, ny, n)
    coords[:, 3] = rng.integers(0, nx, n)
    return dict(head=head, anchors=anchors, corners=corners, coords=coords, grid=(nx, ny), C=C)


def _ahp_device(cuda, case, coords=None, num=None, **cfg):
    import torch
    from paddle3d_b200.ops import anchor_postprocess as ap
    coords = case["coords"] if coords is None else coords
    num = len(coords) if num is None else num
    A = len(case["anchors"])
    pre = cfg["nms_pre_max_size"]
    mask = torch.full((A,), 7, dtype=torch.uint8, device=cuda)
    sb = torch.empty((pre, 7), dtype=torch.float32, device=cuda)
    ss = torch.empty((pre,), dtype=torch.float32, device=cuda)
    ct = _t(cuda, coords) if len(coords) else torch.zeros((0, 4), dtype=torch.int32, device=cuda)
    b, s, l, c = ap.anchor_head_postprocess_device(
        _t(cuda, case["head"]), _t(cuda, case["anchors"]), _t(cuda, case["corners"]), ct,
        torch.tensor([num], dtype=torch.int32, device=cuda), case["grid"], AHP_RANGE, anchor_mask=mask,
        sorted_out=(sb, ss), num_classes=case["C"], **cfg)
    torch.cuda.synchronize()
    cand, k = [int(v) for v in c.cpu()]
    n = min(cand, pre)
    return dict(mask=mask.cpu().numpy(), candidates=cand, cand_boxes=sb[:n].cpu().numpy(),
                cand_scores=ss[:n].cpu().numpy(), boxes=b[:k].cpu().numpy(), scores=s[:k].cpu().numpy(),
                labels=l[:k].cpu().numpy())


AHP_CFG = dict(anchor_area_threshold=1, score_threshold=0.05, nms_iou_threshold=0.5, nms_pre_max_size=1000,
               nms_post_max_size=300)


def _ahp_check(cuda, case, valid=None, coords=None, num=None, **over):
    """Device against the oracle; valid: the pillar coords the oracle sees (default: the case's)."""
    cfg = dict(AHP_CFG, **over)
    got = _ahp_device(cuda, case, coords, num, **cfg)
    want = ppm.anchor_head_postprocess(case["head"], case["anchors"], case["corners"],
                                       case["coords"] if valid is None else valid, case["grid"], AHP_RANGE,
                                       cfg["anchor_area_threshold"], cfg["score_threshold"], cfg["nms_iou_threshold"],
                                       cfg["nms_pre_max_size"], cfg["nms_post_max_size"], num_classes=case["C"])
    assert np.array_equal(got["mask"], want["mask"].astype(np.uint8))
    assert got["candidates"] == want["candidates"] and len(got["boxes"]) == len(want["boxes"]), \
        (got["candidates"], want["candidates"], len(got["boxes"]), len(want["boxes"]))
    for gb, wb in ((got["cand_boxes"], want["cand_boxes"]), (got["boxes"], want["boxes"])):
        assert np.array_equal(gb[:, [0, 1, 6]].view(np.int32), wb[:, [0, 1, 6]].view(np.int32))
        np.testing.assert_allclose(gb[:, 3:6], wb[:, 3:6], rtol=1e-6)
        np.testing.assert_allclose(gb[:, 2], wb[:, 2], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(got["cand_scores"], want["cand_scores"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(got["scores"], want["scores"], rtol=1e-6, atol=0)
    assert np.array_equal(got["labels"], want["labels"])
    return got, want


@pytest.mark.parametrize("ny", [1, 5, 496])
@pytest.mark.parametrize("nx", [1, 31, 32, 33, 432])
def test_ahp_grids_and_pillars(cuda, nx, ny):
    """Pillar grids that reach the row scan's 32-lane carry and the column scan's partial blocks.  The coords hold
    duplicates (counted twice), out-of-grid rows (skipped) and, behind num_coords, in-grid garbage (never read)."""
    case = _ahp_case(nx * 1000 + ny, H=16, W=16, C=3, nx=nx, ny=ny, pillars=0.3)
    valid = case["coords"]
    rng = np.random.default_rng(ny)
    dup = valid[rng.integers(0, max(len(valid), 1), min(len(valid), 50))]
    out = np.zeros((8, 4), np.int32)
    out[:, 2:] = [[-1, 0], [ny, 0], [0, -1], [0, nx], [-5, -5], [ny + 3, nx + 3], [0, 1 << 20], [1 << 20, 0]]
    rows = np.concatenate([valid, dup, out])
    rows = rows[rng.permutation(len(rows))]
    garbage = np.zeros((40, 4), np.int32)
    garbage[:, 2] = rng.integers(0, ny, 40)
    garbage[:, 3] = rng.integers(0, nx, 40)
    inside = (rows[:, 2] >= 0) & (rows[:, 2] < ny) & (rows[:, 3] >= 0) & (rows[:, 3] < nx)
    for thr in (0, 1):
        got, want = _ahp_check(cuda, case, rows[inside], np.concatenate([rows, garbage]), len(rows),
                               anchor_area_threshold=thr)
        assert want["mask"].any() == (nx > 1 and ny > 1)


def test_ahp_no_pillars_and_thresholds(cuda):
    """coords_cap 0 (every area 0); an area equal to the threshold is masked out; score threshold 0 makes every
    unmasked anchor a candidate, sigmoid 0 (logit -200) included."""
    case = _ahp_case(3, H=16, W=16, C=3, nx=40, ny=40)
    empty = np.zeros((0, 4), np.int32)
    got, _ = _ahp_check(cuda, dict(case, coords=empty), anchor_area_threshold=0)
    assert got["mask"].sum() == 0 and got["candidates"] == 0
    got, _ = _ahp_check(cuda, dict(case, coords=empty), anchor_area_threshold=-1)
    assert got["mask"].all()
    areas = ppm.anchor_areas(case["coords"], case["corners"], case["grid"])
    thr = int(np.median(areas[areas > 0]))
    assert (areas == thr).any()
    _ahp_check(cuda, case, anchor_area_threshold=thr)
    zero = dict(case, head=case["head"].copy())
    cls = zero["head"][0, :2 * 3].reshape(-1)
    cls[np.random.default_rng(3).choice(cls.size, cls.size // 2, replace=False)] = -200.0
    cls[: cls.size // 4] = -200.0
    got, want = _ahp_check(cuda, zero, anchor_area_threshold=0, score_threshold=0.0)
    assert got["candidates"] == want["mask"].sum() and (want["cand_scores"] == 0).any()


def _exact_candidates(case, n, seed, lo=8.0):
    """Exactly n candidates: distinct logits lo, lo - 1/64, ... at n random anchors, each in a random class; every
    other logit is far below the threshold."""
    head = case["head"]
    R, C = head.shape[1] // (case["C"] + 9), case["C"]
    cls = head[0, :R * C].reshape(R, C, -1)
    cls[...] = BG
    rng = np.random.default_rng(seed)
    i = rng.choice(len(case["anchors"]), n, replace=False)
    cls[i % R, rng.integers(0, C, n), i // R] = lo - np.arange(n, dtype=F) / 64.0


@pytest.mark.parametrize("pre,n,post", [(64, 63, 64), (64, 64, 1), (64, 65, 65), (65, 64, 64), (65, 65, 300),
                                        (65, 66, 1), (1000, 999, 300), (1000, 1000, 65), (1000, 1001, 64)])
def test_ahp_counts_around_pre_and_post_max(cuda, pre, n, post):
    """Candidate counts around pre_max with post_max cuts, all anchors unmasked."""
    case = _ahp_case(pre * 7 + n, H=24, W=24, R=2, C=2, nx=8, ny=8, extent=25.0)
    _exact_candidates(case, n, n)
    got, want = _ahp_check(cuda, case, anchor_area_threshold=-1, score_threshold=1e-4, nms_pre_max_size=pre,
                           nms_post_max_size=post)
    assert got["candidates"] == n


@pytest.mark.parametrize("kept", [255, 256, 257, 513])
def test_ahp_emit_rounds(cuda, kept):
    """pre_max = post_max = 600 with `kept` boxes that never overlap: the emit's 256-row rounds, with range-filter
    failures in the first and second round."""
    case = _ahp_case(kept, H=24, W=24, R=1, C=1, nx=4, ny=4)
    A = len(case["anchors"])
    i = np.arange(A)
    case["anchors"][:, 0] = (i % 24) * 3.0 - 36.0
    case["anchors"][:, 1] = (i // 24) * 3.0 - 36.0
    case["anchors"][:, 3:5] = 1.0
    case["head"][0, 1:8] = 0.0                                       # box deltas 0: the anchors themselves
    _exact_candidates(case, kept, kept)
    order = np.argsort(-case["head"][0, 0].reshape(-1), kind="stable")
    fail = [r for r in (3, 100, 255, 256, 300, 511) if r < kept]
    zt = case["head"][0, 3].reshape(-1)
    zt[order[fail]] = 100.0                                          # z far above the range
    got, want = _ahp_check(cuda, case, anchor_area_threshold=-1, nms_pre_max_size=600, nms_post_max_size=600)
    assert len(want["keep"]) == kept and len(got["boxes"]) == kept - len(fail)


def test_ahp_ties(cuda):
    """Three logit values only (ties straddle the pre_max cut: ascending anchor), class ties (the lowest class), direction
    ties (0) and an angle of exactly 0 in the direction fix."""
    case = _ahp_case(17, H=32, W=32, R=2, C=3, nx=16, ny=16, extent=30.0)
    rng = np.random.default_rng(17)
    head = case["head"]
    head[0, :6] = rng.choice(np.asarray([-6.0, 0.5, 2.0], F), size=(6, 32, 32), p=[0.5, 0.35, 0.15])
    dirs = head[0, 6 + 14:].reshape(2, 2, -1)                      # cls 2 x 3 | box 7 x 2 | dir 2 x 2 planes
    dirs[:, 1, ::3] = dirs[:, 0, ::3]                               # direction ties
    box = head[0, 6:6 + 14].reshape(2, 7, -1)
    box[:, 6, ::2] = 0.0                                            # rt = 0 with anchor angle 0: theta exactly 0
    for pre in (1000, 300):
        got, want = _ahp_check(cuda, case, anchor_area_threshold=-1, nms_pre_max_size=pre)
        assert len(np.unique(want["cand_scores"])) <= 2 and (got["boxes"][:, 6] == F(np.pi)).any()


def test_ahp_nan_class(cuda):
    """A NaN logit in class 0, 1 or 2 of a three-class head: the anchor is no candidate, whichever class holds it."""
    case = _ahp_case(19, H=16, W=16, R=2, C=3, nx=16, ny=16)
    _exact_candidates(case, 300, 19)
    cls = case["head"][0, :6].reshape(2, 3, -1)
    score = cls.max(1)
    top = np.argwhere(score > 0)
    rng = np.random.default_rng(19)
    pick = top[rng.choice(len(top), 30, replace=False)]
    for j, (a, cell) in enumerate(pick):
        cls[a, j % 3, cell] = np.nan
    got, want = _ahp_check(cuda, case, anchor_area_threshold=-1)
    assert got["candidates"] == 270


def test_ahp_workspace_reuse(cuda):
    """Back-to-back calls on one stream: smaller calls after a large one (432 x 496 grid, pre_max 1000) equal the same
    calls made first on a workspace filled with 0xff."""
    import torch
    from paddle3d_b200 import _lib, _mem
    small = [(_ahp_case(30, H=8, W=8, C=3, nx=33, ny=5), dict(nms_pre_max_size=64, nms_post_max_size=65)),
             (_ahp_case(31, H=16, W=16, C=1, nx=31, ny=17), dict())]
    big = _ahp_case(32, H=64, W=64, C=3, nx=432, ny=496)
    L = _lib.lib()
    need = max(L.p3d_anchor_head_postprocess_workspace_bytes(len(c["anchors"]), *c["grid"], o.get("nms_pre_max_size", 1000))
               for c, o in small)
    st = torch.cuda.Stream(cuda)
    with torch.cuda.stream(st):
        _mem.workspace(need, cuda, "ahp").fill_(0xff)
        first = [_ahp_check(cuda, c, **o)[0] for c, o in small]
        _ahp_check(cuda, big, anchor_area_threshold=0)
        again = [_ahp_device(cuda, c, **dict(AHP_CFG, **o)) for c, o in small]
    for a, b in zip(first, again):
        for k in a:
            assert np.array_equal(np.asarray(a[k]), np.asarray(b[k])), k


# --------------------------------------------------------------------------- p3d_nms / nms_greedy_cta
SIZES = [64 * k + d for k in (1, 2, 3, 64, 781) for d in (-1, 0, 1)]


@pytest.mark.parametrize("normal", [False, True])
@pytest.mark.parametrize("n", SIZES)
def test_nms_known_answers(cuda, n, normal):
    """Chains (alternate boxes kept) crossing the 64-box words at both parities, all-disjoint boxes (all kept) and, up
    to 4097 boxes, all-identical ones (box 0 kept), through nms_gpu and nms_normal_gpu, up to a 313 MB mask."""
    from paddle3d_b200.ops import iou3d_nms
    fn = iou3d_nms.nms_normal_gpu if normal else iou3d_nms.nms_gpu
    cases = [nms_chains.chains(nms_chains.chain_lengths(n, n, p)) for p in (0, 1)] + [nms_chains.disjoint(n)]
    if n <= 4097:
        cases.append(nms_chains.identical(n))
    for boxes, want in cases:
        keep, num = fn(_t(cuda, boxes), nms_chains.THR)
        assert int(num[0]) == len(want)
        assert np.array_equal(keep.numpy()[:len(want)], want)
