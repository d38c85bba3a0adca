"""p3d_anchor3d_postprocess (BEVFusion's Anchor3DHead decode) at its edges, through
ops.anchor3d_postprocess.anchor3d_postprocess_device against bevfusion_oracle.anchor3d_decode_ref, whose per-class
NMS is oracle.nms: the nms_pre cut and its two key forms, the radix select's skipped digits, per-class lists across
the 64-box mask tiles, the greedy pass's stop at max_num, the max_num merge, an IoU exactly at the threshold,
non-finite boxes, the direction fix, and graph replay over heads with different candidate counts.

Inputs are built so that a case states its own answer: class logits are multiples of 1/64 with |logit| <= 8 (equal
logits give equal scores on both sides, different ones scores many ulps apart), and wherever the geometry matters the
box deltas are zero, so a decoded box is its anchor.  Each anchor carries its index in its velocity columns
(vx = index mod 2^20, vy = index >> 20), so an output row names the anchor it came from.  Compared bit for bit:
counts, labels, row order, x, y, vx, vy and the direction-fixed angle; z, w, l, h and the scores at rtol 1e-6 (they
pass through expf).  Every output buffer is poisoned (NaN, -1) and the rows from count to max_num must still hold
the poison.

The tests without the gpu mark check, on the oracle alone, the premise each hand-built GPU case relies on."""
import numpy as np
import pytest

import bevfusion_oracle as bo
import nms_chains
from test_gpu_bevfusion import _anchors, _compare, _run

F = np.float32
BG = -8.0                                    # sigmoid(-8) = 3.4e-4: below every score threshold used here
EXACT = [0, 1, 6, 7, 8]                      # x, y, r, vx, vy
CFG = dict(nms_pre=4096, score_thr=0.05, nms_thr=0.5, max_num=5000, dir_offset=0.7854, dir_limit_offset=0.0)


class Head:
    """A head for A = H * W * R anchors and C classes: every class logit BG, zero deltas and dir logits.  Anchor i is a
    1 x 1 x 1.5 box at heading 0 on a raster 2 m apart (no two overlap), carrying its index in (vx, vy)."""

    def __init__(self, A, C, R=1, H=1):
        HW = A // R
        assert HW * R == A and HW % H == 0
        self.A, self.C, self.R, self.H, self.W = A, C, R, H, HW // H
        self.flat = np.zeros((R * (C + 11), HW), F)
        self.flat[:R * C] = BG
        i = np.arange(A, dtype=np.int64)
        a = np.zeros((A, 9), F)
        a[:, 0] = (i % 1024) * 2.0
        a[:, 1] = (i // 1024) * 2.0
        a[:, 2] = -1.0
        a[:, 3:6] = (1.0, 1.0, 1.5)
        a[:, 7] = i & 0xfffff
        a[:, 8] = i >> 20
        self.anchors = a

    @property
    def planes(self):
        return self.flat.reshape(-1, self.H, self.W)

    def _set(self, base, K, i, k, v):
        i = np.asarray(i, np.int64)
        self.flat[base + (i % self.R) * K + np.asarray(k, np.int64), i // self.R] = v

    def cls(self, i, c, v):
        self._set(0, self.C, i, c, v)

    def reg(self, i, k, v):
        self._set(self.R * self.C, 9, i, k, v)

    def dir(self, i, d0, d1):
        self._set(self.R * (self.C + 9), 2, i, 0, d0)
        self._set(self.R * (self.C + 9), 2, i, 1, d1)

    def place(self, i, xy):
        """Move anchors i to the given (x, y) centres."""
        self.anchors[np.asarray(i, np.int64), :2] = xy

    def ref(self, cfg):
        return bo.anchor3d_decode_ref(self.planes, self.anchors, self.C, self.R, cfg["nms_pre"], cfg["score_thr"],
                                      cfg["nms_thr"], cfg["max_num"], cfg["dir_offset"], cfg["dir_limit_offset"],
                                      details=True)


def ids(boxes):
    """The anchor index each output row came from (zero velocity deltas)."""
    return boxes[:, 7].astype(np.int64) | (boxes[:, 8].astype(np.int64) << 20)


def _same(got, want):
    _compare(got, want)
    gb, wb = got[0], want[0]
    assert np.array_equal(gb[:, EXACT].view(np.int32), wb[:, EXACT].view(np.int32))
    np.testing.assert_allclose(gb[:, 3:6], wb[:, 3:6], rtol=1e-6, atol=0)


def _check(cuda, h, cfg, fill=None):
    """The op into poisoned buffers against the restatement; fill: a byte the workspace is filled with first (1 MB more
    of it than the call needs).  Returns (device rows, restatement rows + details)."""
    import torch
    from paddle3d_b200 import _lib, _mem
    M = cfg["max_num"]
    out = (torch.full((M, 9), float("nan"), device=cuda), torch.full((M,), float("nan"), device=cuda),
           torch.full((M,), -1, dtype=torch.int64, device=cuda), torch.full((1,), -1, dtype=torch.int32, device=cuda))
    if fill is not None:
        need = _lib.lib().p3d_anchor3d_postprocess_workspace_bytes(h.H, h.W, h.R, h.C, cfg["nms_pre"], M)
        _mem.workspace(need + (1 << 20), cuda, "a3d").fill_(fill)
    res, got = _run(cuda, h.planes, h.anchors, h.C, h.R, cfg, out=out)
    want = h.ref(cfg)
    _same(got, want[:3])
    _untouched(res, len(got[0]))
    return got, want


def _untouched(res, k):
    b, s, l, c = [t.cpu().numpy() for t in res]
    assert int(c[0]) == k
    assert np.isnan(b[k:]).all() and np.isnan(s[k:]).all() and (l[k:] == -1).all(), "a row past count was written"


def _rows(got):
    """(anchor index, label) per output row."""
    return list(zip(ids(got[0]).tolist(), got[2].tolist()))


# ---------------------------------------------------------------------------------------- 1. the cut and the key form
PRES = [1, 63, 64, 65, 1000, 4096]


def _cut_case(pre, n):
    """A > pre anchors (R = 3, C = 3), exactly n candidates at random anchors, each in a random class, logits in groups
    of 8 equal values.  Returns (head, expected rows: the top pre candidates by (score, index), class-major)."""
    R, C = 3, 3
    A = R * -(-(2 * pre + 37) // R)
    h = Head(A, C, R)
    rng = np.random.default_rng(pre * 10 + n)
    cand = rng.choice(A, n, replace=False)
    logit = 6.0 - (np.arange(n) // 8) / 64.0
    cls = rng.integers(0, C, n)
    h.cls(cand, cls, logit)
    top = np.lexsort((cand, -logit))[:pre]
    want = []
    for c in range(C):
        t = top[cls[top] == c]
        t = t[np.lexsort((cand[t], -logit[t]))]
        want += [(int(cand[k]), c) for k in t]
    return h, want


@pytest.mark.gpu
@pytest.mark.parametrize("d", [-1, 0, 1])
@pytest.mark.parametrize("pre", PRES)
def test_cut_candidate_counts(cuda, oracle_mod, pre, d):
    """nms_pre - 1, nms_pre and nms_pre + 1 candidates with A > nms_pre: the first two keep every candidate, the last
    runs the radix select and drops the lowest (score, index)."""
    h, want = _cut_case(pre, pre + d)
    got, _ = _check(cuda, h, dict(CFG, nms_pre=pre, max_num=pre + 1))
    assert _rows(got) == want


def _key_form_case(pre):
    """A = pre + 1 anchors (4096 for pre = 4096, the largest nms_pre the op takes), C = 3.  Anchors 0 and A - 1 are the
    same box and tie in class 0 (logit 1); anchor A - 1 also scores 2 in class 1, so in score order it comes first and
    in anchor order last.  The anchors between score 0.5 in class 2.  Returns (head, {nms_pre: expected (anchor, label)
    rows})."""
    A = min(pre + 1, 4096)
    h = Head(A, 3)
    j = A - 1
    h.cls(0, 0, 1.0)
    h.cls(j, 0, 1.0)
    h.cls(j, 1, 2.0)
    h.anchors[j, :7] = h.anchors[0, :7]
    h.cls(np.arange(1, j), 2, 0.5)
    want = {A: [(0, 0), (j, 1)] + [(i, 2) for i in range(1, A - 1)],          # anchor order: 0 first in class 0
            A - 1: [(j, 0), (j, 1)] + [(i, 2) for i in range(1, A - 2)]}      # score order: A - 1 first, A - 2 cut
    return h, want


@pytest.mark.gpu
@pytest.mark.parametrize("pre", PRES)
def test_cut_key_form(cuda, oracle_mod, pre):
    """A == nms_pre keeps anchors in anchor order, A == nms_pre + 1 in score order: on one grid the class-0 survivor
    of a tied, overlapping pair is anchor 0 on one side of the boundary and anchor A - 1 on the other."""
    h, want = _key_form_case(pre)
    for p, rows in want.items():
        got, _ = _check(cuda, h, dict(CFG, nms_pre=p, max_num=h.A + 1))
        assert _rows(got) == rows, p


def test_key_form_premise(oracle_mod):
    for pre in PRES:
        h, want = _key_form_case(pre)
        for p, rows in want.items():
            got = h.ref(dict(CFG, nms_pre=p, max_num=h.A + 1))
            assert _rows(got) == rows
        assert want[h.A][0] != want[h.A - 1][0]


def test_cut_case_premise(oracle_mod):
    for pre in PRES[:5]:
        for d in (-1, 0, 1):
            h, want = _cut_case(pre, pre + d)
            got = h.ref(dict(CFG, nms_pre=pre, max_num=pre + 1))
            assert _rows(got) == want and len(want) == min(pre, pre + d)


# ------------------------------------------------------------------------------------------------- 2. radix digits
RADIX = [255, 257, 65535, 65537, (1 << 24) + 1]


def _radix_case(am1):
    """A = am1 + 1 anchors, R = C = 1; candidates S (more than nms_pre = |S| - 1) all with one logit, among them the
    two highest anchors, so the k-th key (anchor A - 2) has a non-zero digit in the highest low digit the select must
    not skip.  Returns (head, nms_pre, S)."""
    A = am1 + 1
    h = Head(A, 1, H=2 if A > 1 << 20 else 1)
    if A < 4000:
        S = np.setdiff1d(np.arange(A), [3, 40, 100, 128, 200, 250])
    else:
        rng = np.random.default_rng(am1)
        half = 1 << (am1.bit_length() - 1)
        S = np.unique(np.concatenate([rng.choice(A - 2, 3000, replace=False), [0, 1, half - 1, A - 2, A - 1]]))
    h.cls(S, 0, 1.0)
    return h, len(S) - 1, S


def _low_bits(A):
    lb = 1
    while lb < 32 and (A - 1) >> lb:
        lb += 1
    return lb


@pytest.mark.gpu
@pytest.mark.parametrize("am1", RADIX, ids=["2^8-1", "2^8+1", "2^16-1", "2^16+1", "2^24+1"])
def test_radix_select_low_digits(cuda, oracle_mod, am1):
    """Equal scores, more candidates than nms_pre, on both sides of a low_bits boundary: the kept set is the nms_pre
    lowest candidate anchors in index order.  The workspace is zeroed first: 0 is the smallest key, so a scratch slot
    the select ranks without having written it shows as a wrong row.  The A - 1 = 2^24 + 1 case holds 16.8 M anchors
    (1.4 GB on the device)."""
    h, pre, S = _radix_case(am1)
    got, want = _check(cuda, h, dict(CFG, nms_pre=pre, max_num=pre), fill=0)
    assert np.array_equal(want[3]["kept"], S[:pre])
    assert np.array_equal(ids(got[0]), S[:pre])


def test_radix_premise():
    for am1 in RADIX[:4]:
        h, pre, S = _radix_case(am1)
        A, lb = am1 + 1, _low_bits(am1 + 1)
        assert len(S) == pre + 1 <= 4097 and A > pre
        top = (lb - 1) // 8 * 8                       # the highest digit below bit 32 the select reads
        kth = int(S[pre - 1])
        assert kth == A - 2 and (kth >> top) & 255, (am1, kth, top)
        assert S[0] < 1 << (lb - 1) <= S[-1]          # candidates on both sides of the top bit
        cls = bo.split_head(h.planes, 1, 1)[0][:, 0]
        assert np.count_nonzero(cls == 1.0) == len(S) and np.all(cls[np.setdiff1d(np.arange(A), S)] == BG)
    assert _low_bits((1 << 24) + 2) == 25


# ------------------------------------------------------------------------------------------------- 3. NaN at the cut
@pytest.mark.gpu
@pytest.mark.parametrize("n_nan", [150, 99])
def test_nan_at_the_cut(cuda, oracle_mod, n_nan):
    """NaN-scored anchors take kept slots first.  With more of them than nms_pre = 100 no row comes out though 200
    finite candidates exist; with nms_pre - 1 of them the one slot left goes to the best finite candidate."""
    h = Head(600, 3, R=2)
    rng = np.random.default_rng(n_nan)
    perm = rng.permutation(600)
    nan, fin = perm[:n_nan], perm[n_nan:n_nan + 200]
    h.cls(nan, np.arange(n_nan) % 3, np.nan)                # the NaN in any of the three classes
    logit = 4.0 - np.arange(200) / 64.0
    h.cls(fin, rng.integers(0, 3, 200), logit)
    got, want = _check(cuda, h, dict(CFG, nms_pre=100, max_num=50))
    assert np.isnan(bo.sigmoid32(bo.split_head(h.planes, 3, 2)[0]).max(1)).sum() == n_nan
    if n_nan > 100:
        assert len(got[0]) == 0
    else:
        assert ids(got[0]).tolist() == [int(fin[0])]


# ---------------------------------------------------------------------------------- 4. per-class lists across tiles
CHAIN_N = [1, 63, 64, 65, 127, 128, 129, 4096]


def _chain_case(n):
    """C = 64, R = 2, nms_pre = 4096.  Class 37 holds n boxes laid out as nms_chains chains in anchor order, all with
    one logit (so class order = kept order = anchor order); class 0 holds 70 more chain boxes with a lower logit, on
    anchors after them (cut away when n = 4096); every third class-37 box also scores in class 63.  Classes between are
    empty.  Returns (head, {class: expected surviving anchors})."""
    lens = nms_chains.chain_lengths(n, n, n % 2)
    boxes, keep = nms_chains.chains(lens)
    b0, k0 = nms_chains.chains(nms_chains.chain_lengths(70, 7, 1))
    A = 2 * ((n + 70) // 2 + 40)
    h = Head(A, 64, R=2)
    i37 = np.arange(n)
    i0 = n + np.arange(70)
    h.place(i37, boxes[:, :2])
    h.place(i0, b0[:, :2])
    h.cls(i37, 37, 3.0)
    h.cls(i0, 0, 2.0)
    i63 = i37[::3]
    h.cls(i63, 63, 1.0)
    want = {37: i37[keep], 0: i0[k0] if n < 4096 else i0[:0], 63: i63}
    return h, want


@pytest.mark.gpu
@pytest.mark.parametrize("n", CHAIN_N)
def test_class_lists_across_tiles(cuda, oracle_mod, n):
    """One class holds 1 to 4096 boxes whose suppression crosses the 64-box mask words; 64 classes with empty classes
    between the populated ones.  The survivors are the chains' known answers."""
    h, want = _chain_case(n)
    got, _ = _check(cuda, h, dict(CFG, nms_thr=nms_chains.THR, max_num=8192))
    rows = _rows(got)
    for c in range(64):
        assert [i for i, l in rows if l == c] == want.get(c, np.zeros(0)).tolist(), c


def test_chain_premise(oracle_mod):
    """The chains give the stated survivors under oracle.nms, and cross a 64-box word boundary from 65 boxes up."""
    for n in CHAIN_N:
        lens = nms_chains.chain_lengths(n, n, n % 2)
        boxes, keep = nms_chains.chains(lens)
        if n <= 129:
            k, nk = oracle_mod.nms(boxes, nms_chains.THR)
            assert np.array_equal(k[:nk], keep)
        if n > 64:
            ends = np.cumsum(lens)
            assert any(e - L < 64 * m <= e - 1 for e, L in zip(ends, lens) for m in range(1, n // 64 + 1))
    h, want = _chain_case(129)
    rows = _rows(h.ref(dict(CFG, nms_thr=nms_chains.THR, max_num=8192)))
    for c in (0, 37, 63):
        assert [i for i, l in rows if l == c] == want[c].tolist()


# ------------------------------------------------------------------------------------- 5. the greedy pass's stop
def _greedy_case(beside):
    """C = 4.  Class 1 holds 300 chain boxes (150 survivors) with logit 2.  Beside: class 2 with 10 boxes at logit 6
    (higher), class 0 with 5 at logit 2 (equal: before class 1 in class-major order) and class 3 with 8 at logit -1
    (lower), all apart.  Returns (head, every survivor in output order)."""
    b1, k1 = nms_chains.chains(nms_chains.chain_lengths(300, 11, 1))
    h = Head(400, 4)
    i1 = np.arange(300)
    h.place(i1, b1[:, :2] + (0.0, 1000.0))
    h.cls(i1, 1, 2.0)
    order = i1[k1]
    if beside:
        groups = ((2, 6.0, 300 + np.arange(10)), (0, 2.0, 310 + np.arange(5)), (3, -1.0, 315 + np.arange(8)))
        for c, v, i in groups:
            h.cls(i, c, v)
        order = np.concatenate([groups[0][2], groups[1][2], order, groups[2][2]])
    return h, order


@pytest.mark.gpu
@pytest.mark.parametrize("beside", [False, True])
@pytest.mark.parametrize("max_num", [1, 63, 64, 65])
def test_greedy_stop_at_max_num(cuda, oracle_mod, max_num, beside):
    """A class with more survivors than max_num: alone, the total after the per-class cap is exactly max_num (rows in
    class order); beside higher, equal and lower classes, the rank count orders them with ties class-major.  Run on a
    workspace filled with 0x00 and with 0xff: no unwritten workspace word is read."""
    h, order = _greedy_case(beside)
    for fill in (0x00, 0xff):
        got, _ = _check(cuda, h, dict(CFG, nms_thr=nms_chains.THR, max_num=max_num), fill=fill)
        assert ids(got[0]).tolist() == order[:max_num].tolist()


# -------------------------------------------------------------------------------------------- 6. the max_num merge
def _merge_case(layout, d, max_num=100):
    """Survivors in total max_num + d.  spread: class 4 (logit 5) 26 + d boxes, class 0 and class 2 (logit 3, tied
    across classes) 30 and 44; single: class 1 alone with max_num + d.  Returns (head, expected anchors in order)."""
    h = Head(256, 5)
    if layout == "single":
        i = np.arange(max_num + d)
        h.cls(i, 1, 1.5)
        return h, i[:max_num]
    groups = ((0, 3.0, np.arange(30)), (2, 3.0, 30 + np.arange(44)), (4, 5.0, 74 + np.arange(26 + d)))
    for c, v, i in groups:
        h.cls(i, c, v)
    if d <= 0:                                             # class-major
        return h, np.concatenate([g[2] for g in groups])
    return h, np.concatenate([groups[2][2], groups[0][2], groups[1][2]])[:max_num]   # score order, ties class-major


@pytest.mark.gpu
@pytest.mark.parametrize("d", [-1, 0, 1])
@pytest.mark.parametrize("layout", ["spread", "single"])
def test_merge_counts(cuda, oracle_mod, layout, d):
    """max_num - 1 and max_num survivors come out in class-major order; max_num + 1 in score order with ties across
    classes in class order.  A single class of max_num + 1 is capped to max_num and comes out in its own order."""
    h, want = _merge_case(layout, d)
    got, _ = _check(cuda, h, dict(CFG, max_num=100))
    assert ids(got[0]).tolist() == want.tolist()


def test_merge_premise(oracle_mod):
    for layout in ("spread", "single"):
        for d in (-1, 0, 1):
            h, want = _merge_case(layout, d)
            assert ids(h.ref(dict(CFG, max_num=100))[0]).tolist() == want.tolist()


# ---------------------------------------------------------------------------------------- 7. IoU at the threshold
# (dx, dy) of each pair: IoU 0.75 / 1.25, touching edges, touching corners, IoU 0.125 / 1.875
PAIRS = [(0.25, 0.0), (1.0, 0.0), (1.0, 1.0), (0.875, 0.0)]
T06 = F(0.6)


def _threshold_case():
    """C = 1: pair k is two unit squares (dx, dy) apart, the first scoring higher.  Returns (head, first, second)."""
    h = Head(16, 1)
    first, second = np.arange(len(PAIRS)) * 2, np.arange(len(PAIRS)) * 2 + 1
    for k, (dx, dy) in enumerate(PAIRS):
        h.place([first[k], second[k]], [(0.0, 8.0 * k), (dx, 8.0 * k + dy)])
    h.cls(first, 0, 2.0)
    h.cls(second, 0, 1.0)
    return h, first, second


THR_CASES = [(T06, []), (np.nextafter(T06, F(0)), [0]), (F(0), [0, 3])]   # (nms_thr, pairs whose second box goes)


@pytest.mark.gpu
def test_iou_at_the_threshold(cuda, oracle_mod):
    """An IoU equal to nms_thr does not suppress (the test is >); one ulp lower it does.  At nms_thr = 0 touching boxes
    (edge or corner) are kept and overlapping ones suppressed."""
    h, first, second = _threshold_case()
    for thr, gone in THR_CASES:
        got, _ = _check(cuda, h, dict(CFG, nms_thr=thr))
        want = sorted(first.tolist() + [int(s) for k, s in enumerate(second) if k not in gone])
        assert sorted(ids(got[0]).tolist()) == want, thr


def test_threshold_premise(oracle_mod):
    """The pairs' IoUs under oracle.boxes_iou_bev, and oracle.nms's decisions at each threshold."""
    h, first, second = _threshold_case()
    b = h.anchors[:, :7]
    iou = [float(oracle_mod.boxes_iou_bev(b[[f]], b[[s]])[0, 0]) for f, s in zip(first, second)]
    assert F(iou[0]) == T06 and iou[1] == 0.0 and iou[2] == 0.0 and 0 < iou[3] < 0.1
    for thr, gone in THR_CASES:
        for k, (f, s) in enumerate(zip(first, second)):
            keep, nk = oracle_mod.nms(b[[f, s]], float(thr))
            assert nk == (1 if k in gone else 2), (thr, k)


# --------------------------------------------------------------------------------------------- 8. non-finite boxes
def _non_finite_case():
    """C = 2, R = 2.  Each special anchor sits 0.25 m from an ordinary neighbour of its class (IoU 0.6) in a group 4 m
    from the next: NaN and +-inf in each of the nine deltas, a dim delta of 100 (expf overflows), an inf anchor x, y and
    w.  The special scores higher than its neighbour, so were it kept it would suppress it.  Dir logits tie, hold a NaN
    in either bin, or differ.  Returns (head, dropped specials, zero-dim specials, neighbours).  A -inf dim delta gives
    a zero w, l or h: the first two overlap nothing in BEV, the third (h = 0) is a unit square in BEV and suppresses its
    neighbour, the last in the list."""
    specials = [(k, v) for k in range(9) for v in (np.nan, np.inf, -np.inf)]
    specials += [(k, 100.0) for k in (3, 4, 5)] + [("anchor", k) for k in (0, 1, 3)]
    n = len(specials)
    h = Head(4 * n, 2, R=2)
    s, nb = np.arange(n) * 2, np.arange(n) * 2 + 1
    for g in range(n):
        h.place([s[g], nb[g]], [(4.0 * g, 0.0), (4.0 * g + 0.25, 0.0)])
    cls = np.arange(n) % 2
    h.cls(s, cls, 3.0)
    h.cls(nb, cls, 2.0 - (np.arange(n) % 3) / 64.0)
    dirs = [(0.5, 0.5), (np.nan, 0.0), (0.0, np.nan), (0.0, 1.0), (1.0, 0.0)]
    for i in range(4 * n):
        h.dir(i, *dirs[i % len(dirs)])
    zero, dropped = [], []
    for g, (k, v) in enumerate(specials):
        if k == "anchor":
            h.anchors[s[g], v] = np.inf
        else:
            h.reg(s[g], k, v)
        (zero if k in (3, 4, 5) and v == -np.inf else dropped).append(int(s[g]))
    return h, dropped, zero, nb


@pytest.mark.gpu
def test_non_finite_boxes(cuda, oracle_mod):
    """Every box with a non-finite value is dropped and its neighbour survives; a -inf dim delta decodes to a finite
    zero-size box, which is kept, and whose IoU with its neighbour is the oracle's."""
    h, dropped, zero, nb = _non_finite_case()
    got, _ = _check(cuda, h, dict(CFG, nms_thr=0.5))
    out = set(ids(got[0]).tolist())
    assert not out & set(dropped)
    assert set(zero) <= out and set(nb.tolist()) - out == {zero[-1] + 1}
    assert (got[0][:, 3:6] == 0).sum() == 3


def test_non_finite_premise(oracle_mod):
    h, dropped, zero, nb = _non_finite_case()
    _, reg, _ = bo.split_head(h.planes, 2, 2)
    box = bo.decode32(reg, h.anchors)
    fin = np.isfinite(box).all(1)
    assert not fin[dropped].any() and fin[zero].all() and fin[nb].all()
    assert (box[zero, 3:6] == 0).sum() == 3
    iou = [oracle_mod.boxes_iou_bev(box[[a], :7], box[[a + 1], :7])[0, 0] for a in zero]
    assert box[zero[-1], 5] == 0 and iou == [0.0, 0.0, T06]   # w = 0, l = 0: no overlap; h = 0: a unit square in BEV


# ------------------------------------------------------------------------------------------------ 9. the angle fix
def _angle_case(off=F(0.7854)):
    """C = 1, apart boxes at heading 0 whose angle delta rt makes r - dir_offset hit a target v exactly: multiples of
    fp32 pi and one ulp either side (at 0: +-2^-24, the nearest r - dir_offset can get), negative angles, r = 0 and |r|
    near 100.  Dir bins alternate.  Returns (head, targets)."""
    t = []
    for k in range(-4, 5):
        m = F(F(k) * bo.PI32)
        t += [m, np.nextafter(m, F(-np.inf)), np.nextafter(m, F(np.inf))] if k else [m, F(2 ** -24), F(-2 ** -24)]
    t += [F(v) for v in (-0.3, -2.0, -5.5, 1.5, 99.9, -99.9, 100.37, -100.37)] + [-off]
    t = np.asarray(t, F)
    h = Head(2 * len(t), 1)
    i = np.arange(len(t))
    h.cls(i, 0, 1.0)
    for j, v in enumerate(t):
        rt = F(v + off)
        for _ in range(8):                                # nudge rt until fp32(rt - off) == v
            d = F(rt - off)
            if d == v:
                break
            rt = np.nextafter(rt, F(np.inf) if d < v else F(-np.inf))
        h.reg(j, 6, rt)
        h.dir(j, 0.0, 1.0) if j % 2 else h.dir(j, 0.0, 0.0)
    return h, t


@pytest.mark.gpu
@pytest.mark.parametrize("lim", [0.0, 0.5, 1.0])
def test_angle_fix(cuda, oracle_mod, lim):
    """r - dir_offset at multiples of fp32 pi and one ulp off, negative, and near +-100: the fixed angle is bit-equal to
    limit_period32(r - dir_offset, dir_limit_offset) + dir_offset + pi * dir."""
    h, t = _angle_case()
    got, _ = _check(cuda, h, dict(CFG, dir_limit_offset=lim))
    i = ids(got[0])
    assert np.array_equal(np.sort(i), np.arange(len(t)))
    off = F(CFG["dir_offset"])
    want = (bo.limit_period32(t[i], lim) + off).astype(F) + (bo.PI32 * (i % 2).astype(F)).astype(F)
    assert np.array_equal(got[0][:, 6].view(np.int32), want.astype(F).view(np.int32))


def test_angle_premise():
    h, t = _angle_case()
    _, reg, _ = bo.split_head(h.planes, 1, 1)
    v = (reg[:len(t), 6] - F(0.7854)).astype(F)
    assert np.array_equal(v.view(np.int32), t.view(np.int32))
    assert len(np.unique(t)) == len(t)


# ---------------------------------------------------------------------------------------- 10. sync-free replay
def _random_head(rng, H, W, C, R, frac):
    """1/64-grid class logits with a fraction frac above the threshold, small deltas, dir logits with ties."""
    q = rng.integers(-512, -200, (R * C, H, W))
    hot = rng.random((R * C, H, W)) < frac
    q[hot] = rng.integers(-150, 512, int(hot.sum()))
    head = np.zeros((R * (C + 11), H, W), F)
    head[:R * C] = q / 64.0
    head[R * C:R * (C + 9)] = rng.normal(0, 0.3, (R * 9, H, W))
    head[R * (C + 9):] = rng.integers(-2, 3, (R * 2, H, W)) / 2.0
    return head


@pytest.mark.gpu
def test_graph_replay_over_candidate_counts(cuda, oracle_mod):
    """The op captured once in a CUDA graph, replayed over heads with 0 candidates, fewer survivors than max_num and
    more: each replay equals the restatement and leaves the rows past its count alone.  Then one eager call on the
    workspace grown by a larger configuration."""
    import torch
    from paddle3d_b200.ops.anchor3d_postprocess import anchor3d_postprocess_device
    H, W, C, R = 24, 24, 3, 2
    rng = np.random.default_rng(10)
    anchors = _anchors(rng, H, W, R)
    cfg = dict(CFG, nms_pre=500, max_num=100, nms_thr=0.2)
    heads = [_random_head(rng, H, W, C, R, f) for f in (0.3, 0.0, 0.01, 0.3)]
    M = cfg["max_num"]
    out = (torch.empty((M, 9), device=cuda), torch.empty((M,), device=cuda),
           torch.empty((M,), dtype=torch.int64, device=cuda), torch.empty((1,), dtype=torch.int32, device=cuda))
    head_t = torch.from_numpy(heads[0][None]).to(cuda)
    anchors_t = torch.from_numpy(anchors).to(cuda)
    args = (C, R, cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"], M, cfg["dir_offset"], cfg["dir_limit_offset"])
    s = torch.cuda.Stream(cuda)
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        anchor3d_postprocess_device(head_t, anchors_t, *args, out=out)
    torch.cuda.current_stream().wait_stream(s)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=s):
        anchor3d_postprocess_device(head_t, anchors_t, *args, out=out)
    counts = []
    for head in heads:
        head_t.copy_(torch.from_numpy(head[None]))
        out[0].fill_(float("nan"))
        out[1].fill_(float("nan"))
        out[2].fill_(-1)
        out[3].fill_(-1)
        g.replay()
        torch.cuda.synchronize()
        k = int(out[3].item())
        got = tuple(t[:k].cpu().numpy() for t in out[:3])
        want = bo.anchor3d_decode_ref(head, anchors, C, R, cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"], M,
                                      cfg["dir_offset"], cfg["dir_limit_offset"], details=True)
        _same(got, want[:3])
        _untouched(out, k)
        counts.append((k, sum(len(p) for p in want[3]["per_class"])))
    assert counts[1] == (0, 0) and 0 < counts[2][0] == counts[2][1] < M and counts[0][0] == M < counts[0][1], counts
    del g
    big = dict(cfg, nms_pre=4096, max_num=1000)
    _, got = _run(cuda, heads[0], anchors, C, R, big)
    _same(got, bo.anchor3d_decode_ref(heads[0], anchors, C, R, *[big[k] for k in ("nms_pre", "score_thr", "nms_thr",
                                                                                 "max_num", "dir_offset",
                                                                                 "dir_limit_offset")]))
    for head in heads[:3]:
        res, got = _run(cuda, head, anchors, C, R, cfg)
        _same(got, bo.anchor3d_decode_ref(head, anchors, C, R, cfg["nms_pre"], cfg["score_thr"], cfg["nms_thr"], M,
                                          cfg["dir_offset"], cfg["dir_limit_offset"]))
