"""CPU suite for BEVFusion's new device steps: Anchor3DHead's decode restatement (tests/bevfusion_oracle.py) on
hand-built head planes, the anchor layout against an independent restatement of AlignedAnchor3DRangeGenerator, and the
host-side argument checks of p3d_hard_vfe, p3d_se_gate_h16 and p3d_anchor3d_postprocess (every call here is refused
before it reaches the device)."""
import ctypes

import numpy as np
import pytest

import bevfusion_oracle as bo

F = np.float32


def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib.lib()


class Planes:
    """A head on an H x W map with C classes and R anchors per cell: every class logit -10 (below any threshold), zero
    deltas and dir logits; anchors [A, 9] placed 10 m apart along x, 1 m cubes, heading 0."""

    def __init__(self, H=2, W=2, C=3, R=2):
        self.H, self.W, self.C, self.R = H, W, C, R
        self.A = H * W * R
        self.head = np.zeros((R * (C + 11), H, W), F)
        self.head[:R * C] = -10.0
        self.anchors = np.zeros((self.A, 9), F)
        self.anchors[:, 0] = 10.0 * np.arange(self.A)
        self.anchors[:, 3:6] = 1.0

    def _at(self, i, ch_base, K, k):
        cell, a = divmod(i, self.R)
        y, x = divmod(cell, self.W)
        return ch_base + a * K + k, y, x

    def cls(self, i, c, v):
        ch, y, x = self._at(i, 0, self.C, c)
        self.head[ch, y, x] = v

    def reg(self, i, k, v):
        ch, y, x = self._at(i, self.R * self.C, 9, k)
        self.head[ch, y, x] = v

    def dir(self, i, d0, d1):
        for k, v in ((0, d0), (1, d1)):
            ch, y, x = self._at(i, self.R * (self.C + 9), 2, k)
            self.head[ch, y, x] = v

    def run(self, nms_pre=100, score_thr=0.05, nms_thr=0.2, max_num=50, dir_offset=0.7854, dir_limit_offset=0.0,
            details=False):
        return bo.anchor3d_decode_ref(self.head, self.anchors, self.C, self.R, nms_pre, score_thr, nms_thr, max_num,
                                      dir_offset, dir_limit_offset, details=details)


def test_head_layout():
    p = Planes(H=2, W=3, C=4, R=2)
    p.cls(7, 2, 1.0)
    p.reg(7, 8, 2.0)
    p.dir(7, 0.0, 3.0)
    cls, reg, dirl = bo.split_head(p.head, 4, 2)
    assert cls[7, 2] == 1.0 and (cls == -10).sum() == cls.size - 1
    assert reg[7, 8] == 2.0 and np.count_nonzero(reg) == 1
    assert dirl[7, 1] == 3.0 and np.count_nonzero(dirl) == 1


def test_class_major_below_max_num_and_score_sort_above(oracle_mod):
    p = Planes()
    p.cls(0, 2, 3.0)   # highest score, last class
    p.cls(3, 0, 1.0)
    p.cls(5, 1, 2.0)
    b, s, l = p.run(max_num=3)
    assert l.tolist() == [0, 1, 2]                          # class-major, not score order
    np.testing.assert_array_equal(b[:, 0], [30.0, 50.0, 0.0])
    b, s, l = p.run(max_num=2)                              # above max_num: score order, cut
    assert l.tolist() == [2, 1] and b[:, 0].tolist() == [0.0, 50.0]
    assert s[0] > s[1]


def test_ties_at_the_nms_pre_cut(oracle_mod):
    p = Planes()
    for i in (5, 1, 3):
        p.cls(i, 0, 1.0)
    p.cls(6, 1, 0.5)
    b, s, l, d = p.run(nms_pre=2, details=True)
    assert d["kept"].tolist() == [1, 3]                     # equal max scores: the lower anchor indices
    assert sorted(b[:, 0].tolist()) == [10.0, 30.0]
    b, s, l, d = p.run(nms_pre=8, details=True)             # A <= nms_pre: anchor order, every anchor kept
    assert d["kept"].tolist() == list(range(8)) and len(b) == 4


@pytest.mark.parametrize("nms_pre", [8, 4])
def test_ties_within_a_class(oracle_mod, nms_pre):
    """Two identical boxes of one class with equal scores: the first in kept order survives (anchor 2, marked by its
    velocity); a third with a higher score suppresses neither when it is elsewhere."""
    p = Planes()
    p.anchors[6, :3] = p.anchors[2, :3]
    for i, vx in ((2, 1.0), (6, 2.0)):
        p.cls(i, 1, 0.0)
        p.reg(i, 7, vx)
    p.cls(4, 1, 2.0)
    b, s, l = p.run(nms_pre=nms_pre)
    assert l.tolist() == [1, 1]
    assert b[:, 7].tolist() == [0.0, 1.0]                   # anchor 4 first (higher score), then anchor 2


def test_dir_ties_and_limit_period(oracle_mod):
    p = Planes()
    for i in range(4):
        p.cls(i, 0, 1.0)
    k = [-2, -1, 1, 2]
    for i in range(4):
        p.reg(i, 6, F(k[i]) * bo.PI32)                       # exact multiples of fp32(pi)
    p.dir(0, 0.5, 0.5)                                       # tie: bin 0
    p.dir(1, 0.0, 1.0)
    p.dir(2, 1.0, 0.0)
    p.dir(3, -1.0, -1.0)
    want = {0.0: 0.0, 10.0: float(bo.PI32), 20.0: 0.0, 30.0: 0.0}
    for nms_pre in (100, 3):  # every anchor kept in anchor order / the top 3 in score order: labels follow their anchor
        p.cls(3, 0, 1.0 if nms_pre == 100 else -10.0)
        p.cls(0, 0, 1.0 if nms_pre == 100 else 2.0)
        b, s, l = p.run(dir_offset=0.0, nms_pre=nms_pre)
        assert len(b) == (4 if nms_pre == 100 else 3)
        for row in b:
            assert row[6] == want[float(row[0])]
    for m in range(-3, 4):
        assert bo.limit_period32(F(m) * bo.PI32, 0.0) == 0.0
    v = np.linspace(-10, 10, 1001).astype(F)
    lp = bo.limit_period32(v, 0.5)
    assert (lp >= -bo.PI32 / 2 - 1e-6).all() and (lp < bo.PI32 / 2 + 1e-6).all()


def test_empty_class_and_all_empty(oracle_mod):
    p = Planes()
    b, s, l = p.run()
    assert b.shape == (0, 9) and s.shape == (0,) and l.shape == (0,)
    p.cls(1, 0, 1.0)
    b, s, l = p.run()
    assert l.tolist() == [0]


def test_velocity_pass_through(oracle_mod):
    p = Planes()
    p.cls(2, 0, 1.0)
    p.reg(2, 7, 1.5)
    p.reg(2, 8, -2.25)
    b, _, _ = p.run()
    assert b[0, 7:].tolist() == [1.5, -2.25]
    p.anchors[2, 7:] = (0.25, 0.5)
    b, _, _ = p.run()
    assert b[0, 7:].tolist() == [1.75, -1.75]


def test_decode_rules(oracle_mod):
    """DeltaXYZWLHRBBoxCoder on one anchor against the formulas in fp64."""
    p = Planes()
    p.anchors[1, :7] = (3.0, -2.0, -1.8, 1.95, 4.6, 1.7, 1.57)
    p.cls(1, 0, 1.0)
    t = (0.1, -0.2, 0.3, 0.05, -0.1, 0.2, 0.4, 0.0, 0.0)
    for k, v in enumerate(t):
        p.reg(1, k, v)
    b, _, _ = p.run(dir_offset=0.0, dir_limit_offset=1.0)
    xa, ya, za, wa, la, ha, ra = [float(v) for v in p.anchors[1, :7]]
    t = [float(F(v)) for v in t]
    diag = np.hypot(la, wa)
    h = np.exp(t[5]) * ha
    want = [t[0] * diag + xa, t[1] * diag + ya, t[2] * ha + za + ha / 2 - h / 2, np.exp(t[3]) * wa, np.exp(t[4]) * la, h]
    np.testing.assert_allclose(b[0, :6], want, rtol=1e-6, atol=1e-6)
    r = t[6] + ra
    np.testing.assert_allclose(b[0, 6], r - np.floor(r / np.pi + 1.0) * np.pi, rtol=1e-6)


def test_nan_logit_takes_a_kept_slot(oracle_mod):
    """A NaN class logit ranks its anchor first at the nms_pre cut (torch.topk) and its other classes still count."""
    p = Planes()
    p.cls(6, 0, np.nan)
    p.cls(6, 1, 1.0)
    p.cls(2, 0, 2.0)
    p.cls(3, 0, 1.5)
    b, s, l, d = p.run(nms_pre=2, details=True)
    assert d["kept"].tolist() == [6, 2]
    assert sorted(zip(l.tolist(), b[:, 0].tolist())) == [(0, 20.0), (1, 60.0)]


def test_anchor_layout_matches_generator_restatement():
    from paddle3d_b200 import bevfusion as bf
    cfg = bf.CONFIG
    for H, W in ((200, 200), (3, 5)):
        got = bf.make_anchors(cfg, (H, W))
        want = bo.aligned_anchors_loops(H, W, cfg["anchor_xy"], cfg["anchors"], cfg["rotations"], len(cfg["custom_values"]))
        assert got.shape == (H * W * 14, 9)
        np.testing.assert_array_equal(got, want)
    a = bf.make_anchors()
    # anchor ((y W + x) 7 + s) 2 + r: the truck (s = 1) at rotation 1.57 in cell (y 3, x 5)
    i = ((3 * 200 + 5) * 7 + 1) * 2 + 1
    np.testing.assert_allclose(a[i], [-49.6 + 0.496 * 5.5, -49.6 + 0.496 * 3.5, -1.74440365, 2.4560939, 6.73778078,
                                      2.73004906, 1.57, 0, 0], rtol=1e-6)
    assert bf.anchors_per_loc() == 14 and 14 * (10 + 9 + 2) == 294


def test_hard_vfe_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    f = L.p3d_hard_vfe

    def call(n=4, M=8, Fd=4, mid=64, out=64, vox=p, w2=p):
        return f(vox, p, p, None, n, M, Fd, mid, p, p, p, out, w2, p, p, p, p, p, None)
    assert call(vox=None) == -1
    assert call(w2=None) == -1
    assert call(n=-1) == -1
    assert call(mid=0) == -1
    assert call(out=0) == -1
    assert call(M=65) == -4
    assert call(M=0) == -4
    assert call(Fd=2) == -4
    assert call(Fd=9) == -4
    assert call(mid=65) == -4
    assert call(n=0) == 0  # nothing to do: no launch


def test_se_gate_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(4096)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16
    f = L.p3d_se_gate_h16
    need = L.p3d_se_gate_workspace_bytes(1, 4, 4, 64)
    assert need > 0 and L.p3d_se_gate_workspace_bytes(0, 4, 4, 64) == 0

    def call(img=p, B=1, H=4, W=4, C=64, wt=p, status=p, ws=p, ws_bytes=None):
        return f(img, B, H, W, C, wt, p, p, status, ws, need if ws_bytes is None else ws_bytes, None)
    assert call(img=None) == -1
    assert call(wt=None) == -1
    assert call(status=None) == -1
    assert call(img=p + 8) == -1   # 16-byte aligned rows
    assert call(C=48) == -1        # whole 32-channel groups
    assert call(C=0) == -1
    assert call(H=0) == -1
    assert call(C=1056) == -4
    assert call(B=65536) == -4
    assert call(ws_bytes=need - 1) == -2
    assert call(ws=None) == -2


def test_anchor3d_postprocess_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)
    f = L.p3d_anchor3d_postprocess
    ws = L.p3d_anchor3d_postprocess_workspace_bytes
    need = ws(4, 4, 2, 3, 100, 50)
    assert need > 0
    assert ws(0, 4, 2, 3, 100, 50) == 0 and ws(4, 4, 2, 65, 100, 50) == 0 and ws(4, 4, 2, 3, 4097, 50) == 0

    def call(head=p, H=4, W=4, R=2, C=3, pre=100, thr=0.05, nms=0.2, mx=50, out=p, ws_p=p, ws_bytes=None):
        return f(head, H, W, R, C, p, pre, thr, nms, mx, 0.7854, 0.0, out, p, p, p, ws_p,
                 need if ws_bytes is None else ws_bytes, None)
    assert call(head=None) == -1
    assert call(out=None) == -1
    assert call(H=0) == -1
    assert call(R=0) == -1
    assert call(C=0) == -1
    assert call(pre=0) == -1
    assert call(mx=0) == -1
    assert call(thr=float("nan")) == -1
    assert call(thr=-0.5) == -1
    assert call(nms=float("nan")) == -1
    assert call(C=65) == -4
    assert call(pre=4097) == -4
    assert call(H=50000, W=50000) == -4   # A >= 2^31
    assert call(ws_bytes=need - 1) == -2
    assert call(ws_p=None) == -2
