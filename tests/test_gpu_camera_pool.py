"""bev_pool in every kernel instantiation and at every interval length where its pipeline turns, lss_depth_feat at every
block shape, and the LSS view transform at other camera geometries, against exact and float64 references.

Kernels (csrc/bev_pool.cu), ten instantiations behind four entry points:
  * p3d_bev_pool_v2 (host interval count): bev_fwd_warp_kernel<G> when C % 4 == 0, C <= 256 and feat / out are 16-byte
    aligned, with G = 1 for C <= 128 and G = 2 (two float4 channel groups per lane) above; otherwise the round-1 kernel,
    one thread per (interval, channel group): bev_fwd_kernel<4> for aligned C % 4 == 0 above 256, bev_fwd_kernel<1> for
    C % 4 != 0 or a misaligned feat;
  * p3d_bev_pool_v2_dev (count read from counts_dev[1]): bev_fwd_warp_kernel<G, true, PLANAR>, zyx and planar output;
  * p3d_bev_pool_v2_dev_h16: bev_fwd_warp_kernel<2, true, false, true> for every C, pixel fp16-pair rows;
  * p3d_bev_pool_v2_bkwd: bev_bwd_kernel.
The warp kernel walks an interval in batches of 32 points, with the rank words prefetched two batches ahead and the
depth one batch ahead, and keeps U = 16 (G = 1) or 8 (G = 2) feature rows in flight with the index clamped to the
batch's last point.  The interval plans (Plan) hold every length 1..130 plus 191..193, 255..257, 1000, 4099 and 16387,
so every batch count up to five, every partial batch and every partial group of U rows occurs, and the interval count
is not a multiple of the 8 warps of a block.  The channel sweep covers C / 4 = 1..64 across the G boundary (128 / 132)
with a partly owned second group.

References:
  * bit for bit: the C oracle's bev_pool_v2 / bev_pool_v2_bkwd with use_fma=True (the kernels' fp32 FMA chain in index
    order), permuted to each layout; for the pixel rows, oracle.bevdet.split_h16 of it (hi = RN fp16(x), lo' = RN
    fp16((x - hi) 2048), |x| saturated at 65504), compared as bytes, and the status word;
  * float64, on the CPU: every element of the oracle's chain lies within gamma_L sum |d_i f_i| of the exact sum of its
    interval's L terms (gamma_L = L u / (1 - L u), u = 2^-24), which ties the plan's terms to the oracle independently
    of the C code.
Every output is poisoned before the call (NaN floats, fp16 0x7e00), so empty cells and padding channels must come from
the zero fill.  Rank and interval entries past the device count are in range but wrong (a sentinel cell no interval
owns, real depth and feature rows): a kernel that reads them writes a value the comparison catches, and nothing here
can read or write out of bounds if a kernel is wrong.

Which instantiation ran is not restated from the host dispatch: test_every_instantiation_runs records the kernel names
with torch.profiler while it makes one call per instantiation.

lss_depth_feat (csrc/lss_depth_feat.cu, a block of 32 pixels of one camera) runs at shapes with a partial last block, at
the D and C limits (382, 370) and at other camera models' sizes, against oracle.lss.depth_softmax with test_gpu_lss.py's
ulp rules and feat_permute bit for bit, with a NaN guard of 32 max(C, D) floats behind each output.

The LSS view transform (LSSViewTransformer and the captured LSSHotPath) runs at four more camera geometries, checked
stage by stage: coor, ranks, depth, the BEV bit for bit against the oracle's pool of the device's own depth and feat,
end to end against oracle.lss.view_transform, and captured against eager."""
import re

import numpy as np
import pytest

from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
NAN16 = 0x7E00
LENGTHS = list(range(1, 131)) + [191, 192, 193, 255, 256, 257, 1000, 4099, 16387]
WARP_CS = (4, 8, 12, 60, 64, 76, 80, 124, 128, 132, 136, 160, 252, 256)
# (B, Z, Y, X, cells sorted as the prepare emits them)
LAYOUTS = ((1, 1, 13, 17, True), (2, 3, 9, 11, False))


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


def _lib():
    from paddle3d_b200 import _lib
    return _lib.lib()


def _check(rc, what):
    from paddle3d_b200 import _lib
    _lib.check(rc, what)


def _p(t):
    from paddle3d_b200._mem import ptr
    return ptr(t)


def _stream(cuda):
    from paddle3d_b200._mem import stream
    return stream(cuda)


def _nan32(cuda, n):
    import torch
    return torch.full((n,), float("nan"), dtype=torch.float32, device=cuda)


def _nan16(cuda, n):
    import torch
    return torch.full((n,), NAN16, dtype=torch.int16, device=cuda).view(torch.float16)


def _bits_equal(got, want):
    """Bit-equal float tensors / arrays (NaN payloads and signed zeros included)."""
    g = got.cpu().numpy() if hasattr(got, "cpu") else np.asarray(got)
    w = np.ascontiguousarray(want, g.dtype)
    it = {4: np.uint32, 2: np.uint16}[g.dtype.itemsize]
    return g.shape == w.shape and np.array_equal(np.ascontiguousarray(g).view(it), w.view(it))


# ------------------------------------------------------------------------------------------------------- interval plans
class Plan:
    """Rank arrays of a list of interval lengths, laid out as p3d_bev_pool_prepare writes them: interval k is points
    st[k] .. st[k] + ln[k] - 1 of rb / rd / rf, all of one cell, every interval a distinct cell (ascending as the prepare
    emits them, or shuffled); the lengths come in random order.  rd is a random gather of distinct depth entries (the
    depth array has more, in no interval), rf a random gather of n_feat feature rows, shared between intervals as in a
    frustum.  Depth is in (0, 1].
    After the n_pts points and n_int intervals come `spare` points and cap - n_int interval entries that are in range
    but wrong: the points are of cell `sentinel` (a cell no interval owns when there is one) with real depth and feature
    rows, the entries are intervals over them.  All five arrays have cap = n_pts + spare entries, as the prepare's."""

    def __init__(self, seed, lengths, cells, n_feat, sorted_cells, spare=64):
        rng = np.random.default_rng(seed)
        ln = np.array(lengths, np.int64)
        rng.shuffle(ln)
        self.n_int, self.n_pts, self.cells, self.n_feat = len(ln), int(ln.sum()), cells, n_feat
        assert self.n_int <= cells
        cap = self.cap = self.n_pts + spare
        own = rng.choice(cells, self.n_int, replace=False)
        if sorted_cells:
            own.sort()
        free = np.setdiff1d(np.arange(cells), own)
        self.sentinel = int(free[rng.integers(len(free))]) if len(free) else int(own[0])
        st = np.zeros(cap, np.int64)
        st[1:self.n_int] = np.cumsum(ln)[:-1]
        lens = np.zeros(cap, np.int64)
        lens[:self.n_int] = ln
        j = np.arange(cap - self.n_int)
        off = j % spare
        st[self.n_int:] = self.n_pts + off
        lens[self.n_int:] = 1 + j % (spare - off)
        self.st, self.ln = st.astype(np.int32), lens.astype(np.int32)
        self.rb = np.full(cap, self.sentinel, np.int32)
        self.rb[:self.n_pts] = np.repeat(own, ln)
        self.n_depth = cap + 257
        self.rd = rng.permutation(self.n_depth)[:cap].astype(np.int32)
        self.rf = rng.integers(0, n_feat, cap).astype(np.int32)
        self.depth = (1.0 - rng.random(self.n_depth)).astype(np.float32)
        assert (self.depth > 0).all() and (self.depth <= 1).all()
        assert (self.st.astype(np.int64) + self.ln <= cap).all() and self.rb.max() < cells

    def feat(self, C, seed):
        return np.random.default_rng(seed).normal(size=(self.n_feat, C)).astype(np.float32)

    def pool(self, oracle_mod, feat, shape, count=None):
        """The oracle's FMA chain over the first `count` intervals (all of them by default), [B, Z, Y, X, C]."""
        n = self.n_int if count is None else count
        return oracle_mod.bev_pool_v2(self.depth, feat, self.rd, self.rf, self.rb, self.ln[:n], self.st[:n], shape,
                                      use_fma=True)

    def check_fp64(self, feat, want):
        """Every owned cell of want [.., C] (the oracle's chain) within gamma_L sum |d f| of the fp64 interval sum."""
        C = feat.shape[1]
        n, st = self.n_pts, self.st[:self.n_int]
        terms = self.depth[self.rd[:n]].astype(np.float64)[:, None] * feat[self.rf[:n]].astype(np.float64)
        exact = np.add.reduceat(terms, st, axis=0)
        mag = np.add.reduceat(np.abs(terms), st, axis=0)
        L = self.ln[:self.n_int].astype(np.float64)[:, None]
        got = want.reshape(-1, C)[self.rb[st]].astype(np.float64)
        err = np.abs(got - exact)
        assert (err <= L * U32 / (1.0 - L * U32) * mag).all(), "oracle chain off its interval's fp64 sum"
        assert err.max() > 0  # the chain does round somewhere, so the bound is a real check


def layout_plan(B, Z, Y, X, sorted_cells, seed=11):
    plan = Plan(seed + B * Z, LENGTHS, B * Z * Y * X, 3000, sorted_cells)
    assert plan.n_int % 8 and plan.n_int == len(LENGTHS)  # the last block of 8 warps is partial
    return plan


def collapse(pool):
    from oracle import lss
    return lss.collapse_z(pool)


def pixel_rows(planar, out_C):
    """[B, Z C, Y, X] fp32 -> pixel fp16-pair rows [B Y X, 2 out_C] float16: per 32 channels 32 hi halves then 32 lo'
    halves (split_h16, saturated at 65504), channels >= Z C zero."""
    from oracle import bevdet as ob
    B, ZC, Y, X = planar.shape
    v = np.zeros((B, Y, X, out_C), np.float32)
    v[..., :ZC] = planar.transpose(0, 2, 3, 1)
    hi, lo = ob.split_h16(v)
    rows = np.stack([hi.reshape(-1, out_C // 32, 32), lo.reshape(-1, out_C // 32, 32)], 2)
    return rows.reshape(B * Y * X, 2 * out_C)


# ------------------------------------------------------------------------------------------------------ device calls
class Dev:
    """A plan's arrays on the device with one C's feature rows (offset: feat starts one float into its allocation)."""

    def __init__(self, cuda, plan, feat, offset=False):
        import torch
        self.cuda, self.plan, self.C, self.feat_np = cuda, plan, feat.shape[1], feat
        self.depth = _t(cuda, plan.depth)
        if offset:
            buf = torch.empty(feat.size + 1, dtype=torch.float32, device=cuda)
            buf[1:] = _t(cuda, feat.reshape(-1))
            self.feat = buf[1:]
            assert self.feat.data_ptr() % 16 == 4
        else:
            self.feat = _t(cuda, feat)
        self.rd, self.rf, self.rb, self.ln, self.st = [_t(cuda, getattr(plan, k)) for k in ("rd", "rf", "rb", "ln", "st")]

    def _args(self):
        return [_p(t) for t in (self.depth, self.feat, self.rd, self.rf, self.rb, self.ln, self.st)]

    def host(self, n_int=None):
        """p3d_bev_pool_v2 over [cells, C]."""
        out = _nan32(self.cuda, self.plan.cells * self.C)
        n = self.plan.n_int if n_int is None else n_int
        _check(_lib().p3d_bev_pool_v2(*self._args(), n, self.C, _p(out), out.numel(), _stream(self.cuda)), "bev_pool_v2")
        return out

    def _counts(self, count):
        return _t(self.cuda, np.array([self.plan.n_pts, self.plan.n_int if count is None else count], np.int32))

    def dev(self, shape, planar, count=None, capacity=None):
        """p3d_bev_pool_v2_dev, shape (B, Z, Y, X); counts_dev[1] = count (the plan's interval count by default)."""
        B, Z, Y, X = shape
        out = _nan32(self.cuda, B * Z * Y * X * self.C)
        counts = self._counts(count)
        cap = self.plan.cap if capacity is None else capacity
        _check(_lib().p3d_bev_pool_v2_dev(*self._args(), _p(counts), cap, self.C, B, Z, Y, X, int(planar), _p(out),
                                          _stream(self.cuda)), "bev_pool_v2_dev")
        return out

    def h16(self, shape, out_C, status, count=None, capacity=None):
        """p3d_bev_pool_v2_dev_h16 -> rows [B Y X, 2 out_C] float16."""
        B, Z, Y, X = shape
        out = _nan16(self.cuda, B * Y * X * 2 * out_C)
        counts = self._counts(count)
        cap = self.plan.cap if capacity is None else capacity
        _check(_lib().p3d_bev_pool_v2_dev_h16(*self._args(), _p(counts), cap, self.C, B, Z, Y, X, _p(out), out_C,
                                              _p(status), _stream(self.cuda)), "bev_pool_v2_dev_h16")
        return out.view(B * Y * X, 2 * out_C)


def _status(cuda):
    import torch
    return torch.zeros((1,), dtype=torch.int32, device=cuda)


def check_all_layouts(cuda, oracle_mod, d, shape, count=None, capacity=None):
    """Device-count pool in zyx, planar and pixel-row layouts bit-equal to the oracle over the first `count` intervals;
    out_C one 32-channel group wider than Z C rounded up.  Returns the oracle's pool [B, Z, Y, X, C]."""
    import torch
    B, Z, Y, X = shape
    C = d.C
    want = d.plan.pool(oracle_mod, d.feat_np, (B, Z, Y, X, C), count)
    out_C = (Z * C + 31) // 32 * 32 + 32
    status = _status(cuda)
    zyx = d.dev(shape, False, count, capacity)
    planar = d.dev(shape, True, count, capacity)
    rows = d.h16(shape, out_C, status, count, capacity)
    torch.cuda.synchronize()
    what = "C %d shape %s count %s capacity %s" % (C, shape, count, capacity)
    assert _bits_equal(zyx, want.reshape(-1)), "zyx " + what
    assert _bits_equal(planar, collapse(want).reshape(-1)), "planar " + what
    assert _bits_equal(rows, pixel_rows(collapse(want), out_C)), "pixel rows " + what
    assert int(status.item()) == 0, what
    return want


# ------------------------------------------------------------------------------------------------------ forward tests
@pytest.mark.parametrize("C", WARP_CS)
def test_warp_kernel_every_entry_point(cuda, oracle_mod, C):
    """Host count, device count zyx / planar and pixel rows, B 1 / Z 1 on sorted cells and B 2 / Z 3 on shuffled
    cells, bit for bit; the oracle's chain within its fp64 bound."""
    import torch
    for B, Z, Y, X, srt in LAYOUTS:
        plan = layout_plan(B, Z, Y, X, srt)
        feat = plan.feat(C, C)
        d = Dev(cuda, plan, feat)
        want = check_all_layouts(cuda, oracle_mod, d, (B, Z, Y, X))
        plan.check_fp64(feat, want)
        host = d.host()
        torch.cuda.synchronize()
        assert _bits_equal(host, want.reshape(-1)), "host count C %d B %d Z %d" % (C, B, Z)
        assert not np.isnan(want).any() and (want.reshape(-1, C) == 0).all(1).sum() == plan.cells - plan.n_int


@pytest.mark.parametrize("C,offset", [(1, False), (7, False), (260, False), (512, False), (64, True)])
def test_round1_kernel(cuda, oracle_mod, C, offset):
    """p3d_bev_pool_v2's round-1 kernel: bev_fwd_kernel<1> for C % 4 != 0 and for a feat view one float into its
    allocation, bev_fwd_kernel<4> for C > 256."""
    import torch
    for B, Z, Y, X, srt in LAYOUTS:
        plan = layout_plan(B, Z, Y, X, srt)
        feat = plan.feat(C, C + 1000)
        got = Dev(cuda, plan, feat, offset).host()
        torch.cuda.synchronize()
        want = plan.pool(oracle_mod, feat, (B, Z, Y, X, C))
        assert _bits_equal(got, want.reshape(-1)), "C %d offset %s B %d" % (C, offset, B)
        plan.check_fp64(feat, want)


@pytest.mark.parametrize("C", (80, 160))
def test_device_count_edges(cuda, oracle_mod, C):
    """counts_dev[1] = 0, 1, one short of the intervals present (the last interval's cell stays zero), equal to the
    capacity, and equal to the cell count (every cell of a 4 x 4 x 1 grid, B = 2, occupied).  The entries past the count
    are in range but wrong, so a kernel that reads them fails the comparison."""
    B, Z, Y, X = 2, 1, 9, 11
    plan = Plan(23, LENGTHS, B * Z * Y * X, 3000, True)
    feat = plan.feat(C, 7)
    d = Dev(cuda, plan, feat)
    n = plan.n_int
    for count, capacity in ((0, None), (1, None), (n - 1, None), (n, n)):
        want = check_all_layouts(cuda, oracle_mod, d, (B, Z, Y, X), count, capacity)
        assert not want.reshape(-1, C)[plan.sentinel].any()
        if count == n - 1:
            last = plan.rb[plan.st[n - 1]]
            assert not want.reshape(-1, C)[last].any() and want.reshape(-1, C)[plan.rb[plan.st[n - 2]]].any()
    # every cell occupied: the grid is bounded by the cells, not by the capacity
    full = Plan(29, list(range(1, 21)) + [31, 32, 33, 63, 64, 65, 96, 97, 129, 257, 1000, 4099], 32, 500, True)
    assert full.n_int == 32 and full.cap > 32
    feat = full.feat(C, 8)
    d = Dev(cuda, full, feat)
    want = check_all_layouts(cuda, oracle_mod, d, (2, 1, 4, 4), 32)
    assert (want.reshape(32, C) != 0).any(1).all()


def _overflow_plan(values):
    """Plan of two-point intervals with depth 1 on a B = 2, 3 x 5 grid, C = 160: interval k's channel 150 (lane 5 of the
    second channel group) sums the pair values[k], the other channels N(0, 1) products; cells k and 15 + k."""
    n = len(values)
    plan = Plan(31, [2] * (2 * n), 30, 4 * n, True)
    plan.depth[:] = 1.0
    feat = plan.feat(160, 9)
    for k, (a, b) in enumerate(values):
        for half in (0, 1):  # one interval in each batch image
            i = 2 * k + half
            s = plan.st[i]
            plan.rf[s:s + 2] = (2 * i, 2 * i + 1)
            feat[2 * i, 150], feat[2 * i + 1, 150] = a, b
            plan.rb[s:s + 2] = 15 * half + k
    return plan, feat


def test_pixel_rows_overflow(cuda, oracle_mod):
    """Sums of exactly +-65504 leave the status bit clear; just above on either sign sets it and saturates hi; the
    bytes equal split_h16 of the oracle's sums in every case.  The status word is read and reset between cases."""
    import torch
    cases = (([(32752.0, 32752.0), (-32752.0, -32752.0)], 0), ([(32752.0, 32753.0)], 1), ([(-32753.0, -32752.0)], 1))
    status = _status(cuda)
    for values, flag in cases:
        plan, feat = _overflow_plan(values)
        d = Dev(cuda, plan, feat)
        want = plan.pool(oracle_mod, feat, (2, 1, 3, 5, 160))
        sums = [a + b for a, b in values]
        assert sorted(want[..., 150][want[..., 150] != 0].tolist()) == sorted(sums * 2)
        status.zero_()
        rows = d.h16((2, 1, 3, 5), 192, status)
        torch.cuda.synchronize()
        assert _bits_equal(rows, pixel_rows(collapse(want), 192)), values
        assert int(status.item()) == flag, (values, int(status.item()))
        hi = rows.cpu().numpy().reshape(2, 3, 5, 6, 2, 32)[..., 4, 0, 22]  # channel 150's hi
        assert np.abs(hi.astype(np.float32)).max() == 65504.0


# ----------------------------------------------------------------------------------------------------------- backward
BKWD_LENGTHS = list(range(1, 71)) + [127, 128, 129, 1000, 4099]


def bkwd_plan(seed=41):
    """The backward's layout: intervals of points grouped by ranks_feat (one distinct feature row per interval; 20 rows
    in none), ranks_bev random cells of 300, ranks_depth distinct (some depth entries in no interval)."""
    plan = Plan(seed, BKWD_LENGTHS, 300, len(BKWD_LENGTHS) + 20, False)
    rng = np.random.default_rng(seed + 1)
    rows = rng.permutation(plan.n_feat)[:plan.n_int]
    plan.rf[:plan.n_pts] = np.repeat(rows, plan.ln[:plan.n_int])
    plan.rb[:plan.n_pts] = rng.integers(0, plan.cells, plan.n_pts)
    return plan


@pytest.mark.parametrize("C", (1, 7, 31, 32, 33, 80, 256, 260))
def test_backward(cuda, oracle_mod, C):
    """Both gradients bit-equal to the oracle's FMA chains; depth entries and feature rows in no interval are zero."""
    import torch
    plan = bkwd_plan()
    rng = np.random.default_rng(C)
    feat = plan.feat(C, C + 2000)
    og = rng.normal(size=(plan.cells, C)).astype(np.float32)
    n, k = plan.n_pts, plan.n_int
    depth, feat_t, og_t = _t(cuda, plan.depth), _t(cuda, feat), _t(cuda, og)
    rd, rf, rb, ln, st = [_t(cuda, getattr(plan, a)) for a in ("rd", "rf", "rb", "ln", "st")]
    dg, fg = _nan32(cuda, plan.n_depth), _nan32(cuda, feat.size)
    _check(_lib().p3d_bev_pool_v2_bkwd(_p(og_t), _p(depth), _p(feat_t), _p(rd), _p(rf), _p(rb), _p(ln), _p(st), k, C,
                                       _p(dg), dg.numel(), _p(fg), fg.numel(), _stream(cuda)), "bev_pool_v2_bkwd")
    torch.cuda.synchronize()
    wdg, wfg = oracle_mod.bev_pool_v2_bkwd(og, plan.depth, feat, plan.rd, plan.rf, plan.rb, plan.ln[:k], plan.st[:k],
                                           use_fma=True)
    assert _bits_equal(dg, wdg), "depth_grad C %d" % C
    assert _bits_equal(fg, wfg.reshape(-1)), "feat_grad C %d" % C
    unused = np.setdiff1d(np.arange(plan.n_depth), plan.rd[:n])
    assert len(unused) >= 257 and not dg.cpu().numpy()[unused].any()
    free = np.setdiff1d(np.arange(plan.n_feat), plan.rf[:n])
    assert len(free) == 20 and not fg.cpu().numpy().reshape(-1, C)[free].any()
    assert wdg[plan.rd[:n]].all()


# ------------------------------------------------------------------------------------------------ which kernel ran
EXPECTED_KERNELS = {
    "bev_fwd_kernel<1>", "bev_fwd_kernel<4>",
    "bev_fwd_warp_kernel<1,false,false,false>", "bev_fwd_warp_kernel<2,false,false,false>",
    "bev_fwd_warp_kernel<1,true,false,false>", "bev_fwd_warp_kernel<1,true,true,false>",
    "bev_fwd_warp_kernel<2,true,false,false>", "bev_fwd_warp_kernel<2,true,true,false>",
    "bev_fwd_warp_kernel<2,true,false,true>", "bev_bwd_kernel",
}


def kernel_key(name):
    """'void p3d::(anonymous namespace)::bev_fwd_warp_kernel<2, true, false, true>(int, ...)' (or the (int)2 / (bool)1
    spelling) -> 'bev_fwd_warp_kernel<2,true,false,true>'; None for other kernels."""
    m = re.search(r"(bev_(?:fwd_warp|fwd|bwd)_kernel)(<[^>]*>)?", name)
    if m is None:
        return None
    args = (m.group(2) or "").replace("(int)", "").replace("(bool)0", "false").replace("(bool)1", "true")
    return m.group(1) + args.replace(" ", "")


def test_kernel_key():
    assert kernel_key("void p3d::(anonymous namespace)::bev_fwd_warp_kernel<2, true, false, true>(int, int)") == \
        "bev_fwd_warp_kernel<2,true,false,true>"
    assert kernel_key("void p3d::<unnamed>::bev_fwd_warp_kernel<(int)1, (bool)1, (bool)1, (bool)0>(int)") == \
        "bev_fwd_warp_kernel<1,true,true,false>"
    assert kernel_key("p3d::(anonymous namespace)::bev_bwd_kernel(int, int, float const*)") == "bev_bwd_kernel"
    assert kernel_key("void p3d::(anonymous namespace)::bev_fwd_kernel<4>(int)") == "bev_fwd_kernel<4>"
    assert kernel_key("Memset (Device)") is None


def test_every_instantiation_runs(cuda, oracle_mod):
    """One call per instantiation under torch.profiler: the bev_pool kernels seen are exactly the ten."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    plan = Plan(51, list(range(1, 41)), 2 * 3 * 9 * 11, 200, True)
    shape = (2, 3, 9, 11)
    ds = {C: Dev(cuda, plan, plan.feat(C, C)) for C in (7, 80, 160, 260)}
    og = _t(cuda, np.ones((plan.cells, 80), np.float32))
    dg, fg = _nan32(cuda, plan.n_depth), _nan32(cuda, plan.n_feat * 80)
    d80 = ds[80]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for C in (7, 80, 160, 260):
            ds[C].host()                                         # <1>; warp <1>; warp <2>; <4>
        for C in (80, 160):
            ds[C].dev(shape, False)
            ds[C].dev(shape, True)
        d80.h16(shape, 256, _status(cuda))
        _check(_lib().p3d_bev_pool_v2_bkwd(_p(og), *d80._args()[:7], plan.n_int, 80, _p(dg), dg.numel(), _p(fg),
                                           fg.numel(), _stream(cuda)), "bev_pool_v2_bkwd")
        torch.cuda.synchronize()
    names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    if not names:
        pytest.skip("torch.profiler reported no CUDA kernels on this device")
    seen = {k for k in map(kernel_key, names) if k is not None}
    assert seen == EXPECTED_KERNELS, (sorted(seen ^ EXPECTED_KERNELS), sorted(set(names)))


# ------------------------------------------------------------------------------------------------- lss_depth_feat
def _depth_ulp_check(got, want):
    """test_gpu_lss.py's rules: at most 8 ulp and 99 % within 2 ulp on normal results, subnormals absolutely."""
    ulp = np.abs(got.view(np.int32).astype(np.int64) - want.view(np.int32).astype(np.int64))
    normal = want >= np.float32(2.0 ** -126)
    assert ulp[normal].max() <= 8, (ulp[normal].max(), want[normal][np.argmax(ulp[normal])])
    assert (ulp[normal] <= 2).mean() > 0.99
    assert np.abs(got - want)[~normal].max(initial=0.0) < 2.0 ** -126


def special_logits(rng, BN, D, H, W):
    """N(0, 2) logits with a flat pixel, a sharp -80..80 ramp, a pixel of +-1e4, one near -1e4 and one of -1e30 (on
    single-pixel shapes the later ones overwrite the earlier)."""
    x = rng.normal(0, 2, (BN, D, H * W)).astype(np.float32)
    specials = [np.zeros(D), np.linspace(-80, 80, D), rng.choice([-1e4, 1e4], D) + rng.normal(0, 2, D),
                -1e4 + rng.normal(0, 2, D), np.full(D, -1e30)]
    for k, v in enumerate(specials):
        x[k % BN, :, (13 * k + 5) % (H * W)] = v
    return x.reshape(BN, D, H, W)


@pytest.mark.parametrize("BN,D,H,W,C", [
    (1, 1, 1, 1, 1),
    (1, 2, 1, 31, 3),          # one partial block
    (2, 59, 1, 33, 64),        # a full block and a 1-pixel one
    (6, 118, 20, 50, 80),      # H W = 1000: 31 full blocks and 8 pixels
    (12, 59, 32, 88, 64),      # downsample 8
    (1, 382, 3, 11, 370),      # both limits, 33 pixels
])
def test_depth_feat_block_shapes(cuda, BN, D, H, W, C):
    import torch
    from oracle import lss
    from paddle3d_b200.ops import bev_pool_v2 as bp
    rng = np.random.default_rng(D * 1000 + C)
    logits = special_logits(rng, BN, D, H, W)
    tran = rng.normal(size=(BN, C, H, W)).astype(np.float32)
    guard = 32 * max(C, D)
    nd, nf = BN * D * H * W, BN * H * W * C
    dbuf, fbuf = _nan32(cuda, nd + guard), _nan32(cuda, nf + guard)
    depth, feat = bp.lss_depth_feat(_t(cuda, logits), _t(cuda, tran), dbuf[:nd].view(BN, D, H, W),
                                    fbuf[:nf].view(BN, H, W, C))
    torch.cuda.synchronize()
    assert depth.data_ptr() == dbuf.data_ptr() and feat.data_ptr() == fbuf.data_ptr()
    got = depth.cpu().numpy()
    _depth_ulp_check(got, lss.depth_softmax(logits))
    assert (np.abs(got.astype(np.float64).sum(1) - 1.0) <= D * 2.0 ** -23).all()
    assert _bits_equal(feat, lss.feat_permute(tran))
    assert torch.isnan(dbuf[nd:]).all() and torch.isnan(fbuf[nf:]).all(), "a write past the outputs"


# ------------------------------------------------------------------------------------- view transform geometries
GEOMETRIES = {
    # input (H, W), downsample, grid, C, B
    "a_320x800_d59_c64": ((320, 800), 16, dict(synth.LSS_BEVDET, depth=[1.0, 60.0, 1.0]), 64, 1),
    "b_ds8_b2": ((256, 704), 8, synth.LSS_BEVDET, 80, 2),
    "c_z8_c32": ((256, 704), 16, dict(synth.LSS_BEVDET, z=[-5.0, 3.0, 1.0]), 32, 1),
    "d_c160": ((256, 704), 16, synth.LSS_BEVDET, 160, 1),
    # BEVFusion (bevf_pp): 900 / 8 = 112.5 feature rows (floored), 41 depth bins, a 200 x 200 x 16 grid, 1024 channels
    "e_bevf_pp_900x1600_z16": ((900, 1600), 8, dict(synth.LSS_C4, z=[-5.0, 3.0, 0.5], depth=[4.0, 45.0, 1.0]), 64, 1),
}


@pytest.mark.parametrize("geom", sorted(GEOMETRIES))
def test_view_transform_geometry(cuda, oracle_mod, geom):
    """coor bit-equal to the fp32 oracle, ranks = voxel_pooling_prepare_v2 of it, depth within the ulp rules, the BEV
    and the pixel-row fp16-pair pool image (bev_pool_v2_dev_h16, the image the camera encoders read) bit-equal to the
    oracle's pool of the device's depth and feat, within 1e-4 / 1e-5 of oracle.lss.view_transform end to end, and the
    captured frame equal to the eager forward."""
    import torch
    from oracle import lss
    from paddle3d_b200.lss import LSSHotPath, LSSViewTransformer
    from paddle3d_b200.ops import bev_pool_v2 as bp
    size, ds, grid, C, B = GEOMETRIES[geom]
    vt = LSSViewTransformer(grid, size, ds, C, device=cuda)
    X, Y, Z = vt.grid
    rig = synth.camera_rig(70 + C, B=B)
    mats = synth.lss_mats(rig)
    rng = np.random.default_rng(C + B)
    logits = rng.normal(0, 2, (B * 6, vt.D, vt.H, vt.W)).astype(np.float32)
    tran = rng.normal(0, 1, (B * 6, C, vt.H, vt.W)).astype(np.float32)
    tl, tt = _t(cuda, logits), _t(cuda, tran)
    axes = tuple(a.numpy() for a in vt.axes_host)
    cams = bp.unpack_cameras(bp.pack_cameras(*mats), B, 6)
    want, coor_want, prep = lss.view_transform(cams, axes, logits, tran, *vt.grid_args())
    # geometry and ranks
    got = vt._prepare(vt.descriptor(*mats), B, 6, with_coor=True)
    assert _bits_equal(got[6], coor_want), "coor"
    k, m = [int(v) for v in got[5].cpu()]
    rb, rd, rf, st, ln = prep
    assert (k, m) == (len(rb), len(st)) and m > 0
    for g, r, name in zip(got[:5], prep, ("ranks_bev", "ranks_depth", "ranks_feat", "starts", "lengths")):
        assert np.array_equal(g[:len(r)].cpu().numpy(), r), name
    # depth, feat and the pool of the device's own depth and feat
    depth, feat = bp.lss_depth_feat(tl, tt)
    rows = bp.bev_pool_v2_dev_h16(depth, feat, got, vt.bev_feat_shape(B))
    depth, feat = depth.cpu().numpy(), feat.cpu().numpy()
    _depth_ulp_check(depth, lss.depth_softmax(logits))
    assert _bits_equal(feat, lss.feat_permute(tran))
    pool = collapse(oracle_mod.bev_pool_v2(depth, feat, rd, rf, rb, ln, st, (B, Z, Y, X, C), use_fma=True))
    assert _bits_equal(rows, pixel_rows(pool, (Z * C + 31) // 32 * 32)), "pool image != split_h16 of the oracle's pool"
    del rows
    inputs = [torch.zeros((B, 6, 1, 1, 1))] + [rig[n] for n in ("sensor2ego", "ego2global", "cam2imgs", "post_rots",
                                                                   "post_trans", "bda")]
    eager = vt.forward(inputs, tl, tt)
    torch.cuda.synchronize()
    assert eager.shape == (B, Z * C, Y, X)
    assert _bits_equal(eager, pool), "BEV != the oracle's pool of the device's depth and feat"
    np.testing.assert_allclose(eager.cpu().numpy(), want, rtol=1e-4, atol=1e-5)
    frame = LSSHotPath(vt, B, 6, device=cuda).capture()
    bev, counts = frame.infer(mats, tl, tt)
    assert counts == (k, m)
    assert _bits_equal(bev, eager.cpu().numpy()), "captured != eager"
