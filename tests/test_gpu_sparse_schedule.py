"""The sparse fp16-pair convs in every work decomposition they pick on the device, against a float64 reference.

Kernels: `f16::conv_f16_kernel` (csrc/sparse_conv_f16.cu, wgmma; no split, 2-4 tap splits or stream-K, chosen from the
device row count) and `wm::conv_wm_kernel` (csrc/sparse_conv_wm.cu, warp MMA; stream-K over warps).  Both are called
through the C ABI so that the tests control the capacity, the device count, the workspace and `max_splits` directly.

Reference: out[r] = sum_t sum_c X[nbr[r, t], c] W[t, c, :] in float64 on the device, with X the EXACT value of the
fp16-pair input rows (hi + lo' 2^-11, built here from fp32 and checked bit-equal to p3d_rows_convert_h16) and W the fp32
weight (so the weight split error is part of what is checked), then BN scale / shift, residual and ReLU in the
epilogue's order.  Every case also checks that the tolerance REJECTS two wrong answers computed from the reference: the
hi x hi products alone (cross products dropped, ~2^-12 relative) and the result with one tap dropped.

Which decomposition ran is not taken on trust: `choose_splits` / `make_sched`, the host-side split clamp of
p3d_sparse_conv_f16 and the warp ranges of conv_wm_kernel are restated here, the row counts of each regime are searched
with the restatement for this device's SM count, and after every launch the set of partial-sum slab blocks the kernel
wrote (the slab region is NaN-filled before the launch) must be exactly the one the restatement predicts.  If the two
drift apart the test fails instead of quietly covering another path.  Lines starting with "REGIME" (pytest -s) list
the decompositions each instantiation reached on the device."""
import math

import numpy as np
import pytest

from parity import rel_check

KM = 128              # rows per tile of the wgmma kernel (tc::kM)
F16_MAX_SPLITS = 4    # f16::kMaxSplits
SK_FIX = 6            # cost of a stream-K fix-up in taps (f16::kSkFix)
ALIGN = 256           # workspace region alignment (kAlign)
WM_TILE, WM_WARPS = 16, 16
LO = 2.0 ** -11       # weight of lo' in an fp16 pair

# every wgmma instantiation (Cin <= 32: two sub-tiles per stage), and the (3, 1, 1) extra conv
F16_SHAPES = [(16, 16, 27), (16, 32, 27), (32, 32, 27), (32, 64, 27), (64, 64, 27), (64, 128, 27), (128, 128, 27),
              (128, 128, 3)]
WM_SHAPES = [(16, 16, 27), (16, 32, 27), (32, 32, 27)]
F16_CAP = 40000       # capacity of the wgmma cases (313 tiles): every regime is searched below it
WM_CAP = 160000       # level-0 capacity of the full-size frame
WM_ROWS = 149997      # a warp's range spans several whole tiles; not a multiple of 16


# ----------------------------------------------------------------------------------------------- fp16 pairs and reference
def to_h16(x):
    """fp32 rows [n, C] -> fp16-pair rows [n, 2C] (DESIGN.md section 2): groups of KC = min(C, 32) channels, each
    [hi KC | lo' KC] with hi = fp16(x), lo' = fp16((x - hi) 2^11)."""
    import torch
    n, C = x.shape
    KC = min(C, 32)
    hi = x.half()
    lo = ((x - hi.float()) * 2048.0).half()
    return torch.stack([hi.view(n, C // KC, KC), lo.view(n, C // KC, KC)], 2).reshape(n, 2 * C)


def from_h16(h, C):
    """Exact value (float64) of fp16-pair rows."""
    n = h.shape[0]
    KC = min(C, 32)
    g = h.reshape(n, C // KC, 2, KC).double()
    return (g[:, :, 0] + g[:, :, 1] * LO).reshape(n, C)


def gather_gemm(X, nbr, W, taps=None):
    """out[r] = sum_t X[nbr[r, t]] @ W[t] in X's dtype; nbr [n, K], -1 = missing neighbour."""
    import torch
    n, K = nbr.shape
    out = torch.zeros((n, W.shape[2]), dtype=X.dtype, device=X.device)
    for t in (range(K) if taps is None else taps):
        idx = nbr[:, t].long()
        rows = torch.nonzero(idx >= 0).squeeze(1)
        if rows.numel():
            out.index_add_(0, rows, X[idx[rows]] @ W[t])
    return out


def epilogue(acc, scale, shift, res, relu):
    """conv * scale + shift (+ residual) (ReLU), the order of the kernels' epilogue; scale / shift None = 1 / 0."""
    o = acc
    if scale is not None:
        o = o * scale.double()
    if shift is not None:
        o = o + shift.double()
    if res is not None:
        o = o + res
    return o.clamp_min(0.0) if relu else o


def subm_rulebook_torch(coords, spatial, ksize=(3, 3, 3)):
    """SubM neighbour map [n, K] of sites coords [n, 4] (b, z, y, x): column t = (dz * kH + dy) * kW + dx holds the row
    of coord + (dz, dy, dx) - k // 2, or -1.  Sorted linear keys + searchsorted, one offset at a time."""
    import torch
    D, H, W = spatial
    c = coords.long()
    key = ((c[:, 0] * D + c[:, 1]) * H + c[:, 2]) * W + c[:, 3]
    skey, order = torch.sort(key)
    n = c.shape[0]
    cols = []
    for dz in range(ksize[0]):
        for dy in range(ksize[1]):
            for dx in range(ksize[2]):
                z, y, x = c[:, 1] + dz - ksize[0] // 2, c[:, 2] + dy - ksize[1] // 2, c[:, 3] + dx - ksize[2] // 2
                ok = (z >= 0) & (z < D) & (y >= 0) & (y < H) & (x >= 0) & (x < W)
                q = ((c[:, 0] * D + z) * H + y) * W + x
                pos = torch.searchsorted(skey, q).clamp_max(n - 1)
                hit = ok & (skey[pos] == q)
                cols.append(torch.where(hit, order[pos], torch.full_like(pos, -1)))
    return torch.stack(cols, 1).to(torch.int32)


# --------------------------------------------------------------------------------------------- schedule restatement
def _align(x):
    return (x + ALIGN - 1) // ALIGN * ALIGN


def _cdiv(a, b):
    return -(-a // b)


def choose_splits(n_tiles, grid, K, smax):
    """f16::choose_splits: minimise waves x (taps per item + fixed cost)."""
    smax = max(min(smax, K), 1)
    best, best_cost = 1, None
    for s in range(1, smax + 1):
        cost = _cdiv(n_tiles * s, grid) * (_cdiv(K, s) + 4 + (1 if s > 1 else 0))
        if best_cost is None or cost < best_cost:
            best, best_cost = s, cost
    return best


def f16_ws_layout(n_cap, cout):
    """(ticket bytes, bytes of one slab [tiles][128 rows][Cout] fp32) of p3d_sparse_conv_f16's workspace."""
    tiles = _cdiv(n_cap, KM)
    return _align(tiles * 4), tiles * KM * cout * 4


def f16_smax(K, n_cap, cout, max_splits, ws_bytes):
    """The host-side clamp of p3d_sparse_conv_f16: min(max_splits, 4, K, slabs that fit), 1 without two slabs."""
    smax = min(max_splits, F16_MAX_SPLITS, K)
    tick, slab = f16_ws_layout(n_cap, cout)
    if ws_bytes < tick + 2 * slab:  # includes the null workspace
        smax = 1
    if smax > 1:
        smax = min(smax, (ws_bytes - tick) // slab)
    return max(smax, 1)


class Sched:
    def __init__(self, stream, splits, smax, grid, n_tiles, pieces):
        self.stream, self.splits, self.smax, self.grid, self.n_tiles = stream, splits, smax, grid, n_tiles
        self.pieces = pieces  # per tile: partial sums combined through the slabs (1 = none)

    @property
    def key(self):
        if self.stream:
            return "stream%d" % int(self.pieces.max())
        return "split%d" % self.splits

    def label(self):
        if self.stream:
            return "stream-K (tiles in up to %d pieces)" % int(self.pieces.max())
        return "no split" if self.splits == 1 else "%d splits" % self.splits


def f16_sched(sms, n, n_cap, K, cout, max_splits, ws_bytes):
    """f16::launch's grid and f16::make_sched / sched_item for device row count n (clamped to n_cap)."""
    smax = f16_smax(K, n_cap, cout, max_splits, ws_bytes)
    grid = min(_cdiv(n_cap, KM) * (smax if smax > 1 else 1), sms)
    n_tiles = _cdiv(min(n, n_cap), KM)
    splits = choose_splits(n_tiles, grid, K, smax)
    total = n_tiles * K
    if smax >= 4 and total > 0:
        u_min = max((K + 1) // 3, 1)  # ceil((K - 1) / (kMaxSplits - 1))
        g = max(min(total // u_min, grid), 1)
        cost_old = _cdiv(n_tiles * splits, grid) * (_cdiv(K, splits) + 4 + (1 if splits > 1 else 0))
        if _cdiv(total, g) + 4 + SK_FIX < cost_old:
            start = np.arange(n_tiles, dtype=np.int64) * K
            cf, cl = ((start + 1) * g - 1) // total, ((start + K) * g - 1) // total
            return Sched(True, 0, smax, grid, n_tiles, cl - cf + 1)
    return Sched(False, splits, smax, grid, n_tiles, np.full(n_tiles, splits, np.int64))


def f16_expected_blocks(sc, n_slabs, tiles_cap):
    """Slab blocks [piece][tile] the launch writes: piece p of a tile cut into > 1 pieces fills slabs[p][tile]."""
    exp = np.zeros((n_slabs, tiles_cap), bool)
    for p in range(F16_MAX_SPLITS):
        m = (sc.pieces > 1) & (sc.pieces > p)
        if m.any():
            assert p < n_slabs, "restatement needs slab %d, the workspace has %d" % (p, n_slabs)
            exp[p, :sc.n_tiles] = m
    return exp


def f16_search(sms, K, n_cap, cout, max_splits, ws_bytes):
    """First tile count (<= the capacity's) of every decomposition the restatement can reach."""
    found = {}
    for t in range(1, _cdiv(n_cap, KM) + 1):
        found.setdefault(f16_sched(sms, t * KM, n_cap, K, cout, max_splits, ws_bytes).key, t)
    return found


def wm_ranges(sms, n, n_cap, K):
    """wm::launch's grid and conv_wm_kernel's stream-K split: (grid, warps W, units U, tiles)."""
    grid = max(min(sms, _cdiv(n_cap, WM_TILE * WM_WARPS)), 1)
    n_tiles = _cdiv(min(n, n_cap), WM_TILE)
    U = n_tiles * K
    W = grid * WM_WARPS
    if W > U // 8:
        W = U // 8 if U // 8 > 0 else 1
    return grid, W, U, n_tiles


def wm_expected(sms, n, n_cap, K, n_warp_slabs):
    """Per-warp slabs [warp][2] the launch writes: for a tile cut between warps cf..cl, warp cf fills [cf][1] (piece of a
    tile that continues) and warps cf + 1..cl fill [x][0] (piece of a tile begun earlier).  Also the pieces per tile."""
    grid, W, U, n_tiles = wm_ranges(sms, n, n_cap, K)
    exp = np.zeros((n_warp_slabs, 2), bool)
    if U == 0:
        return exp, np.zeros(0, np.int64), W, U
    start = np.arange(n_tiles, dtype=np.int64) * K
    cf, cl = ((start + 1) * W - 1) // U, ((start + K) * W - 1) // U
    split = cl > cf
    exp[cf[split], 1] = True
    for d in range(1, 8):
        m = split & (cf + d <= cl)
        exp[cf[m] + d, 0] = True
    return exp, cl - cf + 1, W, U


# --------------------------------------------------------------------------------------------------- case data
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class Data:
    """Seeded inputs of one (Cin, Cout, K) instantiation: `n_cap` output rows, neighbour map of the given kind
    ('lidar': ~70 % missing taps, 'full', 'empty'), and the float64 reference over the first `n_ref` rows."""

    def __init__(self, dev, cin, cout, K, n_cap, n_ref, seed, kind="lidar", wm=False):
        import torch
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        self.dev, self.cin, self.cout, self.K, self.n_cap, self.n_ref, self.kind = dev, cin, cout, K, n_cap, n_ref, kind
        g = torch.Generator().manual_seed(seed)
        n_in = n_cap + 517
        x = torch.randn(n_in, cin, generator=g)
        nbr = torch.randint(0, n_in, (n_cap, K), generator=g, dtype=torch.int32)
        if kind == "lidar":
            nbr[torch.rand(n_cap, K, generator=g) < 0.7] = -1
        elif kind == "empty":
            nbr.fill_(-1)
        w = torch.randn(K, cin, cout, generator=g) / math.sqrt(K * cin * (0.3 if kind == "lidar" else 1.0))
        self.scale = (torch.rand(cout, generator=g) + 0.5).to(dev)
        self.shift = ((torch.rand(cout, generator=g) - 0.5) * 0.4).to(dev)
        res = torch.randn(n_cap, cout, generator=g).to(dev)
        self.x, self.nbr, self.w = x.to(dev), nbr.to(dev), w.to(dev)
        self.xh, self.resh = to_h16(self.x), to_h16(res)
        self.res64 = from_h16(self.resh[:n_ref], cout)
        L = lib()
        if wm:
            nb = L.p3d_sparse_conv_wm_packed_weight_bytes(K, cin, cout)
            self.packed = torch.empty((nb,), dtype=torch.uint8, device=dev)
            check(L.p3d_sparse_conv_wm_pack_weights(ptr(self.w), K, cin, cout, ptr(self.packed), None, stream(dev)), "wm_pack")
        else:
            nb = L.p3d_sparse_conv_f16_packed_weight_bytes(K, cin, cout)
            self.packed = torch.empty((nb,), dtype=torch.uint8, device=dev)
            check(L.p3d_sparse_conv_f16_pack_weights(ptr(self.w), K, cin, cout, ptr(self.packed), None, stream(dev)),
                  "f16_pack")
        # float64 reference sums and the two wrong answers the tolerance must reject
        nb_ref = self.nbr[:n_ref]
        X, W = from_h16(self.xh, cin), self.w.double()
        self.acc = gather_gemm(X, nb_ref, W)
        self.acc_hh = gather_gemm(self.x.half().double(), nb_ref, self.w.half().double())
        present = (nb_ref >= 0).sum(0)
        self.has_taps = bool(present.sum() > 0)
        t_drop = int(present.argmax())
        self.acc_drop = self.acc - gather_gemm(X, nb_ref, W, taps=[t_drop])


def _np(t):
    return t.double().cpu().numpy()


def _verify(name, d, n, f32, h16, scale, shift, residual, relu, flagged=False):
    """Outputs of rows [0, n) against the reference (fp32 and fp16-pair outputs), the sensitivity guards, and the NaN
    sentinels of the rows at and beyond n (never written)."""
    import torch
    cout = d.cout
    assert n <= d.n_ref
    res = d.res64[:n] if residual else None
    want = epilogue(d.acc[:n], scale, shift, res, relu)
    if n:
        if not flagged:
            rel_check(name + " out_f32", _np(f32[:n]), _np(want))
            rel_check(name + " out_h16", _np(from_h16(h16[:n], cout)), _np(want))
        if d.has_taps and n >= 64 and not flagged:
            for what, acc in (("hi x hi only", d.acc_hh), ("one tap dropped", d.acc_drop)):
                wrong = epilogue(acc[:n], scale, shift, res, relu)
                with pytest.raises(AssertionError):
                    rel_check(name + " guard: " + what, _np(wrong), _np(want))
    assert torch.isnan(f32[n:]).all(), "%s: fp32 rows at or beyond the count were written" % name
    assert torch.isnan(h16[n:]).all(), "%s: fp16-pair rows at or beyond the count were written" % name
    return want


# ---------------------------------------------------------------------------------------------- wgmma kernel case
def run_f16(d, label, n_dev, n_cap, max_splits=4, ws_kind="full", residual=True, relu=True, affine=True,
            scale=None, expect=None):
    """One p3d_sparse_conv_f16 launch (fp32 and fp16-pair outputs at once) checked against the reference, the schedule
    restatement (slab fingerprint), the ticket words and a second launch on the same workspace."""
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    L, dev, cout, K = lib(), d.dev, d.cout, d.K
    sms = _sms()
    tick, slab = f16_ws_layout(n_cap, cout)
    if ws_kind == "full":
        ws_bytes = L.p3d_sparse_conv_f16_workspace_bytes(n_cap, cout, F16_MAX_SPLITS)
    elif ws_kind == "fit2":  # room for exactly two slabs although max_splits allows four
        ws_bytes = tick + 2 * slab
    else:
        ws_bytes = 0
    ws = torch.empty((max(ws_bytes, ALIGN),), dtype=torch.uint8, device=dev) if ws_bytes else None
    n_slabs = (ws_bytes - tick) // slab if ws_bytes >= tick + slab else 0
    tiles_cap = _cdiv(n_cap, KM)
    if ws is not None:
        ws[:tick].zero_()  # tickets: zero on entry
        slabs = ws[tick:tick + n_slabs * slab].view(torch.float32).view(n_slabs, tiles_cap, KM * cout)
        slabs.fill_(float("nan"))
    sc = f16_sched(sms, n_dev, n_cap, K, cout, max_splits, ws_bytes)
    if expect is not None:
        assert sc.key == expect, "%s: restatement picks %s, the case was searched for %s" % (label, sc.key, expect)
    n = min(n_dev, n_cap)
    n_t = torch.tensor([n_dev], dtype=torch.int32, device=dev)
    scale = (d.scale if scale is None else scale) if affine else None
    shift = d.shift if affine else None
    name = "f16 %d->%d K=%d %s n=%d cap=%d" % (d.cin, cout, K, label, n_dev, n_cap)

    def launch():
        f32 = torch.full((d.n_cap, cout), float("nan"), device=dev)
        h16 = torch.full((d.n_cap, 2 * cout), float("nan"), dtype=torch.float16, device=dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        check(L.p3d_sparse_conv_f16(ptr(d.xh), ptr(d.nbr), ptr(n_t), n_cap, K, d.cin, cout, ptr(d.packed), ptr(scale),
                                    ptr(shift), ptr(d.resh if residual else None), int(relu), ptr(f32), ptr(h16),
                                    ptr(ws), ws_bytes, max_splits, ptr(status), stream(dev)), name)
        torch.cuda.synchronize()
        return f32, h16, int(status[0])

    f32, h16, status = launch()
    flagged = scale is not None and bool((scale.abs() > 1e3).any())
    if ws is not None:
        assert not ws[:tick].view(torch.int32).any(), "%s: ticket words not left zero" % name
        fin, nan = torch.isfinite(slabs).all(-1), torch.isnan(slabs).all(-1)
        assert bool((fin | nan).all()), "%s: a slab block was partly written" % name
        got = fin.cpu().numpy()
        exp = f16_expected_blocks(sc, n_slabs, tiles_cap)
        assert np.array_equal(got, exp), "%s: slabs written by the kernel %s != restatement (%s) %s" % (
            name, [tuple(map(int, p)) for p in np.argwhere(got != exp)[:8]], sc.label(), "(piece, tile) differ")
    else:
        assert sc.splits == 1 and not sc.stream
    _verify(name, d, n, f32, h16, scale, shift, residual, relu, flagged)
    assert status == (1 if flagged else 0), "%s: status %d" % (name, status)
    f32b, h16b, _ = launch()
    assert torch.equal(f32.view(torch.int32), f32b.view(torch.int32)) and torch.equal(h16.view(torch.int16), h16b.view(torch.int16)), \
        "%s: second launch on the same workspace differs" % name
    print("REGIME f16 %d->%d K=%d n=%d cap=%d %-16s -> %s" % (
        d.cin, cout, K, n_dev, n_cap, label,
        sc.label() + " (slab fingerprint checked)" if ws is not None else "no split (no workspace, no slabs)"))
    return sc, f32, h16


def _check_overflow(name, d, n, f32, h16, scale, c0):
    """One channel's BN scale drives the outputs past fp16's range: the fp32 output is exact, the pair output
    saturates at +-65504 (status bit 0 checked by the caller)."""
    import torch
    want = epilogue(d.acc[:n], scale, d.shift, d.res64[:n], True)
    big = want[:, c0].abs() > 70000
    assert int(big.sum()) > 10, "%s: overflow case does not overflow" % name
    rel_check(name + " overflowing channel fp32", _np(f32[:n, c0]), _np(want[:, c0]))
    others = [c for c in range(d.cout) if c != c0]
    rel_check(name + " other channels fp32", _np(f32[:n, others]), _np(want[:, others]))
    dec = from_h16(h16[:n], d.cout)
    sat = f32[:n].double().abs() > 65504
    assert bool(sat.any())
    assert torch.equal(dec[sat], torch.sign(f32[:n].double()[sat]) * 65504.0), "%s: pair output does not saturate" % name
    keep = ~sat
    assert bool(((dec[keep] - f32[:n].double()[keep]).abs() <= f32[:n].double()[keep].abs() * 2.0 ** -21 + 2.0 ** -34).all())


# -------------------------------------------------------------------------------------------------- tests
def test_torch_reference_matches_oracle(oracle_mod):
    """CPU: the float64 gather-GEMM and the sorted-key SubM neighbour map above against the C oracle's sparse conv."""
    import torch
    rng = np.random.default_rng(12)
    B, D, H, W = 2, 7, 19, 23
    occ = rng.random((B, D, H, W)) < 0.2
    coords = np.argwhere(occ).astype(np.int32)
    rng.shuffle(coords, axis=0)
    for cin, cout in ((16, 32), (5, 16)):
        feats = rng.normal(size=(len(coords), cin)).astype(np.float32)
        w = (rng.normal(size=(3, 3, 3, cin, cout)) / math.sqrt(27 * cin)).astype(np.float32)
        nbr = subm_rulebook_torch(torch.from_numpy(coords), (D, H, W))
        got = gather_gemm(torch.from_numpy(feats).double(), nbr, torch.from_numpy(w).double().reshape(27, cin, cout))
        oc, of, osp, _ = oracle_mod.sparse_conv3d(coords, feats, B, (D, H, W), w, 1, 1, True)
        assert np.array_equal(oc, coords) and osp == [D, H, W]
        rel_check("torch reference vs oracle %d->%d" % (cin, cout), got.numpy(), of, rtol=1e-6, small_atol=1e-7)
    # every entry points at the site coord + offset
    nb = nbr.numpy()
    for t in range(27):
        off = np.array([0, t // 9 - 1, (t // 3) % 3 - 1, t % 3 - 1], np.int32)
        rows = np.nonzero(nb[:, t] >= 0)[0]
        assert np.array_equal(coords[nb[rows, t]], coords[rows] + off)
    assert (nb >= 0).sum() > 2 * len(coords)


@pytest.mark.gpu
def test_h16_rows_built_here_match_the_library(cuda):
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    g = torch.Generator().manual_seed(1)
    for C in (16, 32, 64, 128):
        x = (torch.randn(3000, C, generator=g) * torch.exp(torch.empty(3000, C).uniform_(-9, 9, generator=g))).to(cuda)
        x[0, :3] = torch.tensor([0.0, -0.0, 65504.0])
        h = torch.empty((3000, 2 * C), dtype=torch.float16, device=cuda)
        check(lib().p3d_rows_convert_h16(ptr(x), 1, None, 3000, C, ptr(h), None, stream(cuda)), "to_h16")
        assert torch.equal(to_h16(x).view(torch.int16), h.view(torch.int16))
        assert bool(((from_h16(h, C) - x.double()).abs() <= x.double().abs() * 2.0 ** -21 + 2.0 ** -34).all())


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,K", F16_SHAPES)
def test_f16_every_schedule(cuda, cin, cout, K):
    """p3d_sparse_conv_f16 in every decomposition the restatement finds below F16_CAP rows on this device: no split,
    2 / 3 / 4 tap splits and stream-K at the automatic cost model; the caps of max_splits 1 / 2 / 3, of a workspace with
    room for two slabs and of a null workspace; counts of 0, above the capacity and equal to a one-tile capacity;
    all-present and all-missing neighbour maps; an fp16 range overflow under split-K and stream-K."""
    import torch
    from paddle3d_b200._lib import lib
    sms = _sms()
    ws_full = lib().p3d_sparse_conv_f16_workspace_bytes(F16_CAP, cout, F16_MAX_SPLITS)
    found = f16_search(sms, K, F16_CAP, cout, F16_MAX_SPLITS, ws_full)

    def rows(t):  # t tiles, never a multiple of 128 rows
        return t * KM - 37

    stream_key = max((k for k in found if k.startswith("stream")), default=None)  # tiles cut the finest
    if K == 27:
        assert {"split1", "split2", "split3", "split4"} <= set(found) and stream_key, found
    else:
        assert stream_key is None and {"split1", "split3"} <= set(found), found
    t_busy = found[stream_key] if stream_key else found["split3"]
    n_ref = max(rows(t) for t in found.values())
    d = Data(cuda, cin, cout, K, F16_CAP, n_ref, seed=cin * 1000 + cout * 10 + K)
    for key, t in sorted(found.items()):
        run_f16(d, key, rows(t), F16_CAP, expect=key)
    # caps where the uncapped choice is stream-K and where it is the most splits
    for t in sorted({t_busy, found["split4" if K == 27 else "split3"]}):
        for ms in (1, 2, 3):
            sc, _, _ = run_f16(d, "max_splits=%d" % ms, rows(t), F16_CAP, max_splits=ms)
            assert sc.smax == min(ms, K) and not sc.stream
        sc, _, _ = run_f16(d, "two-slab workspace", rows(t), F16_CAP, ws_kind="fit2")
        assert sc.smax == 2 and not sc.stream
        run_f16(d, "null workspace", rows(t), F16_CAP, ws_kind="null")
    # counts: none, above the capacity (clamped), capacity of one tile (grid of four CTAs); plain conv epilogue
    run_f16(d, "n=0", 0, F16_CAP)
    run_f16(d, "count above capacity", 10 ** 6, rows(t_busy), residual=False, relu=False, affine=False)
    sc, _, _ = run_f16(d, "one-tile capacity", 91, 91)
    assert sc.grid == min(4, K) and sc.splits == min(4, K)
    # overflow of one channel under split-K and stream-K
    c0 = cout // 3
    for key in ("split4" if K == 27 else "split3", stream_key):
        if key is None:
            continue
        big = d.scale.clone()
        big[c0] = 2.0e6
        n = rows(found[key])
        _, f32, h16 = run_f16(d, "overflow " + key, n, F16_CAP, scale=big, expect=key)
        _check_overflow("f16 %d->%d %s overflow" % (cin, cout, key), d, n, f32, h16, big, c0)
    del d
    # all-present and all-missing maps where the work is cut the finest
    for kind in ("full", "empty"):
        n = rows(t_busy)
        dk = Data(cuda, cin, cout, K, F16_CAP, n, seed=cin + cout + K + 7, kind=kind)
        run_f16(dk, kind + " map", n, F16_CAP)
        torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- warp-MMA kernel case
def run_wm(d, label, n_dev, n_cap, residual=True, relu=True, affine=True, scale=None):
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    L, dev, cout, K = lib(), d.dev, d.cout, d.K
    sms = _sms()
    ws_bytes = L.p3d_sparse_conv_wm_workspace_bytes(n_cap, cout)
    tick = _align(_cdiv(n_cap, WM_TILE) * 4)
    n_ws = sms * WM_WARPS
    assert ws_bytes == tick + _align(n_ws * 2 * 16 * cout * 4)
    ws = torch.empty((ws_bytes,), dtype=torch.uint8, device=dev)
    ws[:tick].zero_()
    slabs = ws[tick:tick + n_ws * 2 * 16 * cout * 4].view(torch.float32).view(n_ws, 2, 16 * cout)
    slabs.fill_(float("nan"))
    exp, pieces, W, U = wm_expected(sms, n_dev, n_cap, K, n_ws)
    n = min(n_dev, n_cap)
    n_t = torch.tensor([n_dev], dtype=torch.int32, device=dev)
    scale = (d.scale if scale is None else scale) if affine else None
    shift = d.shift if affine else None
    name = "wm %d->%d K=%d %s n=%d cap=%d" % (d.cin, cout, K, label, n_dev, n_cap)

    def launch():
        f32 = torch.full((d.n_cap, cout), float("nan"), device=dev)
        h16 = torch.full((d.n_cap, 2 * cout), float("nan"), dtype=torch.float16, device=dev)
        status = torch.zeros((1,), dtype=torch.int32, device=dev)
        check(L.p3d_sparse_conv_wm(ptr(d.xh), ptr(d.nbr), ptr(n_t), n_cap, K, d.cin, cout, ptr(d.packed), ptr(scale),
                                   ptr(shift), ptr(d.resh if residual else None), int(relu), ptr(f32), ptr(h16), ptr(ws),
                                   ws_bytes, ptr(status), stream(dev)), name)
        torch.cuda.synchronize()
        return f32, h16, int(status[0])

    f32, h16, status = launch()
    flagged = scale is not None and bool((scale.abs() > 1e3).any())
    assert not ws[:tick].view(torch.int32).any(), "%s: ticket words not left zero" % name
    fin, nan = torch.isfinite(slabs).all(-1), torch.isnan(slabs).all(-1)
    assert bool((fin | nan).all()), "%s: a warp slab was partly written" % name
    got = fin.cpu().numpy()
    assert np.array_equal(got, exp), "%s: warp slabs written %s != restatement (W=%d, U=%d)" % (
        name, [tuple(map(int, p)) for p in np.argwhere(got != exp)[:8]], W, U)
    _verify(name, d, n, f32, h16, scale, shift, residual, relu, flagged)
    assert status == (1 if flagged else 0), "%s: status %d" % (name, status)
    f32b, h16b, _ = launch()
    assert torch.equal(f32.view(torch.int32), f32b.view(torch.int32)) and torch.equal(h16.view(torch.int16), h16b.view(torch.int16)), \
        "%s: second launch on the same workspace differs" % name
    mp = int(pieces.max()) if pieces.size else 0
    print("REGIME wm %d->%d K=%d n=%d cap=%d %-22s -> %d warps, %.1f units per warp, tiles in up to %d pieces "
          "(slab fingerprint checked)" % (d.cin, cout, K, n_dev, n_cap, label, W, U / W if U else 0.0, mp))
    return W, U, pieces, f32, h16


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,K", WM_SHAPES)
def test_wm_frame_scale(cuda, cin, cout, K):
    """p3d_sparse_conv_wm at the full frame's level-0 size (a warp's range spans several whole tiles and its register
    ring prefetches across them), with the warp count capped at U / 8 (tiles in five pieces), a one-block capacity, a
    count above the capacity, no rows, all-present / all-missing maps and an fp16 range overflow."""
    import torch
    sms = _sms()
    d = Data(cuda, cin, cout, K, WM_CAP, WM_ROWS, seed=cin * 31 + cout, wm=True)
    W, U, pieces, _, _ = run_wm(d, "frame scale", WM_ROWS, WM_CAP)
    assert U / W >= 2 * K and WM_ROWS % 16, (W, U)  # whole tiles inside one warp's range
    grid = wm_ranges(sms, 4997, WM_CAP, K)[0]
    W, U, pieces, _, _ = run_wm(d, "warps capped at U/8", 4997, WM_CAP)
    assert W == U // 8 < grid * WM_WARPS and int(pieces.max()) == 5, (W, U, grid)
    run_wm(d, "one-block capacity", 250, 250)
    run_wm(d, "count above capacity", 10 ** 6, 3001, residual=False, relu=False, affine=False)
    run_wm(d, "n=0", 0, WM_CAP)
    big = d.scale.clone()
    c0 = cout // 3
    big[c0] = 2.0e6
    for n in (4997, WM_ROWS):
        _, _, _, f32, h16 = run_wm(d, "overflow", n, WM_CAP, scale=big)
        _check_overflow("wm %d->%d overflow n=%d" % (cin, cout, n), d, n, f32, h16, big, c0)
    del d
    for kind in ("full", "empty"):
        dk = Data(cuda, cin, cout, K, 40000, 40000 - 5, seed=cin + cout + 3, kind=kind, wm=True)
        run_wm(dk, kind + " map", 40000 - 5, 40000)
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------------- full-size layer and rulebook
@pytest.mark.gpu
def test_full_size_subm_layer_and_rulebook(cuda, oracle_mod):
    """One SubM 64 -> 64 + BN + residual + ReLU layer through sparse_nn (fp16 pairs) on ~60k lidar sites against the C
    oracle; the library's SubM rulebook against a sorted-key one built here; the float64 reference against the oracle."""
    import torch
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import sparse_nn as sp
    cfg = synth.C3
    pts = synth.lidar_cloud(cfg, 21, num_points=250000)
    lo, vs = np.asarray(cfg["point_cloud_range"][:3]), np.asarray(cfg["voxel_size"])
    grid = np.round((np.asarray(cfg["point_cloud_range"][3:]) - lo) / vs).astype(np.int64)  # x, y, z
    ijk = np.floor((pts[:, :3] - lo) / vs).astype(np.int64)
    ijk = ijk[((ijk >= 0) & (ijk < grid)).all(1)]
    sites = np.unique(ijk, axis=0)
    rng = np.random.default_rng(21)
    rng.shuffle(sites, axis=0)
    assert len(sites) >= 60000, len(sites)
    sites = sites[:60000]
    coords = np.concatenate([np.zeros((len(sites), 1), np.int64), sites[:, ::-1]], 1).astype(np.int32)  # b, z, y, x
    spatial = [int(grid[2]), int(grid[1]), int(grid[0])]
    n = len(coords)
    feats = rng.normal(size=(n, 64)).astype(np.float32)
    conv = sp.SubmConv3D(64, 64, 3, padding=1, bias_attr=False, key="full").init_parameters(rng, cuda)
    conv.precision = sp.F16X3
    bn = sp.BatchNorm(64, epsilon=1e-3).init_parameters(rng, cuda, randomize=True)
    x = sp.sparse_coo_tensor(torch.from_numpy(coords).to(cuda).t(), torch.from_numpy(feats).to(cuda), [1] + spatial + [64])
    y = sp.ReLU()(sp.add(bn(conv(x)), x))
    got = y.values()[:n].cpu().numpy()
    mine = subm_rulebook_torch(torch.from_numpy(coords).to(cuda), spatial)
    lib_nbr = x.index.subm_rulebook([3, 3, 3], "full")[:n]
    assert torch.equal(mine, lib_nbr), "SubM rulebook differs from the sorted-key map at %d sites" % n
    assert float((mine >= 0).float().mean()) > 0.1  # surface-like occupancy, not isolated points
    w = conv.weight.cpu().numpy()
    oc, of, _, _ = oracle_mod.sparse_conv3d(coords, feats, 1, spatial, w, 1, 1, True)
    assert np.array_equal(oc, coords)
    acc = gather_gemm(torch.from_numpy(feats).to(cuda).double(), mine, conv.weight.double().reshape(27, 64, 64))
    rel_check("fp64 reference vs oracle at %d sites" % n, acc.cpu().numpy(), of, rtol=1e-6, small_atol=1e-7)
    want = oracle_mod.bn_relu(of, bn.weight.cpu().numpy(), bn.bias.cpu().numpy(), bn._mean.cpu().numpy(),
                              bn._variance.cpu().numpy(), 1e-3, relu=True, residual=feats)
    rel_check("sparse_nn SubM 64->64 + BN + residual + ReLU, %d sites" % n, got, want)
