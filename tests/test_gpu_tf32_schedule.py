"""The tf32-pair convs in every work decomposition they run on the device, against a float64 reference.

These kernels keep the fp32 range: a model whose activations leave fp16's range is sent to them, so no other GPU path
can cross-check their results.  Kernels, called through the C ABI so that the tests control the capacity, the device
row count, the workspace, the N tile and the output buffers:
  `tc::gather_gemm_tf32_kernel<CIN, COUT, SPLIT_ROWS>` + `tc::rows_finalize_kernel` (csrc/sparse_conv_tc.cu;
      p3d_sparse_conv_gather_gemm_tf32x3_ws on fp32 rows, p3d_sparse_conv_gather_gemm_split_ws on split rows),
  `dc::dense_conv_kernel<N>` (csrc/dense_conv_tc.cu; p3d_dense_conv2d_split),
  `head_final_conv_kernel` (csrc/head_final_conv.cu; p3d_head_final_conv).
Both wgmma kernels launch grid = min(items, MIN_CTAS x SMs) persistent CTAs that walk their items round robin, so the
ring position carried across items, the neighbour-map barrier parity and the issue-ahead across item boundaries only
run when a CTA takes a second item.

Reference: float64 on the device from X = hi + lo of the split input (exact) and the fp32 weight (so the weight split
error is part of what is checked), then the epilogue in the kernels' order.  The split itself (`split_tf32`: cvt.rna.tf32,
10 mantissa bits, ties away from zero; lo the same rounding of x - hi) is restated in torch and checked bit-equal to the
library's converters.  Bars: the sparse convs use tests/parity.py's (1e-4 relative above 1e-2 x max, 2e-6 x max below), the
dense and head convs test_gpu_dense_schedule.bar per batch image.  Every case also shows that its bar REJECTS the hi x hi
products alone and the result without one tap (for the split-K sparse convs a tap split 1 owns; for 1x1 and transposed
convs one 32-channel input group; for the head convs the input's hi halves alone).  "BAR" lines (pytest -s) print the
measured error of every check.  Measured on an NVIDIA H100 80GB HBM3 at a 700 W power limit, the same bars as the
fp16-pair kernels hold with room to spare: relative error above the floor at most 1.7e-5 (sparse convs, all cases),
2.1e-5 (dense regime cases), 4.4e-5 (full-size layers), 3.3e-5 (the chained C3 head) and 4.1e-5 (head output convs);
below the floor at most 2.0e-7 / 2.8e-7 / 5.9e-7 / 5.0e-7 / 4.8e-7 x max; std of the error at most 1.4e-7 x max.  These
figures are for the per-tap fp32 totals of the hi x hi products (csrc/sparse_conv_tc.cu, csrc/dense_conv_tc.cu).  With
one tensor-core accumulator over a whole item, the unsplit sparse 128 -> 128 K = 27 conv reached 1.5e-4 (64 -> 128:
1.1e-4) and the dense 128 -> 128 layers 1.1e-4, over the 1e-4 bar.

Which decomposition ran is not taken on trust: the `Cfg` tables, the split-K choice, the grids, the item walk and the
ring start slots of CTA 0 are restated here, the cases are searched with the restatement for this device's SM count,
and the sparse convs' split-K slabs are NaN-filled before every launch: the rows the launch writes must be exactly the
ones the restatement predicts.  "REGIME" lines list the decompositions reached."""
import functools
import math

import numpy as np
import pytest

from test_gpu_dense_schedule import C3_LAYERS, PP_LAYERS, _bits_equal, bar, conv_ref, rel_check_dev
from test_gpu_sparse_schedule import epilogue, gather_gemm, subm_rulebook_torch

KM = 128                # rows of a sparse tile (tc::kM)
TW, TH = 16, 8          # dense output tile (dc::kTW x dc::kTH)
SPARSE_SHAPES = [(16, 16, 27), (16, 32, 27), (32, 32, 27), (32, 64, 27), (64, 64, 27), (64, 128, 27), (128, 128, 27),
                 (128, 128, 3)]
N_MAX_TILES = 4000      # synthetic neighbour maps cover this many 128-row tiles; the searches stay below it
SPARSE_TERMS = 0        # rel_check_dev's bar for sums under 2048 terms == tests/parity.py's defaults
SENTINEL = 7.0


def _cdiv(a, b):
    return -(-a // b)


# ---------------------------------------------------------------------------------------------------- tf32 split
def tf32_rna(x):
    """cvt.rna.tf32.f32 on fp32 x: round to 10 mantissa bits, ties away from zero (low 13 bits cleared)."""
    import torch
    b = x.contiguous().view(torch.int32)
    return ((b + 0x1000) & -0x2000).view(torch.float32)


def split_tf32(x):
    """tc::split_tf32: hi = rna(x), lo = rna(x - hi) (x - hi is exact in fp32)."""
    hi = tf32_rna(x)
    return hi, tf32_rna(x - hi)


def split_rows(x):
    """fp32 rows [n, C] -> split rows [n, 2C] = [hi C | lo C]."""
    import torch
    hi, lo = split_tf32(x)
    return torch.cat([hi, lo], 1).contiguous()


def from_split(s, C, hi_only=False):
    """Exact value (float64) of split rows [n, 2C] (or wider: the first 2C columns of a row of C channels)."""
    s = s.double()
    return s[:, :C] if hi_only else s[:, :C] + s[:, C:2 * C]


def to_pixel_split(x):
    """fp32 NCHW -> pixel split rows [B*H*W, 2C]."""
    B, C, H, W = x.shape
    return split_rows(x.permute(0, 2, 3, 1).reshape(-1, C))


def from_pixel_split(img, B, H, W, C, hi_only=False):
    """Exact value (float64, NHWC) of pixel split rows of C channels."""
    return from_split(img[:B * H * W], C, hi_only).reshape(B, H, W, C)


# --------------------------------------------------------------------------------------------- Cfg restatements
def sparse_cfg(cin, cout, split_rows_):
    """tc::Cfg<CIN, COUT, SPLIT_ROWS> and tc::splits_for: (KC, STAGES, MIN_CTAS, splits)."""
    kc = 32 if split_rows_ and cin >= 32 else 16
    stage = 2 * kc * KM * 4 + 2 * kc * cout * 4
    min_ctas = 2 if cout <= 64 else 1
    s_raw = (96 * 1024 if cout <= 64 else 192 * 1024) // stage
    return kc, 8 if s_raw > 8 else (3 if s_raw < 3 else s_raw), min_ctas, 2 if cout >= 64 else 1


def dense_cfg(n_tile):
    """dc::Cfg<N>: (STAGES, MIN_CTAS)."""
    stage = 2 * 32 * KM * 4 + 2 * 32 * n_tile * 4
    s_raw = (100 * 1024 if n_tile <= 64 else 192 * 1024) // stage
    return 8 if s_raw > 8 else (2 if s_raw < 2 else s_raw), 2 if n_tile <= 64 else 1


# ------------------------------------------------------------------------------------------------ sparse plan
@functools.lru_cache(maxsize=4)
def synth_presence(K, seed):
    """Present entries [N_MAX_TILES * 128, K] of a synthetic neighbour map whose per-tile tap sets vary: each tile uses a
    random subset of 0..K taps (every seventh tile only even taps, so split 1 of a split-K item has no use), a row keeps
    40 % of its tile's taps, and every ninth row has no neighbour.  A prefix of it is the map of a smaller capacity."""
    rng = np.random.default_rng(seed)
    tiles = N_MAX_TILES
    pop = rng.integers(0, K + 1, tiles)
    mask = np.argsort(rng.random((tiles, K)), 1) < pop[:, None]
    mask[3::7, 1::2] = False  # 7: no divisor of the SM counts, so CTAs striding over tiles meet these and others
    present = np.repeat(mask, KM, 0) & (rng.random((tiles * KM, K)) < 0.4)
    present[5::9] = False
    row_bits = (present.astype(np.int64) << np.arange(K, dtype=np.int64)).sum(1)
    tile_bits = np.bitwise_or.reduce(row_bits.reshape(tiles, KM), 1)
    return present, row_bits, tile_bits


def synth_nbr(K, seed, rows, n_in):
    """The map's first `rows` rows with sources in [0, n_in): random rows, one input row repeated at all taps of every
    13th row, the last input row at every 17th row's taps."""
    present = synth_presence(K, seed)[0][:rows]
    rng = np.random.default_rng(seed + 1)
    src = rng.integers(0, n_in, (rows, K), dtype=np.int64)
    src[2::13] = src[2::13, :1]
    src[4::17] = n_in - 1
    return np.where(present, src, -1).astype(np.int32)


def tile_masks(K, seed, n):
    """Active-tap bit masks of the tiles of the first n rows (the last tile's from its rows below n)."""
    _, row_bits, tile_bits = synth_presence(K, seed)
    t = _cdiv(n, KM)
    m = tile_bits[:t].copy()
    if n % KM:
        m[t - 1] = np.bitwise_or.reduce(row_bits[(t - 1) * KM:n])
    return m


class SparsePlan:
    """What p3d_sparse_conv_gather_gemm(_split)_ws launches: split-K taken or not, grid, and the walk of CTA 0 (and of
    CTA 1, which takes the split-1 items under split-K): per item (tile, split, uses, start slot gu % S, full-barrier
    parity of that slot, neighbour-map barrier parity)."""

    def __init__(self, sms, cin, cout, K, split_rows_, n_cap, n_dev, ws_bytes, masks):
        self.kc, self.S, self.min_ctas, s = sparse_cfg(cin, cout, split_rows_)
        self.G = cin // self.kc
        s = min(s, K)
        self.need = s * n_cap * cout * 4
        self.split = s > 1 and ws_bytes is not None and ws_bytes >= self.need
        self.splits = s if self.split else 1
        self.grid = min(_cdiv(n_cap, KM) * self.splits, self.min_ctas * sms)
        self.n = min(n_dev, n_cap)
        self.n_work = _cdiv(self.n, KM) * self.splits
        self.walks = {}
        for c in (0, 1) if self.splits > 1 else (0,):
            gu, walk = 0, []
            for i, w in enumerate(range(c, self.n_work, self.grid)):
                tile, sp = divmod(w, self.splits)
                own = sum(1 << t for t in range(sp, K, self.splits))
                uses = bin(int(masks[tile]) & own).count("1") * self.G
                walk.append((tile, sp, uses, gu % self.S, (gu // self.S) & 1, i & 1))
                gu += uses
            self.walks[c] = walk
        self.reachable = list(range(0, self.S, math.gcd(self.G, self.S)))

    def starts(self, c=0):
        return sorted({it[3] for it in self.walks[c]})

    def covered(self):
        """Every CTA walked takes >= 3 items and they start at every ring slot the per-item use counts can reach
        (uses are multiples of G = Cin / KC, so only the multiples of gcd(G, STAGES) are)."""
        return all(len(w) >= 3 and self.starts(c) == self.reachable for c, w in self.walks.items())

    def describe(self):
        s = "%s, grid %d, %d items (%.2f per CTA)" % ("split-K x%d" % self.splits if self.split else "no split",
                                                       self.grid, self.n_work, self.n_work / max(self.grid, 1))
        for c, w in self.walks.items():
            s += "; CTA %d: %d items, uses %s, start slots %s of %d (reachable %s), parities %s" % (
                c, len(w), [it[2] for it in w][:12], self.starts(c), self.S, self.reachable,
                sorted({it[4] for it in w}))
        return s


def sparse_search(sms, cin, cout, K, seed, regime):
    """(n_dev, n_cap) of a regime: 'multi' the fewest tiles at which both layouts, with split-K where the layer has it,
    cover their ring slots (Plan.covered); 'few' fewer items than CTAs.  n_dev is no multiple of 128, n_cap 300 rows
    above it."""
    wide = min(sparse_cfg(cin, cout, False)[3], K) > 1
    if regime == "few":
        n_dev = 20 * KM - 37
        return n_dev, n_dev + 300
    for t in range(3, N_MAX_TILES - 4):
        n_dev = t * KM - 37
        n_cap = n_dev + 300
        masks = tile_masks(K, seed, n_dev)
        ok = True
        for lay in (False, True):
            p = SparsePlan(sms, cin, cout, K, lay, n_cap, n_dev, 1 << 62 if wide else None, masks)
            if not p.covered():
                ok = False
                break
        if ok:
            return n_dev, n_cap
    return None


def _seed(cin, cout, K):
    return cin * 1000 + cout * 10 + K


# ------------------------------------------------------------------------------------------------- dense plan
class DensePlan:
    """What p3d_dense_conv2d_split launches: items, grid, and for CTA 0 the decoded items (N tile, tap, tile x, tile y,
    batch) and the ring slot each starts at."""

    def __init__(self, sms, B, H, W, cin, cout, n_tile, k, stride, pad, up):
        self.S, self.min_ctas = dense_cfg(n_tile)
        if up > 1:
            self.oH, self.oW, self.out_H, self.out_W = H, W, H * up, W * up
        else:
            self.oH, self.oW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
            self.out_H, self.out_W = self.oH, self.oW
        self.up2 = up * up if up > 1 else 1
        self.n_nt = _cdiv(cout, n_tile)
        self.tiles_x, self.tiles_y = _cdiv(self.oW, TW), _cdiv(self.oH, TH)
        self.items = B * self.tiles_y * self.tiles_x * self.n_nt * self.up2
        self.grid = min(self.items, self.min_ctas * sms)
        self.n_uses = (1 if up > 1 else k * k) * (cin // 32)
        self.n0 = _cdiv(self.items, self.grid)
        self.cta0 = [self.decode(i * self.grid) for i in range(self.n0)]
        self.starts = sorted({i * self.n_uses % self.S for i in range(self.n0)})

    def decode(self, q):
        """dc::decode: N tile fastest, then tap (transposed conv), x, y, batch."""
        nt = q % self.n_nt
        q //= self.n_nt
        tap = q % self.up2
        q //= self.up2
        return nt, tap, q % self.tiles_x, (q // self.tiles_x) % self.tiles_y, q // (self.tiles_x * self.tiles_y)

    def varies(self, field):
        v = [it[field] for it in self.cta0]
        return any(a != b for a, b in zip(v, v[1:]))

    def describe(self):
        return "items %d, grid %d (S %d, MIN_CTAS %d), %.2f items/CTA (CTA 0: %d), %d uses/item, start slots %s of %d" % (
            self.items, self.grid, self.S, self.min_ctas, self.items / self.grid, self.n0, self.n_uses, self.starts,
            self.S)


# (label, N tile, regime, B, cin, N tiles used, k, stride, pad, up): 3x3 s1, 3x3 s2 on odd sizes, 1x1, transposed
# k = s = 2 and 4; per-item uses coprime to the ring depth (Cin 32 / 96 / 160 on the 2-slot rings, 1x1 and transposed
# convs with 1, 2 or 5 channel groups on the 3-slot ring).  R2 needs an odd item count, so B = 1 and no transposed
# conv there.
DENSE_CASES = [
    ("N16 R1 3x3 s1", 16, "R1", 2, 32, 1, 3, 1, 1, 1),
    ("N16 R2 3x3 s2", 16, "R2", 1, 96, 1, 3, 2, 1, 1),
    ("N16 R3 3x3 s2", 16, "R3", 2, 96, 5, 3, 2, 1, 1),
    ("N64 R1 1x1", 64, "R1", 2, 64, 1, 1, 1, 0, 1),
    ("N64 R2 3x3 s1", 64, "R2", 1, 96, 1, 3, 1, 1, 1),
    ("N64 R3 up2", 64, "R3", 2, 160, 5, 2, 2, 0, 2),
    ("N64 R3 3x3 s1", 64, "R3", 2, 32, 7, 3, 1, 1, 1),
    ("N128 R1 3x3 s1", 128, "R1", 2, 64, 1, 3, 1, 1, 1),
    ("N128 R2 3x3 s2", 128, "R2", 1, 32, 1, 3, 2, 1, 1),
    ("N128 R3 1x1", 128, "R3", 2, 160, 5, 1, 1, 0, 1),
    ("N128 R3 up4", 128, "R3", 2, 64, 5, 4, 4, 0, 4),
]


def _dense_cout(n_tile, n_nt):
    return n_nt * n_tile - (16 if n_tile > 16 else 0)


def dense_search(sms, case):
    """(H, W, plan) of a case: output sides that are no multiple of 8 / 16 (ragged tiles); R1 the most items below the
    grid's slots, R2 exactly MIN_CTAS x SMs + 1 items, R3 the fewest items with >= 4 on every CTA, a ragged last round,
    every ring slot as a start slot and the N tile, the batch (and the tap) changing between CTA 0's items."""
    _, nt, regime, B, cin, n_nt, k, stride, pad, up = case
    cout = _dense_cout(nt, n_nt)
    S, mc = dense_cfg(nt)
    slots = mc * sms
    up2 = up * up if up > 1 else 1
    best = None
    for ty in range(1, 120):
        for tx in range(1, 260):  # R2 at 114 SMs: 229 items, a prime
            items = B * ty * tx * n_nt * up2
            if (regime == "R1" and items >= slots) or (regime == "R2" and items != slots + 1) or (
                    regime == "R3" and (items < 4 * slots or (best is not None and items >= best[0]))):
                continue
            oh, ow = TH * ty - 3, TW * tx - 5
            h, w = (oh, ow) if up > 1 else ((oh - 1) * stride + k - 2 * pad, (ow - 1) * stride + k - 2 * pad)
            if h < 1 or w < 1:
                continue
            p = DensePlan(sms, B, h, w, cin, cout, nt, k, stride, pad, up)
            assert (p.oH, p.oW, p.items) == (oh, ow, items)
            if regime == "R3" and not (items % p.grid and p.starts == list(range(S)) and p.varies(0) and p.varies(4)
                                       and (up2 == 1 or p.varies(1))):
                continue
            key = -items if regime == "R1" else items
            if best is None or key < best[0]:
                best = (key, (h, w, p))
    return None if best is None else best[1]


# (label, B, H, W, cin, groups, extra input channels): groups 1 / 36 / 64, Cin 4 / 32 / 64 / 96 / 128, sides no multiple
# of 8 / 16, the C3 head's 36 groups x 64 channels at 180 x 180
HEAD_CASES = [
    ("g1 cin4", 2, 13, 21, 4, 1, 12),
    ("g64 cin32", 2, 37, 45, 32, 64, 32),
    ("g36 cin64 180x180", 2, 180, 180, 64, 36, 32),
    ("g5 cin96", 2, 27, 35, 96, 5, 64),
    ("g3 cin128", 2, 20, 50, 128, 3, 16),
]


# -------------------------------------------------------------------------------------------------- checks
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def check(name, got, want, terms):
    """rel_check_dev on one tensor, with a "BAR" line of the measured error."""
    got, want = got.double(), want.double()
    scale = float(want.abs().max())
    if scale > 0.0:
        floor, small_atol = bar(terms)
        err = (got - want).abs()
        big = want.abs() > floor * scale
        rel = float((err[big] / want[big].abs()).max()) if bool(big.any()) else 0.0
        small = float(err[~big].max()) / scale if bool((~big).any()) else 0.0
        print("BAR %s (%d terms): rel above %.0e x max %.2e (bar 1e-4), below it %.2e x max (bar %.0e), std %.2e x max"
              % (name, terms, floor, rel, small, small_atol, float(err.std()) / scale))
    rel_check_dev(name, got, want, terms)


def rejects(name, wrongs, want, terms, per_image=False):
    """The bar fails each wrong answer."""
    for what, wrong in wrongs:
        with pytest.raises(AssertionError):
            for b in range(want.shape[0]) if per_image else (None,):
                rel_check_dev("%s guard: %s" % (name, what), wrong if b is None else wrong[b],
                              want if b is None else want[b], terms)


def check_images(name, got, want, terms):
    for b in range(want.shape[0]):
        check("%s [b%d]" % (name, b), got[b], want[b], terms)


# ------------------------------------------------------------------------------------------------- CPU tests
def test_split_tf32_restatement():
    """Ties away from zero at 10 mantissa bits, lo the rounding of x - hi, hi + lo within 2^-21 relative."""
    import torch
    u = 2.0 ** -10
    x = torch.tensor([1 + u / 2, -(1 + u / 2), 1 + u / 2 - 2.0 ** -23, 1 + 3 * u / 2, 0.0, -0.0, 3.0e38, -1.5e-30],
                     dtype=torch.float32)
    hi, lo = split_tf32(x)
    assert hi[:4].tolist() == [1 + u, -(1 + u), 1.0, 1 + 2 * u]
    # x - hi = 2^-11 - 2^-23 needs 11 mantissa bits: lo rounds it (a tie) away from zero, so hi + lo != x
    assert lo[2].item() == u / 2 and lo[3].item() == -u / 2
    assert torch.equal(hi[4:6].view(torch.int32), x[4:6].view(torch.int32))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(100000, generator=g) * torch.exp(torch.empty(100000).uniform_(-20, 20, generator=g))
    hi, lo = split_tf32(x)
    assert not bool((hi.view(torch.int32) & 0x1fff).any()) and not bool((lo.view(torch.int32) & 0x1fff).any())
    x64 = x.double()
    assert bool(((hi.double() - x64).abs() <= x64.abs() * 2.0 ** -11).all())
    assert bool(((hi.double() + lo.double() - x64).abs() <= x64.abs() * 2.0 ** -21).all())
    assert torch.equal(hi + lo, (hi.double() + lo.double()).float())  # hi + lo is exact in fp32


def test_restated_cfg_tables():
    """tc::Cfg and dc::Cfg as the kernels' tables list them (a change of the shared-memory plan shows here first)."""
    want = {(16, 16): ((16, 5, 2, 1), (16, 5, 2, 1)), (16, 32): ((16, 4, 2, 1), (16, 4, 2, 1)),
            (32, 32): ((16, 4, 2, 1), (32, 3, 2, 1)), (32, 64): ((16, 4, 2, 2), (32, 3, 2, 2)),
            (64, 64): ((16, 4, 2, 2), (32, 3, 2, 2)), (64, 128): ((16, 6, 1, 2), (32, 3, 1, 2)),
            (128, 128): ((16, 6, 1, 2), (32, 3, 1, 2))}
    assert {k: (sparse_cfg(*k, False), sparse_cfg(*k, True)) for k in want} == want
    assert {n: dense_cfg(n) for n in (16, 64, 128)} == {16: (2, 2), 64: (2, 2), 128: (3, 1)}


def test_sparse_plan_by_hand():
    """The split-K choice at need and need - 1 bytes, the grid cap, the item -> (tile, split) walk and the start slots
    on a hand-built three-tile map."""
    masks = np.array([0b1111, 0b0101, 0b0010], np.int64)  # taps 0-3 | only even taps | only tap 1
    p = SparsePlan(2, 64, 128, 4, True, 3 * KM - 5, 3 * KM - 5, 2 * (3 * KM - 5) * 128 * 4, masks)
    assert p.split and p.splits == 2 and p.grid == 2 and p.n_work == 6 and (p.S, p.G) == (3, 2)
    # CTA 0: items 0, 2, 4 = split 0 of tiles 0, 1, 2: uses 2 x popcount(mask & 0b0101) = 4, 4, 0
    assert [it[:5] for it in p.walks[0]] == [(0, 0, 4, 0, 0), (1, 0, 4, 1, 1), (2, 0, 0, 2, 0)]
    # CTA 1: split 1 of each tile: 4, 0 (only even taps), 2
    assert [it[:4] for it in p.walks[1]] == [(0, 1, 4, 0), (1, 1, 0, 1), (2, 1, 2, 1)]
    q = SparsePlan(2, 64, 128, 4, True, 3 * KM - 5, 3 * KM - 5, p.need - 1, masks)
    assert not q.split and q.grid == 2 and q.n_work == 3
    assert [it[:4] for it in q.walks[0]] == [(0, 0, 8, 0), (2, 0, 2, 2)]  # tiles 0 and 2: 2 x 4 and 2 x 1 uses
    assert SparsePlan(132, 16, 16, 27, False, 10 ** 5, 10 ** 6, None, tile_masks(27, 1, 10 ** 5)).n == 10 ** 5


@pytest.mark.parametrize("sms", [132, 114])
def test_search_finds_every_regime(sms):
    """Both sparse regimes for every instantiation, and every dense case, at 132 and 114 SMs; the synthetic maps have
    tiles whose split 1 has no use and tiles of different use counts."""
    for cin, cout, K in SPARSE_SHAPES:
        seed = _seed(cin, cout, K)
        for regime in ("multi", "few"):
            r = sparse_search(sms, cin, cout, K, seed, regime)
            assert r is not None, (sms, cin, cout, K, regime)
            n_dev, n_cap = r
            assert n_dev % KM and n_dev < n_cap
            for lay in (False, True):
                p = SparsePlan(sms, cin, cout, K, lay, n_cap, n_dev, 1 << 62, tile_masks(K, seed, n_dev))
                if regime == "few":
                    assert p.n_work < p.grid
                else:
                    assert p.covered()
        m = tile_masks(K, seed, 40 * KM)
        odd = sum(1 << t for t in range(1, K, 2))
        assert ((m & odd) == 0).any() and len({bin(int(v)).count("1") for v in m}) > 3
    for case in DENSE_CASES:
        r = dense_search(sms, case)
        assert r is not None, (sms, case[0])
        p = r[2]
        assert p.oH % 8 and p.oW % 16
        if case[2] == "R3":
            assert p.n0 >= 4 and p.starts == list(range(p.S))


def test_synthetic_map_edges():
    """Rows without neighbours, one input row at several taps, the last input row, sources below n_in."""
    nbr = synth_nbr(27, 5, 5000, 7001)
    assert (nbr < 7001).all() and (nbr >= -1).all()
    assert (nbr[5::9] == -1).all() and ((nbr == -1).all(1)).mean() > 0.15
    rep = nbr[2::13]
    rows = [r for r in rep if (r >= 0).sum() >= 3]
    assert rows and all(len(set(r[r >= 0].tolist())) == 1 for r in rows)
    assert (nbr == 7000).sum() > 50


# -------------------------------------------------------------------------------------------------- GPU: split rows
@pytest.mark.gpu
def test_split_rows_built_here_match_the_library(cuda):
    """p3d_rows_convert_layout(..., 0, ...) and p3d_nchw_to_pixel_split against split_tf32, bit for bit."""
    import torch
    from paddle3d_b200._lib import check as ck, lib
    from paddle3d_b200._mem import ptr, stream
    L = lib()
    g = torch.Generator(device=cuda).manual_seed(2)
    for C in (16, 32, 64, 128):
        x = torch.randn((3000, C), generator=g, device=cuda) * torch.exp(
            torch.empty((3000, C), device=cuda).uniform_(-30, 30, generator=g))
        x[0, :4] = torch.tensor([0.0, -0.0, 1 + 2.0 ** -11, -(1 + 2.0 ** -11)])
        s = torch.full((3000, 2 * C), float("nan"), device=cuda)
        ck(L.p3d_rows_convert_layout(ptr(x), 0, None, 3000, C, ptr(s), stream(cuda)), "rows_convert_layout")
        assert torch.equal(s.view(torch.int32), split_rows(x).view(torch.int32))
    for B, C, H, W in ((2, 32, 9, 13), (1, 96, 31, 7), (3, 64, 5, 40)):
        x = torch.randn((B, C, H, W), generator=g, device=cuda) * torch.exp(
            torch.empty((B, C, H, W), device=cuda).uniform_(-30, 30, generator=g))
        s = torch.full((B * H * W, 2 * C), float("nan"), device=cuda)
        ck(L.p3d_nchw_to_pixel_split(ptr(x), B, C, H, W, ptr(s), stream(cuda)), "nchw_to_pixel_split")
        assert torch.equal(s.view(torch.int32), to_pixel_split(x).view(torch.int32))


# -------------------------------------------------------------------------------------------- GPU: sparse convs
class SparseData:
    """Seeded inputs of one instantiation: fp32 input rows and their split rows, the neighbour map's first n_cap rows,
    weights (packed once for both layouts), scale / shift, a residual (split rows; hi + lo for the fp32-row call) and
    the float64 reference over the first n_ref rows with its two wrong answers."""

    def __init__(self, dev, cin, cout, K, n_cap, n_ref, seed, nbr=None, n_in=None):
        import torch
        from paddle3d_b200._lib import check as ck, lib
        from paddle3d_b200._mem import ptr, stream
        self.dev, self.cin, self.cout, self.K, self.n_cap, self.n_ref = dev, cin, cout, K, n_cap, n_ref
        g = torch.Generator(device=dev).manual_seed(seed)
        n_in = n_in or n_cap + n_cap // 3 + 517  # a strided level: more input rows than output rows
        if nbr is None:
            nbr = torch.from_numpy(synth_nbr(K, seed, n_cap, n_in))
        self.nbr = nbr.to(dev).contiguous()
        self.x = torch.randn((n_in, cin), generator=g, device=dev) * 3.0
        self.xs = split_rows(self.x)
        self.w = torch.randn((K, cin, cout), generator=g, device=dev) / math.sqrt(K * cin * 0.4)
        self.scale = torch.rand((cout,), generator=g, device=dev) + 0.5
        self.shift = (torch.rand((cout,), generator=g, device=dev) - 0.5) * 0.4
        self.res_s = split_rows(torch.randn((n_cap, cout), generator=g, device=dev))
        self.res_f = self.res_s[:, :cout] + self.res_s[:, cout:]  # exact: hi + lo has 22 significant bits
        self.packed = torch.empty((lib().p3d_sparse_conv_packed_weight_bytes(K, cin, cout) // 4,), dtype=torch.float32,
                                  device=dev)
        ck(lib().p3d_sparse_conv_pack_weights(ptr(self.w), K, cin, cout, ptr(self.packed), stream(dev)), "pack")
        nb = self.nbr[:n_ref]
        X, W = from_split(self.xs, cin), self.w.double()
        self.acc = gather_gemm(X, nb, W)
        self.acc_hh = gather_gemm(from_split(self.xs, cin, hi_only=True), nb, tf32_rna(self.w).double())
        present = (nb >= 0).sum(0).cpu()
        self.has_taps = bool(present.sum() > 0)
        t_drop = 1 + 2 * int(present[1::2].argmax()) if K > 1 else 0  # a tap split 1 owns
        self.drop = t_drop
        self.acc_drop = self.acc - gather_gemm(X, nb, W, taps=[t_drop])
        self.res64 = from_split(self.res_s[:n_ref], cout)


def run_sparse(d, label, n_dev, n_cap, ws_kind, affine=True, residual=True, relu=True, masks=None):
    """Both row layouts on the same inputs: outputs and slabs NaN-filled, the slab rows written exactly when the
    restatement takes split-K, fp32 outputs bit-equal across layouts, split output = split_tf32(fp32 output), rows at and
    beyond the count untouched, the reference and its guards, a second launch with the same bits."""
    import torch
    from paddle3d_b200._lib import check as ck, lib
    from paddle3d_b200._mem import ptr, stream
    L, dev, cin, cout, K = lib(), d.dev, d.cin, d.cout, d.K
    sms = _sms()
    n = min(n_dev, n_cap)
    masks = tile_masks(K, _seed(cin, cout, K), n) if masks is None else masks
    s = min(sparse_cfg(cin, cout, False)[3], K)
    need = s * n_cap * cout * 4
    if s > 1:
        assert L.p3d_sparse_conv_splitk_workspace_bytes(n_cap, cin, cout) == _cdiv(need, 256) * 256
    ws_bytes = {"none": None, "need": need, "need-1": need - 1}[ws_kind]
    n_t = torch.tensor([n_dev], dtype=torch.int32, device=dev)
    scale, shift = (d.scale, d.shift) if affine else (None, None)
    name = "sparse %d->%d K=%d %s n=%d cap=%d ws=%s" % (cin, cout, K, label, n_dev, n_cap, ws_kind)
    outs, plans = {}, {}
    for lay in (False, True):
        p = SparsePlan(sms, cin, cout, K, lay, n_cap, n_dev, ws_bytes, masks)
        plans[lay] = p

        def launch():
            ws = torch.full((_cdiv(need, 4),), float("nan"), device=dev) if ws_bytes is not None else None
            f32 = torch.full((n_cap, cout), float("nan"), device=dev)
            spl = torch.full((n_cap, 2 * cout), float("nan"), device=dev) if lay else None
            if lay:
                ck(L.p3d_sparse_conv_gather_gemm_split_ws(
                    ptr(d.xs), ptr(d.nbr), ptr(n_t), n_cap, K, cin, cout, ptr(d.packed), ptr(scale), ptr(shift),
                    ptr(d.res_s if residual else None), int(relu), ptr(f32), ptr(spl), ptr(ws), ws_bytes or 0,
                    stream(dev)), name)
            else:
                ck(L.p3d_sparse_conv_gather_gemm_tf32x3_ws(
                    ptr(d.x), ptr(d.nbr), ptr(n_t), n_cap, K, cin, cout, ptr(d.packed), ptr(scale), ptr(shift),
                    ptr(d.res_f if residual else None), int(relu), ptr(f32), ptr(ws), ws_bytes or 0, stream(dev)), name)
            torch.cuda.synchronize()
            return ws, f32, spl

        ws, f32, spl = launch()
        lname = "%s %s rows" % (name, "split" if lay else "fp32")
        if ws is not None:
            slabs = ws[:s * n_cap * cout].view(s, n_cap, cout)
            if p.split:
                assert not bool(torch.isnan(slabs[:, :n]).any()), "%s: split-K predicted, slab rows not written" % lname
            else:
                assert bool(torch.isnan(slabs[:, :n]).all()), "%s: split-K not predicted, slabs written" % lname
            assert bool(torch.isnan(slabs[:, n:]).all()), "%s: slab rows at or beyond the count written" % lname
        assert bool(torch.isnan(f32[n:]).all()), "%s: fp32 rows at or beyond the count were written" % lname
        assert not bool(torch.isnan(f32[:n]).any()), "%s: fp32 rows below the count not written" % lname
        if lay:
            assert bool(torch.isnan(spl[n:]).all()), "%s: split rows at or beyond the count were written" % lname
            assert torch.equal(spl[:n].view(torch.int32), split_rows(f32[:n]).view(torch.int32)), \
                "%s: split output is not split_tf32 of the fp32 output" % lname
        _, f32b, splb = launch()
        assert _bits_equal(f32, f32b) and _bits_equal(spl, splb), "%s: a second launch gives other bits" % lname
        outs[lay] = f32
        print("REGIME %s: %s" % (lname, p.describe()))
    assert torch.equal(outs[False].view(torch.int32), outs[True].view(torch.int32)), \
        "%s: fp32-row and split-row entry points give other bits" % name
    if n:
        assert n <= d.n_ref
        res = d.res64[:n] if residual else None
        want = epilogue(d.acc[:n], scale, shift, res, relu)
        check(name, outs[True][:n], want, SPARSE_TERMS)
        if d.has_taps and n >= 64:
            rejects(name, [("hi x hi only", epilogue(d.acc_hh[:n], scale, shift, res, relu)),
                           ("tap %d dropped" % d.drop, epilogue(d.acc_drop[:n], scale, shift, res, relu))],
                    want, SPARSE_TERMS)
    return plans


@pytest.mark.gpu
@pytest.mark.parametrize("cin,cout,K", SPARSE_SHAPES)
def test_sparse_every_schedule(cuda, cin, cout, K):
    """Each instantiation in both row layouts: CTA 0 walking >= 3 items over every reachable ring start slot, fewer
    items than CTAs, a count of 0 and one above the capacity; the wide layers with no workspace, exactly the split-K
    workspace and one byte less; scale / shift, residual and ReLU on and off."""
    import torch
    sms = _sms()
    seed = _seed(cin, cout, K)
    multi = sparse_search(sms, cin, cout, K, seed, "multi")
    few = sparse_search(sms, cin, cout, K, seed, "few")
    assert multi is not None, "no multi-item case for %d->%d K=%d at %d SMs" % (cin, cout, K, sms)
    d = SparseData(cuda, cin, cout, K, multi[1], multi[0], seed)
    wide = min(sparse_cfg(cin, cout, False)[3], K) > 1
    n_dev, n_cap = multi
    if wide:
        plans = run_sparse(d, "multi-item", n_dev, n_cap, "need")
        assert all(p.split and p.covered() for p in plans.values())
        masks = tile_masks(K, seed, n_dev)
        assert any(it[1] == 1 and it[2] == 0 for it in plans[True].walks[1]) or bool(
            ((masks & sum(1 << t for t in range(1, K, 2))) == 0).any())
        plans = run_sparse(d, "multi-item", n_dev, n_cap, "need-1", affine=False, relu=False)
        assert not any(p.split for p in plans.values())
        plans = run_sparse(d, "multi-item", n_dev, n_cap, "none", residual=False)
        assert not any(p.split for p in plans.values())
    else:
        plans = run_sparse(d, "multi-item", n_dev, n_cap, "none")
        assert all(p.covered() for p in plans.values())
        run_sparse(d, "multi-item", n_dev, n_cap, "none", affine=False, residual=False, relu=False)
    n_dev, n_cap = few
    for ws in ("need", "none") if wide else ("none",):
        plans = run_sparse(d, "fewer items than CTAs", n_dev, n_cap, ws)
        assert all(p.n_work < p.grid for p in plans.values())
    run_sparse(d, "n=0", 0, n_cap, "need" if wide else "none")
    run_sparse(d, "count above capacity", 10 ** 6, n_cap, "need" if wide else "none", affine=False, relu=False)
    del d
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_sparse_level0_rulebook_c3_capacity(cuda):
    """A real level-0 SubM rulebook (synth.lidar_cloud, C3 grid) at the C3 capacity of 160 000 rows, 16 -> 16 in both
    layouts, and 16 -> 32 above it."""
    import torch
    from paddle3d_b200 import synth
    cfg = synth.C3
    pts = synth.lidar_cloud(cfg, 33, num_points=500000)
    lo, vs = np.asarray(cfg["point_cloud_range"][:3]), np.asarray(cfg["voxel_size"])
    grid = np.round((np.asarray(cfg["point_cloud_range"][3:]) - lo) / vs).astype(np.int64)
    ijk = np.floor((pts[:, :3] - lo) / vs).astype(np.int64)
    sites = np.unique(ijk[((ijk >= 0) & (ijk < grid)).all(1)], axis=0)
    np.random.default_rng(33).shuffle(sites, axis=0)
    cap = 160000
    sites = sites[:cap - 1000]
    n = len(sites)
    assert n > 60000 and n % KM
    coords = np.concatenate([np.zeros((n, 1), np.int64), sites[:, ::-1]], 1)
    nbr = torch.full((cap, 27), -1, dtype=torch.int32)
    nbr[:n] = subm_rulebook_torch(torch.from_numpy(coords).to(cuda), [int(grid[2]), int(grid[1]), int(grid[0])]).cpu()
    row_bits = ((nbr[:n] >= 0).long() << torch.arange(27)).sum(1).numpy()
    t = _cdiv(n, KM)
    pad = np.zeros(t * KM, np.int64)
    pad[:n] = row_bits
    masks = np.bitwise_or.reduce(pad.reshape(t, KM), 1)
    for cout in (16, 32):
        d = SparseData(cuda, 16, cout, 27, cap, n, seed=16 + cout, nbr=nbr, n_in=cap)
        run_sparse(d, "level-0 SubM rulebook", n, cap, "none", masks=masks)
        del d
        torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- GPU: dense conv
class DenseCase:
    """Seeded layer: input [B, Cin, H, W] (batch image b scaled by mags[b]), conv or transposed-conv weight (Paddle
    layouts), scale / shift (None with affine=False), its pixel split image and the float64 reference."""

    def __init__(self, dev, B, H, W, cin, cout, k, stride, pad, up, seed, mags=(1.0, 32.0), relu=True, affine=True):
        import torch
        self.dev, self.B, self.H, self.W, self.cin, self.cout = dev, B, H, W, cin, cout
        self.k, self.stride, self.pad, self.up, self.relu = k, stride, pad, up, relu
        g = torch.Generator(device=dev).manual_seed(seed)
        m = torch.tensor([mags[b % len(mags)] for b in range(B)], device=dev).view(B, 1, 1, 1)
        x = torch.randn((B, cin, H, W), generator=g, device=dev) * m
        self.terms = cin if up > 1 else cin * k * k
        self.w = torch.randn((cin, cout, up, up) if up > 1 else (cout, cin, k, k), generator=g, device=dev) / math.sqrt(
            self.terms)
        self.scale = torch.rand((cout,), generator=g, device=dev) + 0.5 if affine else None
        self.shift = (torch.rand((cout,), generator=g, device=dev) - 0.5) * 0.4 if affine else None
        self.xs = to_pixel_split(x)
        del x
        self.drop = ("group", cin // 64) if (up > 1 or k == 1) else ("tap", 4 if k == 3 else 0)

    def plan(self, sms, n_tile):
        return DensePlan(sms, self.B, self.H, self.W, self.cin, self.cout, n_tile, self.k, self.stride, self.pad, self.up)

    def reference(self):
        """(want NHWC, [(what, wrong answer)])."""
        x64 = from_pixel_split(self.xs, self.B, self.H, self.W, self.cin)
        acc, part = conv_ref(x64, self.w.double(), self.k, self.stride, self.pad, self.up, self.drop)
        del x64
        want = epilogue(acc, self.scale, self.shift, None, self.relu)
        dropped = epilogue(acc - part, self.scale, self.shift, None, self.relu)
        del acc, part
        hh, _ = conv_ref(from_pixel_split(self.xs, self.B, self.H, self.W, self.cin, hi_only=True),
                         tf32_rna(self.w).double(), self.k, self.stride, self.pad, self.up)
        return want, [("hi x hi only", epilogue(hh, self.scale, self.shift, None, self.relu)),
                      ("%s %d dropped" % self.drop, dropped)]

    def packed(self, n_tile):
        from paddle3d_b200.ops import dense_conv as dc
        return (dc.pack_deconv_weight if self.up > 1 else dc.pack_conv_weight)(self.w, n_tile)


def run_dense(name, case, n_tile, c0=16, split_out=True, guards=True):
    """One p3d_dense_conv2d_split launch writing split rows at channel c0 of a wider sentinel-filled image (and guard
    pixels after it) together with NaN-filled fp32 planes; both against the reference per batch image, the sentinels,
    the guards and a second launch (same bits).  Returns the plan."""
    import torch
    from paddle3d_b200._lib import check as ck, lib
    from paddle3d_b200._mem import ptr, stream
    p = case.plan(_sms(), n_tile)
    out_C = c0 + case.cout + 12 if split_out else 0
    n_px = case.B * p.out_H * p.out_W
    packed = case.packed(n_tile)
    kk, ss, pp = (case.up, case.up, 0) if case.up > 1 else (case.k, case.stride, case.pad)

    def once():
        img = torch.full((n_px + 37, 2 * out_C), SENTINEL, device=case.dev) if split_out else None
        pl = torch.full((case.B, case.cout, p.out_H, p.out_W), float("nan"), device=case.dev)
        ck(lib().p3d_dense_conv2d_split(ptr(case.xs), case.B, case.H, case.W, case.cin, ptr(packed), case.cout, n_tile,
                                        kk, kk, ss, pp, case.up, ptr(case.scale), ptr(case.shift), int(case.relu),
                                        ptr(img), out_C, c0, ptr(pl), stream(case.dev)), name)
        torch.cuda.synchronize()
        return img, pl

    img, pl = once()
    want, wrongs = case.reference()
    assert not bool(torch.isnan(pl).any()), "%s: fp32 plane elements not written" % name
    check_images(name + " fp32 planes", pl.permute(0, 2, 3, 1), want, case.terms)
    if split_out:
        s = int(torch.tensor(SENTINEL).view(torch.int32))
        bits = img.view(torch.int32)
        assert bool((bits[n_px:] == s).all()), "%s: guard pixels after the image were written" % name
        owned = torch.zeros(2 * out_C, dtype=torch.bool, device=case.dev)
        owned[c0:c0 + case.cout] = True
        owned[out_C + c0:out_C + c0 + case.cout] = True
        assert bool((bits[:n_px][:, ~owned] == s).all()), "%s: channels outside the layer's were written" % name
        sub = torch.cat([img[:n_px, c0:c0 + case.cout], img[:n_px, out_C + c0:out_C + c0 + case.cout]], 1)
        planes_rows = pl.permute(0, 2, 3, 1).reshape(-1, case.cout)
        assert torch.equal(sub.view(torch.int32), split_rows(planes_rows).view(torch.int32)), \
            "%s: split output is not split_tf32 of the fp32 planes" % name
        del sub, planes_rows
    if guards:
        rejects(name, wrongs, want, case.terms, per_image=True)
    del want, wrongs
    img2, pl2 = once()
    assert _bits_equal(img, img2) and _bits_equal(pl, pl2), "%s: a second launch gives other bits" % name
    return p


@pytest.mark.gpu
@pytest.mark.parametrize("case", DENSE_CASES, ids=lambda c: c[0].replace(" ", "_"))
def test_dense_every_regime(cuda, case):
    """Each N tile with fewer items than CTAs, one CTA with two items, and >= 4 items per CTA with ragged tiles, every
    ring slot as a start slot and the N tile, batch (and tap) changing between CTA 0's items; split rows at a channel
    offset of a wider image (20: no multiple of 16 in R3) and fp32 planes from the same launch."""
    import torch
    sms = _sms()
    r = dense_search(sms, case)
    assert r is not None, "no case %s at %d SMs" % (case[0], sms)
    H, W, p = r
    label, nt, regime, B, cin, n_nt, k, stride, pad, up = case
    cout = _dense_cout(nt, n_nt)
    c = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=nt * 7 + cin + 100 * int(regime[1]))
    name = "dense %s B%d %dx%d %d->%d k%d s%d up%d" % (label, B, H, W, cin, cout, k, stride, up)
    got = run_dense(name, c, nt, c0=20 if regime == "R3" else 16)
    assert got.items == p.items and got.starts == p.starts
    print("REGIME %s: %s" % (name, p.describe()))
    del c
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_dense_narrow_cout_planes_only(cuda):
    """Cout 3 on the N = 16 tile (13 padded columns of the tile), fp32 planes only, no scale / shift, no ReLU, >= 4
    items per CTA."""
    sms = _sms()
    c = DenseCase(cuda, 2, 8 * 20 - 3, 16 * 30 - 5, 64, 3, 3, 1, 1, 1, seed=3, relu=False, affine=False)
    p = c.plan(sms, 16)
    assert p.items // p.grid >= 4 and p.items % p.grid
    run_dense("dense Cout 3 planes only", c, 16, split_out=False)
    print("REGIME dense Cout 3 planes only: %s" % p.describe())


def _n_tile(cout):
    from paddle3d_b200.ops import dense_conv as dc
    return dc.n_tile_for(cout)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", C3_LAYERS + PP_LAYERS, ids=lambda l: l[0].replace(" ", "_"))
def test_dense_full_size_layer(cuda, layer):
    """Every dense layer of the CenterPoint (C3) and PointPillars frames at its real size on the tf32-pair kernel."""
    import torch
    name, B, H, W, cin, cout, k, stride, pad, up, relu, bias_only, c0 = layer
    c = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=cin * 13 + cout + H, mags=(1.0,), relu=relu)
    nt = _n_tile(cout)
    p = run_dense("tf32 " + name, c, nt, c0=c0 or 16, split_out=cout % 16 == 0)
    print("REGIME tf32 layer %s (N %d): %s" % (name, nt, p.describe()))
    del c
    torch.cuda.empty_cache()


# --------------------------------------------------------------------------------------------- GPU: head final convs
def run_head(dev, name, B, H, W, cin, groups, extra, seed):
    """One p3d_head_final_conv launch: group g convolves input channels [g Cin, (g + 1) Cin) of an image of
    groups x Cin + extra channels into planes plane0[g] .. + cnt[g] (cnt 1 - 4, plane0 shuffled with gaps); planes no
    group owns keep their NaN."""
    import torch
    from paddle3d_b200._lib import check as ck, lib
    from paddle3d_b200._mem import ptr, stream
    rng = np.random.default_rng(seed)
    g = torch.Generator(device=dev).manual_seed(seed)
    in_C = groups * cin + extra
    cnt = rng.integers(1, 5, groups).astype(np.int32)
    cnt[:min(groups, 4)] = np.arange(1, 5)[:min(groups, 4)]
    slots = rng.permutation(groups)  # planes laid out in a shuffled group order, one spare plane after each group
    plane0 = np.zeros(groups, np.int32)
    p0 = 1
    for gi in slots:
        plane0[gi] = p0
        p0 += int(cnt[gi]) + 1
    planes = p0 + 1
    mags = torch.tensor([1.0, 32.0][:B], device=dev).view(B, 1, 1, 1)
    xs = to_pixel_split(torch.randn((B, in_C, H, W), generator=g, device=dev) * mags)
    w = torch.randn((groups, 4, cin, 3, 3), generator=g, device=dev) / math.sqrt(9 * cin)
    bias = torch.randn((groups, 4), generator=g, device=dev)
    fw = w.permute(0, 3, 4, 2, 1).reshape(groups, 9, cin, 4).contiguous()  # [g][tap][c][k]

    def once():
        out = torch.full((B, planes, H, W), float("nan"), device=dev)
        ck(lib().p3d_head_final_conv(ptr(xs), B, H, W, in_C, cin, groups, ptr(fw), ptr(bias), plane0.ctypes.data,
                                     cnt.ctypes.data, planes, ptr(out), stream(dev)), name)
        torch.cuda.synchronize()
        return out

    out = once()
    X = from_pixel_split(xs, B, H, W, in_C)
    Xh = from_pixel_split(xs, B, H, W, in_C, hi_only=True)
    want = torch.full((B, planes, H, W), float("nan"), dtype=torch.float64, device=dev)
    hh, dropped = want.clone(), want.clone()
    owned = torch.zeros(planes, dtype=torch.bool)
    for gi in range(groups):
        c0, k, p0 = gi * cin, int(cnt[gi]), int(plane0[gi])
        acc, part = conv_ref(X[..., c0:c0 + cin], w[gi, :k].double(), 3, 1, 1, 1, ("tap", 4))
        acc_hh, _ = conv_ref(Xh[..., c0:c0 + cin], w[gi, :k].double(), 3, 1, 1, 1)
        b = bias[gi, :k].double()
        want[:, p0:p0 + k] = (acc + b).permute(0, 3, 1, 2)
        hh[:, p0:p0 + k] = (acc_hh + b).permute(0, 3, 1, 2)
        dropped[:, p0:p0 + k] = (acc - part + b).permute(0, 3, 1, 2)
        owned[p0:p0 + k] = True
    del X, Xh
    owned = owned.to(dev)
    assert bool(torch.isnan(out[:, ~owned]).all()), "%s: planes no group owns were written" % name
    assert not bool(torch.isnan(out[:, owned]).any()), "%s: owned plane elements not written" % name
    check_images(name, out[:, owned], want[:, owned], 9 * cin)
    rejects(name, [("hi halves only", hh[:, owned]), ("tap 4 dropped", dropped[:, owned])], want[:, owned], 9 * cin,
            per_image=True)
    assert _bits_equal(out, once()), "%s: a second launch gives other bits" % name


@pytest.mark.gpu
@pytest.mark.parametrize("case", HEAD_CASES, ids=lambda c: c[0].replace(" ", "_"))
def test_head_final_conv(cuda, case):
    label, B, H, W, cin, groups, extra = case
    name = "head_final_conv %s B%d %dx%d" % (label, B, H, W)
    run_head(cuda, name, B, H, W, cin, groups, extra, seed=cin * 3 + groups)
    blocks = B * _cdiv(H, TH) * _cdiv(W, TW) * groups
    print("REGIME %s: %d blocks of 16 x 8 pixels" % (name, blocks))


# ------------------------------------------------------------------------------------------- chained tf32 C3 head
@pytest.mark.gpu
def test_chained_c3_tf32_frame_eager_and_graph(cuda):
    """The full-size CenterPoint DenseRPNHead on the tf32-pair path (f16=False: every conv on dense_conv_kernel, the 36
    output convs on head_final_conv_kernel) run layer after layer on one stream with no sync in between, once eagerly
    and once captured in a CUDA graph.  Every layer against the float64 reference computed from that layer's actual
    input buffer; eager and graph outputs bit-equal."""
    import torch
    from paddle3d_b200.dense_head import DenseRPNHead
    net = DenseRPNHead(f16=False).init_weight(seed=9, device=cuda, randomize_bn=True, bn_gain=6.0 ** 0.5)
    bp = net._batched_params(cuda)
    big = bp["big"]
    g = torch.Generator(device=cuda).manual_seed(10)
    xs = to_pixel_split(torch.randn((1, net.in_channels, 180, 180), generator=g, device=cuda))

    def chain():
        recs = []  # (conv, input image, its shape, output image, out_C, c0)
        x, sh = xs, (1, 180, 180, net.in_channels)
        feats = []
        for blk in net.blocks:
            for conv in blk:
                y, _, (b, oh, ow) = conv(x, sh)
                recs.append((conv, x, sh, y, conv.cout, 0))
                x, sh = y, (b, oh, ow, conv.cout)
            feats.append((x, sh))
        fpn = net.fpn_channels
        cat = torch.empty((180 * 180, 2 * fpn), dtype=torch.float32, device=cuda)
        c0 = 0
        for (f, fs), de in zip(feats, net.deblocks):
            de(f, fs, out_split=cat, out_channels=fpn, out_c0=c0)
            recs.append((de, f, fs, cat, fpn, c0))
            c0 += de.cout
        s, _, _ = net.shared(cat, (1, 180, 180, fpn))
        recs.append((net.shared, cat, (1, 180, 180, fpn), s, net.shared.cout, 0))
        shape = (1, 180, 180, net.shared.cout)
        mid, _, _ = big(s, shape)
        recs.append((big, s, shape, mid, big.cout, 0))
        planes = net._final_convs(mid, shape, big.cout, bp, bp["planes"], cuda)
        return recs, planes

    recs, planes = chain()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        recs_g, planes_g = chain()
    graph.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(recs, recs_g)):
        assert _bits_equal(a[3], b[3]), "layer %d: graph replay differs from the eager run" % i
    assert _bits_equal(planes, planes_g), "output convs: graph replay differs from the eager run"
    del recs_g, planes_g, graph
    torch.cuda.empty_cache()
    sms = _sms()
    for i, (conv, x, sh, y, out_C, c0) in enumerate(recs):
        b, h, w, cin = sh
        x64 = from_pixel_split(x, b, h, w, cin)
        weight = conv.np["weight"] if conv is not big else np.concatenate([a.np["weight"] for hs in net.heads
                                                                           for _, a, _ in hs], 0)
        acc, _ = conv_ref(x64, torch.from_numpy(weight).to(cuda).double(), conv.k, conv.stride, conv.padding, conv.up)
        del x64
        want = epilogue(acc, conv.dev["scale"], conv.dev["shift"], None, conv.relu)
        del acc
        oh, ow = want.shape[1:3]
        got = (y[:b * oh * ow, c0:c0 + conv.cout].double() + y[:b * oh * ow, out_C + c0:out_C + c0 + conv.cout].double()
               ).reshape(b, oh, ow, conv.cout)
        terms = cin if conv.up > 1 else cin * conv.k * conv.k
        name = "tf32 chain layer %d %d->%d k%d s%d up%d" % (i, cin, conv.cout, conv.k, conv.stride, conv.up)
        check_images(name, got, want, terms)
        p = DensePlan(sms, b, h, w, cin, conv.cout, conv.n_tile, conv.k, conv.stride, conv.padding, conv.up)
        print("REGIME %s (N %d): %s" % (name, conv.n_tile, p.describe()))
        del got, want
    finals = [f for hs in net.heads for _, _, f in hs]
    mid = recs[-1][3]
    X = from_pixel_split(mid, 1, 180, 180, big.cout)
    want = torch.full(tuple(planes.shape), float("nan"), dtype=torch.float64, device=cuda)
    for gi, f in enumerate(finals):
        acc, _ = conv_ref(X[..., gi * 64:(gi + 1) * 64], torch.from_numpy(f.np["weight"]).to(cuda).double(), 3, 1, 1, 1)
        p0 = int(bp["plane0"][gi])
        want[:, p0:p0 + f.cout] = (acc + torch.from_numpy(f.np["bias"]).to(cuda).double()).permute(0, 3, 1, 2)
    assert not bool(torch.isnan(want).any()) and len(finals) == 36
    check_images("tf32 chain output convs (36 groups)", planes, want, 64 * 9)
