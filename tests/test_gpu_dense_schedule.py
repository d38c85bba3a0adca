"""The dense fp16-pair convs in every work decomposition they run on the device, against a float64 reference.

Kernels (csrc/dense_conv_f16.cu): `dcf::dense_conv_f16_kernel<N, MT, HALO>` in its six instantiations and
`dcf::out9::head_out9_kernel` (the CenterHead's output convs, 9 taps in the GEMM's N dimension).  Both launch
grid = min(items, SMs) persistent CTAs that walk their items round robin, so most of their ring, phase and staging logic
only runs when a CTA takes more than one item.  The kernels are called through the C ABI (p3d_dense_conv2d_f16,
p3d_head_out_conv_f16) so that the tests control `mode`, `m_tiles`, the N tile, the output buffers and the status word.

Reference: the conv in float64 on the device (one fp64 GEMM per tap), with X the EXACT value of the fp16-pair input
image (hi + lo' 2^-11, built here from fp32 and checked bit-equal to p3d_nchw_to_pixel_h16) and W the fp32 weight (so
the weight split error is part of what is checked), then scale / shift / ReLU in the epilogue's order.  The bar is the
one of test_gpu_dense.py (tests/parity.py's definition, evaluated on the device): 1e-4 true relative error above a
floor of 1e-2 x max (5e-2 x max for sums of 2048 terms or more, see `bar`), 2e-6 (1e-5) x max below it, per batch
image.  Every
case also shows that the bar REJECTS two wrong answers computed from the reference: the hi x hi products alone, and the
result without one tap (1x1 and transposed convs: without one 32-channel input group).

Which decomposition ran is restated here from the host code (nothing on the device reports it): the item count,
grid = min(items, SMs), the round robin of `decode`, the HALO condition, the MT rule of p3d_dense_conv2d_f16 and the ring
depths NA / NB of `Cfg`.  The regime cases are searched with the restatement for this device's SM count.  Lines starting
with "REGIME" (pytest -s) list the items per CTA and the ring slots at which CTA 0's items start."""
import math

import numpy as np
import pytest

LO = 2.0 ** -11        # weight of lo' in an fp16 pair
TW, TH = 8, 16         # output tile of one M tile (dcf::kTW x dcf::kTH)
PITCH = TW + 2         # haloed tile row (dcf::kPitch)
MAX_A, MAX_B = 6, 12   # dcf::kMaxA, dcf::kMaxB
SMEM = (227 - 6) * 1024  # dcf::kSmemBudget
O9_T, O9_NW, O9_MAXNA = 14, 3, 5  # out9::kOT, kNW, kMaxNA
O9_A, O9_P, O9_WBLK = 256 * 128, 256 * 29 * 4, 64 * 32  # out9::kABytes, kPBytes, kWBlk
GUARD = 37             # sentinel pixels after every fp16-pair output image
SENTINEL = 7.0         # fp16 value of both halves of untouched output channels
INSTS = [(128, 1, True), (128, 1, False), (64, 1, True), (64, 1, False), (64, 2, True), (64, 2, False)]


def _cdiv(a, b):
    return -(-a // b)


# --------------------------------------------------------------------------------------------- schedule restatement
def ring_depths(N, MT, halo):
    """Cfg<N, MT, HALO>::NA and ::NB."""
    a_rows = PITCH * (TH * MT + 2) if halo else 128 * MT
    a_bytes = _cdiv(a_rows * 128, 1024) * 1024
    b_bytes = 128 * N
    avail = SMEM - 2 * MT * 64 * (N + 8) * 4  # less the two staging tiles
    na = 2 if halo else min(avail // (a_bytes + b_bytes), MAX_A)
    return na, min((avail - na * a_bytes) // b_bytes, MAX_B)


class Plan:
    """What p3d_dense_conv2d_f16 launches for a layer: instantiation, items, grid, and for CTA 0 (which takes the most
    items) the decoded items and the activation / weight ring slots each of them starts at."""

    def __init__(self, sms, B, H, W, cin, cout, n_tile, k, stride, pad, up, mode=0, m_tiles=0):
        self.halo = mode == 0 and up == 1 and k == 3 and stride == 1 and pad == 1
        if up > 1:
            self.oH, self.oW, self.out_H, self.out_W = H, W, H * up, W * up
        else:
            self.oH, self.oW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
            self.out_H, self.out_W = self.oH, self.oW
        up2 = up * up if up > 1 else 1
        self.n_nt = _cdiv(cout, n_tile)
        mt = m_tiles
        if mt not in (1, 2):  # the MT rule: fewer M-tile rounds, two M tiles on a tie
            per_row = B * _cdiv(self.oW, TW) * self.n_nt * up2
            i1, i2 = per_row * _cdiv(self.oH, TH), per_row * _cdiv(self.oH, 2 * TH)
            mt = 2 if n_tile <= 64 and 2 * _cdiv(i2, sms) <= _cdiv(i1, sms) else 1
        if n_tile > 64:
            mt = 1
        self.inst = (n_tile, mt, self.halo)
        self.tiles_x, self.tiles_y = _cdiv(self.oW, TW), _cdiv(self.oH, TH * mt)
        self.up2 = up2
        self.items = B * self.tiles_y * self.tiles_x * self.n_nt * up2
        self.grid = min(self.items, sms)
        self.na, self.nb = ring_depths(n_tile, mt, self.halo)
        G = cin // 32
        self.units = G if self.halo else (1 if up > 1 else k * k) * G
        self.steps = self.units * (9 if self.halo else 1)
        self.n0 = _cdiv(self.items, self.grid)
        self.cta0 = [self.decode(i * self.grid) for i in range(self.n0)]  # round robin: item q = blockIdx + idx * grid
        self.a_starts = sorted({i * self.units % self.na for i in range(self.n0)})
        self.b_starts = sorted({i * self.steps % self.nb for i in range(self.n0)})

    def decode(self, q):
        """dcf::decode: (N tile, tap, tile x, tile y, batch) of item q, N tile fastest."""
        nt = q % self.n_nt
        q //= self.n_nt
        tap = q % self.up2
        q //= self.up2
        return nt, tap, q % self.tiles_x, (q // self.tiles_x) % self.tiles_y, q // (self.tiles_x * self.tiles_y)

    @property
    def per_cta(self):
        return self.items / self.grid

    def rings_covered(self):
        """CTA 0's items start at every slot of both rings that the per-item step counts can reach, and those counts are
        coprime to the ring depths as far as the kernel allows (HALO: 9 weight steps per unit, so with NB a multiple of
        3 an item can only start at a multiple of 3 of the weight ring)."""
        ga, gb = math.gcd(self.units, self.na), math.gcd(self.steps, self.nb)
        best_b = math.gcd(9, self.nb) if self.halo else 1
        return (ga == 1 and gb == best_b and self.a_starts == list(range(self.na))
                and self.b_starts == list(range(0, self.nb, gb)))

    def cta0_varies(self, field):
        vals = [it[field] for it in self.cta0]
        return any(a != b for a, b in zip(vals, vals[1:]))

    def describe(self):
        n, mt, halo = self.inst
        return ("(%d, %d, %s) items %d, grid %d, %.2f items/CTA (CTA 0: %d); A ring slots %s of %d, B ring slots %s of %d"
                % (n, mt, "HALO" if halo else "TAP", self.items, self.grid, self.per_cta, self.n0, self.a_starts,
                   self.na, self.b_starts, self.nb))


# per instantiation: (cin, k, stride, pad, up, mode) of the R1 / R2 cases (one N tile, B = 1, so that the item count
# can be SMs + 1) and of the R3 case (several N tiles; per-item unit and step counts coprime to the ring depths)
REGIME_GEOM = {
    (128, 1, True): ((96, 3, 1, 1, 1, 0), (96, 3, 1, 1, 1, 0)),
    (128, 1, False): ((32, 3, 2, 1, 1, 0), (32, 3, 2, 1, 1, 0)),    # stride 2: 9 units per item
    (64, 1, True): ((96, 3, 1, 1, 1, 0), (96, 3, 1, 1, 1, 0)),
    (64, 1, False): ((64, 3, 1, 1, 1, 1), (160, 1, 1, 0, 1, 0)),    # 3x3 forced onto per-tap loads; 1x1, 5 units
    (64, 2, True): ((96, 3, 1, 1, 1, 0), (96, 3, 1, 1, 1, 0)),
    (64, 2, False): ((32, 3, 2, 1, 1, 0), (160, 2, 2, 0, 2, 0)),    # transposed conv k = s = 2: the tap varies per item
}


def _regime_ok(p, regime, sms):
    if regime == "R1":
        return p.items < sms
    if regime == "R2":
        return p.items == sms + 1
    return (p.items // p.grid >= 4 and p.items % p.grid != 0 and p.rings_covered() and p.cta0_varies(4) and p.cta0_varies(0)
            and (p.up2 == 1 or p.cta0_varies(1)))


def search_regime(sms, inst, regime, geom=REGIME_GEOM):
    """Image size (and batch) of a regime for one instantiation: output sides that are no multiple of 8 (ragged last
    tiles); R1 the largest item count below the SM count, R2 exactly SMs + 1 items, R3 the fewest items with at least 4
    on every CTA, a ragged last round, CTA 0's items crossing a batch boundary and changing N tile (and tap) between
    consecutive items, and the ring coverage of Plan.rings_covered.  geom: a table shaped like REGIME_GEOM.  Returns (B,
    H, W, cin, cout, k, stride, pad, up, mode, Plan) or None."""
    N, MT, halo = inst
    cin, k, stride, pad, up, mode = geom[inst][regime == "R3"]
    best = None
    for B in ((2, 3) if regime == "R3" else (1,)):
        for n_nt in ((5, 7) if regime == "R3" else (1,)):
            if regime == "R3" and sms % n_nt == 0:
                continue
            cout = n_nt * N - 16
            for ty in range(1, 80):
                for tx in range(1, 80):
                    items = B * ty * tx * n_nt * (up * up if up > 1 else 1)  # Plan.items, to prune before building one
                    if (regime == "R1" and items >= sms) or (regime == "R2" and items != sms + 1) or (
                            regime == "R3" and (items < 4 * sms or (best is not None and items >= best[0]))):
                        continue
                    oh, ow = TH * MT * ty - 5, TW * tx - 3
                    h, w = (oh, ow) if up > 1 else ((oh - 1) * stride + k - 2 * pad, (ow - 1) * stride + k - 2 * pad)
                    if h < 1 or w < 1:
                        continue
                    p = Plan(sms, B, h, w, cin, cout, N, k, stride, pad, up, mode, MT)
                    assert p.inst == inst and (p.oH, p.oW) == (oh, ow)
                    if not _regime_ok(p, regime, sms):
                        continue
                    key = -p.items if regime == "R1" else p.items
                    if best is None or key < best[0]:
                        best = (key, (B, h, w, cin, cout, k, stride, pad, up, mode, p))
            if best is not None and regime == "R3":
                return best[1]
    return None if best is None else best[1]


class Out9Plan:
    """p3d_head_out_conv_f16's launch: 14 x 14 output tiles x groups, grid = min(items, SMs), activation ring depth NA
    from the shared-memory budget, CTA 0's activation / weight ring start slots."""

    def __init__(self, sms, B, H, W, cin, groups):
        G = cin // 32
        self.na = min((SMEM - 1024 - O9_P - O9_NW * 2 * G * O9_WBLK) // O9_A, O9_MAXNA)
        self.items = B * _cdiv(H, O9_T) * _cdiv(W, O9_T) * groups
        self.grid = min(self.items, sms)
        self.n0 = _cdiv(self.items, self.grid)
        self.a_starts = sorted({i * G % self.na for i in range(self.n0)})
        self.w_starts = sorted({i % O9_NW for i in range(self.n0)})

    def describe(self):
        return "items %d, grid %d, %.2f items/CTA (CTA 0: %d); A ring NA %d slots %s, weight ring slots %s" % (
            self.items, self.grid, self.items / self.grid, self.n0, self.na, self.a_starts, self.w_starts)


def out9_search(sms, B, cin, groups, regime):
    """(H, W) with sides that are no multiple of 14: R1 one item per CTA, R2 about two, R3 more than 3 kNW on every CTA."""
    best = None
    for ty in range(1, 60):
        for tx in range(1, 60):
            H, W = O9_T * ty - 3, O9_T * tx - 5
            p = Out9Plan(sms, B, H, W, cin, groups)
            if regime == "R1":
                ok, key = p.items <= sms, -p.items
            elif regime == "R2":
                ok, key = p.n0 == 2 and p.items % p.grid and p.items / p.grid >= 1.7, p.items
            else:
                ok, key = p.items // p.grid > 3 * O9_NW and p.items % p.grid != 0, p.items
            if ok and (best is None or key < best[0]):
                best = (key, (H, W, p))
    return None if best is None else best[1]


# (label, B, cin, groups [(cnt, plane0, cin0)], in_C, pass cin0, regime): cnt 1 / 2 / 3, planes no group owns (gaps),
# a slice shared by two groups, the g * Cin path (cin0 null), B = 2; Cin 32 / 96 / 128 / 256 / 320 (NA 5 / 4 / 4 / 2 / 2)
OUT9_CASES = [
    ("cin32 gaps", 2, 32, [(3, 0, 64), (1, 4, 0), (2, 6, 64), (3, 9, 32), (2, 13, 96)], 128, True, "R3"),
    ("cin96 null cin0", 1, 96, [(2, 0, 0), (3, 2, 96), (1, 5, 192)], 288, False, "R2"),
    ("cin128", 1, 128, [(3, 1, 128), (1, 0, 0), (2, 4, 0)], 256, True, "R1"),
    ("cin256 B2", 2, 256, [(1, 0, 0), (3, 2, 256)], 512, False, "R2"),
    ("cin320", 1, 320, [(2, 0, 320), (3, 3, 0), (3, 7, 320)], 640, True, "R3"),
]


# ----------------------------------------------------------------------------------------------- fp16 pairs and reference
def to_pixel_h16(x):
    """fp32 NCHW -> pixel fp16-pair rows [B*H*W, 2C]: per pixel groups of 32 channels [hi 32 | lo' 32], hi = fp16(x),
    lo' = fp16((x - hi) 2^11)."""
    import torch
    B, C, H, W = x.shape
    xn = x.permute(0, 2, 3, 1).reshape(-1, C)
    hi = xn.half()
    lo = ((xn - hi.float()) * 2048.0).half()
    n = xn.shape[0]
    return torch.stack([hi.view(n, C // 32, 32), lo.view(n, C // 32, 32)], 2).reshape(n, 2 * C)


def from_pixel_h16(h, B, H, W, C, hi_only=False):
    """Exact value (float64, NHWC [B, H, W, C]) of pixel fp16-pair rows; hi_only: the hi halves alone."""
    g = h[:B * H * W].reshape(-1, C // 32, 2, 32).double()
    v = g[:, :, 0] if hi_only else g[:, :, 0] + g[:, :, 1] * LO
    return v.reshape(B, H, W, C)


def conv_ref(xn, w, k, stride, pad, up, drop=None):
    """Float64 conv of NHWC xn [B, H, W, Cin]: one GEMM per tap.  w: conv weight [Cout, Cin, k, k], or for up > 1 the
    transposed conv's [Cin, Cout, up, up] (out[b, y up + dy, x up + dx] = x[b, y, x] W[:, :, dy, dx]).  Returns
    (out NHWC [B, oH, oW, Cout], the part of out that comes from tap `drop` = ("tap", t) or from 32-channel input group
    ("group", g), or None)."""
    import torch
    import torch.nn.functional as F
    B, H, W, cin = xn.shape
    part = None

    def grp(a, axis):
        g = drop[1]
        return a.narrow(axis, 32 * g, 32)
    if up > 1:
        cout = w.shape[1]
        out = torch.empty((B, H, up, W, up, cout), dtype=torch.float64, device=xn.device)
        flat = xn.reshape(-1, cin)
        if drop is not None:
            part = torch.empty_like(out)
        for dy in range(up):
            for dx in range(up):
                out[:, :, dy, :, dx, :] = (flat @ w[:, :, dy, dx]).view(B, H, W, cout)
                if drop is not None:
                    part[:, :, dy, :, dx, :] = (grp(flat, 1) @ grp(w[:, :, dy, dx], 0)).view(B, H, W, cout)
        out = out.view(B, H * up, W * up, cout)
        return out, None if part is None else part.view(B, H * up, W * up, cout)
    cout = w.shape[0]
    oH, oW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    xp = F.pad(xn, (0, 0, pad, pad, pad, pad)) if pad else xn
    acc = torch.zeros((B * oH * oW, cout), dtype=torch.float64, device=xn.device)
    if drop is not None:
        part = torch.zeros_like(acc)
    for dy in range(k):
        for dx in range(k):
            sl = xp[:, dy:dy + stride * (oH - 1) + 1:stride, dx:dx + stride * (oW - 1) + 1:stride, :].reshape(-1, cin)
            wt = w[:, :, dy, dx].t()
            acc.addmm_(sl, wt)
            if drop is not None and drop[0] == "tap" and drop[1] == dy * k + dx:
                part.addmm_(sl, wt)
            elif drop is not None and drop[0] == "group":
                part.addmm_(grp(sl, 1), grp(wt, 0))
    return acc.view(B, oH, oW, cout), None if part is None else part.view(B, oH, oW, cout)


def epilogue(acc, scale, shift, relu):
    """conv * scale + shift, then ReLU: the order of the kernels' epilogue (scale / shift None = 1 / 0)."""
    o = acc
    if scale is not None:
        o = o * scale.double()
    if shift is not None:
        o = o + shift.double()
    return o.clamp_min(0.0) if relu else o


def bar(terms):
    """(floor, small_atol) of test_gpu_dense.py's two bars for sums of `terms` products, with sums of 2048 terms or more
    (the 3x3 256-channel layers, the 1x1 2048-channel ones) on the 5e-2 floor.  At full size the wgmma fp32 accumulation
    noise is flat in absolute terms (H100, 256 -> 128 at 180 x 180: std 2.6e-7 x max, worst 3.4e-6 x max, the same for
    the haloed and the per-tap loads and the same against the exact pair products without lo' x lo'), so its relative
    error grows as the element shrinks: 1.1e-4 between 1e-2 and 2e-2 x max, 6e-5 up to 5e-2, 2.5e-5 up to 1e-1 (1152
    terms: 6.3e-5 / 3.0e-5 / 1.5e-5).  The same bar holds up to 7200 terms (BEVDet's encoder layers at full size in every decomposition of
    test_gpu_dense_residual.py::test_bevdet_layer_every_decomposition, whose "BAR" lines print these figures, on an
    H100 80GB HBM3 at a 700 W power limit): std of the error 5.2e-7 / 7.0e-7 / 7.5e-7 x max for 4608 / 5760 / 7200
    terms, at most 3.0e-6 / 3.6e-6 / 4.9e-6 x max on the elements below 5e-2 x max, and relative error above 5e-2 x max
    at most 5.6e-5 / 7.3e-5 / 7.0e-5.  The fused CenterHead's planes (a 9 Cin-term conv, its fp16-pair rounding and a
    576-term output conv) stay on the 576-term bar, same card: relative error above 1e-2 x max at most 7.2e-5 and at
    most 1.2e-6 x max below it (test_gpu_head_fused_schedule.py's "BAR" lines).  The 1x1 convs over 2048 channels of
    BEVDet's image encoder (test_gpu_image_encoder_schedule.py, six cameras at 256 x 704, same card) do not hold the
    1e-2 floor: std 1.5e-7 / 2.1e-7 x max (stage-3 conv1 / lateral1), at most 1.3e-6 / 1.2e-6 x max below 5e-2 x max,
    so 1.15e-4 / 1.2e-4 relative at the 1e-2 floor, and relative error above 5e-2 x max at most 2.8e-5 / 2.7e-5, the
    same bits in every decomposition; 1024 terms: std 5.5e-8 to 8.3e-8 x max, at most 9.1e-7 x max below 5e-2 x max.
    BEVFusion's full-size layers (test_gpu_bevfusion_full_size.py, same card and power limit, every decomposition):
    4608 terms std 4.4e-7 x max, relative error above 5e-2 x max at most 4.4e-5; 5760 terms (reduc_conv, seeded input
    and the frame's fusion image) std 6.2e-7 / 6.7e-7 x max, at most 3.8e-6 x max below 5e-2 x max, relative at most
    6.7e-5; 9216 terms (the camera encoder's 1024-channel convs) std 8.9e-7 / 9.6e-7 x max, at most 6.3e-6 x max below,
    relative 9.4e-5 to 1.001e-4 with the whole A_hi x B_hi chain of an item (576 k-steps) in one wgmma accumulator: at
    and past the bar, and not flat (the std doubles from 4608 to 9216 terms).  The tensor core's accumulation does not
    round to nearest, so a launch whose chain is longer than 8192 terms adds the hi partial of every 9 steps into a
    round-to-nearest fp32 total (dcf::kFlush, the FLUSH instantiations); the figures up to 7200 terms are of the single
    accumulator, which those launches keep.  A lost tap or cross product would show a constant relative error instead, which the guards check."""
    return (1e-2, 2e-6) if terms < 2048 else (5e-2, 1e-5)


def rel_check_dev(name, got, want, terms, rtol=1e-4):
    """tests/parity.py's rel_check on the device: true relative error above floor x max|want|, absolute error over
    max|want| below it.  A NaN in `got` fails."""
    floor, small_atol = bar(terms)
    got, want = got.double(), want.double()
    scale = float(want.abs().max())
    err = (got - want).abs()
    if scale == 0.0:
        assert float(err.max()) == 0.0, "%s: reference is zero, output is not" % name
        return
    big = want.abs() > floor * scale
    max_rel = float((err[big] / want[big].abs()).max()) if bool(big.any()) else 0.0
    small = float(err[~big].max()) / scale if bool((~big).any()) else 0.0
    assert max_rel <= rtol, "%s: max relative error %.3e > %.1e (elements above %.0e x max)" % (name, max_rel, rtol, floor)
    assert small <= small_atol, "%s: small-element abs error %.3e x max > %.1e" % (name, small, small_atol)


def check_images(name, got, want, terms):
    """Every batch image on its own bar (images of very different magnitudes: a leak from one into the other shows)."""
    for b in range(want.shape[0]):
        rel_check_dev("%s [b%d]" % (name, b), got[b], want[b], terms)


def check_rejects(name, wrongs, want, terms):
    for what, wrong in wrongs:
        with pytest.raises(AssertionError):
            check_images(name + " guard: " + what, wrong, want, terms)


def owned_halfs(out_C, c0, cout):
    """Mask of the fp16 columns of a pixel row that channels [c0, c0 + cout) occupy (hi and lo')."""
    import torch
    m = torch.zeros(2 * out_C, dtype=torch.bool)
    c = torch.arange(c0, c0 + cout)
    m[(c // 32) * 64 + c % 32] = True
    m[(c // 32) * 64 + 32 + c % 32] = True
    return m


def sentinel_image(n_px, out_C, dev):
    import torch
    return torch.full((n_px + GUARD, 2 * out_C), SENTINEL, dtype=torch.float16, device=dev)


def assert_untouched(name, img, n_px, owned):
    """Guard pixels after the image and the columns no launch owns still hold the sentinel."""
    import torch
    s = int(torch.tensor(SENTINEL, dtype=torch.float16).view(torch.int16))
    bits = img.view(torch.int16)
    assert bool((bits[n_px:] == s).all()), "%s: guard pixels after the image were written" % name
    other = ~owned.to(img.device)
    if bool(other.any()):
        assert bool((bits[:n_px][:, other] == s).all()), "%s: channels outside the layer's were written" % name


def _bits_equal(a, b):
    import torch
    if a is None or b is None:
        return a is None and b is None
    v = torch.int16 if a.dtype == torch.float16 else torch.int32
    return torch.equal(a.view(v), b.view(v))


# --------------------------------------------------------------------------------------------------- dense cases
def _sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


class DenseCase:
    """Seeded layer: input [B, Cin, H, W] (batch image b scaled by mags[b]), conv or transposed-conv weight, BN-like
    scale / shift (bias_only: no scale, shift = bias), its fp16-pair image and the float64 reference."""

    def __init__(self, dev, B, H, W, cin, cout, k, stride, pad, up, seed, mags=(1.0,), relu=True, bias_only=False):
        import torch
        self.dev, self.B, self.H, self.W, self.cin, self.cout = dev, B, H, W, cin, cout
        self.k, self.stride, self.pad, self.up, self.relu = k, stride, pad, up, relu
        g = torch.Generator(device=dev).manual_seed(seed)
        m = torch.tensor([mags[b % len(mags)] for b in range(B)], device=dev).view(B, 1, 1, 1)
        x = torch.randn((B, cin, H, W), generator=g, device=dev) * m
        fan = cin if up > 1 else cin * k * k
        shape = (cin, cout, up, up) if up > 1 else (cout, cin, k, k)
        self.w = torch.randn(shape, generator=g, device=dev) / math.sqrt(fan)
        self.scale = None if bias_only else torch.rand((cout,), generator=g, device=dev) + 0.5
        self.shift = (torch.rand((cout,), generator=g, device=dev) - 0.5) * 0.4
        self.xh = to_pixel_h16(x)
        del x
        self.terms = fan
        self.x64 = from_pixel_h16(self.xh, B, H, W, cin)
        self.drop = ("group", cin // 64) if (up > 1 or k == 1) else ("tap", 4 if k == 3 else 0)
        self._acc = None
        self._packed = {}

    def plan(self, sms, n_tile, mode=0, m_tiles=0):
        return Plan(sms, self.B, self.H, self.W, self.cin, self.cout, n_tile, self.k, self.stride, self.pad, self.up,
                    mode, m_tiles)

    def acc(self):
        if self._acc is None:
            self._acc = conv_ref(self.x64, self.w.double(), self.k, self.stride, self.pad, self.up, self.drop)
        return self._acc

    def want(self, scale=None):
        return epilogue(self.acc()[0], self.scale if scale is None else scale, self.shift, self.relu)

    def wrongs(self):
        """The two wrong answers the bar must reject: hi x hi products only, and one tap (input group) dropped."""
        acc, part = self.acc()
        hh, _ = conv_ref(from_pixel_h16(self.xh, self.B, self.H, self.W, self.cin, hi_only=True),
                         self.w.half().double(), self.k, self.stride, self.pad, self.up)
        return [("hi x hi only", epilogue(hh, self.scale, self.shift, self.relu)),
                ("%s %d dropped" % self.drop, epilogue(acc - part, self.scale, self.shift, self.relu))]

    def packed(self, n_tile):
        from paddle3d_b200.ops import dense_conv as dc
        if n_tile not in self._packed:
            self._packed[n_tile] = (dc.pack_deconv_weight_f16 if self.up > 1 else dc.pack_conv_weight_f16)(self.w, n_tile)
        return self._packed[n_tile]

    def launch(self, n_tile, mode=0, m_tiles=0, out=None, out_C=0, c0=0, planes=True, scale=None, status=None):
        """One p3d_dense_conv2d_f16 launch into `out` (fp16-pair image of out_C channels, written at c0) and fresh
        NaN-filled fp32 planes.  Returns (planes or None, status word)."""
        import torch
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        p = self.plan(_sms(), n_tile, mode, m_tiles)
        pl = (torch.full((self.B, self.cout, p.out_H, p.out_W), float("nan"), device=self.dev) if planes else None)
        st = torch.zeros((1,), dtype=torch.int32, device=self.dev) if status is None else status
        kk, ss, pp = (self.up, self.up, 0) if self.up > 1 else (self.k, self.stride, self.pad)
        check(lib().p3d_dense_conv2d_f16(ptr(self.xh), self.B, self.H, self.W, self.cin, ptr(self.packed(n_tile)),
                                         self.cout, n_tile, kk, kk, ss, pp, self.up,
                                         ptr(self.scale if scale is None else scale), ptr(self.shift), int(self.relu),
                                         ptr(out), out_C, c0, ptr(pl), mode, m_tiles, ptr(st), stream(self.dev)),
              "dense_conv2d_f16")
        return pl, st


def run_dense(name, case, n_tile, mode=0, m_tiles=0, c0=32, h16=True, guards=True, out_C=None):
    """Launch a layer into a sentinel-filled wider fp16-pair image at channel offset c0 and into NaN-filled planes, check
    both against the reference, the sentinels, the status word and a second launch (same bits).  out_C: the image's
    channels (default: 32 more than c0 + cout rounded up to 32).  Returns (plan, image, planes)."""
    import torch
    p = case.plan(_sms(), n_tile, mode, m_tiles)
    if not h16:
        out_C = 0
    elif out_C is None:
        out_C = _cdiv(c0 + case.cout, 32) * 32 + 32
    n_px = case.B * p.out_H * p.out_W

    def once():
        img = sentinel_image(n_px, out_C, case.dev) if h16 else None
        pl, st = case.launch(n_tile, mode, m_tiles, img, out_C, c0)
        torch.cuda.synchronize()
        return img, pl, int(st[0])

    img, pl, st = once()
    want = case.want()
    assert st == 0, "%s: status %d" % (name, st)
    assert not bool(torch.isnan(pl).any()), "%s: fp32 plane elements not written" % name
    check_images(name + " fp32 planes", pl.permute(0, 2, 3, 1), want, case.terms)
    if h16:
        assert_untouched(name, img, n_px, owned_halfs(out_C, c0, case.cout))
        dec = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., c0:c0 + case.cout]
        check_images(name + " fp16-pair image", dec, want, case.terms)
        del dec
    if guards:
        check_rejects(name, case.wrongs(), want, case.terms)
    del want
    img2, pl2, _ = once()
    assert _bits_equal(img, img2) and _bits_equal(pl, pl2), "%s: a second launch gives other bits" % name
    del img2, pl2
    return p, img, pl


# -------------------------------------------------------------------------------------------------------- CPU tests
def test_restated_rings_match_the_kernel_table():
    """Cfg's ring depths as DESIGN's table lists them (a change of the shared-memory plan shows here first)."""
    want = {(128, 1, True): (2, 6), (128, 1, False): (4, 5), (64, 1, True): (2, 12), (64, 1, False): (6, 11),
            (64, 2, True): (2, 7), (64, 2, False): (3, 6)}
    assert {i: ring_depths(*i) for i in INSTS} == want
    assert [Out9Plan(132, 1, 14, 14, c, 1).na for c in (32, 64, 96, 128, 256, 320)] == [5, 5, 4, 4, 2, 2]


@pytest.mark.parametrize("sms", [132, 114])
def test_search_finds_every_regime(sms):
    """The regime search reaches R1 (idle SMs), R2 (one CTA with two items) and R3 (>= 4 items per CTA, ragged, every
    reachable ring slot, batch / N tile / tap changes between CTA 0's items) for all six instantiations, and the three
    head_out9 regimes, at 132 and at 114 SMs."""
    for inst in INSTS:
        for regime in ("R1", "R2", "R3"):
            r = search_regime(sms, inst, regime)
            assert r is not None, (sms, inst, regime)
            p = r[-1]
            assert p.inst == inst and p.oH % 8 and p.out_W % 8
            if regime == "R3":
                assert len({it[4] for it in p.cta0}) > 1 and p.n0 >= 4
    for label, B, cin, groups, in_C, _, regime in OUT9_CASES:
        r = out9_search(sms, B, cin, len(groups), regime)
        assert r is not None and r[0] % O9_T and r[1] % O9_T, (sms, label)


def test_reference_matches_oracle(oracle_mod):
    """The float64 per-tap GEMM reference against the C oracle's conv2d / deconv2d (fp64 sums, fp32 results), with and
    without the dropped tap / input group of the rejection checks."""
    import torch
    from parity import rel_check
    rng = np.random.default_rng(4)
    for cin, cout, k, stride, pad, up, h, w in ((64, 48, 3, 1, 1, 1, 13, 11), (32, 16, 3, 2, 1, 1, 15, 10),
                                                (64, 32, 1, 1, 0, 1, 7, 9), (64, 16, 2, 2, 0, 2, 5, 6),
                                                (32, 16, 4, 4, 0, 4, 3, 5)):
        x = rng.normal(size=(2, cin, h, w)).astype(np.float32)
        wt = rng.normal(size=(cin, cout, k, k) if up > 1 else (cout, cin, k, k)).astype(np.float32)
        want = oracle_mod.deconv2d(x, wt, None, up) if up > 1 else oracle_mod.conv2d(x, wt, None, stride, pad)
        xn = torch.from_numpy(x).double().permute(0, 2, 3, 1)
        drop = ("group", cin // 32 - 1) if (up > 1 or k == 1) else ("tap", 4)
        got, part = conv_ref(xn, torch.from_numpy(wt).double(), k, stride, pad, up, drop)
        rel_check("reference %d->%d k%d s%d up%d" % (cin, cout, k, stride, up), got.permute(0, 3, 1, 2).numpy(), want,
                  rtol=1e-6, small_atol=1e-7)
        xd = x.copy()
        if drop[0] == "group":
            xd[:, 32 * drop[1]:32 * drop[1] + 32] = 0
            wd = wt
        else:
            wd = wt.copy()
            wd[:, :, 1, 1] = 0
        want_d = oracle_mod.deconv2d(xd, wd, None, up) if up > 1 else oracle_mod.conv2d(xd, wd, None, stride, pad)
        rel_check("reference without %s" % (drop,), (got - part).permute(0, 3, 1, 2).numpy(), want_d, rtol=1e-6,
                  small_atol=1e-7)


# -------------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
def test_pixel_h16_built_here_matches_the_library(cuda):
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    g = torch.Generator(device=cuda).manual_seed(3)
    for B, C, H, W in ((2, 32, 9, 13), (1, 96, 31, 7), (3, 64, 5, 40)):
        x = torch.randn((B, C, H, W), generator=g, device=cuda) * torch.exp(
            torch.empty((B, C, H, W), device=cuda).uniform_(-9, 9, generator=g))
        x[0, :3, 0, 0] = torch.tensor([0.0, -0.0, 65504.0])
        h = torch.empty((B * H * W, 2 * C), dtype=torch.float16, device=cuda)
        st = torch.zeros((1,), dtype=torch.int32, device=cuda)
        check(lib().p3d_nchw_to_pixel_h16(ptr(x), B, C, H, W, ptr(h), ptr(st), stream(cuda)), "nchw_to_pixel_h16")
        assert torch.equal(to_pixel_h16(x).view(torch.int16), h.view(torch.int16))
        err = (from_pixel_h16(h, B, H, W, C) - x.permute(0, 2, 3, 1).double()).abs()
        assert bool((err <= x.permute(0, 2, 3, 1).double().abs() * 2.0 ** -21 + 2.0 ** -34).all())
        assert int(st[0]) == 0


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTS, ids=lambda i: "N%d_MT%d_%s" % (i[0], i[1], "HALO" if i[2] else "TAP"))
def test_every_instantiation_in_every_regime(cuda, inst):
    """Each instantiation forced (mode, m_tiles, N tile) in R1, R2 and R3 of this device's SM count.  R3 runs 2 or 3
    batch images of magnitudes 1, 32 and 1/8, several N tiles (the last one partly used) and, for the transposed
    conv, changing taps; its output is written at a channel offset of 16 mod 32."""
    import torch
    sms = _sms()
    N, MT, halo = inst
    for regime in ("R1", "R2", "R3"):
        r = search_regime(sms, inst, regime)
        assert r is not None, "no %s case for %s at %d SMs" % (regime, inst, sms)
        B, H, W, cin, cout, k, stride, pad, up, mode, p = r
        case = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=N * 7 + MT * 3 + halo + 100 * int(regime[1]),
                         mags=(1.0, 32.0, 0.125))
        name = "%s (%d,%d,%s) B%d %dx%d %d->%d k%d s%d up%d mode%d" % (regime, N, MT, "HALO" if halo else "TAP", B, H, W,
                                                                     cin, cout, k, stride, up, mode)
        got, _, _ = run_dense(name, case, N, mode, MT, c0=16 if regime == "R3" else 32)
        assert got.inst == inst and got.items == p.items
        print("REGIME dense %s %s: %s" % (regime, name, p.describe()))
        del case
        torch.cuda.empty_cache()


# full-size layers of both frames: (name, B, H, W, cin, cout, k, stride, pad, up, relu, bias_only, c0)
C3_LAYERS = [
    ("c3 block1 256->128", 1, 180, 180, 256, 128, 3, 1, 1, 1, True, False, 32),
    ("c3 block1 128->128", 1, 180, 180, 128, 128, 3, 1, 1, 1, True, False, 32),
    ("c3 block2 128->256 s2", 1, 180, 180, 128, 256, 3, 2, 1, 1, True, False, 32),
    ("c3 block2 256->256", 1, 90, 90, 256, 256, 3, 1, 1, 1, True, False, 32),
    ("c3 shared 512->64", 1, 180, 180, 512, 64, 3, 1, 1, 1, True, False, 32),
    ("c3 heads 64->2304", 1, 180, 180, 64, 2304, 3, 1, 1, 1, True, False, 32),
]
PP_LAYERS = [
    ("pp block1 64->64 s2", 1, 496, 432, 64, 64, 3, 2, 1, 1, True, False, 32),
    ("pp block1 64->64", 1, 248, 216, 64, 64, 3, 1, 1, 1, True, False, 16),
    ("pp block2 64->128 s2", 1, 248, 216, 64, 128, 3, 2, 1, 1, True, False, 32),
    ("pp block2 128->128", 1, 124, 108, 128, 128, 3, 1, 1, 1, True, False, 32),
    ("pp block3 128->256 s2", 1, 124, 108, 128, 256, 3, 2, 1, 1, True, False, 32),
    ("pp block3 256->256", 1, 62, 54, 256, 256, 3, 1, 1, 1, True, False, 32),
    ("pp head 384->20", 1, 248, 216, 384, 20, 1, 1, 0, 1, False, True, 0),
]
OVERFLOW_LAYERS = {"c3 block1 128->128", "pp block1 64->64 s2"}


def _n_tile(cout):
    return 128 if cout >= 128 else 64


@pytest.mark.gpu
@pytest.mark.parametrize("layer", C3_LAYERS + PP_LAYERS, ids=lambda l: l[0].replace(" ", "_"))
def test_full_size_layer(cuda, layer):
    """A dense layer of the CenterPoint (C3) or PointPillars frame at its real size with automatic mode and MT.  The N = 64
    layers also run with the other MT (same bits expected: MT only regroups pixels, every pixel sees the same k-steps);
    the 3x3 stride-1 layers also run with per-tap loads (mode 1, another summation order) on the fp64 bar; two layers
    drive one channel past fp16's range."""
    import torch
    name, B, H, W, cin, cout, k, stride, pad, up, relu, bias_only, c0 = layer
    sms = _sms()
    nt = _n_tile(cout)
    case = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=cin * 13 + cout + H, relu=relu,
                     bias_only=bias_only)
    h16 = cout % 16 == 0
    p, img, pl = run_dense(name, case, nt, c0=c0, h16=h16)
    print("REGIME layer %s: %s" % (name, p.describe()))
    out_C = _cdiv(c0 + cout, 32) * 32 + 32
    if nt == 64:
        other = 3 - p.inst[1]
        img2 = sentinel_image(B * p.out_H * p.out_W, out_C, cuda) if h16 else None
        pl2, st = case.launch(nt, 0, other, img2, out_C if h16 else 0, c0)
        torch.cuda.synchronize()
        assert int(st[0]) == 0
        assert _bits_equal(img, img2) and _bits_equal(pl, pl2), \
            "%s: MT = %d and MT = %d give other bits" % (name, p.inst[1], other)
        print("REGIME layer %s MT=%d: %s (bit-identical)" % (name, other, case.plan(sms, nt, 0, other).describe()))
        del img2, pl2
    if k == 3 and stride == 1:
        pt, _, _ = run_dense(name + " per-tap loads", case, nt, mode=1, c0=c0, guards=False)
        assert not pt.halo
        print("REGIME layer %s mode=1: %s" % (name, pt.describe()))
    if name in OVERFLOW_LAYERS:
        _check_overflow(name, case, nt, img, pl, out_C, c0)
    del case, img, pl
    torch.cuda.empty_cache()


def _check_overflow(name, case, nt, img0, pl0, out_C, c0):
    """One channel's scale x 2e6: status bit 0 set, that channel saturates at 65504 in the fp16-pair image and stays
    right in the fp32 planes, every other channel gives the bits of the unscaled launch."""
    import torch
    ch = case.cout // 3
    big = case.scale.clone()
    big[ch] = 2.0e6
    p = case.plan(_sms(), nt)
    img = sentinel_image(case.B * p.out_H * p.out_W, out_C, case.dev)
    pl, st = case.launch(nt, 0, 0, img, out_C, c0, scale=big)
    torch.cuda.synchronize()
    assert int(st[0]) & 1, "%s overflow: status bit 0 not set" % name
    want = case.want(big)[..., ch]
    f32 = pl[:, ch]
    rel_check_dev(name + " overflowing channel fp32", f32, want, case.terms)
    dec = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., c0 + ch]
    sat = f32.double().abs() > 65504
    assert int(sat.sum()) > 10, "%s: the overflow case does not overflow" % name
    assert torch.equal(dec[sat], torch.sign(f32.double()[sat]) * 65504.0), "%s: pair output does not saturate" % name
    keep = ~sat
    assert bool(((dec[keep] - f32.double()[keep]).abs() <= f32.double()[keep].abs() * 2.0 ** -21 + 2.0 ** -34).all())
    others = ~owned_halfs(out_C, c0 + ch, 1).to(img.device)
    assert torch.equal(img.view(torch.int16)[:, others], img0.view(torch.int16)[:, others]), \
        "%s overflow: other channels of the pair image changed" % name
    keep_ch = [c for c in range(case.cout) if c != ch]
    assert _bits_equal(pl[:, keep_ch].contiguous(), pl0[:, keep_ch].contiguous()), \
        "%s overflow: other fp32 planes changed" % name


# the necks: deblocks written back to back into one concat image (H, W, cin, cout, k, up) in channel order
NECKS = {
    "c3": (180, 180, [(180, 180, 128, 256, 1, 1), (90, 90, 256, 256, 2, 2)]),
    "pp": (248, 216, [(248, 216, 64, 128, 1, 1), (124, 108, 128, 128, 2, 2), (62, 54, 256, 128, 4, 4)]),
}


@pytest.mark.gpu
@pytest.mark.parametrize("neck", sorted(NECKS))
def test_full_size_neck_concat(cuda, neck):
    """The deblocks of a neck at full size, launched back to back into one concat image (c0 = 0, 256 of 512 for C3;
    0, 128, 256 of 384 for PointPillars) with NaN-filled planes each: every layer against its reference, guard pixels
    untouched, and the same bits from a second round."""
    import torch
    oH, oW, layers = NECKS[neck]
    out_C = sum(l[3] for l in layers)
    cases = [DenseCase(cuda, 1, h, w, cin, cout, k, up if up > 1 else 1, 0, up, seed=cin + cout * 3 + up)
             for h, w, cin, cout, k, up in layers]

    def round_():
        img = sentinel_image(oH * oW, out_C, cuda)
        planes, c0 = [], 0
        st = torch.zeros((1,), dtype=torch.int32, device=cuda)
        for c in cases:
            pl, _ = c.launch(_n_tile(c.cout), 0, 0, img, out_C, c0, status=st)
            planes.append(pl)
            c0 += c.cout
        torch.cuda.synchronize()
        return img, planes, int(st[0])

    img, planes, st = round_()
    assert st == 0
    assert_untouched(neck + " neck", img, oH * oW, torch.ones(2 * out_C, dtype=torch.bool))
    c0 = 0
    for c, pl in zip(cases, planes):
        name = "%s neck %d->%d up%d at c0 %d" % (neck, c.cin, c.cout, c.up, c0)
        p = c.plan(_sms(), _n_tile(c.cout))
        assert (p.out_H, p.out_W) == (oH, oW)
        want = c.want()
        assert not bool(torch.isnan(pl).any()), "%s: plane elements not written" % name
        check_images(name + " fp32 planes", pl.permute(0, 2, 3, 1), want, c.terms)
        check_images(name + " fp16-pair image", from_pixel_h16(img, 1, oH, oW, out_C)[..., c0:c0 + c.cout], want, c.terms)
        check_rejects(name, c.wrongs(), want, c.terms)
        print("REGIME neck %s: %s" % (name, p.describe()))
        c0 += c.cout
    img2, planes2, _ = round_()
    assert _bits_equal(img, img2) and all(_bits_equal(a, b) for a, b in zip(planes, planes2))


# ------------------------------------------------------------------------------------------- chained frame (PDL)
@pytest.mark.gpu
def test_chained_c3_frame_eager_and_graph(cuda):
    """The full-size CenterPoint DenseRPNHead (seeded, fp16 pairs) run layer after layer on one stream with no sync in
    between (programmatic dependent launch: every kernel must wait for its predecessor's output), once eagerly and once
    captured in a CUDA graph.  Every layer's output against the float64 reference computed from that layer's actual
    input buffer, eager and graph outputs bit-equal, status word 0."""
    import torch
    from paddle3d_b200.dense_head import DenseRPNHead
    from paddle3d_b200.ops import dense_conv as dc
    net = DenseRPNHead().init_weight(seed=7, device=cuda, randomize_bn=True, bn_gain=6.0 ** 0.5)
    bp = net._batched_params(cuda)
    big = bp["big"]
    g = torch.Generator(device=cuda).manual_seed(8)
    xh = to_pixel_h16(torch.randn((1, net.in_channels, 180, 180), generator=g, device=cuda))
    status = dc._status(cuda)

    def chain():
        recs = []  # (conv, input image, its shape, output image, out_C, c0)
        x, sh = xh, (1, 180, 180, net.in_channels)
        feats = []
        for blk in net.blocks:
            for conv in blk:
                y, _, (b, oh, ow) = conv(x, sh)
                recs.append((conv, x, sh, y, conv.cout, 0))
                x, sh = y, (b, oh, ow, conv.cout)
            feats.append((x, sh))
        fpn = net.fpn_channels
        cat = torch.empty((180 * 180, 2 * fpn), dtype=torch.float16, device=cuda)
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

    status.zero_()
    recs, planes = chain()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        recs_g, planes_g = chain()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    for i, (a, b) in enumerate(zip(recs, recs_g)):
        assert _bits_equal(a[3], b[3]), "layer %d: graph replay differs from the eager run" % i
    assert _bits_equal(planes, planes_g), "output convs: graph replay differs from the eager run"
    del recs_g, planes_g, graph
    torch.cuda.empty_cache()
    sms = _sms()
    for i, (conv, x, sh, y, out_C, c0) in enumerate(recs):
        b, h, w, cin = sh
        x64 = from_pixel_h16(x, b, h, w, cin)
        weight = conv.np["weight"] if conv is not big else np.concatenate([a.np["weight"] for hs in net.heads
                                                                           for _, a, _ in hs], 0)
        acc, _ = conv_ref(x64, torch.from_numpy(weight).to(cuda).double(), conv.k, conv.stride, conv.padding, conv.up)
        del x64
        want = epilogue(acc, conv.dev["scale"], conv.dev["shift"], conv.relu)
        del acc
        oh, ow = want.shape[1:3]
        got = from_pixel_h16(y, b, oh, ow, out_C)[..., c0:c0 + conv.cout]
        terms = cin if conv.up > 1 else cin * conv.k * conv.k
        name = "chain layer %d %d->%d k%d s%d up%d" % (i, cin, conv.cout, conv.k, conv.stride, conv.up)
        check_images(name, got, want, terms)
        p = Plan(sms, b, h, w, cin, conv.cout, conv.n_tile, conv.k, conv.stride, conv.padding, conv.up)
        print("REGIME chain %s: %s" % (name, p.describe()))
        del got, want
    # output convs: 36 groups of 3x3 64 -> 1..3 with bias over the heads' 2304-channel image
    finals = [f for hs in net.heads for _, _, f in hs]
    mid = recs[-1][3]
    X = from_pixel_h16(mid, 1, 180, 180, big.cout)
    want = torch.full(tuple(planes.shape), float("nan"), dtype=torch.float64, device=cuda)
    for gi, f in enumerate(finals):
        acc, _ = conv_ref(X[..., gi * 64:(gi + 1) * 64], torch.from_numpy(f.np["weight"]).to(cuda).double(), 3, 1, 1, 1)
        p0 = int(bp["plane0"][gi])
        want[:, p0:p0 + f.cout] = (acc + torch.from_numpy(f.np["bias"]).to(cuda).double()).permute(0, 3, 1, 2)
    assert not bool(torch.isnan(want).any())
    check_images("chain output convs (36 groups)", planes, want, 64 * 9)
    o9 = Out9Plan(sms, 1, 180, 180, 64, len(finals))
    print("REGIME chain head_out9 36 groups Cin 64 180x180: %s" % o9.describe())


# ------------------------------------------------------------------------------------------------ head_out9
def run_out9(dev, name, B, H, W, cin, groups, in_C, pass_cin0, seed):
    """One p3d_head_out_conv_f16 launch: group g convolves channels [cin0, cin0 + Cin) with its own 3x3 weights (all 3
    columns random, only cnt used) + bias into planes [plane0, plane0 + cnt); planes no group owns keep their NaN."""
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    from paddle3d_b200.ops import dense_conv as dc
    L = lib()
    gen = torch.Generator(device=dev).manual_seed(seed)
    n_planes = max(p0 + c for c, p0, _ in groups) + 2
    mags = torch.tensor([1.0, 32.0][:B], device=dev).view(B, 1, 1, 1)
    xh = to_pixel_h16(torch.randn((B, in_C, H, W), generator=gen, device=dev) * mags)
    w = torch.randn((len(groups), 3, cin, 3, 3), generator=gen, device=dev) / math.sqrt(9 * cin)
    bias = torch.randn((len(groups), 4), generator=gen, device=dev)
    blk = cin * 32 * 4
    packed = torch.zeros((len(groups) * blk,), dtype=torch.uint8, device=dev)
    for g in range(len(groups)):
        w2 = torch.zeros((cin, 32), device=dev)
        w2[:, :27] = w[g].permute(1, 2, 3, 0).reshape(cin, 27)  # W2[c][tap * 3 + j]
        check(L.p3d_dense_conv2d_f16_pack_weights(ptr(w2), 1, cin, 32, ptr(packed[g * blk:(g + 1) * blk]),
                                                  ptr(dc._status(dev)), stream(dev)), "pack_weights")
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=dev)  # noqa: E731
    cin0 = [c0 if pass_cin0 else g * cin for g, (_, _, c0) in enumerate(groups)]
    cin0_t, plane0_t, cnt_t = i32(cin0), i32([p0 for _, p0, _ in groups]), i32([c for c, _, _ in groups])

    def once():
        out = torch.full((B, n_planes, H, W), float("nan"), device=dev)
        check(L.p3d_head_out_conv_f16(ptr(xh), B, H, W, in_C, cin, len(groups), ptr(packed), ptr(bias),
                                      ptr(cin0_t if pass_cin0 else None), ptr(plane0_t), ptr(cnt_t), n_planes, ptr(out),
                                      stream(dev)), name)
        torch.cuda.synchronize()
        return out

    out = once()
    X = from_pixel_h16(xh, B, H, W, in_C)
    Xh = from_pixel_h16(xh, B, H, W, in_C, hi_only=True)
    want = torch.full((B, n_planes, H, W), float("nan"), dtype=torch.float64, device=dev)
    hh, dropped = want.clone(), want.clone()
    owned = torch.zeros(n_planes, dtype=torch.bool)
    for g, (cnt, p0, _) in enumerate(groups):
        c0 = cin0[g]
        wg = w[g].double()
        acc, part = conv_ref(X[..., c0:c0 + cin], wg, 3, 1, 1, 1, ("tap", 4))
        acc_hh, _ = conv_ref(Xh[..., c0:c0 + cin], w[g].half().double(), 3, 1, 1, 1)
        b = bias[g, :cnt].double()
        want[:, p0:p0 + cnt] = (acc[..., :cnt] + b).permute(0, 3, 1, 2)
        hh[:, p0:p0 + cnt] = (acc_hh[..., :cnt] + b).permute(0, 3, 1, 2)
        dropped[:, p0:p0 + cnt] = ((acc - part)[..., :cnt] + b).permute(0, 3, 1, 2)
        owned[p0:p0 + cnt] = True
    owned = owned.to(dev)
    assert bool(torch.isnan(out[:, ~owned]).all()), "%s: planes no group owns were written" % name
    assert not bool(torch.isnan(out[:, owned]).any()), "%s: owned plane elements not written" % name
    check_images(name, out[:, owned], want[:, owned], 9 * cin)
    check_rejects(name, [("hi x hi only", hh[:, owned]), ("tap 4 dropped", dropped[:, owned])], want[:, owned], 9 * cin)
    assert _bits_equal(out, once()), "%s: a second launch gives other bits" % name


@pytest.mark.gpu
@pytest.mark.parametrize("case", OUT9_CASES, ids=lambda c: c[0].replace(" ", "_"))
def test_head_out9_regimes(cuda, case):
    """head_out9 with one item per CTA, about two, and more than 3 kNW (the weight ring refilled by next_w many times),
    for Cin 32 / 96 / 128 / 256 / 320, groups of 1 / 2 / 3 planes with gaps, shared input slices, cin0 null, B = 2 and
    image sides that are no multiple of 14."""
    label, B, cin, groups, in_C, pass_cin0, regime = case
    sms = _sms()
    H, W, p = out9_search(sms, B, cin, len(groups), regime)
    name = "head_out9 %s %s B%d %dx%d" % (regime, label, B, H, W)
    run_out9(cuda, name, B, H, W, cin, groups, in_C, pass_cin0, seed=cin + len(groups))
    print("REGIME %s: %s" % (name, p.describe()))
