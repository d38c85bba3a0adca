"""The fused CenterHead path in every work decomposition it runs on the device, its tap sum bit for bit, and the frames'
heads at their real size, against a float64 reference.

Kernels (csrc/dense_conv_f16.cu): `dcf::dense_conv_f16_kernel<128, 1, HALO, FUSE_P>` (p3d_head_conv_p_f16), the
CenterHead's batched ConvModule conv, which also runs the output convs' tap-as-N GEMM on its staged fp16-pair rows and
stores P [B][Cout / 64][H][W][28] fp32 instead of the heads' pixel fp16-pair image, and `dcf::tapsum::head_tap_sum_kernel`
(p3d_head_tap_sum), which adds P's 9 taps into the output planes.  On top of the plain <128, 1, HALO> kernel the fused
one has one more weight-ring fill per item (the N tile's two W2 images: 9 G + 1 weight steps per item, G = Cin / 32), a
second GEMM between two warpgroup barriers after the pair split, and a P store of one TMA box per consumer warpgroup at
4th coordinate (b n_ntiles + nt) 2, clipped at the bottom and right edges.  The launches go through the C ABI so that the
tests control B, H, W, Cin, Cout, the P buffer and the status word.

Reference, in float64 with X the EXACT value of the fp16-pair input and W / scale / shift / W2 / bias the fp32 values
the kernels were given: mid = relu(conv3x3(X) scale + shift); per head P[px][tap 3 + co] = sum_c mid[px][c]
W2[c][tap 3 + co]; plane = bias + sum_tap P[px shifted by the tap], 0 outside the image, which is the 3x3 output conv of
mid (test_tap_as_n_reference_is_the_output_conv).  Two checks per launch:
  * P alone against the exact value of the pair image p3d_dense_conv2d_f16 writes for the same conv times W2 (64 terms,
    bar(64)): this isolates the second GEMM from the conv, which test_gpu_dense_schedule.py covers;
  * the planes end to end against the reference from X (the composition of a 9 Cin-term conv, its pair rounding and a
    576-term output conv, on bar(9 x 64); the "BAR" lines print the measured figures).
Every batch image is checked on its own bar, and every case shows that the bar REJECTS the wrong answers of
FusedCase.wrongs and FusedCase.p_wrongs.

Which decomposition ran is restated here from the host code (nothing on the device reports it): FusedPlan is
test_gpu_dense_schedule.Plan for <128, 1, HALO> with the fused kernel's weight steps.  The regime cases are searched with
the restatement for this device's SM count.  Lines starting with "REGIME" (pytest -s) list the items per CTA and the
ring slots at which CTA 0's items start; lines starting with "BAR" the error figures against the bar."""
import math

import pytest

from test_gpu_dense_schedule import (TH, TW, Plan, _bits_equal, _sms, bar, check_images, check_rejects, conv_ref, epilogue,
                                     from_pixel_h16, rel_check_dev, to_pixel_h16)

PPITCH = 28                   # dcf::kPPitch: fp32 columns of a P row (27 used, column 27 zero)
TS_TX, TS_TY = 32, 8          # dcf::tapsum::kTX, kTY: output tile of one tap-sum block
P_GUARD = 37 * PPITCH         # NaN floats after every P buffer
MAGS = (1.0, 32.0, 0.125)     # batch image b of an input is scaled by MAGS[b]
CINS = (32, 64, 96)
PLANE_TERMS = 9 * 64          # the output convs' terms: the planes' bar


# --------------------------------------------------------------------------------------------- schedule restatement
class FusedPlan(Plan):
    """What p3d_head_conv_p_f16 launches: Plan's <128, 1, HALO> decomposition of a Cout = 128 n_nt conv, with 9 G + 1
    weight-ring steps per item (the producer's extra W2 fill), so the weight slot at which each of CTA 0's items starts
    is not the plain kernel's."""

    def __init__(self, sms, B, H, W, cin, cout):
        super().__init__(sms, B, H, W, cin, cout, 128, 3, 1, 1, 1)
        assert self.inst == (128, 1, True)
        self.steps = 9 * self.units + 1
        self.b_starts = sorted({i * self.steps % self.nb for i in range(self.n0)})

    def rings_covered(self):
        """CTA 0's items start at every slot of both rings the per-item counts can reach: multiples of gcd(G, NA) of the
        activation ring, of gcd(9 G + 1, NB) of the weight ring (NB = 6: every slot for Cin 64, every second one for Cin 32
        and 96)."""
        ga, gb = math.gcd(self.units, self.na), math.gcd(self.steps, self.nb)
        return self.a_starts == list(range(0, self.na, ga)) and self.b_starts == list(range(0, self.nb, gb))


# H = 16 ty - dh: R1 and R2 have H mod 16 in 9..15 (both warpgroups' P boxes reach into the last tile row), R3 in 1..8
# (the second warpgroup's box lies wholly below the image); W = 8 tx - 3 everywhere, so W mod 8 = 5 and W is odd
REGIME_DH = {"R1": 5, "R2": 3, "R3": 13}


def fused_search(sms, cin, regime):
    """(B, H, W, n_nt, FusedPlan) of a regime, at least 2 x 2 tiles per image: R1 the most items below the SM count (B 2,
    2 N tiles), R2 exactly SMs + 1
    items (B 1, one N tile), R3 the fewest items with at least 4 on every CTA, a ragged last round, B 2 or 3 and 5 or 7 N
    tiles (no divisor of the SM count), CTA 0's items changing batch image and N tile, and the ring coverage of
    FusedPlan.rings_covered.  None if there is no such case."""
    dh = REGIME_DH[regime]
    r3 = regime == "R3"
    best = None
    for B in ((2, 3) if r3 else (2,) if regime == "R1" else (1,)):
        for n_nt in ((5, 7) if r3 else (2,) if regime == "R1" else (1,)):
            if r3 and sms % n_nt == 0:
                continue
            for ty in range(2, 80):  # at least two tile rows and columns: items meet at tile and image edges
                for tx in range(2, 80):
                    items = B * ty * tx * n_nt
                    if (regime == "R1" and items >= sms) or (regime == "R2" and items != sms + 1) or (
                            r3 and (items < 4 * sms or (best is not None and items >= best[0]))):
                        continue
                    H, W = TH * ty - dh, TW * tx - 3
                    p = FusedPlan(sms, B, H, W, cin, 128 * n_nt)
                    assert p.items == items
                    if r3 and not (p.items // p.grid >= 4 and p.items % p.grid and p.rings_covered()
                                   and p.cta0_varies(4) and p.cta0_varies(0)):
                        continue
                    key = -items if regime == "R1" else items
                    if best is None or key < best[0]:
                        best = (key, (B, H, W, n_nt, p))
            if best is not None and r3:
                return best[1]
    return None if best is None else best[1]


# R1 cases that the search does not give: a 1 x 1 image and one smaller than an 8 x 16 tile, several batch images
# (B, H, W, n_nt)
SMALL_CASES = [(2, 1, 1, 2), (3, 5, 7, 1)]


def regime_cases(sms, cin):
    """[(label, B, H, W, n_nt, FusedPlan)]: the two small R1 cases, then R1, R2 and R3 of fused_search."""
    out = [("R1 small", B, H, W, n, FusedPlan(sms, B, H, W, cin, 128 * n)) for B, H, W, n in SMALL_CASES]
    for regime in ("R1", "R2", "R3"):
        r = fused_search(sms, cin, regime)
        assert r is not None, "no %s case for Cin %d at %d SMs" % (regime, cin, sms)
        out.append((regime,) + r)
    return out


# ----------------------------------------------------------------------------------------------------- reference
def tap_sum_ref(P, bias, plane0, cnt, n_planes, clamp=False, skip_tap=None):
    """Float64 planes [B, n_planes, H, W] of P [B, G, H, W, >= 27]: group g writes planes plane0[g] + co, co < cnt[g], as
    bias[g][co] + sum over the taps t = 3 dy + dx of P[y + dy - 1][x + dx - 1][3 t + co], with 0 for pixels outside the
    image (clamp: the nearest pixel inside instead; skip_tap: without that tap).  Planes no group writes are NaN."""
    import torch
    import torch.nn.functional as F
    B, G, H, W = P.shape[:4]
    P = P[..., :27].double()
    if clamp:
        ys = torch.arange(-1, H + 1, device=P.device).clamp(0, H - 1)
        xs = torch.arange(-1, W + 1, device=P.device).clamp(0, W - 1)
        Pp = P[:, :, ys][:, :, :, xs]
    else:
        Pp = F.pad(P, (0, 0, 1, 1, 1, 1))
    s = torch.zeros((B, G, H, W, 3), dtype=torch.float64, device=P.device)
    for t in range(9):
        if t != skip_tap:
            s += Pp[:, :, t // 3:t // 3 + H, t % 3:t % 3 + W, 3 * t:3 * t + 3]
    s += bias[:, :3].double().to(P.device).view(1, G, 1, 1, 3)
    out = torch.full((B, n_planes, H, W), float("nan"), dtype=torch.float64, device=P.device)
    for g in range(G):
        out[:, plane0[g]:plane0[g] + cnt[g]] = s[:, g, ..., :cnt[g]].permute(0, 3, 1, 2)
    return out


def tap_sum_f32(P, bias, plane0, cnt, n_planes):
    """head_tap_sum_kernel's sums restated in fp32 in its order: s = bias, then s += tap 0 .. tap 8, +0 outside."""
    import torch
    import torch.nn.functional as F
    B, G, H, W = P.shape[:4]
    Pp = F.pad(P[..., :27], (0, 0, 1, 1, 1, 1))
    s = bias[:, :3].reshape(1, G, 1, 1, 3).expand(B, G, H, W, 3).clone()
    for t in range(9):
        s = s + Pp[:, :, t // 3:t // 3 + H, t % 3:t % 3 + W, 3 * t:3 * t + 3]
    out = torch.full((B, n_planes, H, W), float("nan"), dtype=torch.float32, device=P.device)
    for g in range(G):
        out[:, plane0[g]:plane0[g] + cnt[g]] = s[:, g, ..., :cnt[g]].permute(0, 3, 1, 2)
    return out


def w2_image(wf):
    """Tap-as-N weights W2 [Cin][32] of an output conv wf [cnt <= 3, Cin, 3, 3]: W2[c][tap 3 + co] = wf[co][c][dy][dx]
    with tap = 3 dy + dx (dense_head._group_params' layout), the other columns zero."""
    import torch
    cnt, cin = wf.shape[:2]
    w2 = torch.zeros((cin, 9, 3), dtype=wf.dtype, device=wf.device)
    w2[..., :cnt] = wf.permute(1, 2, 3, 0).reshape(cin, 9, cnt)
    return torch.cat([w2.reshape(cin, 27), torch.zeros((cin, 5), dtype=wf.dtype, device=wf.device)], 1)


def figures(got, want, terms):
    """Worst over the batch images of the bar's figures: the std of the error over max|want|, the largest error below the
    floor over max|want|, and the largest relative error above it."""
    floor = bar(terms)[0]
    worst = [0.0, 0.0, 0.0]
    for b in range(want.shape[0]):
        g, w = got[b].double(), want[b].double()
        scale = float(w.abs().max())
        err = (g - w).abs()
        big = w.abs() > floor * scale
        f = [float(err.std()) / scale if err.numel() > 1 else 0.0,
             float(err[~big].max()) / scale if bool((~big).any()) else 0.0,
             float((err[big] / w[big].abs()).max()) if bool(big.any()) else 0.0]
        worst = [max(a, c) for a, c in zip(worst, f)]
    return tuple(worst)


def bar_line(label, got, want, terms):
    floor, small_atol = bar(terms)
    std, small, rel = figures(got, want, terms)
    return ("BAR %s, %d terms: error std %.2e x max, %.2e x max below %.0e x max (bar %.0e), relative %.2e above (bar 1e-4)"
            % (label, terms, std, small, floor, small_atol, rel))


# --------------------------------------------------------------------------------------------------------- cases
class FusedCase:
    """Seeded CenterHead conv of Cout = 128 n_nt channels (2 n_nt 64-channel heads), generated on the host so that every
    device gets the same values: input [B, Cin, H, W] with batch image b scaled by MAGS[b], ConvModule weights with a
    BN-like scale / shift, per head a W2 [64][32] with all 27 tap-as-N columns random and columns 27..31 zero and a bias
    [4], and groups of cnt 3, 1, 2, 3, ... planes in head order."""

    def __init__(self, dev, B, H, W, cin, n_nt, seed):
        import torch
        g = torch.Generator().manual_seed(seed)
        self.dev, self.B, self.H, self.W, self.cin = dev, B, H, W, cin
        self.cout, self.G = 128 * n_nt, 2 * n_nt
        m = torch.tensor([MAGS[b % len(MAGS)] for b in range(B)]).view(B, 1, 1, 1)
        x = torch.randn((B, cin, H, W), generator=g) * m
        self.w = (torch.randn((self.cout, cin, 3, 3), generator=g) / math.sqrt(9 * cin)).to(dev)
        self.scale = (torch.rand((self.cout,), generator=g) + 0.5).to(dev)
        self.shift = ((torch.rand((self.cout,), generator=g) - 0.5) * 0.4).to(dev)
        w2 = torch.zeros((self.G, 64, 32))
        w2[..., :27] = torch.randn((self.G, 64, 27), generator=g) / 8.0
        self.w2 = w2.to(dev)
        self.bias = (torch.randn((self.G, 4), generator=g) * 0.1).to(dev)
        self.cnt = [(3, 1, 2)[h % 3] for h in range(self.G)]
        self.plane0 = [sum(self.cnt[:h]) for h in range(self.G)]
        self.n_planes = sum(self.cnt)
        self.xh = to_pixel_h16(x.to(dev))
        self.x64 = from_pixel_h16(self.xh, B, H, W, cin)
        self._acc = self._packed = self._packed_w2 = None

    def plan(self, sms):
        return FusedPlan(sms, self.B, self.H, self.W, self.cin, self.cout)

    # ---- reference
    def acc(self):
        if self._acc is None:
            self._acc = conv_ref(self.x64, self.w.double(), 3, 1, 1, 1, ("tap", 4))
        return self._acc

    def mid(self, drop_tap=False, relu=True):
        acc, part = self.acc()
        return epilogue(acc - part if drop_tap else acc, self.scale, self.shift, relu)

    def p_of(self, mid, w2=None):
        """P [B, G, H, W, 27] of a mid image [B, H, W, Cout] (float64)."""
        import torch
        w2 = (self.w2 if w2 is None else w2)[..., :27].double()
        return torch.einsum("bhwgc,gcn->bghwn", mid.reshape(self.B, self.H, self.W, self.G, 64), w2)

    def planes_of(self, P, **kw):
        return tap_sum_ref(P, self.bias, self.plane0, self.cnt, self.n_planes, **kw)

    def owned(self):
        import torch
        m = torch.zeros(self.n_planes, dtype=torch.bool)
        for p0, c in zip(self.plane0, self.cnt):
            m[p0:p0 + c] = True
        return m.to(self.dev)

    @staticmethod
    def swap_heads(P):
        """The two heads of every N tile swapped."""
        B, G = P.shape[:2]
        return P.reshape((B, G // 2, 2) + tuple(P.shape[2:])).flip(2).reshape(P.shape)

    def p_wrongs(self, mid_k):
        """Wrong P answers from the pair image mid_k: the hi x hi products alone, the heads of each N tile swapped, another
        batch image's P, every N tile's P made with the next N tile's W2 images."""
        import torch
        P = self.p_of(mid_k)
        yield "hi x hi only", self.p_of(mid_k.half().double(), self.w2.half().double())
        yield "heads of an N tile swapped", self.swap_heads(P)
        if self.B > 1:
            yield "another batch image's P", P.roll(1, 0)
        if self.G > 2:
            yield "the next N tile's W2", self.p_of(mid_k, torch.roll(self.w2, -2, 0))

    def wrongs(self):
        """Wrong planes from the reference: the P GEMM with hi x hi products only, one ConvModule tap dropped, one output
        conv tap dropped, the two heads of each N tile swapped, another batch image's P, mid without ReLU, neighbours
        outside the image read as the nearest pixel inside (clamped) instead of 0."""
        mid = self.mid()
        P = self.p_of(mid)
        yield "P GEMM hi x hi only", self.planes_of(self.p_of(mid.half().double(), self.w2.half().double()))
        yield "ConvModule tap 4 dropped", self.planes_of(self.p_of(self.mid(drop_tap=True)))
        yield "output conv tap 4 dropped", self.planes_of(P, skip_tap=4)
        yield "heads of an N tile swapped", self.planes_of(self.swap_heads(P))
        if self.B > 1:
            yield "another batch image's P", self.planes_of(P.roll(1, 0))
        yield "mid without ReLU", self.planes_of(self.p_of(self.mid(relu=False)))
        yield "clamped neighbours", self.planes_of(P, clamp=True)

    # ---- launches
    def packed(self):
        from paddle3d_b200.ops import dense_conv as dc
        if self._packed is None:
            self._packed = dc.pack_conv_weight_f16(self.w, 128)
        return self._packed

    def packed_w2(self):
        """Per head p3d_dense_conv2d_f16_pack_weights(taps 1, Cin 64, n_tile 32) of its W2, as run_out9 packs it; head h at
        byte 8192 h, so N tile nt's two images are bytes [16384 nt, 16384 (nt + 1))."""
        import torch
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        from paddle3d_b200.ops import dense_conv as dc
        if self._packed_w2 is None:
            blk = 64 * 32 * 4
            out = torch.zeros((self.G * blk,), dtype=torch.uint8, device=self.dev)
            for h in range(self.G):
                wt = self.w2[h].contiguous()
                check(lib().p3d_dense_conv2d_f16_pack_weights(ptr(wt), 1, 64, 32, ptr(out[h * blk:(h + 1) * blk]),
                                                              ptr(dc._status(self.dev)), stream(self.dev)), "pack_weights")
            self._packed_w2 = out
        return self._packed_w2

    def group_tensors(self):
        import torch
        i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=self.dev)  # noqa: E731
        return i32(self.plane0), i32(self.cnt)

    def conv_p(self, status):
        """One p3d_head_conv_p_f16 launch into a NaN-filled P buffer with P_GUARD NaN floats after it (flat)."""
        import torch
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        n = self.B * self.G * self.H * self.W * PPITCH
        pbuf = torch.full((n + P_GUARD,), float("nan"), device=self.dev)
        check(lib().p3d_head_conv_p_f16(ptr(self.xh), self.B, self.H, self.W, self.cin, ptr(self.packed()), self.cout,
                                        ptr(self.scale), ptr(self.shift), ptr(self.packed_w2()), ptr(pbuf), ptr(status),
                                        stream(self.dev)), "head_conv_p_f16")
        return pbuf

    def p_view(self, pbuf):
        return pbuf[:self.B * self.G * self.H * self.W * PPITCH].view(self.B, self.G, self.H, self.W, PPITCH)

    def tap_sum(self, P):
        """p3d_head_tap_sum of P [B, G, H, W, 28] into NaN-filled planes."""
        return run_tap_sum(P, self.bias, *self.group_tensors(), self.n_planes)

    def pair_image(self, status):
        """The same conv by p3d_dense_conv2d_f16 (its <128, 1, HALO> instantiation): the pixel fp16-pair image that the
        fused kernel stages instead of storing."""
        import torch
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        img = torch.empty((self.B * self.H * self.W, 2 * self.cout), dtype=torch.float16, device=self.dev)
        check(lib().p3d_dense_conv2d_f16(ptr(self.xh), self.B, self.H, self.W, self.cin, ptr(self.packed()), self.cout,
                                         128, 3, 3, 1, 1, 1, ptr(self.scale), ptr(self.shift), 1, ptr(img), self.cout, 0,
                                         None, 0, 0, ptr(status), stream(self.dev)), "dense_conv2d_f16")
        return img


def run_tap_sum(P, bias, plane0_t, cnt_t, n_planes):
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    B, G, H, W, _ = P.shape
    out = torch.full((B, n_planes, H, W), float("nan"), device=P.device)
    check(lib().p3d_head_tap_sum(ptr(P), B, H, W, G, ptr(bias), ptr(plane0_t), ptr(cnt_t), n_planes, ptr(out),
                                 stream(P.device)), "head_tap_sum")
    return out


def run_fused(name, case):
    """Launch the fused conv and the tap sum and check: P written exactly where it should be (columns 0..26 finite,
    column 27 zero, the guard tail still NaN), P against the exact pair image times W2, the planes against the reference
    from X, the rejected wrong answers of both, status 0, and a second launch giving the same bits."""
    import torch
    st = torch.zeros((1,), dtype=torch.int32, device=case.dev)
    pbuf = case.conv_p(st)
    P = case.p_view(pbuf)
    planes = case.tap_sum(P)
    torch.cuda.synchronize()
    assert int(st[0]) == 0, "%s: status %d" % (name, int(st[0]))
    assert bool(torch.isfinite(P[..., :27]).all()), "%s: P elements not written (or not finite)" % name
    assert bool((P[..., 27] == 0).all()), "%s: P column 27 is not zero" % name
    assert bool(torch.isnan(pbuf[P.numel():]).all()), "%s: the P buffer's guard tail was written" % name
    owned = case.owned()
    assert bool(torch.isnan(planes[:, ~owned]).all()), "%s: planes no group owns were written" % name
    assert not bool(torch.isnan(planes[:, owned]).any()), "%s: owned plane elements not written" % name

    # P alone: the exact pair image of the plain conv (checked against fp64 here too) times the fp32 W2
    img = case.pair_image(st)
    torch.cuda.synchronize()
    assert int(st[0]) == 0, "%s: status %d after the plain conv" % (name, int(st[0]))
    mid_k = from_pixel_h16(img, case.B, case.H, case.W, case.cout)
    del img
    mid = case.mid()
    check_images(name + " plain conv's pair image", mid_k, mid, 9 * case.cin)
    want_p = case.p_of(mid_k)
    print(bar_line(name + " P", P[..., :27], want_p, 64))
    check_images(name + " P", P[..., :27], want_p, 64)
    check_rejects(name + " P", case.p_wrongs(mid_k), want_p, 64)
    del want_p, mid_k

    # the planes end to end
    want = case.planes_of(case.p_of(mid))[:, owned]
    del mid
    print(bar_line(name + " planes", planes[:, owned], want, PLANE_TERMS))
    check_images(name + " planes", planes[:, owned], want, PLANE_TERMS)
    check_rejects(name + " planes", ((w, x[:, owned]) for w, x in case.wrongs()), want, PLANE_TERMS)
    del want

    pbuf2 = case.conv_p(st)
    planes2 = case.tap_sum(case.p_view(pbuf2))
    torch.cuda.synchronize()
    assert int(st[0]) == 0
    assert _bits_equal(pbuf, pbuf2) and _bits_equal(planes, planes2), "%s: a second launch gives other bits" % name


# -------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("sms", [132, 114])
def test_fused_search_finds_every_regime(sms):
    """For Cin 32, 64 and 96 the search reaches R1 (idle SMs; with a 1 x 1 image and one smaller than a tile), R2 (SMs
    + 1 items) and R3 (>= 4 items per CTA, ragged, B 2 or 3, 5 or 7 N tiles, batch and N tile changes between CTA 0's
    items, every reachable ring slot: all six weight slots for Cin 64, every second one for Cin 32 and 96); over the
    cases the image heights put the second warpgroup's P box both inside and wholly below the last tile row, and the
    widths and heights are ragged against the conv's 8 x 16 and the tap sum's 8 x 32 tiles."""
    for cin in CINS:
        cases = regime_cases(sms, cin)
        for label, B, H, W, n_nt, p in cases:
            assert p.inst == (128, 1, True) and p.steps == 9 * cin // 32 + 1 and (p.na, p.nb) == (2, 6)
            assert W % TW and W % TS_TX and H % TS_TY, (sms, cin, label)
            if label == "R1" or label == "R1 small":
                assert p.items < sms
            elif label == "R2":
                assert p.items == sms + 1 and p.n0 == 2
            else:
                assert B in (2, 3) and n_nt in (5, 7) and sms % n_nt
                assert p.items // p.grid >= 4 and p.items % p.grid and p.cta0_varies(4) and p.cta0_varies(0)
                assert p.rings_covered()
                assert p.b_starts == (list(range(6)) if cin == 64 else [0, 2, 4]), (sms, cin, p.b_starts)
                assert p.a_starts == ([0] if cin == 64 else [0, 1])
        assert {H % TH for _, _, H, _, _, _ in cases} & set(range(1, 9))
        assert {H % TH for _, _, H, _, _, _ in cases} & set(range(9, 16))
        assert any(H == 1 and W == 1 for _, _, H, W, _, _ in cases)
        assert any(H < TH and W < TW and (H, W) != (1, 1) for _, _, H, W, _, _ in cases)


def test_fused_plan_weight_slots():
    """The extra W2 fill moves CTA 0's items' weight-ring starts off the plain kernel's: with 2 items per CTA a Cin 64
    conv's second item starts at slot 19 mod 6 = 1 (plain: 18 mod 6 = 0)."""
    p = FusedPlan(132, 1, 16, 8 * 133, 64, 128)
    q = Plan(132, 1, 16, 8 * 133, 64, 128, 128, 3, 1, 1, 1)
    assert p.items == q.items == 133 and p.n0 == q.n0 == 2
    assert (p.steps, p.b_starts) == (19, [0, 1]) and (q.steps, q.b_starts) == (18, [0])


def test_tap_as_n_reference_is_the_output_conv(oracle_mod):
    """P[px][tap 3 + co] = sum_c mid[px][c] W2[c][tap 3 + co], then bias + sum_tap P[shifted px] with 0 outside the
    image, equals in float64 the direct 3x3 conv of mid by the output conv's weights (cnt 1, 2 and 3, ragged images and
    a 1 x 1 one), which equals oracle.conv2d: this pins the W2 layout [c][tap 3 + co] that the tests pack."""
    import numpy as np
    import torch
    from parity import rel_check
    rng = np.random.default_rng(11)
    for cnt, (B, H, W) in zip((1, 2, 3, 3), ((2, 9, 13), (1, 17, 5), (2, 6, 33), (1, 1, 1))):
        mid = np.maximum(rng.normal(size=(B, 64, H, W)), 0).astype(np.float32)
        wf = rng.normal(size=(cnt, 64, 3, 3)).astype(np.float32)
        bias = rng.normal(size=(cnt,)).astype(np.float32)
        want = oracle_mod.conv2d(mid, wf, bias, 1, 1)
        m64 = torch.from_numpy(mid).double().permute(0, 2, 3, 1)
        direct, _ = conv_ref(m64, torch.from_numpy(wf).double(), 3, 1, 1, 1)
        direct = direct + torch.from_numpy(bias).double()
        rel_check("direct conv cnt %d %dx%d" % (cnt, H, W), direct.permute(0, 3, 1, 2).numpy(), want, rtol=1e-6,
                  small_atol=1e-7)
        w2 = w2_image(torch.from_numpy(wf).double())
        assert w2.shape == (64, 32) and not bool(w2[:, 27:].any())
        P = torch.einsum("bhwc,cn->bhwn", m64, w2).unsqueeze(1)
        b4 = torch.zeros((1, 4), dtype=torch.float64)
        b4[0, :cnt] = torch.from_numpy(bias).double()
        got = tap_sum_ref(P, b4, [1], [cnt], cnt + 2)
        assert bool(torch.isnan(got[:, 0]).all()) and bool(torch.isnan(got[:, cnt + 1]).all())
        got = got[:, 1:cnt + 1]
        assert float((got - direct.permute(0, 3, 1, 2)).abs().max()) <= 1e-12 * float(direct.abs().max())
        # the clamped tap sum (a wrong answer of the GPU tests) differs from the zero-padded one
        assert float((tap_sum_ref(P, b4, [0], [cnt], cnt, clamp=True) - got).abs().max()) > 1e-3


# -------------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("cin", CINS)
def test_fused_conv_p_every_regime(cuda, cin):
    """p3d_head_conv_p_f16 and p3d_head_tap_sum in the two small R1 cases and in R1, R2 and R3 of this device's SM
    count: P and the planes against fp64, the rejected wrong answers, the P buffer's edges, status 0 and repeatable
    bits."""
    import torch
    sms = _sms()
    for label, B, H, W, n_nt, p in regime_cases(sms, cin):
        case = FusedCase(cuda, B, H, W, cin, n_nt, seed=cin * 5 + n_nt + H + W)
        name = "fused %s cin%d B%d %dx%d %d->%d" % (label, cin, B, H, W, cin, case.cout)
        assert case.plan(sms).items == p.items
        print("REGIME %s: %s" % (name, p.describe()))
        run_fused(name, case)
        del case
        torch.cuda.empty_cache()


# (H, W): the 8 x 32 tap-sum tile, ragged against it both ways, a single row / column / pixel
TAP_SUM_SHAPES = [(8, 32), (13, 70), (17, 33), (1, 1), (1, 40), (37, 1)]
# (cnt, plane0) per group: cnt 1, 2 and 3, planes out of order, planes 3, 5, 8, 11 and 15 owned by no group
TAP_SUM_GROUPS = [(2, 9), (3, 0), (1, 4), (3, 12), (2, 6)]


@pytest.mark.gpu
@pytest.mark.parametrize("hw", TAP_SUM_SHAPES, ids=lambda s: "%dx%d" % s)
def test_tap_sum_bit_for_bit(cuda, hw):
    """p3d_head_tap_sum on a synthetic P buffer of B = 3 is bit-equal to the fp32 restatement in its order; the P
    columns a group does not use (column 27 and the columns of co >= cnt) and the bias entries past cnt hold NaN and
    reach no plane; planes that no group owns stay NaN."""
    import torch
    H, W = hw
    B, n_planes = 3, 16
    G = len(TAP_SUM_GROUPS)
    g = torch.Generator().manual_seed(H * 100 + W)
    P = torch.randn((B, G, H, W, PPITCH), generator=g)
    bias = torch.randn((G, 4), generator=g)
    P[..., 27] = float("nan")
    for gi, (cnt, _) in enumerate(TAP_SUM_GROUPS):
        for co in range(cnt, 3):
            P[:, gi, ..., co::3][..., :9] = float("nan")
        bias[gi, cnt:] = float("nan")
    P, bias = P.to(cuda), bias.to(cuda)
    plane0 = [p0 for _, p0 in TAP_SUM_GROUPS]
    cnt = [c for c, _ in TAP_SUM_GROUPS]
    i32 = lambda v: torch.tensor(v, dtype=torch.int32, device=cuda)  # noqa: E731
    got = run_tap_sum(P, bias, i32(plane0), i32(cnt), n_planes)
    want = tap_sum_f32(P, bias, plane0, cnt, n_planes)
    torch.cuda.synchronize()
    owned = torch.zeros(n_planes, dtype=torch.bool, device=cuda)
    for c, p0 in TAP_SUM_GROUPS:
        owned[p0:p0 + c] = True
    assert bool(torch.isnan(got[:, ~owned]).all()), "planes no group owns were written"
    assert not bool(torch.isnan(got[:, owned]).any()), "an unused P column or bias entry reached a plane"
    assert _bits_equal(got, want), "tap sum differs from its fp32 restatement"
    # and within fp32 rounding of the float64 sums (the restatement is the tap sum, not a second copy of a mistake)
    ref = tap_sum_ref(P.nan_to_num(0.0), bias.nan_to_num(0.0), plane0, cnt, n_planes)
    rel_check_dev("tap sum %dx%d" % hw, got[:, owned], ref[:, owned], 9)


# full-size heads: (label, model, B)
FULL_HEADS = [("voxel 180x180", "voxel", 1), ("pillars 128x128", "pillars", 1), ("pillars 128x128 B2", "pillars", 2)]


@pytest.mark.gpu
@pytest.mark.parametrize("head", FULL_HEADS, ids=lambda h: h[0].replace(" ", "_"))
def test_full_size_head_fused(cuda, head):
    """DenseRPNHead.forward through the fused path with its own packed parameters (bp["big"], packed9, bias9, plane0_9,
    cnt9) on the CenterPoint-voxel head at 180 x 180 and the CenterPoint-pillars / BEVDet head at 128 x 128 (B 1 and 2):
    every output, by name and task, against the float64 reference from the module's fp32 parameters and the exact value
    of its trunk output."""
    import torch
    from paddle3d_b200.dense_head import DenseRPNHead
    label, model, B = head
    if model == "voxel":
        net = DenseRPNHead(256).init_weight(seed=5, device=cuda, randomize_bn=True)
        shape_in = (B, 256, 180, 180)
    else:
        from paddle3d_b200.centerpoint_pillars import CenterPointPillars
        m = CenterPointPillars()
        net = m.head.init_weight(seed=6, device=cuda, randomize_bn=True)
        shape_in = (B, m.C, m.grid[1], m.grid[0])
    bp = net._batched_params(cuda)
    assert net.fused_heads(bp)
    g = torch.Generator().manual_seed(7 + B)
    bev = torch.randn(shape_in, generator=g).to(cuda)
    s, shape = net._trunk(bev)
    got = net.forward(bev)
    torch.cuda.synchronize()
    b, H, W, cin = shape
    assert (b, H, W) == ((B, 180, 180) if model == "voxel" else (B, 128, 128))
    heads = [(name, a, f) for hs in net.heads for name, a, f in hs]
    S = from_pixel_h16(s, b, H, W, cin)
    wbig = torch.cat([torch.from_numpy(a.np["weight"]) for _, a, _ in heads], 0).to(cuda).double()
    acc, _ = conv_ref(S, wbig, 3, 1, 1, 1)
    del S, wbig
    mid = epilogue(acc, torch.cat([a.dev["scale"] for _, a, _ in heads]), torch.cat([a.dev["shift"] for _, a, _ in heads]),
                   True)
    del acc
    want = {}
    for i, (name, _, f) in enumerate(heads):
        o, _ = conv_ref(mid[..., 64 * i:64 * (i + 1)], torch.from_numpy(f.np["weight"]).to(cuda).double(), 3, 1, 1, 1)
        want.setdefault(name, []).append((o + torch.from_numpy(f.np["bias"]).to(cuda).double()).permute(0, 3, 1, 2))
    del mid
    assert sorted(want) == sorted(got) and all(len(want[n]) == len(got[n]) == len(net.tasks) for n in want)
    for name in sorted(want):
        worst = [0.0, 0.0, 0.0]
        for t, (gt, wt) in enumerate(zip(got[name], want[name])):
            assert tuple(gt.shape) == tuple(wt.shape)
            worst = [max(a, c) for a, c in zip(worst, figures(gt, wt, PLANE_TERMS))]
        print("BAR full-size head %s %s (%d tasks), %d terms: error std %.2e x max, %.2e x max below 1e-2 x max, "
              "relative %.2e above" % ((label, name, len(net.tasks), PLANE_TERMS) + tuple(worst)))
        for t, (gt, wt) in enumerate(zip(got[name], want[name])):
            check_images("%s %s task %d" % (label, name, t), gt, wt, PLANE_TERMS)
