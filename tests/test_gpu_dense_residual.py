"""The residual fp16-pair dense conv in every work decomposition it runs on the device, BEVDet's encoder layers at their
real size, and BEVDet's chained encoder, against a float64 reference.

Kernel (csrc/dense_conv_f16.cu): `dcf::dense_conv_f16_kernel<N, MT, HALO, false, true>` in its six instantiations,
reached through p3d_dense_conv2d_f16_residual.  Its pair-tile epilogue reads each item's residual rows from global
memory at offsets computed from the item's batch image, tile origin and N tile, adds them after scale / shift and before
ReLU, and skips the channels of the last N tile past cout.  The launches here go through the C ABI so that the tests
control `mode`, `m_tiles`, the N tile, the output image (out_C, out_c0) and the status word.

Reference: relu(conv * scale + shift + R) in float64, with conv as in test_gpu_dense_schedule.py (the exact value of the
fp16-pair input against the fp32 weight) and R the exact value of the residual image (hi + lo' 2^-11).  The residual
image is wider than the layer (res_C > cout, channels past cout fp16 NaN in both halves: never read) and batch image b
is scaled like that image's conv output, so a residual read from the wrong place is never negligible.  Besides the two
wrong answers of test_gpu_dense_schedule.py, every case shows that the bar rejects six residual mistakes (see
ResidualCase.wrongs).

The regimes are those of test_gpu_dense_schedule.search_regime with RES_GEOM in place of REGIME_GEOM: the residual
entry point takes no transposed conv, so (64, 2, TAP) runs its R3 case as a 1x1 conv.  Lines starting with "REGIME"
(pytest -s) list the items per CTA and the ring slots at which CTA 0's items start; lines starting with "BAR" the error
figures of each full-size BEVDet launch that test_gpu_dense_schedule.bar quotes."""
import numpy as np
import pytest

from test_gpu_dense_schedule import (INSTS, REGIME_GEOM, DenseCase, Plan, _bits_equal, _cdiv, _n_tile, _sms,
                                     assert_untouched, check_images, check_rejects, conv_ref, epilogue, from_pixel_h16,
                                     owned_halfs, run_dense, search_regime, sentinel_image, to_pixel_h16)
from test_gpu_dense_tma_store import run_pairs

# REGIME_GEOM with the transposed R3 case of (64, 2, TAP) replaced by a 1x1 conv over 5 input groups (5 units per item:
# coprime to that instantiation's ring depths NA 3 / NB 6)
RES_GEOM = dict(REGIME_GEOM)
RES_GEOM[(64, 2, False)] = (REGIME_GEOM[(64, 2, False)][0], (160, 1, 1, 0, 1, 0))


def _round32(c):
    return _cdiv(c, 32) * 32


def zero_pad_input(case, cin_real):
    """Input channels [cin_real, cin) zero and the weights zero there: BEVDet's 96-channel pool image, whose channels
    80..95 are zero, and the weights _Conv(cin_pad=96) packs.  Call before the case's reference or packed weights."""
    pad = owned_halfs(case.cin, cin_real, case.cin - cin_real).to(case.dev)
    case.xh[:, pad] = 0
    case.x64 = from_pixel_h16(case.xh, case.B, case.H, case.W, case.cin)
    case.w[:, cin_real:] = 0
    case.terms = cin_real * case.k * case.k


class ResidualCase(DenseCase):
    """DenseCase (up = 1) with a residual: the pixel fp16-pair image rh [B*oH*oW, 2*res_C] of a seeded fp32 tensor whose
    batch image b is scaled by mags[b], channels [cout, res_C) fp16 NaN in both halves; r64 its exact value in channels
    [0, cout)."""

    def __init__(self, dev, B, H, W, cin, cout, k, stride, pad, seed, res_C, mags=(1.0,), relu=True, cin_real=None):
        import torch
        super().__init__(dev, B, H, W, cin, cout, k, stride, pad, 1, seed, mags, relu)
        if cin_real is not None:
            zero_pad_input(self, cin_real)
        self.oH, self.oW = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
        self.res_C = res_C
        g = torch.Generator(device=dev).manual_seed(seed + 1)
        m = torch.tensor([mags[b % len(mags)] for b in range(B)], device=dev).view(B, 1, 1, 1)
        self.rh = to_pixel_h16(torch.randn((B, res_C, self.oH, self.oW), generator=g, device=dev) * m)
        if res_C > cout:
            self.rh[:, owned_halfs(res_C, cout, res_C - cout).to(dev)] = float("nan")
        self.r64 = self.residual(self.rh)

    def residual(self, rh, hi_only=False):
        return from_pixel_h16(rh, self.B, self.oH, self.oW, self.res_C, hi_only)[..., :self.cout]

    def result(self, acc, r, scale=None, shift=None, relu=None, after_relu=False):
        """acc * scale + shift + r, then ReLU (after_relu: ReLU, then + r); scale / shift / relu None: the case's."""
        relu = self.relu if relu is None else relu
        o = epilogue(acc, self.scale if scale is None else scale, self.shift if shift is None else shift,
                     relu and after_relu) + r
        return o.clamp_min(0.0) if relu and not after_relu else o

    def want(self, scale=None):
        return self.result(self.acc()[0], self.r64, scale=scale)

    def wrongs(self):
        """The two wrong convs of DenseCase.wrongs, and the residual omitted, added after ReLU, hi halves only (lo'
        dropped), read from the neighbouring pixel column, read 8 channels off, taken from the other batch image."""
        import torch
        acc, part = self.acc()
        r = self.r64
        hh, _ = conv_ref(from_pixel_h16(self.xh, self.B, self.H, self.W, self.cin, hi_only=True), self.w.half().double(),
                         self.k, self.stride, self.pad, 1)
        out = [("hi x hi only", self.result(hh, r)),
               ("%s %d dropped" % self.drop, self.result(acc - part, r)),
               ("residual omitted", self.result(acc, torch.zeros_like(r))),
               ("residual hi halves only", self.result(acc, self.residual(self.rh, hi_only=True))),
               ("residual of the neighbouring pixel column", self.result(acc, r.roll(-1, 2))),
               ("residual 8 channels off", self.result(acc, r.roll(-8, 3)))]
        if self.relu:
            out.append(("residual after ReLU", self.result(acc, r, after_relu=True)))
        if self.B >= 2:
            out.append(("residual of the other batch image", self.result(acc, r.roll(1, 0))))
        return out

    def launch(self, n_tile, mode=0, m_tiles=0, out=None, out_C=0, c0=0, rh=None, scale=None, shift=None, relu=None,
               status=None):
        """One p3d_dense_conv2d_f16_residual launch into `out` (fp16-pair image of out_C channels, written at c0).
        Returns the status word."""
        import torch
        from paddle3d_b200._lib import check, lib
        from paddle3d_b200._mem import ptr, stream
        st = torch.zeros((1,), dtype=torch.int32, device=self.dev) if status is None else status
        check(lib().p3d_dense_conv2d_f16_residual(
            ptr(self.xh), self.B, self.H, self.W, self.cin, ptr(self.packed(n_tile)), self.cout, n_tile, self.k, self.k,
            self.stride, self.pad, 1, ptr(self.scale if scale is None else scale),
            ptr(self.shift if shift is None else shift),
            int(self.relu if relu is None else relu), ptr(out), out_C, c0, None, ptr(self.rh if rh is None else rh),
            self.res_C, mode, m_tiles, ptr(st), stream(self.dev)), "dense_conv2d_f16_residual")
        return st


def run_residual(name, case, n_tile, mode=0, m_tiles=0, c0=32, guards=True):
    """Launch into a sentinel-filled fp16-pair image wider than the layer (out_C > c0 + cout, out_C != res_C) at channel
    offset c0: status 0, sentinels untouched, no NaN, the fp64 bar, the rejected wrong answers, and a second launch
    giving the same bits.  Returns (plan, image, out_C)."""
    import torch
    p = case.plan(_sms(), n_tile, mode, m_tiles)
    out_C = _round32(c0 + case.cout) + 64
    assert out_C != case.res_C
    n_px = case.B * p.out_H * p.out_W

    def once():
        img = sentinel_image(n_px, out_C, case.dev)
        st = case.launch(n_tile, mode, m_tiles, img, out_C, c0)
        torch.cuda.synchronize()
        return img, int(st[0])

    img, st = once()
    assert st == 0, "%s: status %d" % (name, st)
    assert_untouched(name, img, n_px, owned_halfs(out_C, c0, case.cout))
    dec = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., c0:c0 + case.cout]
    assert not bool(torch.isnan(dec).any()), "%s: NaN in the output (a residual channel past cout was read)" % name
    want = case.want()
    check_images(name + " fp16-pair image", dec, want, case.terms)
    del dec
    if guards:
        check_rejects(name, case.wrongs(), want, case.terms)
    del want
    img2, _ = once()
    assert _bits_equal(img, img2), "%s: a second launch gives other bits" % name
    return p, img, out_C


# -------------------------------------------------------------------------------------------------------- CPU tests
@pytest.mark.parametrize("sms", [132, 114])
def test_residual_search_finds_every_regime(sms):
    """RES_GEOM reaches R1, R2 and R3 (>= 4 items per CTA, a ragged last round, batch and N tile changes between CTA 0's
    items, every reachable ring slot) for all six instantiations with convs the residual entry point takes (up = 1),
    the last N tile 16 channels short."""
    for inst in INSTS:
        for regime in ("R1", "R2", "R3"):
            r = search_regime(sms, inst, regime, RES_GEOM)
            assert r is not None, (sms, inst, regime)
            B, H, W, cin, cout, k, stride, pad, up, mode, p = r
            assert up == 1 and p.inst == inst and p.oH % 8 and p.oW % 8 and cout == p.n_nt * inst[0] - 16
            if regime == "R3":
                assert p.items // p.grid >= 4 and p.items % p.grid and p.rings_covered()
                assert p.cta0_varies(4) and p.cta0_varies(0)


# -------------------------------------------------------------------------------------------------------- GPU tests
@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTS, ids=lambda i: "N%d_MT%d_%s" % (i[0], i[1], "HALO" if i[2] else "TAP"))
def test_residual_every_instantiation_in_every_regime(cuda, inst):
    """Each residual instantiation forced (mode, m_tiles, N tile) in R1, R2 and R3 of this device's SM count, written at
    channel offset 32 of a wider image (R3 also at 0), residual rows 32 channels wider than the layer's N tiles.  R3 runs
    2 or 3 batch images of magnitudes 1, 32 and 1/8 and several N tiles, the last one 16 channels short (its last group
    goes through the ordinary stores)."""
    import torch
    sms = _sms()
    N, MT, halo = inst
    for regime in ("R1", "R2", "R3"):
        r = search_regime(sms, inst, regime, RES_GEOM)
        assert r is not None, "no %s case for %s at %d SMs" % (regime, inst, sms)
        B, H, W, cin, cout, k, stride, pad, up, mode, p = r
        case = ResidualCase(cuda, B, H, W, cin, cout, k, stride, pad, seed=N * 7 + MT * 3 + halo + 100 * int(regime[1]),
                            res_C=_round32(cout) + 32, mags=(1.0, 32.0, 0.125))
        name = "%s residual (%d,%d,%s) B%d %dx%d %d->%d k%d s%d mode%d res_C %d" % (
            regime, N, MT, "HALO" if halo else "TAP", B, H, W, cin, cout, k, stride, mode, case.res_C)
        got, _, _ = run_residual(name, case, N, mode, MT, c0=32)
        assert got.inst == inst and got.items == p.items
        if regime == "R3":
            run_residual(name + " c0 0", case, N, mode, MT, c0=0, guards=False)
        print("REGIME residual %s: %s" % (name, p.describe()))
        del case
        torch.cuda.empty_cache()


def error_stats(got, want):
    """The figures test_gpu_dense_schedule.bar quotes: the std of the error and its largest value on the elements below
    5e-2 x max (both over max|want|), and the largest relative error on the elements above."""
    got, want = got.double(), want.double()
    scale = float(want.abs().max())
    err = (got - want).abs()
    big = want.abs() > 5e-2 * scale
    return float(err.std()) / scale, float(err[~big].max()) / scale, float((err[big] / want[big].abs()).max())


def decomposition_runs(case):
    """(N tile, mode, m_tiles) of a full-size layer's every-decomposition runs: the frame's N tile with the MT rule's
    choice, N = 64 with both M tilings where the layer has at least 128 channels (else the other M tiling), and for the
    3x3 stride-1 layers the forced per-tap loads."""
    nt = _n_tile(case.cout)
    runs = [(nt, 0, 0)]
    if case.cout >= 128:
        runs += [(64, 0, 1), (64, 0, 2)]
    else:
        runs += [(64, 0, 3 - case.plan(_sms(), 64).inst[1])]
    if case.up == 1 and case.k == 3 and case.stride == 1:
        runs.append((nt, 1, 0))
    return runs


# BEVDet's encoder (bevdet.BEVDetEncoder) at full size: (name, H, W, cin, cout, k, stride, pad, relu, bias_only,
# residual, cin_real).  Per stage: the first block's conv1 and identity conv (3x3 stride 2 with bias, no ReLU) on the
# previous stage's output, conv1 of the second block, conv2 with the residual; then FPN_LSS and the head's shared conv.
BEVDET_LAYERS = [
    ("s1 conv1 96->160 s2", 128, 128, 96, 160, 3, 2, 1, True, False, False, 80),
    ("s1 identity 96->160 s2", 128, 128, 96, 160, 3, 2, 1, False, True, False, 80),
    ("s1 conv1 160->160", 64, 64, 160, 160, 3, 1, 1, True, False, False, None),
    ("s1 conv2 160->160 residual", 64, 64, 160, 160, 3, 1, 1, True, False, True, None),
    ("s2 conv1 160->320 s2", 64, 64, 160, 320, 3, 2, 1, True, False, False, None),
    ("s2 identity 160->320 s2", 64, 64, 160, 320, 3, 2, 1, False, True, False, None),
    ("s2 conv1 320->320", 32, 32, 320, 320, 3, 1, 1, True, False, False, None),
    ("s2 conv2 320->320 residual", 32, 32, 320, 320, 3, 1, 1, True, False, True, None),
    ("s3 conv1 320->640 s2", 32, 32, 320, 640, 3, 2, 1, True, False, False, None),
    ("s3 identity 320->640 s2", 32, 32, 320, 640, 3, 2, 1, False, True, False, None),
    ("s3 conv1 640->640", 16, 16, 640, 640, 3, 1, 1, True, False, False, None),
    ("s3 conv2 640->640 residual", 16, 16, 640, 640, 3, 1, 1, True, False, True, None),
    ("fpn 800->512", 64, 64, 800, 512, 3, 1, 1, True, False, False, None),
    ("fpn 512->512", 64, 64, 512, 512, 3, 1, 1, True, False, False, None),
    ("fpn 512->256 at 128", 128, 128, 512, 256, 3, 1, 1, True, False, False, None),
    ("fpn 1x1 256->256 bias", 128, 128, 256, 256, 1, 1, 0, False, True, False, None),
    ("head shared 256->64", 128, 128, 256, 64, 3, 1, 1, True, False, False, None),
]


@pytest.mark.gpu
@pytest.mark.parametrize("layer", BEVDET_LAYERS, ids=lambda l: l[0].replace(" ", "_").replace(">", ""))
def test_bevdet_layer_every_decomposition(cuda, layer):
    """Each encoder layer at full size (B = 1, written at channel offset 0 as the frame writes it): the frame's N tile
    with the MT rule's choice, N = 64 with both M tilings where the layer has at least 128 channels (else the other M
    tiling), and for the 3x3 stride-1 layers the forced per-tap loads.  Residual layers (residual rows of exactly cout
    channels, as the frame passes them) go through run_residual; the others check the fp32 planes and the image of the
    launch with planes against fp64, and the H16-only image bit-identical to it."""
    import torch
    name, H, W, cin, cout, k, stride, pad, relu, bias_only, res, cin_real = layer
    seed = cin * 7 + cout + H
    if res:
        case = ResidualCase(cuda, 1, H, W, cin, cout, k, stride, pad, seed, res_C=cout, relu=relu, cin_real=cin_real)
    else:
        case = DenseCase(cuda, 1, H, W, cin, cout, k, stride, pad, 1, seed, relu=relu, bias_only=bias_only)
        if cin_real is not None:
            zero_pad_input(case, cin_real)
    for i, (n, mode, mt) in enumerate(decomposition_runs(case)):
        label = "bevdet %s N%d mode%d MT%d" % (name, n, mode, mt)
        if res:
            p, img, out_C = run_residual(label, case, n, mode, mt, c0=0, guards=i == 0)
            got = from_pixel_h16(img, 1, p.out_H, p.out_W, out_C)[..., :cout]
        else:
            p, _, pl = run_dense(label, case, n, mode, mt, c0=0, guards=i == 0)
            run_pairs(label + " H16-only", case, n, mode, mt, c0=0, reference=False)
            got = pl.permute(0, 2, 3, 1)
        assert p.inst[0] == n and (mt == 0 or p.inst[1] == mt) and p.halo == (mode == 0 and k == 3 and stride == 1)
        print("REGIME bevdet %s: %s" % (label, p.describe()))
        print("BAR bevdet %s, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
              % ((label, case.terms) + error_stats(got, case.want())))
        del got
    del case
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- chained encoder (PDL)
@pytest.mark.gpu
def test_chained_bevdet_encoder_eager_and_graph(cuda):
    """BEVDet's encoder (seeded, BN gain sqrt(6)) on a real pool image (empty cells included), restated launch by launch
    on one stream with no sync in between (programmatic dependent launch: conv2 reads a residual written two launches
    earlier), once eagerly and once captured in a CUDA graph.  The chain's output is bit-equal to BEVDet.encode; graph
    and eager give the same bits in every buffer and status 0; every conv against the float64 reference computed from
    its actual input and residual buffers; every upsample bit-equal to oracle.bevdet.upsample_bilinear_fp32 of its
    actual input, at its channel offset of the concat."""
    import torch
    from oracle import bevdet as ob
    from paddle3d_b200 import synth
    from paddle3d_b200.bevdet import BEVDet
    from paddle3d_b200.ops import dense_conv as dc
    from test_gpu_bevdet import _pairs
    m = BEVDet(device=cuda).init_weight(seed=11, bn_gain=6.0 ** 0.5)
    vt = m.vt
    rng = np.random.default_rng(12)
    logits = torch.from_numpy(rng.normal(0, 2, (m.N, vt.D, vt.H, vt.W)).astype(np.float32)).to(cuda)
    tran = torch.from_numpy(rng.normal(0, 1, (m.N, vt.out_channels, vt.H, vt.W)).astype(np.float32)).to(cuda)
    img = m.image(synth.lss_mats(synth.camera_rig(31)), logits, tran)
    torch.cuda.synchronize()
    empty = (img == 0).all(1)
    assert bool(empty.any()) and not bool(empty.all()), "the pool image should have empty and filled cells"
    enc = m.encoder
    status = dc._status(cuda)

    def chain():
        convs = []  # (conv, input, its shape, residual or None, output)
        ups = []    # (input, its shape, scale, output, out_C, c0)
        x, sh = img, m.image_shape
        feats = []
        for stage in enc.stages:
            for blk in stage:
                c1, c2, down = blk["conv1"], blk["conv2"], blk["down"]
                t, _, (b, oh, ow) = c1(x, sh)
                convs.append((c1, x, sh, None, t))
                idn = x
                if down is not None:
                    idn, _, _ = down(x, sh)
                    convs.append((down, x, sh, None, idn))
                tsh = (b, oh, ow, c1.cout)
                y, _, _ = c2(t, tsh, residual=idn, res_channels=c1.cout)
                convs.append((c2, t, tsh, idn, y))
                x, sh = y, (b, oh, ow, c2.cout)
            feats.append((x, sh))
        (x0, s0), (x2, s2) = feats[enc.index[0]], feats[enc.index[1]]
        b, h, w, ch0 = s0
        cat_c = enc.cat_channels
        cat = torch.empty((b * h * w, 2 * cat_c), dtype=torch.float16, device=cuda)
        dc.upsample_bilinear_h16(x0, s0, 1, out_h16=cat, out_channels=cat_c, out_c0=0)
        ups.append((x0, s0, 1, cat, cat_c, 0))
        dc.upsample_bilinear_h16(x2, s2, enc.scale_factor, out_h16=cat, out_channels=cat_c, out_c0=ch0)
        ups.append((x2, s2, enc.scale_factor, cat, cat_c, ch0))
        f0, f1, f2, f3 = enc.fpn
        sh = (b, h, w, cat_c)
        y, _, _ = f0(cat, sh)
        convs.append((f0, cat, sh, None, y))
        sh = (b, h, w, f0.cout)
        y1, _, _ = f1(y, sh)
        convs.append((f1, y, sh, None, y1))
        sh = (b, h, w, f1.cout)
        u, (b, h, w) = dc.upsample_bilinear_h16(y1, sh, enc.extra_upsample)
        ups.append((y1, sh, enc.extra_upsample, u, f1.cout, 0))
        sh = (b, h, w, f1.cout)
        y2, _, _ = f2(u, sh)
        convs.append((f2, u, sh, None, y2))
        sh = (b, h, w, f2.cout)
        y3, _, _ = f3(y2, sh)
        convs.append((f3, y2, sh, None, y3))
        return convs, ups

    status.zero_()
    convs, ups = chain()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    out, shape = m.encode(img)
    torch.cuda.synchronize()
    assert shape == (1, 128, 128, enc.fpn_channels)
    assert _bits_equal(convs[-1][4], out), "the restated chain is not BEVDet.encode's launch sequence"
    del out
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        convs_g, ups_g = chain()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    for i, (a, g) in enumerate(zip(convs, convs_g)):
        assert _bits_equal(a[4], g[4]), "conv %d: graph replay differs from the eager run" % i
    for i, (a, g) in enumerate(zip(ups, ups_g)):
        assert _bits_equal(a[3], g[3]), "upsample %d: graph replay differs from the eager run" % i
    del convs_g, ups_g, graph
    torch.cuda.empty_cache()
    for i, (conv, x, sh, r, y) in enumerate(convs):
        b, h, w, cin = sh
        x64 = from_pixel_h16(x, b, h, w, cin)[..., :conv.cin]  # stage 1: the pool image's 80 of 96 channels
        acc, _ = conv_ref(x64, torch.from_numpy(conv.np["weight"]).to(cuda).double(), conv.k, conv.stride, conv.padding, 1)
        del x64
        o = epilogue(acc, conv.dev["scale"], conv.dev["shift"], False)
        del acc
        oh, ow = o.shape[1:3]
        if r is not None:
            o = o + from_pixel_h16(r, b, oh, ow, conv.cout)
        want = o.clamp_min(0.0) if conv.relu else o
        got = from_pixel_h16(y, b, oh, ow, conv.cout)
        name = "encoder conv %d %d->%d k%d s%d%s" % (i, conv.cin, conv.cout, conv.k, conv.stride,
                                                     " + residual" if r is not None else "")
        check_images(name, got, want, conv.cin * conv.k * conv.k)
        p = Plan(_sms(), b, h, w, cin, conv.cout, conv.n_tile, conv.k, conv.stride, conv.padding, 1)
        print("REGIME chain %s: %s" % (name, p.describe()))
        del o, want, got
    for x, (b, h, w, c), s, out, out_C, c0 in ups:
        hi, lo = _pairs(x, b, h, w, c)
        whi, wlo = (hi, lo) if s == 1 else ob.split_h16(ob.upsample_bilinear_fp32(ob.merge_h16(hi, lo), s))
        ghi, glo = _pairs(out, b, h * s, w * s, out_C)
        name = "encoder upsample x%d %d channels at c0 %d of %d" % (s, c, c0, out_C)
        assert np.array_equal(ghi[..., c0:c0 + c].view(np.int16), whi.view(np.int16)), name + ": hi halves"
        assert np.array_equal(glo[..., c0:c0 + c].view(np.int16), wlo.view(np.int16)), name + ": lo' halves"
    assert [(u[5], u[1][3]) for u in ups[:2]] == [(0, 160), (160, 640)] and ups[0][4] == 800


# ------------------------------------------------------------------------------------------- overflow semantics
@pytest.mark.gpu
@pytest.mark.parametrize("sign,relu", [(1, True), (1, False), (-1, True), (-1, False)],
                         ids=["positive_relu", "positive_no_relu", "negative_relu", "negative_no_relu"])
def test_residual_overflow(cuda, sign, relu):
    """One channel's residual set to sign * 6e4 and its shift moved by sign * 1e4 (positive) or sign * 2e4 (negative), so
    that the sum before ReLU is near 7e4 / -8e4 on every pixel: without ReLU, or with a positive sum, status bit 0 is
    set and the channel saturates at +-65504; with ReLU a negative sum clamps to 0 and leaves the bit clear.  Every other
    channel keeps the bits of the launch without the large residual."""
    import torch
    case = ResidualCase(cuda, 2, 37, 45, 160, 144, 3, 1, 1, seed=21 + sign, res_C=192, mags=(1.0, 32.0), relu=relu)
    nt, c0 = 64, 32
    p = case.plan(_sms(), nt)
    out_C = _round32(c0 + case.cout) + 64
    n_px = case.B * p.out_H * p.out_W
    base = sentinel_image(n_px, out_C, cuda)
    assert int(case.launch(nt, out=base, out_C=out_C, c0=c0)[0]) == 0
    ch = case.cout // 3
    rh = case.rh.clone()
    hi_col, lo_col = (ch // 32) * 64 + ch % 32, (ch // 32) * 64 + 32 + ch % 32
    rh[:n_px, hi_col] = sign * 6.0e4
    rh[:n_px, lo_col] = 0.0
    shift = case.shift.clone()
    shift[ch] += sign * (1.0e4 if sign > 0 else 2.0e4)
    img = sentinel_image(n_px, out_C, cuda)
    st = int(case.launch(nt, out=img, out_C=out_C, c0=c0, rh=rh, shift=shift)[0])
    torch.cuda.synchronize()
    want = case.result(case.acc()[0], case.residual(rh), shift=shift)[..., ch]
    got = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., c0 + ch]
    name = "residual overflow sign %d relu %d" % (sign, relu)
    if relu and sign < 0:
        assert bool((want == 0).all()), "%s: the case does not clamp every pixel" % name
        assert st == 0, "%s: a sum that ReLU clamps set the status bit" % name
        assert bool((got == 0).all()), "%s: clamped channel not zero" % name
    else:
        assert bool((want.abs() > 65504).all()), "%s: the case does not overflow every pixel" % name
        assert st & 1, "%s: status bit 0 not set" % name
        assert bool((got == sign * 65504.0).all()), "%s: the channel does not saturate" % name
    others = ~owned_halfs(out_C, c0 + ch, 1).to(cuda)
    assert torch.equal(img.view(torch.int16)[:, others], base.view(torch.int16)[:, others]), \
        "%s: other channels changed" % name
