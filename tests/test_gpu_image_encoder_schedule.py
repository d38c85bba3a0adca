"""BEVDet's image encoder (bevdet.BEVDetImageEncoder: ResNet-50, CustomFPN and the depth net) on the dense fp16-pair
conv in every work decomposition, layer by layer at full size and as the chained encoder, against a float64 reference.

The encoder issues 56 p3d_dense_conv2d_f16{,_residual} launches per frame, 27 distinct ones (IMAGE_LAYERS), at shapes no
other schedule test reaches: 1x1 stride-2 pad-0 convs (the downsample identities, on the per-tap path with a TMA element
stride of 2), Cin 1024 and 2048 (32 and 64 k-units per item), six batch images (cameras), M tiles mostly empty (oH 8 and
4 against a 16-row tile), a 1x1 conv3 whose residual is the downsample conv launched just before it, lateral0 whose
residual rows are the nearest-upsampled lateral1, and the depth net's 208 computed channels (198 real) written into
224-channel rows.

Machinery, reference and bar are those of test_gpu_dense_schedule.py (DenseCase, run_dense, Plan, search_regime, bar)
and test_gpu_dense_residual.py (ResidualCase, run_residual): X the exact value of the fp16-pair input, W the fp32
weight, the epilogue in the kernels' order, per batch image 1e-4 true relative error above bar()'s floor.  Every
guarded case shows that the bar rejects the "hi x hi only" answer and a dropped tap or input group (residual cases also
the six residual mistakes).  Lines starting with "REGIME" (pytest -s) list the items per CTA and the ring slots at
which CTA 0's items start; lines starting with "BAR" the error figures of each full-size launch that
test_gpu_dense_schedule.bar quotes."""
import numpy as np
import pytest

from test_gpu_dense_residual import ResidualCase, error_stats, run_residual
from test_gpu_dense_schedule import (REGIME_GEOM, SENTINEL, DenseCase, Plan, _bits_equal, _n_tile, _sms, check_images,
                                     check_rejects, conv_ref, epilogue, from_pixel_h16, run_dense, search_regime,
                                     sentinel_image)
from test_gpu_dense_tma_store import run_pairs

CAM_MAGS = (1.0, 32.0, 0.125, 4.0, 0.5, 2.0)  # one magnitude per camera: a leak from one camera into another shows
TAP_INSTS = [(128, 1, False), (64, 1, False), (64, 2, False)]

# REGIME_GEOM with every per-tap instantiation running a 1x1 stride-2 pad-0 conv (forced mode 1), the downsample
# identity of the ResNet's stages 1-3.  Cin coprime to the instantiation's ring depths: 224 (7 units; NA 4, NB 5) for
# (128, 1), 160 (5 units; NA 6 / NB 11 and NA 3 / NB 6) for (64, 1) and (64, 2).
IMG_GEOM = dict(REGIME_GEOM)
for _inst, _cin in zip(TAP_INSTS, (224, 160, 160)):
    IMG_GEOM[_inst] = ((_cin, 1, 2, 0, 1, 1), (_cin, 1, 2, 0, 1, 1))

# The distinct launches of the encoder at 256 x 704, six cameras: (name, H, W, cin, cout, k, stride, pad, relu,
# bias_only, residual).  H x W is the layer's input; the depth net computes cout_pad 208 channels (198 real).
IMAGE_LAYERS = [
    ("s0 conv1 64->64", 64, 176, 64, 64, 1, 1, 0, True, False, False),
    ("s0 conv1 256->64", 64, 176, 256, 64, 1, 1, 0, True, False, False),
    ("s0 conv2 64->64", 64, 176, 64, 64, 3, 1, 1, True, False, False),
    ("s0 down 64->256", 64, 176, 64, 256, 1, 1, 0, False, False, False),
    ("s0 conv3 64->256 residual", 64, 176, 64, 256, 1, 1, 0, True, False, True),
    ("s1 conv1 256->128", 64, 176, 256, 128, 1, 1, 0, True, False, False),
    ("s1 conv2 128->128 s2", 64, 176, 128, 128, 3, 2, 1, True, False, False),
    ("s1 down 256->512 s2", 64, 176, 256, 512, 1, 2, 0, False, False, False),
    ("s1 conv3 128->512 residual", 32, 88, 128, 512, 1, 1, 0, True, False, True),
    ("s1 conv1 512->128", 32, 88, 512, 128, 1, 1, 0, True, False, False),
    ("s1 conv2 128->128", 32, 88, 128, 128, 3, 1, 1, True, False, False),
    ("s2 conv1 512->256", 32, 88, 512, 256, 1, 1, 0, True, False, False),
    ("s2 conv2 256->256 s2", 32, 88, 256, 256, 3, 2, 1, True, False, False),
    ("s2 down 512->1024 s2", 32, 88, 512, 1024, 1, 2, 0, False, False, False),
    ("s2 conv3 256->1024 residual", 16, 44, 256, 1024, 1, 1, 0, True, False, True),
    ("s2 conv1 1024->256", 16, 44, 1024, 256, 1, 1, 0, True, False, False),
    ("s2 conv2 256->256", 16, 44, 256, 256, 3, 1, 1, True, False, False),
    ("s3 conv1 1024->512", 16, 44, 1024, 512, 1, 1, 0, True, False, False),
    ("s3 conv2 512->512 s2", 16, 44, 512, 512, 3, 2, 1, True, False, False),
    ("s3 down 1024->2048 s2", 16, 44, 1024, 2048, 1, 2, 0, False, False, False),
    ("s3 conv3 512->2048 residual", 8, 22, 512, 2048, 1, 1, 0, True, False, True),
    ("s3 conv1 2048->512", 8, 22, 2048, 512, 1, 1, 0, True, False, False),
    ("s3 conv2 512->512", 8, 22, 512, 512, 3, 1, 1, True, False, False),
    ("lateral1 2048->512 bias", 8, 22, 2048, 512, 1, 1, 0, False, True, False),
    ("lateral0 1024->512 bias residual", 16, 44, 1024, 512, 1, 1, 0, False, True, True),
    ("fpn 512->512 bias", 16, 44, 512, 512, 3, 1, 1, False, True, False),
    ("depth net 512->208 bias", 16, 44, 512, 208, 1, 1, 0, False, True, False),
]
DEPTH_REAL = 198  # D + C of the depth net: 118 depth bins + 80 context channels


def _out_hw(conv, h, w):
    return (h + 2 * conv.padding - conv.k) // conv.stride + 1, (w + 2 * conv.padding - conv.k) // conv.stride + 1


def _entry(conv, h, w, residual):
    """A launch of `conv` on an h x w input as IMAGE_LAYERS lists it (without the name)."""
    return (h, w, conv.cin, conv.cout_pad or conv.cout, conv.k, conv.stride, conv.padding, conv.relu,
            conv.has_bias and conv.bn_eps is None, residual)


def encoder_launches(enc, H, W):
    """Every dense-conv launch of BEVDetImageEncoder `enc` on H x W images, in launch order (the stem excluded)."""
    from paddle3d_b200.ops import dense_conv as dc
    h, w = dc.stem_shape(H, W)
    out, sizes = [], []
    for stage in enc.stages:
        for blk in stage:
            oh, ow = _out_hw(blk["conv2"], h, w)
            out += [_entry(blk["conv1"], h, w, False), _entry(blk["conv2"], h, w, False)]
            if blk["down"] is not None:
                out.append(_entry(blk["down"], h, w, False))
            out.append(_entry(blk["conv3"], oh, ow, True))
            h, w = oh, ow
        sizes.append((h, w))
    (h0, w0), (h1, w1) = sizes[enc.out_indices[0]], sizes[enc.out_indices[1]]
    l0, l1 = enc.lateral
    return out + [_entry(l1, h1, w1, False), _entry(l0, h0, w0, True), _entry(enc.fpn_conv, h0, w0, False),
                  _entry(enc.depth_net, h0, w0, False)]


def _image_encoder():
    from paddle3d_b200.bevdet import DEPTH_NET, IMG_BACKBONE, IMG_NECK, BEVDetImageEncoder
    return BEVDetImageEncoder(IMG_BACKBONE, IMG_NECK, DEPTH_NET, 118, 80)


# -------------------------------------------------------------------------------------------------------- CPU tests
def test_layer_table_matches_the_model():
    """IMAGE_LAYERS is the set of distinct launches of the encoder at 256 x 704 (56 launches, 27 distinct)."""
    enc = _image_encoder()
    launches = encoder_launches(enc, 256, 704)
    assert len(launches) == 56
    table = [l[1:] for l in IMAGE_LAYERS]
    assert len(set(table)) == len(table) == 27
    assert set(table) == set(launches)
    assert enc.out_C == 224 and enc.depth_net.cout == DEPTH_REAL and enc.depth_net.cout_pad == 208


@pytest.mark.parametrize("sms", [132, 114])
def test_search_finds_every_regime_1x1_stride2(sms):
    """IMG_GEOM reaches R1, R2 and R3 (>= 4 items per CTA, a ragged last round, batch and N tile changes between CTA 0's
    items, every ring slot) with a 1x1 stride-2 pad-0 conv for all three per-tap instantiations."""
    for inst in TAP_INSTS:
        for regime in ("R1", "R2", "R3"):
            r = search_regime(sms, inst, regime, IMG_GEOM)
            assert r is not None, (sms, inst, regime)
            B, H, W, cin, cout, k, stride, pad, up, mode, p = r
            assert (k, stride, pad, up, mode) == (1, 2, 0, 1, 1) and p.inst == inst and p.oH % 8 and p.oW % 8
            assert H == 2 * p.oH - 1 and W == 2 * p.oW - 1
            if regime == "R3":
                assert p.items // p.grid >= 4 and p.items % p.grid and p.rings_covered()
                assert p.a_starts == list(range(p.na)) and p.b_starts == list(range(p.nb))
                assert p.cta0_varies(4) and p.cta0_varies(0)


# -------------------------------------------------------------------------------------------------------- GPU tests
def _even_input(case):
    """The case with one more input row and column, fp16 NaN in both halves: a 1x1 stride-2 conv never reads them, so
    the output (and the reference) is the case's own."""
    import copy

    import torch
    B, H, W, cin = case.B, case.H, case.W, case.cin
    even = copy.copy(case)
    xh = torch.full((B, H + 1, W + 1, 2 * cin), float("nan"), dtype=torch.float16, device=case.dev)
    xh[:, :H, :W] = case.xh.view(B, H, W, 2 * cin)
    even.H, even.W, even.xh = H + 1, W + 1, xh.view(-1, 2 * cin)
    even.x64 = from_pixel_h16(even.xh, B, H + 1, W + 1, cin)
    return even


@pytest.mark.gpu
@pytest.mark.parametrize("inst", TAP_INSTS, ids=lambda i: "N%d_MT%d_TAP" % (i[0], i[1]))
def test_1x1_stride2_every_regime(cuda, inst):
    """Each per-tap instantiation forced (mode 1, m_tiles, N tile) on a 1x1 stride-2 pad-0 conv in R1, R2 and R3 of this
    device's SM count (fp32 planes and fp16-pair image against fp64, sentinels and guard pixels, rejected wrong answers,
    same bits twice, and the H16-only epilogue bit-identical), then the same case with one more input row and column
    (the frame's even sizes): the same bits, the extra row and column (NaN) never read."""
    import torch
    sms = _sms()
    N, MT, _ = inst
    for regime in ("R1", "R2", "R3"):
        r = search_regime(sms, inst, regime, IMG_GEOM)
        assert r is not None, "no %s case for %s at %d SMs" % (regime, inst, sms)
        B, H, W, cin, cout, k, stride, pad, up, mode, p = r
        case = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=N * 7 + MT * 3 + 100 * int(regime[1]),
                         mags=CAM_MAGS)
        name = "%s (%d,%d,TAP) B%d %dx%d %d->%d 1x1 s2 mode%d" % (regime, N, MT, B, H, W, cin, cout, mode)
        c0 = 16 if regime == "R3" else 32
        got, img, pl = run_dense(name, case, N, mode, MT, c0=c0)
        assert got.inst == inst and got.items == p.items
        run_pairs(name + " H16-only", case, N, mode, MT, c0=c0, reference=False)
        print("REGIME image encoder %s: %s" % (name, p.describe()))
        even = _even_input(case)
        name_e = "%s (%d,%d,TAP) B%d %dx%d (even) %d->%d 1x1 s2 mode%d" % (regime, N, MT, B, H + 1, W + 1, cin, cout,
                                                                            mode)
        pe, img_e, pl_e = run_dense(name_e, even, N, mode, MT, c0=c0, guards=False)
        assert (pe.oH, pe.oW, pe.items) == (p.oH, p.oW, p.items)
        assert _bits_equal(img, img_e) and _bits_equal(pl, pl_e), "%s: other bits than the odd-sized input" % name_e
        run_pairs(name_e + " H16-only", even, N, mode, MT, c0=c0, reference=False)
        del case, even, img, pl, img_e, pl_e
        torch.cuda.empty_cache()


def _layer_case(dev, layer, seed):
    name, H, W, cin, cout, k, stride, pad, relu, bias_only, res = layer
    if res:
        case = ResidualCase(dev, 6, H, W, cin, cout, k, stride, pad, seed, res_C=cout, mags=CAM_MAGS, relu=relu)
        if bias_only:
            case.scale = None  # lateral0: a conv with bias, no BatchNorm
        return case
    return DenseCase(dev, 6, H, W, cin, cout, k, stride, pad, 1, seed, mags=CAM_MAGS, relu=relu, bias_only=bias_only)


@pytest.mark.gpu
@pytest.mark.parametrize("layer", IMAGE_LAYERS, ids=lambda l: l[0].replace(" ", "_").replace(">", ""))
def test_image_encoder_layer_every_decomposition(cuda, layer):
    """Each distinct encoder launch at 256 x 704, six cameras of magnitudes CAM_MAGS (each on its own bar), written at
    channel offset 0 as the frame writes it: the frame's N tile with the MT rule's choice, N = 64 with both M tilings
    where the layer has at least 128 channels (else the other M tiling), and for the 3x3 stride-1 layers the forced
    per-tap loads.  Residual layers (residual rows of exactly cout channels, as the frame passes them) go through
    run_residual; the others check the fp32 planes and the image against fp64, and the H16-only image bit-identical to
    the image of the launch with planes."""
    import torch
    name, H, W, cin, cout, k, stride, pad, relu, bias_only, res = layer
    case = _layer_case(cuda, layer, seed=cin * 7 + cout + H)
    nt = _n_tile(cout)
    runs = [(nt, 0, 0)]
    if cout >= 128:
        runs += [(64, 0, 1), (64, 0, 2)]
    else:
        runs += [(64, 0, 3 - case.plan(_sms(), 64).inst[1])]
    if k == 3 and stride == 1:
        runs.append((nt, 1, 0))
    for i, (n, mode, mt) in enumerate(runs):
        label = "image %s N%d mode%d MT%d" % (name, n, mode, mt)
        if res:
            p, img, out_C = run_residual(label, case, n, mode, mt, c0=0, guards=i == 0)
            got = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., :cout]
        else:
            p, _, pl = run_dense(label, case, n, mode, mt, c0=0, guards=i == 0)
            run_pairs(label + " H16-only", case, n, mode, mt, c0=0, reference=False)
            got = pl.permute(0, 2, 3, 1)
        assert p.inst[0] == n and (mt == 0 or p.inst[1] == mt) and p.halo == (mode == 0 and k == 3 and stride == 1)
        print("REGIME %s: %s" % (label, p.describe()))
        print("BAR %s, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
              % ((label, case.terms) + error_stats(got, case.want())))
        del got
    del case
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_depth_net_frame_layout(cuda):
    """The depth net as the frame runs it: 208 computed outputs whose weights and bias past the 198 real ones are zero,
    H16-only at channel offset 0 of sentinel-filled 224-channel rows (the second N tile holds 80 channels and ends in a
    half-filled 32-channel group).  Channels 0..197 within the bar on every camera, 198..207 exactly zero in both
    halves, 208..223 untouched."""
    import torch
    layer = IMAGE_LAYERS[-1]
    name, H, W, cin, cout, k, stride, pad, relu, bias_only, res = layer
    case = DenseCase(cuda, 6, H, W, cin, cout, k, stride, pad, 1, seed=5, mags=CAM_MAGS, relu=relu, bias_only=bias_only)
    case.w[DEPTH_REAL:] = 0
    case.shift[DEPTH_REAL:] = 0
    out_C = _image_encoder().out_C
    p = case.plan(_sms(), _n_tile(cout))
    n_px = case.B * p.out_H * p.out_W
    img = sentinel_image(n_px, out_C, cuda)
    _, st = case.launch(_n_tile(cout), out=img, out_C=out_C, c0=0, planes=False)
    torch.cuda.synchronize()
    assert int(st[0]) == 0
    rows = img[:n_px].view(n_px, out_C // 32, 2, 32).view(torch.int16)
    ch = torch.arange(out_C, device=cuda)
    bits = rows.permute(0, 1, 3, 2).reshape(n_px, out_C, 2)  # [pixel, channel, (hi, lo')]
    assert bool((bits[:, (ch >= DEPTH_REAL) & (ch < cout)] == 0).all()), "depth net: padding outputs are not +0"
    s = int(torch.tensor(SENTINEL, dtype=torch.float16).view(torch.int16))
    assert bool((bits[:, cout:] == s).all()), "depth net: channels past the computed 208 were written"
    assert bool((img[n_px:].view(torch.int16) == s).all()), "depth net: guard pixels after the image were written"
    dec = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., :DEPTH_REAL]
    want = case.want()[..., :DEPTH_REAL]
    check_images("depth net frame layout", dec, want, case.terms)
    check_rejects("depth net frame layout", [(w, v[..., :DEPTH_REAL]) for w, v in case.wrongs()], want, case.terms)
    print("REGIME image depth net frame layout: %s" % p.describe())


# ------------------------------------------------------------------------------------------- chained encoder (PDL)
@pytest.mark.gpu
@pytest.mark.parametrize("size", [(256, 704), (128, 352)], ids=["256x704", "128x352"])
def test_chained_image_encoder_eager_and_graph(cuda, oracle_mod, size):
    """BEVDetFromImages' image encoder (seeded, BN gain sqrt(6)) on synth.camera_images, restated launch by launch on
    one stream with no sync in between (programmatic dependent launch: conv3 reads a residual written one or three
    launches earlier, lateral0 one written by the upsample), once eagerly and once captured in a CUDA graph.  The chain's
    output is bit-equal to image_encoder(imgs); graph and eager give the same bits in every buffer and status 0; the stem
    against fp64; every one of the 56 convs against the float64 reference computed from its actual input and residual
    buffers, per camera, with the "hi x hi only" answer rejected; the upsample bit-equal to indexing its input."""
    import torch
    from bevdet_images_oracle import max_pool_3x3_s2_p1
    from parity import rel_check
    from paddle3d_b200 import synth
    from paddle3d_b200.bevdet import CONFIG_IMG, BEVDetFromImages
    from paddle3d_b200.ops import dense_conv as dc
    from test_gpu_bevdet_images import BN_GAIN
    H, W = size
    m = BEVDetFromImages(dict(CONFIG_IMG, input_size=size), device=cuda).init_weight(seed=13, bn_gain=BN_GAIN)
    enc = m.image_encoder
    imgs_np = synth.camera_images(14, 6, H, W)
    imgs = torch.from_numpy(imgs_np).to(cuda)
    status = dc._status(cuda)

    def chain():
        convs = []  # (conv, input, its shape, residual or None, output, its channels)
        x, sh = enc.stem_forward(imgs)
        stem = x
        feats = []
        for stage in enc.stages:
            for blk in stage:
                c1, c2, c3, down = blk["conv1"], blk["conv2"], blk["conv3"], blk["down"]
                b = sh[0]
                t, _, (_, h, w) = c1(x, sh)
                convs.append((c1, x, sh, None, t, c1.cout))
                tsh = (b, h, w, c1.cout)
                t2, _, (_, oh, ow) = c2(t, tsh)
                convs.append((c2, t, tsh, None, t2, c2.cout))
                idn = x
                if down is not None:
                    idn, _, _ = down(x, sh)
                    convs.append((down, x, sh, None, idn, down.cout))
                t2sh = (b, oh, ow, c2.cout)
                y, _, _ = c3(t2, t2sh, residual=idn, res_channels=c3.cout)
                convs.append((c3, t2, t2sh, idn, y, c3.cout))
                x, sh = y, (b, oh, ow, c3.cout)
            feats.append((x, sh))
        (x0, s0), (x1, s1) = feats[enc.out_indices[0]], feats[enc.out_indices[1]]
        l0c, l1c = enc.lateral
        oc = l0c.cout
        l1, _, _ = l1c(x1, s1)
        convs.append((l1c, x1, s1, None, l1, oc))
        l1sh = (s1[0], s1[1], s1[2], oc)
        up, (b, h, w) = dc.upsample_nearest_h16(l1, l1sh, s0[1] // s1[1])
        l0, _, _ = l0c(x0, s0, residual=up, res_channels=oc)
        convs.append((l0c, x0, s0, up, l0, oc))
        y, _, _ = enc.fpn_conv(l0, (b, h, w, oc))
        convs.append((enc.fpn_conv, l0, (b, h, w, oc), None, y, oc))
        dn = enc.depth_net
        d = torch.zeros((b * h * w, 2 * enc.out_C), dtype=torch.float16, device=cuda)
        dn(y, (b, h, w, oc), out_h16=d, out_channels=enc.out_C)
        convs.append((dn, y, (b, h, w, oc), None, d, enc.out_C))
        return stem, convs, (l1, l1sh, up)

    status.zero_()
    stem, convs, ups = chain()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    assert len(convs) == 56
    rows, shape = enc(imgs)
    torch.cuda.synchronize()
    assert shape == (6, H // 16, W // 16, enc.out_C)
    assert _bits_equal(convs[-1][4], rows), "the restated chain is not the image encoder's launch sequence"
    del rows
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        stem_g, convs_g, ups_g = chain()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    assert _bits_equal(stem, stem_g), "stem: graph replay differs from the eager run"
    for i, (a, g) in enumerate(zip(convs, convs_g)):
        assert _bits_equal(a[4], g[4]), "conv %d: graph replay differs from the eager run" % i
    assert _bits_equal(ups[2], ups_g[2]), "upsample: graph replay differs from the eager run"
    del stem_g, convs_g, ups_g, graph
    torch.cuda.empty_cache()

    # the stem against fp64 (as test_gpu_bevdet_images.test_stem_vs_fp64 computes it)
    sd = enc.stem_dev
    ref = oracle_mod.conv2d(imgs_np, enc.stem.np["weight"], None, 2, 3).astype(np.float64)
    sc, sf = sd["scale"].cpu().numpy().reshape(1, -1, 1, 1), sd["shift"].cpu().numpy().reshape(1, -1, 1, 1)
    ref = max_pool_3x3_s2_p1(np.maximum(ref * sc + sf, 0.0))
    sh0 = (6,) + dc.stem_shape(H, W) + (64,)
    got = dc.pixel_h16_to_nchw(stem, sh0).cpu().numpy()
    rel_check("chain stem %dx%d" % size, got, ref, floor=1e-2, small_atol=2e-6)  # test_gpu_dense.py's floor, 147 terms
    del ref

    # the upsample: the pairs of pixel (Y / 2, X / 2), bit for bit
    l1, (b, h1, w1, c), up = ups
    s = 2
    src = l1.view(b, h1, w1, 2 * c)
    yi = torch.arange(h1 * s, device=cuda) // s
    xi = torch.arange(w1 * s, device=cuda) // s
    want_up = src[:, yi][:, :, xi].reshape(-1, 2 * c)
    assert torch.equal(up.view(torch.int16), want_up.view(torch.int16)), "upsample: not the nearest pixel's pairs"

    sms = _sms()
    for i, (conv, x, sh, r, y, out_C) in enumerate(convs):
        b, h, w, cin = sh
        cout = conv.cout
        wt = torch.from_numpy(conv.np["weight"]).to(cuda).double()
        sc = conv.dev["scale"]
        sf = conv.dev["shift"]
        sc = None if sc is None else sc[:cout]
        sf = None if sf is None else sf[:cout]

        def result(acc):
            o = epilogue(acc, sc, sf, False)
            if r is not None:
                o = o + from_pixel_h16(r, b, o.shape[1], o.shape[2], cout)
            return o.clamp_min(0.0) if conv.relu else o
        acc, _ = conv_ref(from_pixel_h16(x, b, h, w, cin), wt, conv.k, conv.stride, conv.padding, 1)
        want = result(acc)
        del acc
        oh, ow = want.shape[1:3]
        got = from_pixel_h16(y, b, oh, ow, out_C)
        terms = conv.cin * conv.k * conv.k
        name = "chain %dx%d conv %d %d->%d k%d s%d%s" % (H, W, i, conv.cin, cout, conv.k, conv.stride,
                                                        " + residual" if r is not None else "")
        check_images(name, got[..., :cout], want, terms)
        if out_C > cout:  # the depth net: computed padding outputs and untouched row channels, all zero
            assert bool((got[..., cout:] == 0).all()), "%s: channels past the real outputs are not zero" % name
        hh, _ = conv_ref(from_pixel_h16(x, b, h, w, cin, hi_only=True), wt.float().half().double(), conv.k, conv.stride,
                         conv.padding, 1)
        check_rejects(name, [("hi x hi only", result(hh))], want, terms)
        del hh, want, got
        p = Plan(sms, b, h, w, cin, conv.cout_pad or cout, conv.n_tile, conv.k, conv.stride, conv.padding, 1)
        print("REGIME chain %s: %s" % (name, p.describe()))
