"""The dense fp16-pair conv's pair-tile epilogue: launches that write only the pixel H16 image (no fp32 planes).

Such a launch of `dcf::dense_conv_f16_kernel<N, MT, HALO>` applies scale / shift / ReLU and the fp16-pair split in the
consumer warpgroups and stores the rows with TMA (or, for 32-channel groups the layer owns only in part, with ordinary
stores from the epilogue warps); a launch with fp32 planes keeps the fp32 staging and the epilogue-warp stores.  Both do
the same operations in the same order, so the image of an H16-only launch must be bit-identical to the image of the same
launch with planes.  This file drives the H16-only path wherever test_gpu_dense_schedule.py drives the other one: every
instantiation in the regimes of its search, the full-size layers and necks of both frames, the overflow case, and the
chained CenterPoint head (programmatic dependent launch, eager and captured in a CUDA graph)."""
import pytest

from test_gpu_dense_schedule import (C3_LAYERS, INSTS, NECKS, OVERFLOW_LAYERS, PP_LAYERS, DenseCase, _bits_equal, _cdiv,
                                     _n_tile, _sms, assert_untouched, check_images, from_pixel_h16, owned_halfs,
                                     search_regime, sentinel_image)


def _image_pair(case, n_tile, mode, m_tiles, out_C, c0, scale=None):
    """The same launch H16-only and with fp32 planes, each into its own sentinel image.  Returns (H16-only image, its
    status word, image of the launch with planes, its planes, its status word)."""
    import torch
    p = case.plan(_sms(), n_tile, mode, m_tiles)
    n_px = case.B * p.out_H * p.out_W
    img = sentinel_image(n_px, out_C, case.dev)
    _, st = case.launch(n_tile, mode, m_tiles, img, out_C, c0, planes=False, scale=scale)
    ref = sentinel_image(n_px, out_C, case.dev)
    pl, st_ref = case.launch(n_tile, mode, m_tiles, ref, out_C, c0, scale=scale)
    torch.cuda.synchronize()
    return img, int(st[0]), ref, pl, int(st_ref[0])


def run_pairs(name, case, n_tile, mode=0, m_tiles=0, c0=32, reference=True, out_C=None):
    """H16-only launch against the launch with planes (same bits, same status), sentinels untouched, a second H16-only
    launch gives the same bits; with `reference` also the fp64 bar.  out_C: the image's channels (default: 32 more than
    c0 + cout rounded up to 32).  Returns (plan, H16-only image, out_C)."""
    import torch
    p = case.plan(_sms(), n_tile, mode, m_tiles)
    if out_C is None:
        out_C = _cdiv(c0 + case.cout, 32) * 32 + 32
    n_px = case.B * p.out_H * p.out_W
    img, st, ref, _, st_ref = _image_pair(case, n_tile, mode, m_tiles, out_C, c0)
    assert st == 0 and st_ref == 0, "%s: status %d / %d" % (name, st, st_ref)
    assert _bits_equal(img, ref), "%s: the H16-only image differs from the image of the launch with planes" % name
    del ref
    assert_untouched(name, img, n_px, owned_halfs(out_C, c0, case.cout))
    if reference:
        dec = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., c0:c0 + case.cout]
        check_images(name + " H16-only image", dec, case.want(), case.terms)
        del dec
    img2 = sentinel_image(n_px, out_C, case.dev)
    case.launch(n_tile, mode, m_tiles, img2, out_C, c0, planes=False)
    torch.cuda.synchronize()
    assert _bits_equal(img, img2), "%s: a second H16-only launch gives other bits" % name
    return p, img, out_C


@pytest.mark.gpu
@pytest.mark.parametrize("inst", INSTS, ids=lambda i: "N%d_MT%d_%s" % (i[0], i[1], "HALO" if i[2] else "TAP"))
def test_every_instantiation_in_every_regime_h16_only(cuda, inst):
    """Each instantiation forced in R1, R2 and R3 of this device's SM count (test_gpu_dense_schedule.search_regime),
    H16-only.  R3: 2 or 3 batch images, several N tiles with the last one partly used, output at a channel offset of
    16 mod 32 (every group owned in part) and changing taps for the transposed conv; R1 / R2 at offset 32 (TMA boxes)."""
    import torch
    N, MT, halo = inst
    for regime in ("R1", "R2", "R3"):
        r = search_regime(_sms(), inst, regime)
        assert r is not None, "no %s case for %s" % (regime, inst)
        B, H, W, cin, cout, k, stride, pad, up, mode, p = r
        case = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=N * 7 + MT * 3 + halo + 100 * int(regime[1]),
                         mags=(1.0, 32.0, 0.125))
        name = "%s (%d,%d,%s) B%d %dx%d %d->%d k%d s%d up%d mode%d H16-only" % (
            regime, N, MT, "HALO" if halo else "TAP", B, H, W, cin, cout, k, stride, up, mode)
        got, _, _ = run_pairs(name, case, N, mode, MT, c0=16 if regime == "R3" else 32)
        assert got.inst == inst and got.items == p.items
        if regime == "R3":  # the same items with every group whole: the last N tile's partly used group on the TMA path
            run_pairs(name + " c0 0", case, N, mode, MT, c0=0)
        del case
        torch.cuda.empty_cache()


H16_LAYERS = [l for l in C3_LAYERS + PP_LAYERS if l[5] % 16 == 0]


@pytest.mark.gpu
@pytest.mark.parametrize("layer", H16_LAYERS, ids=lambda l: l[0].replace(" ", "_"))
def test_full_size_layer_h16_only(cuda, layer):
    """A dense layer of the CenterPoint (C3) or PointPillars frame at its real size, H16-only, bit-identical to the
    launch with planes; the two overflow layers drive one channel past fp16's range."""
    import torch
    name, B, H, W, cin, cout, k, stride, pad, up, relu, bias_only, c0 = layer
    nt = _n_tile(cout)
    case = DenseCase(cuda, B, H, W, cin, cout, k, stride, pad, up, seed=cin * 13 + cout + H, relu=relu,
                     bias_only=bias_only)
    _, img, out_C = run_pairs(name, case, nt, c0=c0, reference=False)
    if name in OVERFLOW_LAYERS:
        _check_overflow(name, case, nt, img, out_C, c0)
    del case, img
    torch.cuda.empty_cache()


def _check_overflow(name, case, nt, img0, out_C, c0):
    """One channel's scale x 2e6, H16-only: status bit 0 set, that channel saturates at 65504 where the fp32 planes of
    the launch with planes pass it, every other channel keeps the bits of the unscaled launch, and the image is the one
    of the launch with planes."""
    import torch
    ch = case.cout // 3
    big = case.scale.clone()
    big[ch] = 2.0e6
    p = case.plan(_sms(), nt)
    img, st, ref, pl, st_ref = _image_pair(case, nt, 0, 0, out_C, c0, scale=big)
    assert st & 1 and st_ref & 1, "%s overflow: status bit 0 not set (%d / %d)" % (name, st, st_ref)
    assert _bits_equal(img, ref), "%s overflow: the H16-only image differs from the launch with planes" % name
    f32 = pl[:, ch].double()
    dec = from_pixel_h16(img, case.B, p.out_H, p.out_W, out_C)[..., c0 + ch]
    sat = f32.abs() > 65504
    assert int(sat.sum()) > 10, "%s: the overflow case does not overflow" % name
    assert torch.equal(dec[sat], torch.sign(f32[sat]) * 65504.0), "%s: pair output does not saturate" % name
    others = ~owned_halfs(out_C, c0 + ch, 1).to(img.device)
    assert torch.equal(img.view(torch.int16)[:, others], img0.view(torch.int16)[:, others]), \
        "%s overflow: other channels of the pair image changed" % name


@pytest.mark.gpu
@pytest.mark.parametrize("neck", sorted(NECKS))
def test_full_size_neck_concat_h16_only(cuda, neck):
    """The deblocks of a neck at full size launched back to back into one concat image, H16-only, against the same
    launches with planes: the whole images bit-identical, guard pixels untouched, a second round the same bits."""
    import torch
    oH, oW, layers = NECKS[neck]
    out_C = sum(l[3] for l in layers)
    cases = [DenseCase(cuda, 1, h, w, cin, cout, k, up if up > 1 else 1, 0, up, seed=cin + cout * 3 + up)
             for h, w, cin, cout, k, up in layers]

    def round_(planes):
        img = sentinel_image(oH * oW, out_C, cuda)
        st = torch.zeros((1,), dtype=torch.int32, device=cuda)
        c0 = 0
        for c in cases:
            c.launch(_n_tile(c.cout), 0, 0, img, out_C, c0, planes=planes, status=st)
            c0 += c.cout
        torch.cuda.synchronize()
        return img, int(st[0])

    img, st = round_(False)
    ref, st_ref = round_(True)
    assert st == 0 and st_ref == 0
    assert_untouched(neck + " neck H16-only", img, oH * oW, torch.ones(2 * out_C, dtype=torch.bool))
    assert _bits_equal(img, ref), "%s neck: the H16-only concat image differs from the launches with planes" % neck
    img2, _ = round_(False)
    assert _bits_equal(img, img2), "%s neck: a second H16-only round gives other bits" % neck


@pytest.mark.gpu
def test_chained_c3_head_h16_only_matches_planes(cuda):
    """The full-size CenterPoint DenseRPNHead chain (every conv H16-only, back to back on one stream with programmatic
    dependent launch) eagerly and captured in a CUDA graph: the same bits; and every layer's image bit-identical to the
    same layer relaunched with planes on the same input."""
    import torch
    from paddle3d_b200.dense_head import DenseRPNHead
    from test_gpu_dense_schedule import to_pixel_h16
    net = DenseRPNHead().init_weight(seed=7, device=cuda, randomize_bn=True, bn_gain=6.0 ** 0.5)
    big = net._batched_params(cuda)["big"]
    g = torch.Generator(device=cuda).manual_seed(8)
    xh = to_pixel_h16(torch.randn((1, net.in_channels, 180, 180), generator=g, device=cuda))

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
        mid, _, _ = big(s, (1, 180, 180, net.shared.cout))
        recs.append((big, s, (1, 180, 180, net.shared.cout), mid, big.cout, 0))
        return recs

    recs = chain()
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        recs_g = chain()
    graph.replay()
    torch.cuda.synchronize()
    for i, (a, b) in enumerate(zip(recs, recs_g)):
        assert _bits_equal(a[3], b[3]), "layer %d: graph replay differs from the eager run" % i
    del recs_g, graph
    for i, (conv, x, sh, y, out_C, c0) in enumerate(recs):
        ref = torch.empty_like(y)
        if out_C != conv.cout:  # a deblock of the concat: the other deblocks' channels from the chain's image
            ref.copy_(y)
        conv(x, sh, out_split=ref, out_channels=out_C, out_c0=c0, want_nchw=True)
        torch.cuda.synchronize()
        assert _bits_equal(y, ref), "chain layer %d: the H16-only image differs from the launch with planes" % i
        del ref
