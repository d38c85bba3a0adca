"""CenterPoint-pillars and both PointPillars models (car, cyclist / pedestrian), the benchmarked frames, at full size stage
by stage against float64 references; CenterPoint-pillars also at its pillar cap, past the nms_pre cut, out of fp16's
range, in lanes and on the sweep stream.

The frames are the bench tools': CenterPointPillarsHotPath(synth.CP_PILLARS, seed=0, bn_gain=bench.BN_GAIN) and
PointPillarsHotPath(cfg, seed=0, bn_gain=bench.BN_GAIN, model_cfg=...), each head calibrated on bench.frame_pool(cfg, .)[0]
and run on that cloud.  cp_pillars_chain and pointpillars_chain restate the models' encode / dense / postprocess on the
current stream with no sync in between and keep every buffer: hard_voxelize, the pillar encoder's fp32 rows, the pixel
fp16-pair image, every dense conv with its input and output image (cp_chain_convs / pp_chain_convs, tied to the models'
conv lists and to the written-out tables CP_CHAIN / PP_CHAIN by a CPU test), the head and the postprocess.  Every stage
is checked from its actual input buffer:

  * hard_voxelize bit for bit against oracle.hard_voxelize over its whole capacity (zero rows past the count), with
    the pillar counts of the tables below;
  * the pillar encoder against oracle.centerpoint_pillars.pillar_feature_net2 / oracle.pillar_feature_net (fp64, 1e-4);
  * the pixel image bit for bit against the fp16-pair split (to_pixel_h16) of the encoder rows scattered to their pixels
    (lidar_front_end_oracle.scatter_dense);
  * every dense conv against the float64 conv and epilogue on test_gpu_dense_schedule's bar, which rejects the hi x hi
    products alone and the result without one tap (1x1 and transposed convs: one 32-channel input group);
  * CenterPoint-pillars' fused head planes against the tap-sum reference of test_gpu_head_fused_schedule, and bit for
    bit against the fp32 tap sum of the P buffer its conv launch wrote; PointPillars' head planes against a float64
    1x1 conv plus bias;
  * the postprocess against oracle.centerpoint_postprocess / oracle.pointpillars(_multiclass).anchor_head_postprocess of
    the actual planes (PointPillars: also its decoded candidates in score order).

No pillar stage numbers its rows with atomics (hard_voxelize keeps pillars in point order, the dense convs' work
decomposition depends on shapes only), so the eager chain, the captured chain and the hot path's captured frame are
the same bits in the default mode.  Lines starting with "REGIME" (pytest -s) name each conv's work decomposition,
"BAR" its error figures, "POST" the postprocess counts, "MEM" each test's peak device memory and wall time."""
import numpy as np
import pytest

import bench
import lidar_front_end_oracle as lfo
from paddle3d_b200 import io as p3d_io
from paddle3d_b200 import synth
from parity import rel_check
from test_gpu_centerpoint_full_size import _clean_status_and_peak_memory, check_postprocess  # noqa: F401 (autouse)
from test_gpu_centerpoint_pillars import _frame_inputs
from test_gpu_dense_residual import error_stats
from test_gpu_dense_schedule import (Plan, _bits_equal, bar, check_images, check_rejects, conv_ref, epilogue,
                                     from_pixel_h16, to_pixel_h16)
from test_gpu_head_fused_schedule import PLANE_TERMS, FusedPlan, tap_sum_f32, tap_sum_ref, w2_image

FP16_GAIN = 6.0  # BatchNorm gain that drives the activations far past 65504 (sqrt(6) keeps them O(1))

# The dense convs before the head in launch order: (Cin, Cout, k, stride, up, transposed).  SecondBackbone
# [3, 5, 5] / [64, 128, 256], then the SecondFPN deblocks into the 384-channel concat image.
_TRUNK = ([(64, 128, 3, 2, 1, False)] + [(128, 128, 3, 1, 1, False)] * 5
          + [(128, 256, 3, 2, 1, False)] + [(256, 256, 3, 1, 1, False)] * 5)
# CenterPoint-pillars: first block stride 2, upsample strides (0.5, 1, 2) with use_conv_for_no_stride (a 2x2 stride-2
# conv, a 1x1 conv, a 2x2 transposed conv), then the shared conv
CP_CHAIN = ([(64, 64, 3, 2, 1, False)] + [(64, 64, 3, 1, 1, False)] * 3 + _TRUNK
            + [(64, 128, 2, 2, 1, False), (128, 128, 1, 1, 1, False), (256, 128, 2, 2, 2, True)]
            + [(384, 64, 3, 1, 1, False)])
# PointPillars: upsample strides (1, 2, 4) without use_conv_for_no_stride (a 1x1 transposed conv, 2x2 and 4x4
# transposed convs), then the 1x1 SSD head with bias; car: first block stride 2, cyclist / pedestrian: stride 1
_PP_DEBLOCKS = [(64, 128, 1, 1, 1, True), (128, 128, 2, 2, 2, True), (256, 128, 4, 4, 4, True)]
PP_CHAIN = {
    "car": [(64, 64, 3, 2, 1, False)] + [(64, 64, 3, 1, 1, False)] * 3 + _TRUNK + _PP_DEBLOCKS
    + [(384, 20, 1, 1, 1, False)],
    "ped_cyclist": [(64, 64, 3, 1, 1, False)] + [(64, 64, 3, 1, 1, False)] * 3 + _TRUNK + _PP_DEBLOCKS
    + [(384, 44, 1, 1, 1, False)],
}
# (H, W) of the pixel image, after each backbone block, and of the concat image
CP_SIZES = ((512, 512), [(256, 256), (128, 128), (64, 64)], (128, 128))
PP_SIZES = {"car": ((496, 432), [(248, 216), (124, 108), (62, 54)], (248, 216)),
            "ped_cyclist": ((248, 296), [(248, 296), (124, 148), (62, 74)], (248, 296))}

# hard_voxelize on the bench clouds (oracle.hard_voxelize): (points in range, pillars kept, pillars at max_points,
# 1-point pillars)
CP_BENCH_PILLARS = (300000, 7449, 4061, 800)
# uniform_cloud(CP_PILLARS, 0): points in range, occupied pillars, of which the first 60 000 in point order are kept,
# with at most 7 points each and 24 610 with one point
CP_UNIFORM = (266411, 166820, 60000, 7, 24610)
PP_BENCH_PILLARS = {"car": (9724, 2109, 31, 635), "ped_cyclist": (9381, 470, 64, 62)}


# ------------------------------------------------------------------------------------------------- the models' chains
def cp_chain_convs(head):
    """CenterPointPillars.head's convs before the CenterHead in launch order: the trunk blocks, the deblocks, the shared
    conv."""
    return [c for blk in head.blocks for c in blk] + list(head.deblocks) + [head.shared]


def pp_chain_convs(m):
    """PointPillars' convs in launch order: SecondTrunk's blocks and deblocks, the head."""
    return [c for blk in m.trunk.blocks for c in blk] + list(m.trunk.deblocks) + [m.head]


def _table(convs):
    return [(c.cin, c.cout, c.k, c.stride, c.up, c.transposed) for c in convs]


def _sizes(convs, blocks, hw):
    """(H, W) after each backbone block and of every deblock's output, walking the conv geometry from the pixel image."""
    h, w = hw
    it = iter(convs)
    feats = []
    for blk in blocks:
        for _ in blk:
            c = next(it)
            h, w = (h + 2 * c.padding - c.k) // c.stride + 1, (w + 2 * c.padding - c.k) // c.stride + 1
        feats.append((h, w))
    outs = []
    for (h, w), _ in zip(feats, blocks):
        c = next(it)
        outs.append((h * c.up, w * c.up) if c.up > 1 else ((h - c.k) // c.stride + 1, (w - c.k) // c.stride + 1))
    return feats, outs


def _encode_front(m, pts_dev, pfn):
    """hard_voxelize, the pillar encoder (pfn(voxels, npv, coors, nv)) and the pixel image, buffers kept."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox
    cfg = m.cfg
    voxels, co, npv, nv = vox.hard_voxelize(pts_dev, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                            cfg["max_voxels"])
    coors = torch.nn.functional.pad(co, (1, 0))
    feats = pfn(voxels, npv, coors, nv)
    nx, ny = m.grid
    image, shape = sp.sparse_coo_tensor(coors, feats, [1, 1, ny, nx, m.C], num=nv).to_pixel_h16()
    return dict(voxels=voxels, co=co, npv=npv, nv=nv, coors=coors, feats=feats, image=image, shape=shape)


def _trunk_chain(blocks, deblocks, fpn, x, sh, dev):
    """SecondTrunk.__call__ conv by conv: ([(conv, input image, its shape, output image, out_C, c0)], concat image, its
    shape)."""
    import torch
    from paddle3d_b200.dense_head import SecondTrunk
    convs, feats = [], []
    for blk in blocks:
        for conv in blk:
            y, _, (b, oh, ow) = conv(x, sh)
            convs.append((conv, x, sh, y, conv.cout, 0))
            x, sh = y, (b, oh, ow, conv.cout)
        feats.append((x, sh))
    b = sh[0]
    hws = {SecondTrunk.deblock_out_hw(de, fs[1], fs[2]) for (_, fs), de in zip(feats, deblocks)}
    assert len(hws) == 1
    H, W = hws.pop()
    cat = torch.empty((b * H * W, 2 * fpn), dtype=torch.float16, device=dev)
    c0 = 0
    for (f, fs), de in zip(feats, deblocks):
        de(f, fs, out_split=cat, out_channels=fpn, out_c0=c0)
        convs.append((de, f, fs, cat, fpn, c0))
        c0 += de.cout
    return convs, cat, (b, H, W, fpn)


def cp_pillars_chain(hot, pts_dev):
    """CenterPointPillars.encode / dense / postprocess restated on the current stream, every buffer kept: hard_voxelize,
    the two-layer PFN's fp32 rows, the pixel image, the trunk, the deblocks into the concat image, the shared conv, the
    fused CenterHead conv + tap sum, the postprocess and the status word."""
    from paddle3d_b200.ops import centerpoint_postprocess as cpp
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import sparse_nn as sp
    m = hot.model
    d, dev, cfg = m.head, pts_dev.device, m.cfg
    r = _encode_front(m, pts_dev, lambda v, n, c, nv: pe.pillar_feature_net2(
        v, n, c, m.pfn_dev, cfg["voxel_size"], cfg["point_cloud_range"], num_voxels=nv, folded=m.pfn_folded))
    convs, cat, cshape = _trunk_chain(d.blocks, d.deblocks, d.fpn_channels, r["image"], r["shape"], dev)
    s, _, _ = d.shared(cat, cshape)
    convs.append((d.shared, cat, cshape, s, d.shared.cout, 0))
    bp = d._batched_params(dev)
    assert d.fused_heads(bp)
    shape = cshape[:3] + (d.shared.cout,)
    P = d._heads_conv_p(s, shape, bp, dev)
    planes = d._tap_sum(P, bp, dev)
    h = {}
    for name, p0, k in zip(bp["names"], bp["plane0"], bp["cnt"]):
        h.setdefault(name, []).append(planes[:, int(p0):int(p0) + int(k)])
    post = cpp.centerpoint_postprocess_heads(h, cfg["voxel_size"][:2], cfg["point_cloud_range"], m.test_cfg,
                                             m.label_off)
    r.update(convs=convs, shared=s, head_shape=shape, P=P, planes=planes, heads=h, post=post, bp=bp,
             status=sp.status_tensor(dev).clone())
    return r


def pointpillars_chain(hot, pts_dev):
    """PointPillars.encode / dense / postprocess restated on the current stream, every buffer kept: hard_voxelize, the
    one-layer PFN's fp32 rows, the pixel image, SecondTrunk's convs and deblocks, the 1x1 head conv with bias into fp32
    NCHW planes (its record in convs has the planes as output image), anchor_head_postprocess_device with its decoded
    candidates in score order (sorted_out, "cand") and the status word."""
    import torch
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import sparse_nn as sp
    m = hot.model
    dev, cfg, p = pts_dev.device, m.cfg, m.pfn
    r = _encode_front(m, pts_dev, lambda v, n, c, nv: pe.pillar_feature_net(
        v, n, c, m.pfn_weight, p["gamma"], p["beta"], p["mean"], p["var"], p["eps"], cfg["voxel_size"],
        cfg["point_cloud_range"], num_voxels=nv, folded=m.pfn_folded))
    convs, cat, cshape = _trunk_chain(m.trunk.blocks, m.trunk.deblocks, m.trunk.fpn_channels, r["image"], r["shape"],
                                      dev)
    _, planes, _ = m.head(cat, cshape, want_nchw=True)
    convs.append((m.head, cat, cshape, planes, m.head.cout, 0))
    pre = m.mc["test"]["nms_pre_max_size"]
    cand = (torch.empty((pre, 7), dtype=torch.float32, device=dev), torch.empty((pre,), dtype=torch.float32, device=dev))
    post = m.postprocess(planes, r["coors"], r["nv"], sorted_out=cand)
    r.update(convs=convs, planes=planes, cand=cand, post=post, status=sp.status_tensor(dev).clone())
    return r


def _run_chains(chain, hot, pts_d):
    """chain once eagerly on the current stream, and once captured by torch.cuda.graph (on its own capture stream)
    and replayed."""
    import torch
    eager = chain(hot, pts_d)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = chain(hot, pts_d)
    graph.replay()
    torch.cuda.synchronize()
    return eager, captured, graph


# ----------------------------------------------------------------------------------------------- references / checks
def _hard_voxelize_into(pts_dev, cfg, fill):
    """p3d_hard_voxelize (the launch of ops.voxelize.hard_voxelize) into output buffers filled with the byte `fill`."""
    import torch
    from paddle3d_b200._lib import check, host_floats, lib
    from paddle3d_b200._mem import ptr, stream
    n, f = pts_dev.shape
    P, V, dev = cfg["max_points"], cfg["max_voxels"], pts_dev.device
    out = [torch.full(s, fill, dtype=torch.uint8, device=dev).view(t)
           for s, t in (((V, P, 4 * f), torch.float32), ((V, 12), torch.int32), ((4 * V,), torch.int32),
                        ((4,), torch.int32))]
    ws = torch.empty((max(1, lib().p3d_hard_voxelize_workspace_bytes(n, P, V)),), dtype=torch.uint8, device=dev)
    check(lib().p3d_hard_voxelize(ptr(pts_dev), n, f, host_floats(cfg["voxel_size"]),
                                  host_floats(cfg["point_cloud_range"]), P, V, *[ptr(t) for t in out], ptr(ws),
                                  ws.numel(), stream(dev)), "hard_voxelize")
    return out


def check_voxelize(name, oracle_mod, r, pts, cfg):
    """voxels, coors, points per pillar and the count bit-equal oracle.hard_voxelize over the whole capacity: the rows
    past the count are zero, as the reference's op leaves them (its outputs are sized by max_voxels and zero-filled).
    The same launch into buffers filled with 0xFF bytes gives the same bits, so every row is written, none is left
    as it was.  Returns (pillars, pillars at max_points, 1-point pillars, most points in a pillar)."""
    import torch
    want = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                    cfg["max_voxels"])
    vox, co, npv, nv = want
    k = int(nv[0])
    assert int(r["nv"][0]) == k, "%s: pillar count %d, oracle %d" % (name, int(r["nv"][0]), k)
    assert not co[k:].any() and not npv[k:].any() and not vox[k:].any()
    got = [r[key] for key in ("voxels", "co", "npv", "nv")]
    for what, g, w in zip(("voxels", "coors", "points per pillar"), got, want):
        g = g.cpu().numpy()
        assert np.array_equal(g.view(np.uint32), w.view(np.uint32)), "%s: %s, %d of %d rows differ (%d past the count)" % (
            name, what, int((g != w).reshape(len(w), -1).any(1).sum()), len(w),
            int((g[k:] != w[k:]).reshape(len(w) - k, -1).any(1).sum()))
    pts_dev = torch.from_numpy(pts).to(r["nv"].device)
    again = _hard_voxelize_into(pts_dev, cfg, 0xFF)
    torch.cuda.synchronize()
    assert all(torch.equal(a.view(torch.int32), b.view(torch.int32)) for a, b in zip(again[:3], got[:3])), \
        "%s: hard_voxelize into 0xFF-filled buffers gives other bits: a row is not written" % name
    assert int(again[3][0]) == k and not bool((again[3][1:] != -1).any()), "%s: count word" % name
    c = npv[:k]
    return k, int((c == cfg["max_points"]).sum()), int((c == 1).sum()), int(c.max())


def points_in_range(pts, cfg):
    """Points of the cloud inside the grid, and the occupied cells (hard_voxelize's floor((p - lo) / size) in fp32)."""
    lo, vs = np.asarray(cfg["point_cloud_range"][:3], np.float32), np.asarray(cfg["voxel_size"], np.float32)
    grid = np.round((np.asarray(cfg["point_cloud_range"][3:], np.float32) - lo) / vs).astype(np.int64)
    ijk = np.floor((pts[:, :3] - lo) / vs).astype(np.int64)
    ok = ((ijk >= 0) & (ijk < grid)).all(1)
    return int(ok.sum()), len(np.unique(ijk[ok], axis=0))


def check_pfn(name, r, want, two_layer):
    """The encoder's rows against the fp64 reference `want` [k, C], on the 1e-4 bar of the encoder's own test (two-layer:
    test_gpu_centerpoint_pillars' true relative 1e-4; one layer: test_gpu_voxelize's 1e-4 of the element or of the
    largest one); rows past the count zero."""
    k = len(want)
    got = r["feats"].cpu().numpy()
    if two_layer:
        rel_check("%s PFN" % name, got[:k], want, rtol=1e-4)
    else:
        np.testing.assert_allclose(got[:k], want, rtol=1e-4, atol=1e-4 * np.abs(want).max())
    assert not got[k:].any(), "%s: PFN rows past the pillar count were written" % name


def check_pixel_image(name, m, r):
    """The pixel image bit-equal to_pixel_h16 of the encoder rows scattered to their (y, x) pixels (scatter_dense).
    Returns the occupied pixels."""
    import torch
    nx, ny = m.grid
    n = int(r["nv"][0])
    canvas = lfo.scatter_dense(r["feats"].cpu().numpy(), r["coors"].cpu().numpy(), n, 1, 1, ny, nx, use_z=False)
    want = to_pixel_h16(torch.from_numpy(canvas.reshape(1, m.C, ny, nx)).to(r["image"].device))
    assert r["shape"] == (1, ny, nx, m.C) and r["image"].shape == want.shape
    assert _bits_equal(r["image"], want), "%s: pixel image" % name
    return int((r["image"].view(torch.int16) != 0).any(1).sum())


def conv_weight(conv, dev):
    """The float32 weight in conv_ref's layout: a stride-1 Conv2DTranspose's [Cin, Cout, 1, 1] becomes [Cout, Cin, 1, 1]."""
    import torch
    w = torch.from_numpy(conv.np["weight"]).to(dev)
    return w.transpose(0, 1).contiguous() if conv.transposed and conv.up == 1 else w


def check_convs(name, r, sms):
    """Every dense conv of r["convs"] from its actual input image against the float64 conv and epilogue on the dense bar,
    and the bar rejecting the hi x hi products alone and the result without one tap (centre tap of a 3x3 conv, tap 0
    of the 2x2 stride-2 conv, 32-channel input group Cin / 64 of a 1x1 or transposed conv, as DenseCase drops)."""
    import torch
    for i, (conv, x, sh, y, out_C, c0) in enumerate(r["convs"]):
        b, h, w, cin = sh
        k, s, p, up = conv.k, conv.stride, conv.padding, conv.up
        w32 = conv_weight(conv, x.device)
        drop = ("group", cin // 64) if (up > 1 or k == 1) else ("tap", 4 if k == 3 else 0)
        acc, part = conv_ref(from_pixel_h16(x, b, h, w, cin), w32.double(), k, s, p, up, drop)
        scale, shift = conv.dev["scale"], conv.dev["shift"]
        want = epilogue(acc, scale, shift, conv.relu)
        oh, ow = want.shape[1:3]
        if y.dtype == torch.float32:  # PointPillars' head: fp32 NCHW planes
            got = y.permute(0, 2, 3, 1)
        else:
            got = from_pixel_h16(y, b, oh, ow, out_C)[..., c0:c0 + conv.cout]
        terms = cin if up > 1 else cin * k * k
        label = "%s conv %d %d->%d k%d s%d up%d%s at c0 %d" % (name, i, cin, conv.cout, k, s, up,
                                                               " transposed" if conv.transposed else "", c0)
        check_images(label, got, want, terms)
        hh, _ = conv_ref(from_pixel_h16(x, b, h, w, cin, hi_only=True), w32.half().double(), k, s, p, up)
        check_rejects(label, [("hi x hi only", epilogue(hh, scale, shift, conv.relu)),
                              ("%s %d dropped" % drop, epilogue(acc - part, scale, shift, conv.relu))], want, terms)
        floor, _ = bar(terms)
        print("BAR %s, %d terms (floor %.0e): error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
              % ((label, terms, floor) + error_stats(got, want)))
        pl = Plan(sms, b, h, w, cin, conv.cout, conv.n_tile, k, s, p, up)
        print("REGIME %s: %s" % (label, pl.describe()))
        del acc, part, hh, want, got


def check_fused_head(name, d, r, sms):
    """The fused head's planes against the tap-sum reference of the float64 ConvModule output of the actual shared map."""
    import torch
    dev = r["planes"].device
    bp = r["bp"]
    heads = [(n, a, f) for hs in d.heads for n, a, f in hs]
    b, H, W, cin = r["head_shape"]
    wbig = torch.cat([torch.from_numpy(a.np["weight"]) for _, a, _ in heads], 0).to(dev).double()
    acc, _ = conv_ref(from_pixel_h16(r["shared"], b, H, W, cin), wbig, 3, 1, 1, 1)
    mid = epilogue(acc, bp["big"].dev["scale"], bp["big"].dev["shift"], True)
    del acc, wbig
    P = torch.stack([torch.einsum("bhwc,cn->bhwn", mid[..., 64 * g:64 * (g + 1)],
                                  w2_image(torch.from_numpy(f.np["weight"]).to(dev).double()))
                     for g, (_, _, f) in enumerate(heads)], 1)
    del mid
    want = tap_sum_ref(P, bp["bias9"], [int(v) for v in bp["plane0_9"]], [int(v) for v in bp["cnt9"]], bp["planes"])
    del P
    assert not bool(torch.isnan(want).any()) and want.shape[1] == 70
    check_images("%s fused head planes" % name, r["planes"], want, PLANE_TERMS)
    # the second launch alone: the planes are the fp32 tap sum of the P buffer the first launch wrote, in its order
    f32 = tap_sum_f32(r["P"], bp["bias9"], [int(v) for v in bp["plane0_9"]], [int(v) for v in bp["cnt9"]], bp["planes"])
    assert _bits_equal(r["planes"], f32), "%s: planes differ from the fp32 tap sum of the fused conv's P" % name
    print("BAR %s fused head planes, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
          % ((name, PLANE_TERMS) + error_stats(r["planes"], want)))
    print("REGIME %s fused head conv %d->%d: %s" % (name, cin, bp["big"].cout,
                                                    FusedPlan(sms, b, H, W, cin, bp["big"].cout).describe()))


def check_pp_postprocess(name, oracle_mod, m, r):
    """anchor_head_postprocess (oracle.pointpillars for one class, oracle.pointpillars_multiclass for several) of the
    actual planes: candidate and box counts and labels exact; the decoded candidates in score order (the first
    nms_pre), the boxes and the scores on test_gpu_pointpillars' tolerances.
    Returns (candidates, boxes)."""
    import oracle.pointpillars as opp
    import oracle.pointpillars_multiclass as opm
    tc = m.mc["test"]
    n = int(r["nv"][0])
    planes = r["planes"].cpu().numpy()
    coors = r["coors"][:n].cpu().numpy()
    args = (planes, m.anchors_np, m.corners_np, coors, m.grid, tc["post_center_limit_range"], tc["anchor_area_threshold"],
            tc["nms_score_threshold"], tc["nms_iou_threshold"], tc["nms_pre_max_size"], tc["nms_post_max_size"])
    want = opp.anchor_head_postprocess(*args) if m.num_classes == 1 else \
        opm.anchor_head_postprocess(*args, num_classes=m.num_classes)
    boxes, scores, labels, counts = r["post"]
    ncand, k = [int(v) for v in counts.cpu()]
    assert ncand == want["candidates"] and k == len(want["boxes"]), "%s: counts %d / %d, oracle %d / %d" % (
        name, ncand, k, want["candidates"], len(want["boxes"]))
    nc = min(ncand, tc["nms_pre_max_size"])
    cb, cs = (t[:nc].cpu().numpy() for t in r["cand"])
    np.testing.assert_allclose(cb, want["cand_boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(cs, want["cand_scores"], rtol=1e-6, atol=0)
    np.testing.assert_allclose(boxes[:k].cpu().numpy(), want["boxes"], rtol=1e-6, atol=1e-6)
    np.testing.assert_allclose(scores[:k].cpu().numpy(), want["scores"], rtol=1e-6, atol=0)
    assert np.array_equal(labels[:k].cpu().numpy(), want["labels"]), "%s: labels" % name
    return ncand, k


# -------------------------------------------------------------------------------------------------------- CPU tests
def test_restated_chains_are_the_models():
    """cp_chain_convs plus the CenterHead's 36 ConvModule / output-conv pairs are CenterPointPillars.head.all_convs() in
    order, and pp_chain_convs is PointPillars.trunk.convs() + [head], for both PointPillars models; the lists match the
    tables CP_CHAIN / PP_CHAIN and the feature sizes CP_SIZES / PP_SIZES.  A conv removed from, added to or moved in a
    model fails here instead of leaving a stale restatement."""
    from paddle3d_b200.centerpoint_pillars import CenterPointPillars
    from paddle3d_b200.dense_head import COMMON_HEADS
    from paddle3d_b200.pointpillars import CONFIG, CONFIG_PED_CYCLIST, PointPillars
    m = CenterPointPillars(synth.CP_PILLARS)
    d = m.head
    chain, allc = cp_chain_convs(d), d.all_convs()
    assert len(allc) == len(chain) + 2 * 36 and all(a is b for a, b in zip(chain, allc))
    pairs = [c for hs in d.heads for _, a, f in hs for c in (a, f)]
    assert all(a is b for a, b in zip(allc[len(chain):], pairs))
    assert _table(chain) == CP_CHAIN and len(chain) == 20
    names = [n for n, _ in COMMON_HEADS] + ["hm"]
    assert len(d.heads) == 6 and all([n for n, _, _ in hs] == names for hs in d.heads)
    pix, blocks, cat = CP_SIZES
    assert (m.grid[1], m.grid[0]) == pix and m.feat_hw == blocks and m.cat_hw == cat
    feats, outs = _sizes(chain, d.blocks, pix)
    assert feats == blocks and outs == [cat] * 3
    assert d.fpn_channels == 384 and d.shared.cin == 384 and d.shared.cout == 64 and d.head_planes() == 70
    assert d.bev_depth == 1 and m.C == 64 and m.cfg["max_voxels"] == 60000 and m.cfg["max_points"] == 20

    for key, cfg, mc in (("car", synth.C2, CONFIG), ("ped_cyclist", synth.C2_PED_CYCLIST, CONFIG_PED_CYCLIST)):
        m = PointPillars(cfg, mc)
        chain = pp_chain_convs(m)
        allc = m.trunk.convs() + [m.head]
        assert len(chain) == len(allc) == 20 and all(a is b for a, b in zip(chain, allc)), key
        assert _table(chain) == PP_CHAIN[key], key
        assert m.head.has_bias and m.head.bn_eps is None and not m.head.relu
        pix, blocks, cat = PP_SIZES[key]
        feats, outs = _sizes(chain, m.trunk.blocks, pix)
        assert (m.grid[1], m.grid[0]) == pix and feats == blocks and outs == [cat] * 3 and m.feat_hw == cat, key
        assert m.trunk.fpn_channels == 384 and m.head_channels == m.head.cout
        assert m.anchors_np.shape[0] == cat[0] * cat[1] * mc["anchors_per_loc"]


# -------------------------------------------------------------------------------------------------------- GPU tests
def _cp_hot(cuda, **kw):
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    return CenterPointPillarsHotPath(synth.CP_PILLARS, cuda, seed=0, bn_gain=kw.pop("bn_gain", bench.BN_GAIN), **kw)


def _cp_bench_frame(cuda):
    """The bench tool's frame: head calibrated on bench.frame_pool(CP_PILLARS, .)[0] (= lidar_cloud(CP_PILLARS, 0)),
    captured on that cloud.  Returns (hot, points, device points)."""
    import torch
    pts = bench.frame_pool(synth.CP_PILLARS, 1)[0]
    pts_d = torch.from_numpy(pts).to(cuda)
    hot = _cp_hot(cuda)
    hot.calibrate_head(pts_d)
    hot.points.copy_(pts_d)
    return hot, pts, pts_d


def _cp_stages(name, oracle_mod, hot, r, pts, sms):
    """Every stage of a CenterPoint-pillars chain against its reference.  Returns (pillar stats, occupied pixels, cells
    above the score threshold per task, boxes per task)."""
    from oracle.centerpoint_pillars import pillar_feature_net2
    m = hot.model
    cfg = m.cfg
    stats = check_voxelize(name, oracle_mod, r, pts, cfg)
    k = stats[0]
    want = pillar_feature_net2(r["voxels"][:k].cpu().numpy(), r["npv"][:k].cpu().numpy(), r["coors"][:k].cpu().numpy(),
                               m.pfn, cfg["voxel_size"], cfg["point_cloud_range"])
    check_pfn(name, r, want, True)
    del want
    occupied = check_pixel_image(name, m, r)
    assert [c for c, *_ in r["convs"]] == cp_chain_convs(m.head)
    check_convs(name, r, sms)
    check_fused_head(name, m.head, r, sms)
    passing, per_task = check_postprocess(name, oracle_mod, m, r)
    return stats, occupied, passing, per_task


@pytest.mark.gpu
def test_cp_pillars_bench_frame_stage_by_stage(cuda, oracle_mod):
    """The bench frame restated (cp_pillars_chain) eagerly and captured: status 0; the two chains and
    CenterPointPillarsHotPath's captured frame bit-equal (pixel image and every conv output between the chains, head
    planes and boxes with the hot path); every stage of the eager chain from its actual input buffer against its
    reference, with the pillar counts of CP_BENCH_PILLARS and about 97 % of the pixels empty."""
    import torch
    hot, pts, pts_d = _cp_bench_frame(cuda)
    hot.capture()
    want = [t.clone() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    assert not hot.h_status.any()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    eager, captured, graph = _run_chains(cp_pillars_chain, hot, pts_d)
    for label, r in (("eager", eager), ("captured", captured)):
        assert not r["status"].any(), "%s chain: status %s" % (label, r["status"].tolist())
        assert _bits_equal(r["image"], eager["image"]), "%s chain: pixel image" % label
        for i, (a, b) in enumerate(zip(eager["convs"], r["convs"])):
            assert _bits_equal(a[3], b[3]), "%s chain: conv %d differs from the eager chain's" % (label, i)
        for key, planes in hot.out["head"].items():
            for t, p in enumerate(planes):
                assert _bits_equal(r["heads"][key][t], p), "%s chain: %s planes of task %d differ from the hot " \
                                                           "path's" % (label, key, t)
        boxes, scores, labels, counts = r["post"]
        k = int(counts[-1])
        assert k == len(want[2]), "%s chain: box count %d, hot path %d" % (label, k, len(want[2]))
        assert _bits_equal(boxes[:k].cpu(), want[0]) and _bits_equal(scores[:k].cpu(), want[1])
        assert torch.equal(labels[:k].cpu(), want[2])
    del captured, graph
    torch.cuda.empty_cache()

    (k, at_max, one, _), occupied, passing, per_task = _cp_stages("cp_pillars", oracle_mod, hot, eager, pts, sms)
    assert (points_in_range(pts, synth.CP_PILLARS)[0], k, at_max, one) == CP_BENCH_PILLARS
    assert occupied == k
    empty = 1.0 - occupied / (512 * 512)
    assert 0.97 < empty < 0.975, empty
    tc = hot.model.test_cfg
    print("POST cp_pillars bench frame: %d pillars (%d at %d points), %.1f %% of the pixels empty; cells above the score "
          "threshold per task %s (nms_pre %d); boxes per task %s (nms_post %d)" % (
              k, at_max, synth.CP_PILLARS["max_points"], 100 * empty, passing, tc["nms_pre_max_size"], per_task,
              tc["nms_post_max_size"]))
    # the calibration puts 1.4 % of each task's 128 x 128 cells above the threshold (measured on an H100: 229 or 230),
    # fewer than nms_pre: the frame never takes the nms_pre cut, and every task takes the nms_post cut
    assert all(p in (229, 230) for p in passing) and max(passing) < tc["nms_pre_max_size"], passing
    assert per_task == [tc["nms_post_max_size"]] * 6 and sum(per_task) == len(want[2]), per_task


@pytest.mark.gpu
def test_cp_pillars_at_pillar_cap(cuda, oracle_mod):
    """uniform_cloud(CP_PILLARS, 0) on the bench-calibrated model: hard_voxelize keeps the first 60 000 of 166 820
    occupied pillars in point order (at most 7 points each), bit-equal to the oracle; the PFN on all 60 000 rows, a
    pixel image with 60 000 occupied pixels, the 20 convs, the head and the postprocess on their bars.  Dropping
    pillars at the cap is the reference's silent behaviour: infer() returns with status 0."""
    import torch
    hot, _, _ = _cp_bench_frame(cuda)
    pts = synth.uniform_cloud(synth.CP_PILLARS, 0)
    pts_d = torch.from_numpy(pts).to(cuda)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    r = cp_pillars_chain(hot, pts_d)
    torch.cuda.synchronize()
    assert not r["status"].any()
    (k, at_max, one, most), occupied, passing, per_task = _cp_stages("cp_pillars uniform", oracle_mod, hot, r, pts, sms)
    in_range, cells = points_in_range(pts, synth.CP_PILLARS)
    assert (in_range, cells, k, most, one) == CP_UNIFORM and at_max == 0
    assert occupied == k == synth.CP_PILLARS["max_voxels"]
    boxes, _, labels = hot.infer(torch.from_numpy(pts).pin_memory())
    assert not hot.h_status.any(), "dropping pillars at the cap is not an error"
    assert len(labels) == sum(per_task)
    tc = hot.model.test_cfg
    cut = [p > tc["nms_pre_max_size"] for p in passing]
    print("POST cp_pillars uniform: %d of %d occupied pillars kept, %d occupied pixels; cells above the score threshold "
          "per task %s (nms_pre %d: cut in %d tasks); boxes per task %s (nms_post %d)" % (
              k, cells, occupied, passing, tc["nms_pre_max_size"], sum(cut), per_task, tc["nms_post_max_size"]))
    # with 23 % of the pixels occupied instead of 2.8 %, the bench calibration lets 3 500 to 13 700 cells per task
    # through (measured on an H100): both NMS cuts bind in every task
    assert all(cut) and per_task == [tc["nms_post_max_size"]] * 6, (passing, per_task)


@pytest.mark.gpu
def test_cp_pillars_nms_pre_cut(cuda, oracle_mod):
    """The bench frame with the heat maps calibrated to 8 % of the 16 384 cells per task (about 1 300, more than
    nms_pre 1000): the postprocess of the actual planes against the oracle, and the nms_pre cut taken in every task."""
    import torch
    hot, pts, pts_d = _cp_bench_frame(cuda)
    hot.model.calibrate_heatmap_bias(pts_d, target_frac=0.08)
    r = cp_pillars_chain(hot, pts_d)
    torch.cuda.synchronize()
    assert not r["status"].any()
    passing, per_task = check_postprocess("cp_pillars 8 %", oracle_mod, hot.model, r)
    tc = hot.model.test_cfg
    print("POST cp_pillars calibrated to 8 %%: cells above the score threshold per task %s (nms_pre %d); boxes per task "
          "%s (nms_post %d)" % (passing, tc["nms_pre_max_size"], per_task, tc["nms_post_max_size"]))
    # measured on an H100: 1 311 cells in every task, then 83 boxes in every task
    assert all(1300 < p < 1320 for p in passing) and min(passing) > tc["nms_pre_max_size"], passing
    assert per_task == [tc["nms_post_max_size"]] * 6, per_task


@pytest.mark.gpu
def test_cp_pillars_fp16_range_raises(cuda):
    """The bench cloud with BatchNorm gain 6: the fp16-pair path saturates (status bit 0) and infer() raises the
    fp16-range error."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    pts = torch.from_numpy(bench.frame_pool(synth.CP_PILLARS, 1)[0]).pin_memory()
    hot = _cp_hot(cuda, bn_gain=FP16_GAIN)
    with pytest.raises(RuntimeError, match="left fp16's range"):
        hot.infer(pts)
    st = int(hot.h_status[0])
    assert st & 1, st
    print("FP16 cp_pillars gain %.1f: status word %d" % (FP16_GAIN, st))
    sp.status_tensor(cuda).zero_()  # the device's word is sticky: it would carry the overflow into the next frame


@pytest.mark.gpu
def test_cp_pillars_lanes_full_size(cuda):
    """CenterPointSweep with four CenterPointPillarsHotPath lanes, infer_many over six distinct bench.frame_pool clouds
    (twice, so both staging sets of each lane are reused): every frame bit-equal to the single-lane captured frame."""
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    cfg = synth.CP_PILLARS
    frames = bench.frame_pool(cfg, 6)
    pinned = [torch.from_numpy(f).pin_memory() for f in frames]
    dev0 = torch.from_numpy(frames[0]).to(cuda)
    sweep = CenterPointSweep(4, frame_cls=CenterPointPillarsHotPath, cfg=cfg, device=cuda, seed=0, bn_gain=bench.BN_GAIN)
    sweep.calibrate_head(dev0)
    sweep.capture(dev0)
    single = _cp_hot(cuda)
    single.share_model(sweep.lanes[0])
    single.points.copy_(dev0)
    single.capture()
    want = [[t.clone() for t in single.infer(f)] for f in pinned]
    assert len({float(w[0].sum()) for w in want}) == len(want)
    for rnd in range(2):
        got = list(sweep.infer_many(iter(pinned)))
        assert len(got) == len(want)
        for i, (g, w) in enumerate(zip(got, want)):
            assert len(g[2]) == len(w[2]), "round %d frame %d: box count" % (rnd, i)
            assert _bits_equal(g[0], w[0]) and _bits_equal(g[1], w[1]) and torch.equal(g[2], w[2]), \
                "round %d frame %d differs from the single-lane frame" % (rnd, i)
    print("LANES cp_pillars 4 lanes, %d frames x 2 rounds: boxes per frame %s" % (len(want), [len(w[2]) for w in want]))


@pytest.mark.gpu
def test_cp_pillars_sweep_stream_full_size(cuda):
    """sweep_input at its defaults (10 sweeps into 300 000 rows, default slot_cap) on a synth.sweep_sequence of about
    29 500 points per sweep: the device merge bit-equal to io.merge_sweeps (NaN rows after it), merge status 0, and
    one frame's infer_sweeps equal to infer on io.merge_sweeps' cloud; infer_stream on two lanes sharing one ring equals
    the single lane."""
    import torch
    from paddle3d_b200.centerpoint_pillars import CenterPointPillarsHotPath
    from paddle3d_b200.pipeline import CenterPointSweep
    K = 10
    seq = synth.sweep_sequence(K + 3, 2)
    ref, _, _ = _cp_bench_frame(cuda)
    pipe = _cp_hot(cuda, sweep_input=dict())
    pipe.share_model(ref)
    assert pipe.n == 300000 and pipe.sweep_input["max_sweeps"] == K and pipe.h_status.numel() == 2
    key, sweeps = _frame_inputs(seq, K - 1, K)
    merged = p3d_io.merge_sweeps(key, sweeps, use_dim=4, use_time_lag=True, sweep_remove_radius=1.0)
    assert 0.9 * pipe.n < len(merged) <= pipe.n, len(merged)
    full = np.full((pipe.n, 5), np.nan, np.float32)
    full[:len(merged)] = merged
    want = [t.clone() for t in ref.infer(torch.from_numpy(full).pin_memory())]
    eager = [t.clone() for t in pipe.infer_sweeps(key, sweeps)]
    assert not pipe.h_status.any(), pipe.h_status.tolist()
    assert pipe.merged_rows() == len(merged) and len(eager[0]) > 0
    # the device merge transforms in fp64 and rounds once to fp32, as the host merge does: the same rows, the same bits
    rows = pipe.points.cpu().numpy()
    assert np.array_equal(rows[:len(merged)].view(np.uint32), merged.view(np.uint32)), "device merge != host merge"
    assert np.isnan(rows[len(merged):]).all()
    assert all(_bits_equal(a, b) for a, b in zip(eager[:2], want[:2])) and torch.equal(eager[2], want[2])
    pipe.capture()
    got = pipe.infer_sweeps(key, sweeps)
    assert all(_bits_equal(a, b) for a, b in zip(got[:2], eager[:2])) and torch.equal(got[2], eager[2])
    single = list(pipe.infer_stream(iter(seq)))
    lanes = CenterPointSweep(2, frame_cls=CenterPointPillarsHotPath, cfg=synth.CP_PILLARS, device=cuda, seed=0,
                             bn_gain=bench.BN_GAIN, sweep_input=dict())
    assert lanes.lanes[1].ring is lanes.lanes[0].ring
    for p in lanes.lanes:
        p.share_model(ref)
        p.infer_sweeps(*_frame_inputs(seq, 0, K))
        p.capture()
    got = list(lanes.infer_stream(iter(seq)))
    assert len(got) == len(single) == len(seq)
    for j, (g, w) in enumerate(zip(got, single)):
        assert all(_bits_equal(a, b) for a, b in zip(g[:2], w[:2])) and torch.equal(g[2], w[2]), j
    print("SWEEPS cp_pillars: %d merged rows of %d, bit-equal to the host merge; %d stream frames, boxes %s" % (
        len(merged), pipe.n, len(single), [len(s[2]) for s in single]))


PP_MODELS = ["car", "ped_cyclist"]
PP_CANDIDATES = {"car": 2143, "ped_cyclist": 3864}  # anchors above the score threshold on the bench frame


@pytest.mark.gpu
@pytest.mark.parametrize("key", PP_MODELS)
def test_pointpillars_bench_frame_stage_by_stage(cuda, oracle_mod, key):
    """The bench frame of tools/pointpillars_bench.py (seed 0, bench.BN_GAIN, classes calibrated on
    bench.frame_pool(cfg, .)[0], run on that cloud) restated (pointpillars_chain) eagerly and captured: status 0, the two
    chains and PointPillarsHotPath's captured frame bit-equal in the head planes and the boxes; hard_voxelize bit for
    bit with PP_BENCH_PILLARS' counts, the PFN against oracle.pillar_feature_net, the pixel image bit for bit, the 16
    convs, 3 deblocks and the head on the dense bar with its guards, the postprocess against the oracle of the actual
    planes, with more candidates than nms_pre (the cut runs)."""
    import torch
    from paddle3d_b200.pointpillars import CONFIG, CONFIG_PED_CYCLIST, PointPillarsHotPath
    cfg, mc = (synth.C2, CONFIG) if key == "car" else (synth.C2_PED_CYCLIST, CONFIG_PED_CYCLIST)
    pts = bench.frame_pool(cfg, 1)[0]
    pts_d = torch.from_numpy(pts).to(cuda)
    hot = PointPillarsHotPath(cfg, cuda, seed=0, bn_gain=bench.BN_GAIN, model_cfg=mc)
    hot.calibrate_head(pts_d)
    hot.points.copy_(pts_d)
    hot.capture()
    want = [t.clone() for t in hot.infer(torch.from_numpy(pts).pin_memory())]
    assert not hot.h_status.any()
    hot_planes = hot.out["planes"].clone()
    hot_counts = hot.h_counts.clone()
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    eager, captured, graph = _run_chains(pointpillars_chain, hot, pts_d)
    for label, r in (("eager", eager), ("captured", captured)):
        assert not r["status"].any(), "%s chain: status %s" % (label, r["status"].tolist())
        assert _bits_equal(r["image"], eager["image"]), "%s chain: pixel image" % label
        for i, (a, b) in enumerate(zip(eager["convs"], r["convs"])):
            assert _bits_equal(a[3], b[3]), "%s chain: conv %d differs from the eager chain's" % (label, i)
        assert _bits_equal(r["planes"], hot_planes), "%s chain: head planes differ from the hot path's" % label
        boxes, scores, labels, counts = r["post"]
        assert torch.equal(counts.cpu(), hot_counts), "%s chain: counts %s, hot path %s" % (label, counts, hot_counts)
        k = int(counts[-1])
        assert _bits_equal(boxes[:k].cpu(), want[0]) and _bits_equal(scores[:k].cpu(), want[1])
        assert torch.equal(labels[:k].cpu(), want[2])
    del captured, graph
    torch.cuda.empty_cache()

    m, r = hot.model, eager
    name = "pointpillars %s" % key
    k, at_max, one, _ = check_voxelize(name, oracle_mod, r, pts, cfg)
    assert (points_in_range(pts, cfg)[0], k, at_max, one) == PP_BENCH_PILLARS[key]
    p = m.pfn
    want_pfn = oracle_mod.pillar_feature_net(r["voxels"][:k].cpu().numpy(), r["npv"][:k].cpu().numpy(),
                                             r["coors"][:k].cpu().numpy(), p["weight"], p["gamma"], p["beta"], p["mean"],
                                             p["var"], p["eps"], cfg["voxel_size"], cfg["point_cloud_range"])
    check_pfn(name, r, want_pfn, False)
    occupied = check_pixel_image(name, m, r)
    assert occupied == k
    assert [c for c, *_ in r["convs"]] == pp_chain_convs(m)
    assert m.head.dev["scale"] is None  # the head's epilogue adds the bias only
    check_convs(name, r, sms)
    ncand, nbox = check_pp_postprocess(name, oracle_mod, m, r)
    tc = m.mc["test"]
    nx, ny = m.grid
    print("POST %s: %d pillars (%d at %d points), %.1f %% of the pixels empty; %d candidates of %d anchors (nms_pre %d); "
          "%d boxes (nms_post %d)" % (name, k, at_max, cfg["max_points"], 100 * (1 - occupied / (nx * ny)), ncand,
                                      m.anchors_np.shape[0], tc["nms_pre_max_size"], nbox, tc["nms_post_max_size"]))
    # calibrate_cls_bias puts round(2 % of the anchors / C) above the threshold in each class, 2 143 for the car; the
    # two classes of the cyclist / pedestrian model share 2 008 of their 2 x 2 936 anchors (measured on an H100).  Both
    # exceed nms_pre, so the cut runs; NMS leaves fewer boxes than nms_post (235 car, 185 cyclist / pedestrian)
    assert ncand == PP_CANDIDATES[key] > tc["nms_pre_max_size"], ncand
    assert nbox < tc["nms_post_max_size"], nbox
