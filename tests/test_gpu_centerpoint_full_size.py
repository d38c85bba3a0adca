"""CenterPoint-voxel, the benchmarked frame, at full size stage by stage, its strided levels at and past their row
capacities, its two status branches and its sweep lanes, against float64 references.

The frame is bench.py's: CenterPointHotPath(cfg, precision=F16X3, with_head=True, keep_bev=False, bn_gain=bench.BN_GAIN)
with the head calibrated on the 300 k-point synth.lidar_cloud it then runs.  frame_chain restates forward_device's launch
chain on one stream with no sync in between and keeps every buffer: voxelize_mean, the 21 sparse convs of
SparseResNet3D (sparse_steps, tied to SparseResNet3D.all_layers() by a CPU test) with the input and output rows of each,
the BEV pixel image, the dense trunk, the deblocks and the shared conv (dense_chain_convs, tied to DenseRPNHead by a CPU
test), the fused CenterHead conv + tap sum, and the postprocess.  Every stage is checked from its actual input buffer:

  * voxelize_mean against oracle.hard_voxelize (bit for bit) and the fp32 slot-order mean (lidar_front_end_oracle);
  * the level-0 SubM map, each strided level's site set, counters and taps, and each level's fused SubM map against
    maps built here (numpy candidate sets, lidar_front_end_oracle.nbr_map, subm_rulebook_torch);
  * every sparse conv against the float64 gather-GEMM of test_gpu_sparse_schedule on the rel_check bar, which rejects
    the hi x hi products alone and the result without one tap;
  * the BEV pixel image bit for bit against rows_to_pixel_h16 of the last level's rows;
  * the dense convs on test_gpu_dense_schedule's bar, the head planes against the tap-sum reference of
    test_gpu_head_fused_schedule, the postprocess against oracle.centerpoint_postprocess of the actual planes.

The strided levels number their rows with atomics (DESIGN section 8), so a row's place in the work decomposition
changes from run to run.  A conv's result is then the same bits only where its decomposition does not depend on the
row's place: not on the warp-MMA kernel (stream-K over warps, in row order) and not under the wgmma kernel's stream-K
(a tile's taps are cut at points that follow the tile's index; the 2-4 tap splits cut every tile at the same taps and
sum the pieces in index order).  Measured on an H100: with NARROW_WM off alone, level 1's 16 -> 32 conv (stream-K at
39 526 rows) already differs in a quarter of its rows between two runs.  So the float64 checks run in the default mode
(the one bench.py times), and the bit-equality of the eager chain, the captured chain and CenterPointHotPath's captured
frame in a second pass with NARROW_WM off and at most 3 splits (no stream-K); the level counts are the same in both.
Lines starting with "REGIME" (pytest -s) name each conv's work decomposition at its real row count, "BAR" the sparse
convs' error figures, "LEVELS" the site counts, "MEM" each test's peak device memory and wall time."""
import time

import numpy as np
import pytest

import bench
import lidar_front_end_oracle as lfo
from paddle3d_b200 import synth
from parity import rel_check
from test_gpu_boxes import RTOL
from test_gpu_dense_schedule import Plan, _bits_equal, bar, check_images, conv_ref, from_pixel_h16
from test_gpu_dense_schedule import epilogue as dense_epilogue
from test_gpu_head_fused_schedule import PLANE_TERMS, FusedPlan, tap_sum_ref, w2_image
from test_gpu_sparse_schedule import epilogue, f16_sched, from_h16, gather_gemm, subm_rulebook_torch, wm_ranges

V = 160000  # max_voxels of both geometries
# (id, cfg, voxels kept from lidar_cloud(cfg, 0), sites of the four strided levels)
GEOMS = [("C3", synth.C3, 67517, [39526, 16141, 6547, 5535]),
         ("C3_01", synth.C3_01, 54675, [34171, 15176, 6516, 5635])]
# uniform_cloud(C3, 0): occupied cells, and the levels' exact site counts from the 160 000 kept voxels
UNIFORM_CELLS, UNIFORM_LEVELS = 266007, [525805, 635490, 161278, 64800]
WIDE_CAPS = [4 * V, 4 * V, 2 * V, V]
FP16_GAIN = 6.0  # BatchNorm gain that drives the backbone's activations far past 65504 (sqrt(6) keeps them O(1))

# The 21 steps of SparseResNet3D: (Cin, Cout, SubM, residual) with residual the step whose output the conv adds before
# its ReLU; every step is conv -> BN (-> + residual) -> ReLU, one fused launch
SPARSE_CHAIN = ([(5, 16, True, None)]
                + [(16, 16, True, None), (16, 16, True, 0), (16, 16, True, None), (16, 16, True, 2)]
                + [(16, 32, False, None), (32, 32, True, None), (32, 32, True, 5), (32, 32, True, None), (32, 32, True, 7)]
                + [(32, 64, False, None), (64, 64, True, None), (64, 64, True, 10), (64, 64, True, None), (64, 64, True, 12)]
                + [(64, 128, False, None), (128, 128, True, None), (128, 128, True, 15), (128, 128, True, None),
                   (128, 128, True, 17)]
                + [(128, 128, False, None)])
# the strided steps' (kernel, stride, padding) and the rulebook key of the SubM map fused into their rulebook launch
STRIDED = {5: ((3, 3, 3), (2, 2, 2), (1, 1, 1), "res1"), 10: ((3, 3, 3), (2, 2, 2), (1, 1, 1), "res2"),
           15: ((3, 3, 3), (2, 2, 2), (0, 1, 1), "res3"), 20: ((3, 1, 1), (2, 1, 1), (0, 0, 0), None)}
# DenseRPNHead(256)'s convs before the CenterHead, in launch order: (Cin, Cout, k, stride, up)
DENSE_CHAIN = ([(256, 128, 3, 1, 1)] + [(128, 128, 3, 1, 1)] * 5 + [(128, 256, 3, 2, 1)] + [(256, 256, 3, 1, 1)] * 5
               + [(128, 256, 1, 1, 1), (256, 256, 2, 2, 2)] + [(512, 64, 3, 1, 1)])


@pytest.fixture(autouse=True)
def _clean_status_and_peak_memory(request):
    """Each test starts from a zero device status word (the word is per device and sticky: any earlier overflow in the
    process would show in every later frame) and prints its peak device memory and wall time ("MEM" lines)."""
    import torch
    gpu = torch.cuda.is_available()
    if gpu:
        from paddle3d_b200.ops import sparse_nn as sp
        sp.status_tensor(torch.device("cuda:0")).zero_()
        torch.cuda.reset_peak_memory_stats()
    t0 = time.perf_counter()
    yield
    if gpu:
        torch.cuda.synchronize()
        print("MEM %s: peak device memory %.2f GiB, wall time %.1f s" % (
            request.node.name, torch.cuda.max_memory_allocated() / 2 ** 30, time.perf_counter() - t0))


# ------------------------------------------------------------------------------------------------- the model's chain
def sparse_steps(net):
    """[(conv, bn, residual)] of a SparseResNet3D in launch order (residual: as in SPARSE_CHAIN)."""
    steps = [(net.conv_input[0], net.conv_input[1], None)]

    def blocks(bl):
        for b in bl:
            i = len(steps) - 1
            steps.append((b.conv1, b.bn1, None))
            steps.append((b.conv2, b.bn2, i))
    blocks(net.blocks0)
    for down, bl in net.stages:
        steps.append((down[0], down[1], None))
        blocks(bl)
    steps.append((net.extra_conv[0], net.extra_conv[1], None))
    return steps


def dense_chain_convs(dense):
    """DenseRPNHead's convs before the CenterHead in launch order: the trunk blocks, the deblocks, the shared conv."""
    return [c for blk in dense.blocks for c in blk] + list(dense.deblocks) + [dense.shared]


def sparse_chain(net, mean, coors, nv):
    """SparseResNet3D.forward_sparse step by step (sparse_steps): the input tensor and every step's output tensor, and
    every step's pending launch (kept: the tensor drops it when it runs)."""
    from paddle3d_b200.ops import sparse_nn as sp
    x = sp.sparse_coo_tensor(coors, mean, [1] + net.sparse_shape + [net.in_channels], num=nv)
    outs, pend = [x], []
    for conv, bn, res in sparse_steps(net):
        y = bn(conv(outs[-1]))
        if res is not None:
            y = sp.add(y, outs[res + 1])
        y = sp.ReLU()(y)
        pend.append(y._pending)
        outs.append(y)
    return outs, pend


def strided_levels(net, outs):
    """The index sets of the four strided levels."""
    return [outs[i + 1].index for i, (conv, _, _) in enumerate(sparse_steps(net)) if not conv.subm]


def sparse_frame(hot, pts_dev):
    """voxelize_mean, the 21 sparse convs and the BEV pixel image of forward_device, buffers kept."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox
    cfg = hot.cfg
    mean, coors, npv, nv = vox.voxelize_mean(pts_dev, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                             cfg["max_voxels"], 0)
    outs, pend = sparse_chain(hot.net, mean, coors, nv)
    rows, shape = outs[-1].to_pixel_h16()
    status = torch.stack([sp.status_tensor(mean.device)[0]] + [ix.counters[1] for ix in strided_levels(hot.net, outs)])
    return dict(mean=mean, coors=coors, npv=npv, nv=nv, outs=outs, pend=pend, bev=rows, bev_shape=shape, status=status)


def frame_chain(hot, pts_dev):
    """forward_device of the bench frame restated on the current stream, every buffer kept: sparse_frame, then the
    dense trunk (first conv: the (z, c)-permuted image), the deblocks into the concat image, the shared conv, the fused
    CenterHead conv + tap sum, and the postprocess.  convs: (conv, input image, its shape, output image, out_C, c0)."""
    import torch
    from paddle3d_b200.ops import centerpoint_postprocess as cpp
    r = sparse_frame(hot, pts_dev)
    d, dev = hot.dense, pts_dev.device
    convs, feats = [], []
    x, sh = r["bev"], r["bev_shape"]
    for bi, blk in enumerate(d.blocks):
        for ci, conv in enumerate(blk):
            c = d._first_zc if bi == ci == 0 else conv
            y, _, (b, oh, ow) = c(x, sh)
            convs.append((c, x, sh, y, c.cout, 0))
            x, sh = y, (b, oh, ow, c.cout)
        feats.append((x, sh))
    b = sh[0]
    H, W = d.trunk.deblock_out_hw(d.deblocks[0], *feats[0][1][1:3])
    fpn = d.fpn_channels
    cat = torch.empty((b * H * W, 2 * fpn), dtype=torch.float16, device=dev)
    c0 = 0
    for (f, fs), de in zip(feats, d.deblocks):
        de(f, fs, out_split=cat, out_channels=fpn, out_c0=c0)
        convs.append((de, f, fs, cat, fpn, c0))
        c0 += de.cout
    s, _, _ = d.shared(cat, (b, H, W, fpn))
    convs.append((d.shared, cat, (b, H, W, fpn), s, d.shared.cout, 0))
    bp = d._batched_params(dev)
    assert d.fused_heads(bp)
    shape = (b, H, W, d.shared.cout)
    planes = d._tap_sum(d._heads_conv_p(s, shape, bp, dev), bp, dev)
    h = {}
    for name, p0, k in zip(bp["names"], bp["plane0"], bp["cnt"]):
        h.setdefault(name, []).append(planes[:, int(p0):int(p0) + int(k)])
    post = cpp.centerpoint_postprocess_heads(h, hot.cfg["voxel_size"][:2], hot.cfg["point_cloud_range"], hot.test_cfg,
                                             hot.label_off)
    r.update(convs=convs, shared=s, head_shape=shape, planes=planes, heads=h, post=post, bp=bp)
    return r


# ----------------------------------------------------------------------------------------------- references / checks
def strided_sites(coords, spatial, ksize, stride, padding):
    """The exact output site set of a strided sparse conv over input sites coords [n, 4] (b, z, y, x): every
    o = (c + pad - k) / stride that is integral, >= 0 and inside the output grid.  Returns (sites sorted by their
    linear key, output spatial shape)."""
    c, bt = np.asarray(coords, np.int64)[:, 1:], np.asarray(coords, np.int64)[:, 0]
    k, s, p = (np.asarray(v, np.int64) for v in (ksize, stride, padding))
    osp = (np.asarray(spatial, np.int64) + 2 * p - k) // s + 1
    keys = []
    for dz in range(k[0]):
        for dy in range(k[1]):
            for dx in range(k[2]):
                o = c + p - np.asarray([dz, dy, dx])
                ok = (o >= 0).all(1) & (o % s == 0).all(1)
                o = o // s
                ok &= (o < osp).all(1)
                keys.append(((bt[ok] * osp[0] + o[ok, 0]) * osp[1] + o[ok, 1]) * osp[2] + o[ok, 2])
    u = np.unique(np.concatenate(keys))
    vol = osp[0] * osp[1] * osp[2]
    return np.stack([u // vol, u // (osp[1] * osp[2]) % osp[0], u // osp[2] % osp[1], u % osp[2]], 1), osp


def _site_keys(coords, spatial):
    c = np.asarray(coords, np.int64)
    return ((c[:, 0] * spatial[0] + c[:, 1]) * spatial[1] + c[:, 2]) * spatial[2] + c[:, 3]


def check_voxelize(name, oracle_mod, r, pts, cfg):
    """coors, npv, num_voxels bit-equal oracle.hard_voxelize; the mean bit-equal the fp32 slot-order restatement (rows
    past the count zero) and within 1e-6 of oracle.voxel_mean."""
    vox, co, npv, nv = oracle_mod.hard_voxelize(pts, cfg["voxel_size"], cfg["point_cloud_range"], cfg["max_points"],
                                                cfg["max_voxels"])
    k = int(nv[0])
    assert int(r["nv"][0]) == k, name
    coors = r["coors"].cpu().numpy()
    assert np.array_equal(coors[:k, 1:], co[:k]) and not coors[:k, 0].any(), "%s: coors" % name
    assert np.array_equal(r["npv"][:k].cpu().numpy(), npv[:k]), "%s: points per voxel" % name
    mean = r["mean"].cpu().numpy()
    want = lfo.voxel_mean_f32(vox, npv, k)
    assert np.array_equal(mean.view(np.uint32), want.view(np.uint32)), "%s: mean differs from the fp32 restatement" % name
    np.testing.assert_allclose(mean[:k], oracle_mod.voxel_mean(vox, npv, k), rtol=1e-6, atol=1e-6)
    return k


def level_sites(net, r):
    """(counters, sorted site keys) of each strided level."""
    out = []
    for ix in strided_levels(net, r["outs"]):
        cnt = ix.counters.cpu().numpy().copy()
        out.append((cnt, np.sort(_site_keys(ix.coords[:int(cnt[0])].cpu().numpy(), ix.spatial))))
    return out


def check_rulebooks(name, net, r, levels=4, caps_hold=True):
    """The level-0 SubM map; per strided level the site set (exact, or with caps_hold=False a subset of the exact set
    with the overflow flagged), the counters [clamped n, overflow, raw n], every tap, and the fused SubM map.  Returns
    the exact site counts."""
    import torch
    outs, pend = r["outs"], r["pend"]
    ix0 = outs[0].index
    n0 = int(ix0.num[0])
    assert torch.equal(ix0.subm_rulebooks[("res0", (3, 3, 3))][:n0], subm_rulebook_torch(ix0.coords[:n0], ix0.spatial)), \
        "%s: level-0 SubM map" % name
    prev, counts = ix0, []
    for i, (conv, _, _) in enumerate(sparse_steps(net)):
        if conv.subm:
            continue
        if len(counts) == levels:
            break
        ix = outs[i + 1].index
        lvl = "%s level %d" % (name, len(counts) + 1)
        cnt = ix.counters.cpu().numpy()
        n = int(cnt[0])
        pc = prev.coords[:int(prev.num[0])].cpu().numpy()
        want, osp = strided_sites(pc, prev.spatial, conv.kernel_size, conv.stride, conv.padding)
        assert list(osp) == ix.spatial, lvl
        got = ix.coords[:n].cpu().numpy()
        gk, wk = _site_keys(got, osp), _site_keys(want, osp)
        assert len(np.unique(gk)) == n, "%s: a site is listed twice" % lvl
        assert int(cnt[2]) == len(want), "%s: raw count %d, exact set %d" % (lvl, cnt[2], len(want))
        if caps_hold:
            assert n == len(want) and int(cnt[1]) == 0, "%s: counters %s, exact set %d" % (lvl, cnt[:3], len(want))
            assert np.array_equal(np.sort(gk), wk), "%s: site set differs from the exact one" % lvl
        else:
            assert n == min(len(want), ix.cap) and int(cnt[1]) == int(len(want) > ix.cap), "%s: counters %s" % (lvl, cnt[:3])
            assert np.isin(gk, wk).all(), "%s: a kept site is not in the exact set" % lvl
        nbr = pend[i].nbr[:n].cpu().numpy()
        assert np.array_equal(nbr, lfo.nbr_map(pc, got, prev.spatial, conv.kernel_size, conv.stride, conv.padding)), \
            "%s: strided taps" % lvl
        fuse = getattr(conv, "fuse_subm", None)
        if fuse is not None:
            m = ix.subm_rulebooks[(fuse[1], tuple(fuse[0]))]
            assert torch.equal(m[:n], subm_rulebook_torch(ix.coords[:n], ix.spatial)), "%s: fused SubM map" % lvl
        counts.append(len(want))
        prev = ix
    return counts


def check_sparse_convs(name, net, r, sms):
    """Every sparse conv from its actual input rows against the float64 gather-GEMM, BN, residual and ReLU in the
    epilogue's order, on the rel_check bar; the bar rejects the hi x hi products alone and the result without the
    most-used tap.  Prints each conv's decomposition at its real row count."""
    from paddle3d_b200._lib import lib
    from paddle3d_b200.ops import sparse_nn as sp
    assert len(r["pend"]) == 21
    for i, ((conv, _, _), q) in enumerate(zip(sparse_steps(net), r["pend"])):
        n, n_in = int(q.num[0]), int(q.x.index.num[0])
        label = "%s conv %d %d->%d K=%d" % (name, i, q.cin, q.cout, q.K)
        if q.precision == sp.F16X3:
            X = from_h16(q.x._vals[sp.ROWS_H16][:n_in], q.cin)
        else:
            assert q.precision == sp.FP32 and q.cin == 5, label  # the few-channel input layer: exact fp32 FMAs
            X = q.x._vals[sp.ROWS_F32][:n_in].double()
        W = conv.weight.double().reshape(q.K, q.cin, q.cout)
        nbr = q.nbr[:n]
        res = from_h16(q.residual._vals[sp.ROWS_H16][:n], q.cout) if q.residual is not None else None
        acc = gather_gemm(X, nbr, W)
        want = epilogue(acc, q.scale, q.shift, res, q.relu).cpu().numpy()
        got = from_h16(r["outs"][i + 1]._vals[sp.ROWS_H16][:n], q.cout).cpu().numpy()
        floor, small_atol = bar(q.K * q.cin)
        e = rel_check(label, got, want, floor=floor, small_atol=small_atol)
        print("BAR %s, %d terms: relative %.2e above %.0e x max, %.2e x max below" % (
            label, q.K * q.cin, e["max_rel"], floor, e["max_small_abs_over_scale"]))
        hh = gather_gemm(X.float().half().double(), nbr, conv.weight.half().double().reshape(q.K, q.cin, q.cout))
        t_drop = int((nbr >= 0).sum(0).argmax())
        for what, a in (("hi x hi only", hh), ("one tap dropped", acc - gather_gemm(X, nbr, W, taps=[t_drop]))):
            with pytest.raises(AssertionError):
                rel_check(label + " guard: " + what, epilogue(a, q.scale, q.shift, res, q.relu).cpu().numpy(), want,
                          floor=floor, small_atol=small_atol)
        del X, acc, hh, want, got
        if q.precision == sp.FP32:
            regime = "small_cin (fp32 FMA, pair rows out)"
        elif q.wm:
            grid, Wp, U, tiles = wm_ranges(sms, n, q.cap, q.K)
            regime = "warp MMA, %d warps over %d tiles, %.1f units per warp" % (Wp, tiles, U / Wp if Wp else 0.0)
        else:
            ws = lib().p3d_sparse_conv_f16_workspace_bytes(q.cap, q.cout, sp.F16_MAX_SPLITS)
            regime = "wgmma, " + f16_sched(sms, n, q.cap, q.K, q.cout, sp.F16_MAX_SPLITS, ws).label()
        print("REGIME %s rows %d of %d: %s" % (label, n, q.cap, regime))


def check_pixel_image(name, net, r):
    """The BEV pixel image bit-equal rows_to_pixel_h16 of the last level's rows ((z, c) channel order, empty pixels
    zero).  Returns the share of empty pixels."""
    from paddle3d_b200.ops import sparse_nn as sp
    last = r["outs"][-1]
    ix = last.index
    n = int(ix.num[0])
    D, Hb, Wb = ix.spatial
    rows = last._vals[sp.ROWS_H16].cpu().numpy().view(np.uint16)
    want = lfo.rows_to_pixel_h16(rows, ix.coords.cpu().numpy(), n, last.channels, 1, D, Hb, Wb)
    got = r["bev"].cpu().numpy().view(np.uint16)
    assert r["bev_shape"] == (1, Hb, Wb, D * last.channels)
    assert np.array_equal(got, want), "%s: BEV pixel image" % name
    return float((got == 0).all(1).mean())


def check_dense(name, hot, r, sms):
    """The trunk, deblocks and shared conv from their actual input images on the dense bar; the fused head's planes
    against the tap-sum reference of the float64 ConvModule output of the actual shared feature map."""
    import torch
    dev = r["planes"].device
    assert [c for c, *_ in r["convs"]] == [hot.dense._first_zc] + dense_chain_convs(hot.dense)[1:]
    for i, (conv, x, sh, y, out_C, c0) in enumerate(r["convs"]):
        b, h, w, cin = sh
        acc, _ = conv_ref(from_pixel_h16(x, b, h, w, cin), torch.from_numpy(conv.np["weight"]).to(dev).double(), conv.k,
                          conv.stride, conv.padding, conv.up)
        want = dense_epilogue(acc, conv.dev["scale"], conv.dev["shift"], conv.relu)
        del acc
        oh, ow = want.shape[1:3]
        got = from_pixel_h16(y, b, oh, ow, out_C)[..., c0:c0 + conv.cout]
        label = "%s dense conv %d %d->%d k%d s%d up%d" % (name, i, cin, conv.cout, conv.k, conv.stride, conv.up)
        check_images(label, got, want, cin if conv.up > 1 else cin * conv.k * conv.k)
        p = Plan(sms, b, h, w, cin, conv.cout, conv.n_tile, conv.k, conv.stride, conv.padding, conv.up)
        print("REGIME %s: %s" % (label, p.describe()))
        del got, want
    bp = r["bp"]
    heads = [(n, a, f) for hs in hot.dense.heads for n, a, f in hs]
    b, H, W, cin = r["head_shape"]
    wbig = torch.cat([torch.from_numpy(a.np["weight"]) for _, a, _ in heads], 0).to(dev).double()
    acc, _ = conv_ref(from_pixel_h16(r["shared"], b, H, W, cin), wbig, 3, 1, 1, 1)
    mid = dense_epilogue(acc, bp["big"].dev["scale"], bp["big"].dev["shift"], True)
    del acc, wbig
    P = torch.stack([torch.einsum("bhwc,cn->bhwn", mid[..., 64 * g:64 * (g + 1)],
                                  w2_image(torch.from_numpy(f.np["weight"]).to(dev).double()))
                     for g, (_, _, f) in enumerate(heads)], 1)
    del mid
    want = tap_sum_ref(P, bp["bias9"], [int(v) for v in bp["plane0_9"]], [int(v) for v in bp["cnt9"]], bp["planes"])
    del P
    assert not bool(torch.isnan(want).any())
    check_images("%s fused head planes" % name, r["planes"], want, PLANE_TERMS)
    print("REGIME %s fused head conv %d->%d: %s" % (name, cin, bp["big"].cout,
                                                    FusedPlan(sms, b, H, W, cin, bp["big"].cout).describe()))


def check_postprocess(name, oracle_mod, hot, r):
    """oracle.centerpoint_postprocess of the actual head planes: labels, order and counts exact, scores and boxes on
    test_gpu_boxes' tolerances.  Returns the score-passing cells per task and the per-task box counts."""
    h = {k: [t.cpu().numpy() for t in v] for k, v in r["heads"].items()}
    cfg, tc = hot.cfg, hot.test_cfg
    wb, ws, wl, wc = oracle_mod.centerpoint_postprocess(
        h["hm"], h["reg"], h["height"], h["dim"], h["vel"], h["rot"], cfg["voxel_size"][:2], cfg["point_cloud_range"],
        tc["post_center_limit_range"], hot.label_off, tc["down_ratio"], tc["score_threshold"], tc["nms_iou_threshold"],
        tc["nms_pre_max_size"], tc["nms_post_max_size"], True)
    boxes, scores, labels, counts = (t.cpu().numpy() for t in r["post"])
    k = int(counts[-1])
    assert np.array_equal(counts[:-1], wc) and k == len(wl), "%s: counts %s, oracle %s" % (name, counts, wc)
    assert np.array_equal(labels[:k], wl), "%s: labels / order" % name
    np.testing.assert_allclose(scores[:k], ws, rtol=RTOL)
    np.testing.assert_allclose(boxes[:k], wb, rtol=RTOL, atol=1e-5)
    passing = [int((1.0 / (1.0 + np.exp(-hm.astype(np.float64).max(1))) > tc["score_threshold"]).sum()) for hm in h["hm"]]
    return passing, [int(c) for c in wc]


# -------------------------------------------------------------------------------------------------------- CPU tests
def test_restated_chain_is_the_model():
    """sparse_steps walks SparseResNet3D.all_layers() in order (every conv and BN once) and matches SPARSE_CHAIN and
    STRIDED; dense_chain_convs plus the CenterHead's ConvModule / output-conv pairs are DenseRPNHead.all_convs() in
    order and match DENSE_CHAIN.  A change of either model fails here instead of leaving a stale restatement."""
    from paddle3d_b200.dense_head import COMMON_HEADS, DenseRPNHead
    from paddle3d_b200.layers import SparseResNet3D
    from paddle3d_b200.ops import sparse_nn as sp
    for cfg in (synth.C3, synth.C3_01):
        net = SparseResNet3D(cfg["point_dim"], cfg["voxel_size"], cfg["point_cloud_range"])
        steps = sparse_steps(net)
        flat = [l for c, b, _ in steps for l in (c, b)]
        assert len(flat) == len(net.all_layers()) and all(a is b for a, b in zip(flat, net.all_layers()))
        assert [(c.in_channels, c.out_channels, c.subm, res) for c, _, res in steps] == SPARSE_CHAIN
        assert all(isinstance(b, sp.BatchNorm) and b.num_features == c.out_channels for c, b, _ in steps)
        for i, (c, _, _) in enumerate(steps):
            if c.subm:
                assert c.kernel_size == [3, 3, 3] and i not in STRIDED
            else:
                k, s, p, key = STRIDED[i]
                assert (tuple(c.kernel_size), tuple(c.stride), tuple(c.padding)) == (k, s, p)
                fuse = getattr(c, "fuse_subm", None)
                assert (fuse is None and key is None) or tuple(fuse) == ((3, 3, 3), key)
        # the keys of the SubM layers: each level's blocks share the map the strided conv's launch builds
        keys = [c.key for c, _, _ in steps if c.subm]
        assert keys == ["res0"] * 5 + ["res1"] * 4 + ["res2"] * 4 + ["res3"] * 4
        # every step ends in a ReLU; the residual steps are the blocks' second convs, adding the block input
        assert isinstance(net.conv_input[2], sp.ReLU) and isinstance(net.extra_conv[2], sp.ReLU)
        assert all(isinstance(d[2], sp.ReLU) for d, _ in net.stages)
        blocks = list(net.blocks0) + [b for _, bl in net.stages for b in bl]
        conv2 = {id(b.conv2) for b in blocks}
        assert all((res is not None) == (id(c) in conv2) for c, _, res in steps)
        assert net.sparse_shape == [41, 1440, 1440]
    dense = DenseRPNHead(in_channels=256)
    chain = dense_chain_convs(dense)
    allc = dense.all_convs()
    assert all(a is b for a, b in zip(chain, allc)) and len(allc) == len(chain) + 2 * 36
    assert [(c.cin, c.cout, c.k, c.stride, c.up) for c in chain] == DENSE_CHAIN
    pairs = [c for hs in dense.heads for _, a, f in hs for c in (a, f)]
    assert all(a is b for a, b in zip(allc[len(chain):], pairs))
    names = [n for n, _ in COMMON_HEADS] + ["hm"]
    assert all([n for n, _, _ in hs] == names for hs in dense.heads) and len(dense.heads) == 6
    assert all(a.cin == a.cout == 64 and a.k == 3 and f.cin == 64 and f.cout <= 3 for hs in dense.heads for _, a, f in hs)
    assert dense.bev_depth == 2 and dense.in_channels == 256


class _LevelsOnly:
    level_counters = [None] * 4


def _status_frame():
    from paddle3d_b200.pipeline import CenterPointHotPath
    p = CenterPointHotPath.__new__(CenterPointHotPath)
    p.net, p.n = _LevelsOnly(), 300000
    return p


def test_check_status_branches():
    """CenterPointHotPath.check_status on fabricated status words: zero passes; bit 0 raises the fp16-range message
    (before any level); a set overflow flag of level N names level N; with sweep input (six words) the merge's word is
    read from index 5 and raised first, and a five-word status never reads a level flag as the merge's."""
    from paddle3d_b200.ops import sweep_merge as sm
    p = _status_frame()
    p.check_status([0, 0, 0, 0, 0])
    p.check_status([0, 0, 0, 0, 0, 0])
    for st in ([1, 0, 0, 0, 0], [1, 1, 1, 1, 1], [5, 0, 0, 0, 0]):
        with pytest.raises(RuntimeError, match="left fp16's range"):
            p.check_status(st)
    for lvl in range(1, 5):
        st = [0] * 5
        st[lvl] = 1
        with pytest.raises(RuntimeError, match="strided level %d overflowed" % lvl):
            p.check_status(st)
        with pytest.raises(RuntimeError, match="strided level %d overflowed" % lvl):
            p.check_status(st + [0])
    with pytest.raises(RuntimeError, match="strided level 2 overflowed"):
        p.check_status([0, 0, 1, 1, 0])
    with pytest.raises(RuntimeError, match="point capacity"):
        p.check_status([1, 1, 0, 0, 0, sm.OVERFLOW])
    with pytest.raises(RuntimeError, match="descriptor entry"):
        p.check_status([0, 0, 0, 0, 0, sm.BAD_ENTRY | sm.OVERFLOW])
    with pytest.raises(RuntimeError, match="strided level 4 overflowed"):
        p.check_status([0, 0, 0, 0, sm.OVERFLOW])


def test_strided_sites_reference():
    """The numpy candidate set against oracle.sparse_conv3d's output sites on a small grid, for the four strided
    geometries of the model (odd sides, so the last output row sees fewer taps)."""
    import oracle
    rng = np.random.default_rng(3)
    spatial = (9, 13, 11)
    occ = rng.random(spatial) < 0.15
    coords = np.concatenate([np.zeros((int(occ.sum()), 1), np.int64), np.argwhere(occ)], 1).astype(np.int32)
    feats = rng.normal(size=(len(coords), 1)).astype(np.float32)
    for k, s, p, _ in STRIDED.values():
        w = np.ones(k + (1, 1), np.float32)
        oc, _, osp, _ = oracle.sparse_conv3d(coords, feats, 1, spatial, w, s, p, False)
        want, mine = strided_sites(coords, spatial, k, s, p)
        assert list(mine) == list(osp)
        assert np.array_equal(want, oc[np.argsort(_site_keys(oc, osp))])


# -------------------------------------------------------------------------------------------------------- GPU tests
def _bench_frame(cuda, cfg, **kw):
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointHotPath
    kw = dict(dict(precision=sp.F16X3, with_head=True, keep_bev=False, bn_gain=bench.BN_GAIN), **kw)
    return CenterPointHotPath(cfg, cuda, **kw)


def _run_chains(hot, pts_d):
    """frame_chain once eagerly and once captured (and replayed) on the default stream."""
    import torch
    eager = frame_chain(hot, pts_d)
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = frame_chain(hot, pts_d)
    graph.replay()
    torch.cuda.synchronize()
    return eager, captured, graph


@pytest.mark.gpu
@pytest.mark.parametrize("geom", GEOMS, ids=[g[0] for g in GEOMS])
def test_full_size_frame_stage_by_stage(cuda, oracle_mod, geom, monkeypatch):
    """The bench frame on lidar_cloud(cfg, 0), restated (frame_chain) eagerly and captured: every stage from its actual
    input buffer against its reference, the exact level counts of GEOMS, status 0; then without the row-order
    dependent decompositions (NARROW_WM off, at most 3 splits) the eager
    chain, the captured chain and CenterPointHotPath's captured frame bit-equal in the pixel image and the boxes (the
    two chains also in the head planes), with the same level counts as the default mode."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    name, cfg, n_vox, n_levels = geom
    pts = synth.lidar_cloud(cfg, 0)
    pts_d = torch.from_numpy(pts).to(cuda)
    pin = torch.from_numpy(pts).pin_memory()
    hot = _bench_frame(cuda, cfg)
    hot.calibrate_head(pts_d)
    hot.points.copy_(pts_d)
    hot.capture()
    hot.infer(pin)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    assert not hot.h_status.any()

    # ---- default mode (the one bench.py times): the float64 checks
    eager, captured, graph = _run_chains(hot, pts_d)
    assert not eager["status"].any() and not captured["status"].any()
    sites = level_sites(hot.net, eager)
    assert [int(c[0]) for c, _ in sites] == n_levels
    for which, other in (("captured chain", level_sites(hot.net, captured)),
                         ("CenterPointHotPath", [(c.cpu().numpy(), None) for c in hot.net.level_counters])):
        for (a, ka), (b, kb) in zip(sites, other):
            assert np.array_equal(a[:3], b[:3]), "%s: level counters %s != %s" % (which, b[:3], a[:3])
            assert kb is None or np.array_equal(ka, kb), "%s: a level's site set differs" % which
    del captured, graph
    assert check_voxelize(name, oracle_mod, eager, pts, cfg) == n_vox
    assert check_rulebooks(name, hot.net, eager) == n_levels
    print("LEVELS %s: %d voxels, strided levels %s of capacities %s" % (
        name, n_vox, n_levels, [c.out_cap for c in (d[0] for d, _ in hot.net.stages)] + [hot.net.extra_conv[0].out_cap]))
    check_sparse_convs(name, hot.net, eager, sms)
    empty = check_pixel_image(name, hot.net, eager)
    assert empty > 0.8, "%s: only %.1f %% of the BEV pixels are empty" % (name, 100 * empty)
    check_dense(name, hot, eager, sms)
    passing, per_task = check_postprocess(name, oracle_mod, hot, eager)
    tc = hot.test_cfg
    print("POST %s: %.1f %% of the BEV pixels empty; cells above the score threshold per task %s (nms_pre %d); boxes "
          "per task %s (nms_post %d)" % (name, 100 * empty, passing, tc["nms_pre_max_size"], per_task,
                                         tc["nms_post_max_size"]))
    # the calibration puts 1.4 % of each task's cells above the threshold (454 of 180 x 180), fewer than nms_pre: the
    # frame never takes the nms_pre cut (test_gpu_boxes' hm_mean -4.0 case does), and every task takes the nms_post cut
    cells = eager["head_shape"][1] * eager["head_shape"][2]
    assert all(0.01 * cells < p < 0.02 * cells for p in passing) and max(passing) < tc["nms_pre_max_size"], passing
    assert per_task == [tc["nms_post_max_size"]] * len(per_task), per_task
    del eager
    torch.cuda.empty_cache()

    # ---- no decomposition that follows the row order: the three runs of the frame bit-equal
    monkeypatch.setattr(sp, "NARROW_WM", [False])
    monkeypatch.setattr(sp, "F16_MAX_SPLITS", 3)
    hot.capture()
    want = [t.clone() for t in hot.infer(pin)]
    assert not hot.h_status.any()
    hot_bev = hot.out["bev_h16"][0].clone()
    eager, captured, graph = _run_chains(hot, pts_d)
    assert [int(c[0]) for c, _ in level_sites(hot.net, eager)] == n_levels
    for label, r in (("eager", eager), ("captured", captured)):
        assert not r["status"].any()
        assert _bits_equal(r["bev"], hot_bev), "%s chain: BEV pixel image differs from CenterPointHotPath's" % label
        assert _bits_equal(r["planes"], eager["planes"]), "%s chain: head planes differ from the eager chain's" % label
        boxes, scores, labels, counts = r["post"]
        k = int(counts[-1])
        assert k == len(want[2]), "%s chain: box count" % label
        assert _bits_equal(boxes[:k].cpu(), want[0]) and _bits_equal(scores[:k].cpu(), want[1])
        assert torch.equal(labels[:k].cpu(), want[2])
    check_pixel_image(name + " row-order independent", hot.net, eager)


@pytest.mark.gpu
def test_full_size_uniform_cloud_at_capacity(cuda, oracle_mod):
    """A 300 k-point uniform_cloud on C3: the voxelizer keeps the first 160 000 of 266 007 occupied cells.  Default caps:
    level 1 holds 480 000 of its 525 805 sites (overflow flagged, kept sites a subset of the exact set with correct taps)
    and infer() raises the level-1 error.  Caps [4V, 4V, 2V, V]: status 0, every level exact (level 2: 635 490 of
    640 000 rows), every sparse conv on the float64 bar and the pixel image bit-exact."""
    import torch
    pts = synth.uniform_cloud(synth.C3, 0)
    pts_d = torch.from_numpy(pts).to(cuda)
    hot = _bench_frame(cuda, synth.C3)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    r = sparse_frame(hot, pts_d)
    torch.cuda.synchronize()
    assert check_voxelize("uniform", oracle_mod, r, pts, synth.C3) == V
    lo, vs = np.asarray(synth.C3["point_cloud_range"][:3], np.float32), np.asarray(synth.C3["voxel_size"], np.float32)
    ijk = np.floor((pts[:, :3] - lo) / vs).astype(np.int64)
    grid = np.round((np.asarray(synth.C3["point_cloud_range"][3:], np.float32) - lo) / vs).astype(np.int64)
    assert len(np.unique(ijk[((ijk >= 0) & (ijk < grid)).all(1)], axis=0)) == UNIFORM_CELLS
    cnt = strided_levels(hot.net, r["outs"])[0].counters.cpu().numpy()
    assert list(cnt[:3]) == [3 * V, 1, UNIFORM_LEVELS[0]], cnt
    assert int(r["status"][1]) == 1
    assert check_rulebooks("uniform default caps", hot.net, r, levels=1, caps_hold=False) == UNIFORM_LEVELS[:1]
    del r
    with pytest.raises(RuntimeError, match="strided level 1 overflowed its row capacity"):
        hot.infer(torch.from_numpy(pts).pin_memory())
    torch.cuda.empty_cache()

    hot.net.set_level_caps(WIDE_CAPS)
    r = sparse_frame(hot, pts_d)
    torch.cuda.synchronize()
    assert not r["status"].any()
    assert check_rulebooks("uniform wide caps", hot.net, r) == UNIFORM_LEVELS
    ix = strided_levels(hot.net, r["outs"])
    assert [x.cap for x in ix] == WIDE_CAPS and WIDE_CAPS[1] - int(ix[1].counters[0]) == 4510
    print("LEVELS uniform: %d of %d occupied cells kept, strided levels %s of capacities %s" % (
        V, UNIFORM_CELLS, UNIFORM_LEVELS, WIDE_CAPS))
    check_sparse_convs("uniform", hot.net, r, sms)
    empty = check_pixel_image("uniform", hot.net, r)
    print("POST uniform: %.1f %% of the BEV pixels empty" % (100 * empty))


@pytest.mark.gpu
def test_fp16_range_raises(cuda):
    """The bench cloud with BatchNorm gain 6: on the fp16-pair path the backbone saturates (status bit 0) and infer()
    raises the fp16-range error; the same frame at TF32X3_SPLIT runs with status 0 and a BEV far past 65504."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    pts = torch.from_numpy(synth.lidar_cloud(synth.C3, 0)).pin_memory()
    f16 = _bench_frame(cuda, synth.C3, with_head=False, bn_gain=FP16_GAIN)
    with pytest.raises(RuntimeError, match="left fp16's range"):
        f16.infer(pts)
    assert int(f16.h_status[0]) & 1 and not f16.h_status[1:].any()
    del f16
    sp.status_tensor(cuda).zero_()  # the device's word is sticky: it would carry the overflow into the next frame
    tf = _bench_frame(cuda, synth.C3, precision=sp.TF32X3_SPLIT, with_head=False, bn_gain=FP16_GAIN)
    boxes, _, labels = tf.infer(pts)
    assert not tf.h_status.any() and len(labels) >= 6
    top = float(tf.out["bev"].abs().max())
    assert 65504 < top < 1e30, top
    print("FP16 gain %.1f: BEV max |x| %.3e at TF32X3_SPLIT" % (FP16_GAIN, top))
    sp.status_tensor(cuda).zero_()


@pytest.mark.gpu
def test_sweep_lanes_full_size(cuda, monkeypatch):
    """CenterPointSweep with bench.py's four lanes, infer_many over six distinct full-size clouds of bench.frame_pool
    (twice, so both staging sets of each lane are reused), NARROW_WM off and at most 3 splits (see the module
    docstring): every frame bit-equal to the single-lane captured frame on the same cloud."""
    import torch
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.pipeline import CenterPointSweep
    monkeypatch.setattr(sp, "NARROW_WM", [False])
    monkeypatch.setattr(sp, "F16_MAX_SPLITS", 3)
    cfg = synth.C3
    frames = bench.frame_pool(cfg, 6)
    pinned = [torch.from_numpy(f).pin_memory() for f in frames]
    dev0 = torch.from_numpy(frames[0]).to(cuda)
    sweep = CenterPointSweep(4, cfg=cfg, device=cuda, precision=sp.F16X3, seed=0, with_head=True, keep_bev=False,
                             bn_gain=bench.BN_GAIN)
    sweep.calibrate_head(dev0)
    sweep.capture(dev0)
    single = _bench_frame(cuda, cfg)
    single.share_model(sweep.lanes[0])
    single.points.copy_(dev0)
    single.capture()
    want = [[t.clone() for t in single.infer(f)] for f in pinned]
    assert len({len(w[2]) for w in want}) > 1 or len({float(w[0].sum()) for w in want}) == len(want)
    for rnd in range(2):
        got = list(sweep.infer_many(iter(pinned)))
        assert len(got) == len(want)
        for i, (g, w) in enumerate(zip(got, want)):
            assert len(g[2]) == len(w[2]), "round %d frame %d: box count" % (rnd, i)
            assert _bits_equal(g[0], w[0]) and _bits_equal(g[1], w[1]) and torch.equal(g[2], w[2]), \
                "round %d frame %d differs from the single-lane frame" % (rnd, i)
    print("LANES 4 lanes, %d frames x 2 rounds: boxes per frame %s" % (len(want), [len(w[2]) for w in want]))
