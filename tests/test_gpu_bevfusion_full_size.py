"""BEVFusion (bevf_pp) at full size: every dense conv of the frame in every work decomposition, the 640-channel fusion
image as the frame builds it, HardVFE on a full-size cloud, and the frame's launch chain stage by stage, against a
float64 reference.

The dense convs run at B = 1 with the frame's channel offset and output width (BEVFUSION_LAYERS, tied to
bevfusion.BEVFusion's convs by a CPU test), through the C ABI in the decompositions of
test_gpu_dense_residual.decomposition_runs, on the bar of test_gpu_dense_schedule.bar; every case shows that the bar
rejects the hi x hi products alone and the result without one tap (1x1 and transposed convs: one 32-channel input group).
The camera encoder's first two convs sum 9216 terms per output and reduc_conv 5760, the longest reductions of the
project.  Lines starting with "REGIME" (pytest -s) give each launch's decomposition, lines starting with "BAR" the error
figures that test_gpu_dense_schedule.bar quotes, and "MEM" the peak device memory of each test.

The camera view transform at bevf_pp's geometry is a GEOMETRIES entry of test_gpu_camera_pool.py."""
import numpy as np
import pytest

import bevfusion_oracle as bo
from test_gpu_dense_residual import decomposition_runs, error_stats
from test_gpu_dense_schedule import (DenseCase, Plan, _bits_equal, _n_tile, _sms, assert_untouched, check_images,
                                     check_rejects, conv_ref, epilogue, from_pixel_h16, run_dense,
                                     sentinel_image)
from test_gpu_dense_tma_store import run_pairs

# The distinct conv shapes of BEVFusion(CONFIG) (one of each run of repeated trunk convs): (name, H, W in, cin, cout, k,
# stride, pad, up, relu, bias_only, c0, out_C).  c0 / out_C: where the frame writes the output (out_C 0: fp32 planes
# only, the head's 294 channels are no multiple of 16).  The camera encoder's last conv and the three SECONDFPN deblocks
# write channels [0, 256), [256, 384), [384, 512) and [512, 640) of the fusion image.
FUSE_C = 640
BEVFUSION_LAYERS = [
    ("cam conv1 1024->1024", 200, 200, 1024, 1024, 3, 1, 1, 1, True, False, 0, 1024),
    ("cam conv2 1024->512", 200, 200, 1024, 512, 3, 1, 1, 1, True, False, 0, 512),
    ("cam conv3 512->256", 200, 200, 512, 256, 3, 1, 1, 1, True, False, 0, FUSE_C),
    ("trunk b1 first 64->64 s2", 400, 400, 64, 64, 3, 2, 1, 1, True, False, 0, 64),
    ("trunk b1 64->64", 200, 200, 64, 64, 3, 1, 1, 1, True, False, 0, 64),
    ("trunk b2 first 64->128 s2", 200, 200, 64, 128, 3, 2, 1, 1, True, False, 0, 128),
    ("trunk b2 128->128", 100, 100, 128, 128, 3, 1, 1, 1, True, False, 0, 128),
    ("trunk b3 first 128->256 s2", 100, 100, 128, 256, 3, 2, 1, 1, True, False, 0, 256),
    ("trunk b3 256->256", 50, 50, 256, 256, 3, 1, 1, 1, True, False, 0, 256),
    ("fpn 1x1 64->128", 200, 200, 64, 128, 1, 1, 0, 1, True, False, 256, FUSE_C),
    ("fpn up2 128->128", 100, 100, 128, 128, 2, 2, 0, 2, True, False, 384, FUSE_C),
    ("fpn up4 256->128", 50, 50, 256, 128, 4, 4, 0, 4, True, False, 512, FUSE_C),
    ("reduc_conv 640->384", 200, 200, 640, 384, 3, 1, 1, 1, True, False, 0, 384),
    ("head 384->294 bias", 200, 200, 384, 294, 1, 1, 0, 1, False, True, 0, 0),
]
# the automatic plan's work items at 132 SMs (DESIGN's layer table)
ITEMS_132 = [2600, 1300, 650, 325, 325, 91, 91, 56, 56, 325, 364, 448, 975, 975]


def model_layers(m):
    """(H, W in, cin, cout, k, stride, pad, up, relu, bias_only, c0, out_C) of every dense conv of a BEVFusion, in launch
    order, from its convs, its pillar grid and its BEV size."""
    Y, X = m.bev_hw
    seen = []

    def row(cv, h, w, c0, out_C):
        seen.append(cv)
        bias_only = cv.has_bias and cv.bn_eps is None
        return (h, w, cv.cin, cv.cout, cv.k, cv.stride, cv.padding, cv.up, cv.relu, bias_only, c0, out_C)
    out = [row(cv, Y, X, 0, cv.cout) for cv in m.cam_convs[:-1]] + [row(m.cam_convs[-1], Y, X, 0, m.fuse_C)]
    h, w = m.grid[1], m.grid[0]
    sizes = []
    for blk in m.trunk.blocks:
        for cv in blk:
            out.append(row(cv, h, w, 0, cv.cout))
            h, w = (h + 2 * cv.padding - cv.k) // cv.stride + 1, (w + 2 * cv.padding - cv.k) // cv.stride + 1
        sizes.append((h, w))
    c0 = m.cam_C
    for (h, w), de in zip(sizes, m.trunk.deblocks):
        assert m.trunk.deblock_out_hw(de, h, w) == (Y, X)
        out.append(row(de, h, w, c0, m.fuse_C))
        c0 += de.cout
    out.append(row(m.reduc, Y, X, 0, m.reduc.cout))
    out.append(row(m.head, Y, X, 0, 0 if m.head.cout % 16 else m.head.cout))
    # the rows are the model's convs() one for one, in its order: a conv the walk above misses (or adds) shows here
    convs = m.convs()
    order = m.cam_convs + [cv for blk in m.trunk.blocks for cv in blk] + list(m.trunk.deblocks) + [m.reduc, m.head]
    assert len(seen) == len(convs) and all(a is b for a, b in zip(seen, order))
    assert sorted(map(id, seen)) == sorted(map(id, convs))
    return out


def _terms(cin, k, up):
    return cin if up > 1 else cin * k * k


@pytest.fixture(autouse=True)
def _peak_memory():
    """Print each GPU test's peak device memory ("MEM" lines)."""
    import torch
    gpu = torch.cuda.is_available()
    if gpu:
        torch.cuda.reset_peak_memory_stats()
    yield
    if gpu:
        print("MEM peak device memory %.2f GiB" % (torch.cuda.max_memory_allocated() / 2 ** 30))


# -------------------------------------------------------------------------------------------------------- CPU tests
def test_layer_table_matches_the_model():
    """BEVFUSION_LAYERS is the set of BEVFusion(CONFIG)'s conv shapes (a CONFIG change shows here before the GPU tests
    check stale shapes), with the frame's N tiles, the sum lengths and the automatic plan's work items at 132 SMs."""
    from paddle3d_b200 import bevfusion as bf
    m = bf.BEVFusion(device="cpu")
    derived = model_layers(m)
    table = [l[1:] for l in BEVFUSION_LAYERS]
    assert len(derived) == len(m.convs()) == 24
    assert sorted(set(derived), key=derived.index) == table
    assert [cv.n_tile for cv in m.convs()] == [_n_tile(cv.cout) for cv in m.convs()]
    assert max(_terms(l[3], l[5], l[8]) for l in BEVFUSION_LAYERS) == 9216
    assert [_terms(l[3], l[5], l[8]) for l in BEVFUSION_LAYERS if l[0].startswith(("cam", "reduc"))] == [
        9216, 9216, 4608, 5760]
    plans = [Plan(132, 1, H, W, cin, cout, _n_tile(cout), k, s, p, up)
             for _, H, W, cin, cout, k, s, p, up, _, _, _, _ in BEVFUSION_LAYERS]
    assert [p.items for p in plans] == ITEMS_132
    assert [(p.out_H, p.out_W) for p in plans] == [(200, 200), (200, 200), (200, 200), (200, 200), (200, 200),
                                                   (100, 100), (100, 100), (50, 50), (50, 50), (200, 200), (200, 200),
                                                   (200, 200), (200, 200), (200, 200)]
    assert plans[0].inst == (128, 1, True) and plans[-1].inst == (128, 1, False)
    assert 294 - (plans[-1].n_nt - 1) * 128 == 38
    # the fusion image: the four launches that write it own its 640 channels exactly once
    writers = [l for l in BEVFUSION_LAYERS if l[12] == FUSE_C]
    assert [(l[11], l[11] + l[4]) for l in writers] == [(0, 256), (256, 384), (384, 512), (512, 640)]
    assert FUSE_C == m.fuse_C and m.reduc.cin == FUSE_C


# -------------------------------------------------------------------------------------------------------- GPU tests
def _case(cuda, layer):
    name, H, W, cin, cout, k, stride, pad, up, relu, bias_only, c0, out_C = layer
    return DenseCase(cuda, 1, H, W, cin, cout, k, stride, pad, up, seed=cin * 7 + cout + H + up, relu=relu,
                     bias_only=bias_only)


def _plane_guard(case, n_tile, mode, m_tiles, planes):
    """The launch again into a NaN-filled plane buffer one N tile longer than the layer: channels [0, cout) the bits of
    `planes`, nothing written past channel cout - 1 (the last N tile is partly used)."""
    import torch
    from paddle3d_b200._lib import check, lib
    from paddle3d_b200._mem import ptr, stream
    assert case.up == 1, "the launch below passes the conv geometry of a convolution"
    p = case.plan(_sms(), n_tile, mode, m_tiles)
    hw = p.out_H * p.out_W
    buf = torch.full(((p.n_nt + 1) * n_tile * hw,), float("nan"), device=case.dev)
    st = torch.zeros((1,), dtype=torch.int32, device=case.dev)
    check(lib().p3d_dense_conv2d_f16(ptr(case.xh), 1, case.H, case.W, case.cin, ptr(case.packed(n_tile)), case.cout,
                                     n_tile, case.k, case.k, case.stride, case.pad, case.up, ptr(case.scale),
                                     ptr(case.shift), int(case.relu), ptr(None), 0, 0, ptr(buf), mode, m_tiles, ptr(st),
                                     stream(case.dev)), "dense_conv2d_f16")
    torch.cuda.synchronize()
    assert int(st[0]) == 0
    assert bool(torch.isnan(buf[case.cout * hw:]).all()), "planes past channel %d were written" % (case.cout - 1)
    assert _bits_equal(buf[:case.cout * hw], planes.reshape(-1)), "a plane buffer with room past cout gives other bits"


@pytest.mark.gpu
@pytest.mark.parametrize("layer", BEVFUSION_LAYERS, ids=lambda l: l[0].replace(" ", "_").replace(">", ""))
def test_bevfusion_layer_every_decomposition(cuda, layer):
    """Each distinct conv of the frame at full size, written where the frame writes it: the frame's N tile with the MT
    rule's choice, N = 64 with both M tilings (Cout >= 128; else the other M tiling), and for the 3x3 stride-1 layers
    the forced per-tap loads.  Every run: fp32 planes and the fp16-pair image against fp64, sentinels and guard pixels
    untouched, a second launch the same bits, the H16-only launch bit-equal to the launch with planes; the head (planes
    only) writes no plane past its 294 channels."""
    import torch
    name, H, W, cin, cout, k, stride, pad, up, relu, bias_only, c0, out_C = layer
    case = _case(cuda, layer)
    h16 = out_C > 0
    runs = decomposition_runs(case)
    want = case.want()
    for n, mode, mt in runs:  # every run's figures first, so that a run off the bar does not hide the others'
        pl, _ = case.launch(n, mode, mt)
        print("BAR bevfusion %s N%d mode%d MT%d, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, "
              "relative %.2e above" % ((name, n, mode, mt, case.terms) + error_stats(pl.permute(0, 2, 3, 1), want)))
        del pl
    del want
    for i, (n, mode, mt) in enumerate(runs):
        label = "bevfusion %s N%d mode%d MT%d" % (name, n, mode, mt)
        p, _, pl = run_dense(label, case, n, mode, mt, c0=c0, h16=h16, guards=i == 0, out_C=out_C)
        if h16:
            run_pairs(label + " H16-only", case, n, mode, mt, c0=c0, reference=False, out_C=out_C)
        else:
            _plane_guard(case, n, mode, mt, pl)
        assert p.inst[0] == n and (mt == 0 or p.inst[1] == mt)
        assert p.halo == (mode == 0 and up == 1 and k == 3 and stride == 1)
        print("REGIME bevfusion %s: %s" % (label, p.describe()))
        del pl
    del case
    torch.cuda.empty_cache()


@pytest.mark.gpu
def test_fusion_image_and_reduc_conv(cuda):
    """The camera encoder's last conv and the three deblocks launched back to back into one sentinel-filled 640-channel
    image at c0 = 0, 256, 384, 512, each from its own seeded input: every channel range against its own fp64 reference,
    the guard pixels untouched, a second round the same bits.  Then reduc_conv (3x3, 640 -> 384, 5760 terms) on the
    image that was written, against fp64 from that image, in every decomposition."""
    import torch
    writers = [l for l in BEVFUSION_LAYERS if l[12] == FUSE_C]
    cases = [_case(cuda, l) for l in writers]
    n_px = 200 * 200

    def round_():
        img = sentinel_image(n_px, FUSE_C, cuda)
        st = torch.zeros((1,), dtype=torch.int32, device=cuda)
        planes = [c.launch(_n_tile(c.cout), 0, 0, img, FUSE_C, l[11], status=st)[0] for c, l in zip(cases, writers)]
        torch.cuda.synchronize()
        return img, planes, int(st[0])

    img, planes, st = round_()
    assert st == 0
    assert_untouched("fusion image", img, n_px, torch.ones(2 * FUSE_C, dtype=torch.bool))
    for c, l, pl in zip(cases, writers, planes):
        name = "fusion image %s at c0 %d" % (l[0], l[11])
        p = c.plan(_sms(), _n_tile(c.cout))
        assert (p.out_H, p.out_W) == (200, 200)
        want = c.want()
        check_images(name + " fp32 planes", pl.permute(0, 2, 3, 1), want, c.terms)
        got = from_pixel_h16(img, 1, 200, 200, FUSE_C)[..., l[11]:l[11] + c.cout]
        check_images(name + " fp16-pair image", got, want, c.terms)
        check_rejects(name, c.wrongs(), want, c.terms)
        print("REGIME %s: %s" % (name, p.describe()))
        del want, got
    img2, planes2, _ = round_()
    assert _bits_equal(img, img2) and all(_bits_equal(a, b) for a, b in zip(planes, planes2)), \
        "a second round gives other bits"
    del cases, planes, planes2, img2
    reduc = [l for l in BEVFUSION_LAYERS if l[0].startswith("reduc")][0]
    rc = _case(cuda, reduc)
    rc.xh = img[:n_px]
    rc.x64 = from_pixel_h16(rc.xh, 1, 200, 200, FUSE_C)
    assert bool((rc.x64 >= 0).all()) and float(rc.x64.amax()) > 0  # ReLU outputs of all four writers
    for i, (n, mode, mt) in enumerate(decomposition_runs(rc)):
        label = "bevfusion reduc_conv on the fusion image N%d mode%d MT%d" % (n, mode, mt)
        p, _, pl = run_dense(label, rc, n, mode, mt, c0=0, guards=i == 0, out_C=reduc[12])
        print("REGIME %s: %s" % (label, p.describe()))
        print("BAR %s, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
              % ((label, rc.terms) + error_stats(pl.permute(0, 2, 3, 1), rc.want())))
    torch.cuda.empty_cache()


def _vfe_layers(rng, Fd, mid, out):
    layers = []
    for cin, cout in ((Fd + 6, mid), (2 * mid, out)):
        layers.append(dict(weight=rng.normal(0, 0.3, (cin, cout)).astype(np.float32),
                           gamma=rng.uniform(0.5, 1.5, cout).astype(np.float32),
                           beta=rng.normal(0, 0.5, cout).astype(np.float32),
                           mean=rng.normal(0, 0.1, cout).astype(np.float32),
                           var=rng.uniform(0.5, 1.5, cout).astype(np.float32), eps=1e-3))
    return layers


def _hard_vfe_ref(voxels, npv, coors, layers, vs, pcr, chunk=4096):
    """bevfusion_oracle.hard_vfe_ref over chunks of voxels (its fp64 intermediates of 40 000 voxels would take GBs)."""
    return np.concatenate([bo.hard_vfe_ref(voxels[i:i + chunk], npv[i:i + chunk], coors[i:i + chunk], layers, vs, pcr)
                           for i in range(0, len(npv), chunk)], 0)


@pytest.mark.gpu
def test_hard_vfe_full_size_cloud(cuda):
    """p3d_hard_vfe on the device's own voxels of a 300 k-point cloud at bevf_pp's voxel size (max_voxels 40 000, 64
    points per voxel): every voxel against the fp64 HardVFE at 1e-4, rows past the device count untouched."""
    import torch
    from paddle3d_b200 import bevfusion as bf
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import voxelize as vox
    c = bf.CONFIG
    vs, pcr, M, V = c["voxel_size"], c["point_cloud_range"], c["max_points"], c["max_voxels"]
    cloud = dict(num_points=300000, point_dim=4, point_cloud_range=list(pcr))
    pts = torch.from_numpy(synth.lidar_cloud(cloud, 41, 300000).astype(np.float32)).to(cuda)
    voxels, co, npv, nv = vox.hard_voxelize(pts, vs, pcr, M, V)
    coors = torch.nn.functional.pad(co, (1, 0))
    layers = _vfe_layers(np.random.default_rng(42), 4, *c["vfe"]["feat_channels"])
    lay = [dict(l, weight=torch.from_numpy(l["weight"]).to(cuda)) for l in layers]
    folded = [pe.fold_bn(l["gamma"], l["beta"], l["mean"], l["var"], l["eps"], cuda) for l in layers]
    out = torch.full((V, c["vfe"]["feat_channels"][1]), float("nan"), device=cuda)
    got = pe.hard_vfe(voxels, npv, coors, lay, vs, pcr, num_voxels=nv, folded=folded, out=out)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    k = int(nv[0])
    cnt = npv[:k].cpu().numpy()
    assert 1000 < k <= V and cnt.max() == M and cnt.min() >= 1, (k, cnt.min(), cnt.max())
    g = got.cpu().numpy()
    assert np.isnan(g[k:]).all(), "rows past the device count were written"
    want = _hard_vfe_ref(voxels[:k].cpu().numpy(), cnt, coors[:k].cpu().numpy(), layers, vs, pcr)
    np.testing.assert_allclose(g[:k], want, rtol=1e-4, atol=1e-4)
    print("HardVFE full-size cloud: %d voxels, %d with all %d points" % (k, int((cnt == M).sum()), M))


# ------------------------------------------------------------------------------------------------ the full-size frame
@pytest.mark.gpu
def test_full_size_frame_stage_by_stage(cuda, oracle_mod):
    """A seeded BEVFusion(CONFIG) with calibrated class biases on a 300 k-point cloud and random depth-net outputs.  The
    frame's launch chain is restated on one stream with no sync in between, keeping every buffer: the LiDAR branch, the
    camera pool, the three encoder convs, reduc_conv, the SE gate, the head and the decode; once eagerly and once
    captured.  Both are bit-equal to BEVFusionHotPath's captured frame (whose two branches write the fusion image
    concurrently) in the fused image, the SE output, the planes and the decode, with status 0; every conv is on the fp64
    bar from its actual input buffer, HardVFE on the fp64 restatement, the gate within 1e-5 of se_gate_ref, the scaled
    image bit-equal to se_scale_ref, and the decode's order, labels and counts those of anchor3d_decode_ref of the
    actual planes, with both the nms_pre and the max_num cut taken."""
    import torch
    from paddle3d_b200 import bevfusion as bf
    from paddle3d_b200.ops import bev_pool_v2 as bp
    from paddle3d_b200.ops import pillar_encoder as pe
    from paddle3d_b200.ops import sparse_nn as sp
    from paddle3d_b200.ops import voxelize as vox
    from paddle3d_b200.ops.se_gate import se_gate_h16
    from test_gpu_bevfusion import _compare, _frame_inputs, _t
    m = bf.BEVFusion(device=cuda).init_weight(seed=5)
    c = m.cfg
    pts, mats, logits, tran = _frame_inputs(m, 9, n=300000)
    pts_d, tl, tt = _t(cuda, pts), _t(cuda, logits), _t(cuda, tran)
    m.calibrate_cls_bias(pts_d, mats, tl, tt)
    hot = bf.BEVFusionHotPath(m, num_points=300000, device=cuda).capture()
    hot_res = [t.clone() for t in hot.infer(pts, mats, tl, tt)]
    hot_status = int(hot.out["status"].reshape(-1)[0])
    hot_bufs = dict(fused=hot.fused.clone(), se=hot.out["se"].clone(), planes=hot.out["planes"].clone())
    desc = m.vt.descriptor(*mats)
    Y, X = m.bev_hw
    fc = c["fusion_channels"]
    status = sp.status_tensor(cuda)

    def chain():
        r = dict(convs=[])  # convs: (conv, input image, its shape, output image, out_C, c0)
        convs = r["convs"]
        fused = r["fused"] = m.fused_image()
        voxels, co, npv, nv = vox.hard_voxelize(pts_d, c["voxel_size"], c["point_cloud_range"], c["max_points"],
                                                c["max_voxels"])
        coors = torch.nn.functional.pad(co, (1, 0))
        vfe = pe.hard_vfe(voxels, npv, coors, m.vfe_dev, c["voxel_size"], c["point_cloud_range"], num_voxels=nv,
                          folded=m.vfe_folded)
        r.update(voxels=voxels, npv=npv, coors=coors, nv=nv, vfe=vfe)
        nx, ny = m.grid
        x, sh = sp.sparse_coo_tensor(coors, vfe, [1, 1, ny, nx, m.vfe_C[1]], num=nv).to_pixel_h16()
        feats = []
        for blk in m.trunk.blocks:
            for conv in blk:
                y, _, (b, oh, ow) = conv(x, sh)
                convs.append((conv, x, sh, y, conv.cout, 0))
                x, sh = y, (b, oh, ow, conv.cout)
            feats.append((x, sh))
        c0 = m.cam_C
        for (f, fs), de in zip(feats, m.trunk.deblocks):
            de(f, fs, out_split=fused, out_channels=m.fuse_C, out_c0=c0)
            convs.append((de, f, fs, fused, m.fuse_C, c0))
            c0 += de.cout
        prepared = m.vt._prepare(desc, 1, m.N)
        depth, feat = bp.lss_depth_feat(tl, tt)
        x = r["pool"] = m.pool(depth, feat, prepared)
        sh = (1, Y, X, m.pool_C)
        for cv in m.cam_convs[:-1]:
            y, _, _ = cv(x, sh)
            convs.append((cv, x, sh, y, cv.cout, 0))
            x, sh = y, (1, Y, X, cv.cout)
        m.cam_convs[-1](x, sh, out_h16=fused, out_channels=m.fuse_C, out_c0=0)
        convs.append((m.cam_convs[-1], x, sh, fused, m.fuse_C, 0))
        se, _, _ = m.reduc(fused, (1, Y, X, m.fuse_C))
        r["reduc"] = se.clone()
        convs.append((m.reduc, fused, (1, Y, X, m.fuse_C), r["reduc"], fc, 0))
        r["gate"] = torch.empty((1, fc), dtype=torch.float32, device=cuda)
        se_gate_h16(se, (1, Y, X, fc), m.se_dev["weight"], m.se_dev["bias"], gate=r["gate"])
        _, planes, _ = m.head(se, (1, Y, X, fc), want_nchw=True)
        r.update(se=se, planes=planes, decode=m.postprocess(planes))
        return r

    status.zero_()
    eager = chain()
    torch.cuda.synchronize()
    assert int(status[0]) == 0 and hot_status == 0
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        captured = chain()
    graph.replay()
    torch.cuda.synchronize()
    assert int(status[0]) == 0
    k = int(hot.out["counts"].reshape(-1)[0])
    for label, r in (("eager", eager), ("captured", captured)):
        for key in ("fused", "se", "planes"):
            assert _bits_equal(r[key], hot_bufs[key]), "%s chain: %s differs from BEVFusionHotPath's" % (label, key)
        boxes, scores, labels, counts = r["decode"]
        assert int(counts.reshape(-1)[0]) == k, "%s chain: decode count" % label
        assert _bits_equal(boxes[:k].cpu(), hot_res[0]) and _bits_equal(scores[:k].cpu(), hot_res[1])
        assert np.array_equal(labels[:k].cpu().numpy(), hot_res[2].numpy()), "%s chain: decode labels" % label
        for i, (a, b) in enumerate(zip(eager["convs"], r["convs"])):
            assert _bits_equal(a[3], b[3]), "conv %d: the %s chain differs from the eager one" % (i, label)
    del captured, graph
    torch.cuda.empty_cache()
    r = eager
    # HardVFE on the device's own voxels
    nv = int(r["nv"][0])
    cnt = r["npv"][:nv].cpu().numpy()
    assert nv > 1000
    want = _hard_vfe_ref(r["voxels"][:nv].cpu().numpy(), cnt, r["coors"][:nv].cpu().numpy(), m.vfe,
                         c["voxel_size"], c["point_cloud_range"])
    np.testing.assert_allclose(r["vfe"][:nv].cpu().numpy(), want, rtol=1e-4, atol=1e-4)
    del want
    # every conv from its actual input buffer
    sms = _sms()
    for i, (conv, x, sh, y, out_C, c0) in enumerate(r["convs"]):
        b, h, w, cin = sh
        x64 = from_pixel_h16(x, b, h, w, cin)
        acc, _ = conv_ref(x64, torch.from_numpy(conv.np["weight"]).to(cuda).double(), conv.k, conv.stride,
                          conv.padding, conv.up)
        del x64
        want = epilogue(acc, conv.dev["scale"], conv.dev["shift"], conv.relu)
        del acc
        oh, ow = want.shape[1:3]
        got = from_pixel_h16(y, b, oh, ow, out_C)[..., c0:c0 + conv.cout]
        terms = _terms(cin, conv.k, conv.up)
        name = "frame conv %d %d->%d k%d s%d up%d at c0 %d" % (i, cin, conv.cout, conv.k, conv.stride, conv.up, c0)
        check_images(name, got, want, terms)
        p = Plan(sms, b, h, w, cin, conv.cout, conv.n_tile, conv.k, conv.stride, conv.padding, conv.up)
        print("REGIME %s: %s" % (name, p.describe()))
        print("BAR %s, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
              % ((name, terms) + error_stats(got, want)))
        del got, want
    assert len(r["convs"]) == len(m.convs()) - 1
    # SE gate: the gate in fp64 from the reduc_conv output, the scale bit for bit
    rows = r["reduc"].cpu().numpy()
    hi, lo = bo.pair_to_hilo(rows, fc)
    xs = bo.merge_h16(hi, lo).reshape(1, Y, X, fc)
    gate = r["gate"].cpu().numpy()
    np.testing.assert_allclose(gate, bo.se_gate_ref(xs, m.se["weight"], m.se["bias"]), rtol=0, atol=1e-5)
    want_rows, ovf = bo.se_scale_ref(rows, fc, np.repeat(gate, Y * X, 0))
    assert not ovf
    assert np.array_equal(r["se"].cpu().numpy().view(np.uint16), want_rows.view(np.uint16)), "SE scale"
    del rows, hi, lo, xs, want_rows
    # head: bias-only 1x1 conv of the SE output into fp32 planes
    acc, _ = conv_ref(from_pixel_h16(r["se"], 1, Y, X, fc), torch.from_numpy(m.head.np["weight"]).to(cuda).double(),
                      1, 1, 0, 1)
    want = epilogue(acc, None, m.head.dev["shift"], False)
    del acc
    check_images("frame head planes", r["planes"].permute(0, 2, 3, 1), want, fc)
    print("BAR frame head 384->294, %d terms: error std %.2e x max, %.2e x max below 5e-2 x max, relative %.2e above"
          % ((fc,) + error_stats(r["planes"].permute(0, 2, 3, 1), want)))
    del want
    # decode of the actual planes, with both cuts taken
    planes = r["planes"].cpu().numpy()
    t = c["test"]
    scores = bo.sigmoid32(bo.split_head(planes, m.num_classes, m.R)[0]).max(1)
    passing = int((scores > np.float32(t["score_thr"])).sum())
    assert passing > t["nms_pre"], passing
    want = bo.anchor3d_decode_ref(planes, m.anchors_np, m.num_classes, m.R, **t)
    assert len(want[0]) == k == t["max_num"]
    _compare([v.numpy() for v in hot_res], want)
    print("frame: %d voxels, %d of %d anchors pass score_thr, %d boxes" % (nv, passing, len(scores), k))
