"""CPU: CenterPoint-pillars KITTI (centerpoint_pillars.CONFIG_KITTI with synth.CP_PILLARS_KITTI) — the wide two-layer
pillar encoder's argument limits, the model built from its config against a written-out conv table and flop sum, its
checkpoint table (no velocity head, two tasks), the CenterPoint-to-KITTI box conversion, and the default common_heads
building the same heads and seeded parameters as before common_heads existed."""
import ctypes as C
import hashlib
import os
import re
import subprocess
import tempfile

import numpy as np
import pytest

from conftest import ROOT
from paddle3d_b200 import centerpoint_pillars as cpp
from paddle3d_b200 import checkpoint, kitti, synth
from paddle3d_b200.dense_head import COMMON_HEADS, DenseRPNHead

ERR_INVALID, ERR_UNSUPPORTED = -1, -4


def _model(seed=0):
    return cpp.CenterPointPillars(synth.CP_PILLARS_KITTI, cpp.CONFIG_KITTI).init_weight(seed=seed, device=None)


def test_wide_pfn_entry_limits():
    from paddle3d_b200 import _lib
    L = _lib.lib()
    p = C.c_void_p(256)  # non-null dummy address: every call returns before touching it
    vs, pcr = _lib.host_floats([0.16, 0.16, 4.0]), _lib.host_floats(synth.CP_PILLARS_KITTI["point_cloud_range"])
    wide, narrow = L.p3d_pillar_feature_net2_wide, L.p3d_pillar_feature_net2
    # n_cap 0: an accepted call has nothing to do and returns 0 after its checks
    for m in (1, 64, 65, 100, 128):
        assert wide(p, p, p, None, 0, m, 4, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == 0, m
    for m in (0, 129, 256):
        assert wide(p, p, p, None, 10, m, 4, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED, m
    assert wide(p, p, p, None, 10, 100, 9, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert wide(p, p, p, None, 10, 100, 2, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert wide(p, p, p, None, 10, 100, 4, 65, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED
    assert wide(p, p, p, None, 10, 100, 4, 32, None, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_INVALID
    assert wide(p, p, p, None, 10, 100, 4, 32, p, p, p, 0, p, p, p, vs, pcr, p, None) == ERR_INVALID
    # the existing entries keep their 64-point limit
    for m in (65, 100):
        assert narrow(p, p, p, None, 10, m, 4, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED, m
        assert L.p3d_pillar_feature_net(p, p, p, None, 10, m, 4, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED, m
        assert L.p3d_hard_vfe(p, p, p, None, 10, m, 4, 32, p, p, p, 64, p, p, p, vs, pcr, p, None) == ERR_UNSUPPORTED, m


# (Cin, Cout, k, stride, up) of every dense conv before the CenterHead, in launch order: SecondBackbone [3, 5, 5] at
# strides [2, 2, 2], then SecondFPN upsample strides [1, 2, 4] (a 1x1 conv, 2x2 and 4x4 transposed convs)
TRUNK = ([(64, 64, 3, 2, 1)] + [(64, 64, 3, 1, 1)] * 3 + [(64, 128, 3, 2, 1)] + [(128, 128, 3, 1, 1)] * 5
         + [(128, 256, 3, 2, 1)] + [(256, 256, 3, 1, 1)] * 5 + [(64, 128, 1, 1, 1), (128, 128, 2, 2, 2), (256, 128, 4, 4, 4)])
HEADS = [("reg", 2), ("height", 1), ("dim", 3), ("rot", 2)]


def test_config_builds_the_model():
    m = cpp.CenterPointPillars(synth.CP_PILLARS_KITTI, cpp.CONFIG_KITTI)
    assert m.grid == (432, 496) and m.F == 4 and m.pfn_shapes() == [(9, 32), (64, 64)]
    assert synth.CP_PILLARS_KITTI["max_points"] == 100 and synth.CP_PILLARS_KITTI["max_voxels"] == 40000
    assert [(c.cin, c.cout, c.k, c.stride, c.up) for c in m.head.trunk.convs()] == TRUNK
    assert m.feat_hw == [(248, 216), (124, 108), (62, 54)] and m.cat_hw == (248, 216)
    assert m.head.fpn_channels == 384
    sh = m.head.shared
    assert (sh.cin, sh.cout, sh.k) == (384, 64, 3)
    assert [[(n, a.cin, a.cout, f.cout) for n, a, f in hs] for hs in m.head.heads] == [
        [(n, 64, 64, k) for n, k in HEADS + [("hm", t)]] for t in (1, 2)]
    assert sum(len(hs) for hs in m.head.heads) == 10  # ten ConvModules
    assert m.head.head_planes() == 19 and m.label_off == [0, 1]
    assert not m.head.with_velocity
    assert m.test_cfg["down_ratio"] == 2 and m.test_cfg["nms_post_max_size"] == 83
    # flops written out at the shapes above (2 x MACs)
    px1, px2, px3 = 248 * 216, 124 * 108, 62 * 54
    backbone = (2 * px1 * 9 * 64 * 64 * 4 + 2 * px2 * 9 * (64 * 128 + 5 * 128 * 128)
                + 2 * px3 * 9 * (128 * 256 + 5 * 256 * 256))
    fpn = 2 * px1 * (64 * 128 + 128 * 128 + 256 * 128)
    shared, modules, outputs = 2 * px1 * 9 * 384 * 64, 10 * 2 * px1 * 9 * 64 * 64, 2 * px1 * 9 * 64 * 19
    fl = m.flops()
    assert fl["backbone"] == backbone and fl["fpn"] == fpn
    assert (fl["head_shared"], fl["head_convmodules"], fl["head_output"]) == (shared, modules, outputs)
    assert fl["backbone"] + fl["fpn"] + fl["head"] == backbone + fpn + shared + modules + outputs
    assert round(backbone / 1e9) == 59 and round(fpn / 1e9) == 6 and round(shared / 1e9) == 24
    assert round(modules / 1e8) == 395 and round(outputs / 1e8) == 12
    assert 129e9 < backbone + fpn + shared + modules + outputs < 131e9


def test_checkpoint_table():
    m = _model(seed=2)
    sd = m.state_dict()
    assert not [k for k in sd if ".vel." in k]
    assert {k.split(".")[2] for k in sd if k.startswith("bbox_head.tasks.")} == {"0", "1"}
    assert {k.split(".")[3] for k in sd if k.startswith("bbox_head.tasks.")} == {"reg", "height", "dim", "rot", "hm"}
    # the table covers every parameter: both PFN layers and every dense conv, each once; a round trip through a model
    # of another seed gives the same state dict
    table = checkpoint.centerpoint_pillars(m)
    assert len(table) == 2 + len(m.head.all_convs())
    assert sorted(id(g.l) for g in table[2:]) == sorted(id(c) for c in m.head.all_convs())
    assert len(sd) == sum(len(g.shapes()) for g in table)
    other = _model(seed=7)
    other.load_state_dict(sd, device=None)
    got = other.state_dict()
    assert list(got) == list(sd) and all(np.array_equal(got[k], sd[k]) for k in sd)
    # errors name their key; the nuScenes table asks for velocity keys this model does not hold
    bad = dict(sd)
    del bad["bbox_head.tasks.1.hm.3.bias"]
    bad["bbox_head.tasks.0.vel.0.weight"] = np.zeros((64, 64, 3, 3), np.float32)
    bad["bbox_head.tasks.0.dim.3.weight"] = np.zeros((2, 64, 3, 3), np.float32)
    with pytest.raises(ValueError) as e:
        _model(seed=7).load_state_dict(bad, device=None)
    msg = str(e.value)
    assert "missing keys: bbox_head.tasks.1.hm.3.bias" in msg
    assert "unexpected keys: bbox_head.tasks.0.vel.0.weight" in msg
    assert "bbox_head.tasks.0.dim.3.weight: shape (2, 64, 3, 3), expected (3, 64, 3, 3)" in msg
    nusc = cpp.CenterPointPillars(synth.CP_PILLARS_KITTI, dict(cpp.CONFIG_KITTI, head=dict(
        tasks=(1, 2), share_conv_channel=64)))
    with pytest.raises(ValueError, match=r"missing keys: .*bbox_head\.tasks\.0\.vel\.0\.weight"):
        nusc.load_state_dict(sd, device=None)


def test_centerpoint_box_conversion_and_labels():
    # (x, y, z_centre, d0, d1, d2, rot) -> (x, y, z - d2 / 2, d1, d0, d2, -(rot + pi / 2)), worked by hand
    cp_boxes = np.array([[10.0, 2.0, -0.5, 4.0, 1.6, 1.5, 0.0],
                         [20.0, -3.0, -1.0, 0.8, 0.6, 1.8, -np.pi / 2],
                         [30.0, 5.0, -0.2, 1.7, 0.5, 1.7, 1.0]], np.float32)
    want = np.array([[10.0, 2.0, -1.25, 1.6, 4.0, 1.5, -np.pi / 2],
                     [20.0, -3.0, -1.9, 0.6, 0.8, 1.8, 0.0],
                     [30.0, 5.0, -1.05, 0.5, 1.7, 1.7, -1.0 - np.pi / 2]])
    got = kitti.centerpoint_to_lidar_boxes(cp_boxes)
    assert got.dtype == np.float64 and got.shape == (3, 7)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-6)
    assert kitti.centerpoint_to_lidar_boxes(np.zeros((0, 7), np.float32)).shape == (0, 7)
    names = kitti.CLASS_NAMES["centerpoint"]
    assert names == ("Car", "Pedestrian", "Cyclist") and len(names) == sum(synth.CP_PILLARS_KITTI_TASKS)
    calib = kitti.parse_calib(synth.KITTI_CALIB)
    annos = kitti.to_kitti(got, np.array([0.9, 0.5, 0.3]), np.array([0, 1, 2]), calib, class_names=names)
    assert list(annos["name"]) == ["Car", "Pedestrian", "Cyclist"]
    # KITTI dimensions (h, w, l): h = d2, w = d1, l = d0; rotation_y is the converted heading -(rot + pi / 2)
    np.testing.assert_allclose(annos["dimensions"], want[:, [5, 3, 4]], atol=1e-9)
    np.testing.assert_allclose(annos["rotation_y"], -(cp_boxes[:, 6].astype(np.float64) + np.pi / 2), atol=1e-6)
    # location: the bottom centre, about 1.5 m below a centre at z_centre in camera y (down)
    bottom = kitti.lidar_to_camera(want[:, :3], calib["R0_rect"], calib["Tr_velo_to_cam"])
    np.testing.assert_allclose(annos["location"], bottom, atol=1e-9)
    lines = kitti.format_label_lines(annos)
    assert lines[0].split()[:3] == ["Car", "0.0000", "0"]
    assert lines[1].split()[8:11] == ["%.4f" % v for v in (1.8, 0.6, 0.8)]
    assert len(lines[2].split()) == 16


def test_default_common_heads_unchanged():
    """The default head list and seeded parameters are those of the parent commit (digests taken there)."""
    assert COMMON_HEADS == (("reg", 2), ("height", 1), ("dim", 3), ("rot", 2), ("vel", 2))
    m = cpp.CenterPointPillars().init_weight(seed=3, device=None)
    assert [n for n, _, _ in m.head.heads[0]] == ["reg", "height", "dim", "rot", "vel", "hm"]
    assert m.head.head_planes() == 70 and m.head.with_velocity
    h = hashlib.sha256()
    sd = m.state_dict()
    for k in sorted(sd):
        h.update(k.encode())
        h.update(np.ascontiguousarray(sd[k], np.float32).tobytes())
    assert h.hexdigest() == "a1823a425b9345f618327ffec1f8dd4371e041045dcf250932d3250e10512495"
    head = DenseRPNHead(in_channels=64, out_channels=(64,), layer_nums=(1,), downsample_strides=(1,),
                        fpn_out_channels=(64,), upsample_strides=(1,)).init_weight(seed=5, device=None, randomize_bn=True)
    h = hashlib.sha256()
    for c in head.all_convs():
        for k in ("weight", "bias"):
            if c.np[k] is not None:
                h.update(c.np[k].tobytes())
        if c.np["bn"] is not None:
            for k in ("gamma", "beta", "mean", "var"):
                h.update(c.np["bn"][k].tobytes())
    assert h.hexdigest() == "249a654b06f10a1636d20d630188c9ad63a5e1b39f2094e2209bbac66d1c1519"
    # an explicit velocity flag still overrides, as tests/test_nms_utils.py uses it; asking for one without a head fails
    assert not DenseRPNHead(with_velocity=False).with_velocity
    with pytest.raises(ValueError, match="vel"):
        DenseRPNHead(with_velocity=True, common_heads=HEADS)


# SASS of the existing pfn_kernel instantiations at the parent commit (cuobjdump -sass, instruction text only; nvcc 12.9):
# one layer, two layers, HardVFE.  The row bound became a template parameter; these three must not change.
PARENT_SASS = {"Li1ELb0": "8cfc5d79f1b386712ce04504f1c47e8280fdb4fd2f72a9ae7cfb6c913d0bdb10",
               "Li2ELb0": "c1a4777cc02d8fec96d5e815d7f05a34074c122516f03cf3ddd5d42ac70cc4d8",
               "Li2ELb1": "0f375b5fb068d8e4910c3ed6a7ec35a31ea57a2d4953eee2177fbb76c104f909"}


def test_existing_pfn_instantiations_keep_their_sass():
    from paddle3d_b200 import build
    nvcc = build.NVCC
    try:
        ver = subprocess.run([nvcc, "--version"], capture_output=True, text=True).stdout
    except OSError:
        pytest.skip("no nvcc")
    if "release 12.9" not in ver:
        pytest.skip("the parent's SASS digests were taken with nvcc 12.9")
    with tempfile.TemporaryDirectory() as d:
        obj = os.path.join(d, "pillar_encoder.o")
        subprocess.run([nvcc] + build.FLAGS + ["-c", os.path.join(ROOT, "paddle3d_b200", "csrc", "pillar_encoder.cu"),
                                               "-o", obj], check=True, capture_output=True)
        sass = subprocess.run([os.path.join(os.path.dirname(nvcc), "cuobjdump"), "-sass", obj], check=True,
                              capture_output=True, text=True).stdout
    funcs, name = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : \S*pfn_kernelI(Li\d+ELb\d)(ELi(\d+))?", line)
        if m:
            name = (m.group(1), int(m.group(3) or 64))
            funcs[name] = []
            continue
        if "Function :" in line:
            name = None
        if name and re.search(r"/\*[0-9a-f]{4}\*/", line):
            funcs[name].append(re.sub(r"\s+", " ", line.split(";")[0]).strip())
    assert set(funcs) == {(k, 64) for k in PARENT_SASS} | {("Li2ELb0", 128)}
    for k, want in PARENT_SASS.items():
        assert hashlib.sha256("\n".join(funcs[(k, 64)]).encode()).hexdigest() == want, k
