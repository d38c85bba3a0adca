"""CPU suite for BEVDet's box decode: the numpy oracle (tests/bevdet_postprocess_oracle.py) on hand-made cases, the C ABI
of p3d_bevdet_postprocess without a device (symbols, signatures, every refused argument), the Python layer's argument
checks and the Paddle registration."""
import ctypes
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT

T_CH = [1, 2, 2, 1, 2, 2]   # car | truck, cv | bus, trailer | barrier | motorcycle, bicycle | pedestrian, cone
OFF = [0, 1, 3, 5, 6, 8]
H = W = 16


def _cfg(**over):
    """TEST_CFG_BEVDET on a 16 x 16 map of exact 1 m cells (0.125 m voxels x 8) from -8 m: every centre below is exact
    in fp32."""
    from paddle3d_b200.bevdet import TEST_CFG_BEVDET
    return dict(TEST_CFG_BEVDET, voxel_size=(0.125, 0.125), point_cloud_range=[-8.0, -8.0, -5.0, 8.0, 8.0, 3.0], **over)


def _empty():
    h = dict(hm=[], reg=[], height=[], dim=[], vel=[], rot=[])
    for c in T_CH:
        h["hm"].append(np.full((1, c, H, W), -20.0, np.float32))
        for name, k in (("reg", 2), ("height", 1), ("dim", 3), ("vel", 2), ("rot", 2)):
            h[name].append(np.zeros((1, k, H, W), np.float32))
    return h


def _put(h, t, c, x, y, dims=(1.0, 1.0, 1.0), logit=2.0, z=0.0, yaw=0.0, reg=None):
    """A box of class c of task t centred at (x, y) metres; reg overrides the (cell, offset) split of the centre."""
    u, v = x + 8.0, y + 8.0
    xs, ys = int(np.floor(u)), int(np.floor(v))
    rx, ry = (u - xs, v - ys) if reg is None else reg
    h["hm"][t][0, c, ys, xs] = logit
    h["reg"][t][0, :, ys, xs] = (rx, ry)
    h["height"][t][0, 0, ys, xs] = z
    h["dim"][t][0, :, ys, xs] = np.log(np.asarray(dims, np.float64))
    h["rot"][t][0, :, ys, xs] = (np.sin(yaw), np.cos(yaw))
    h["vel"][t][0, :, ys, xs] = (0.5, -0.25)
    return h


def _ref(h, cfg):
    from bevdet_postprocess_oracle import bevdet_postprocess_ref
    return bevdet_postprocess_ref(h, cfg, OFF)


def _factors(task, value):
    from paddle3d_b200.bevdet import TEST_CFG_BEVDET
    f = list(TEST_CFG_BEVDET["nms_rescale_factor"])
    f[task] = value
    return f


def test_truck_scale_factor_decides(oracle_mod):
    """Two 4 x 2 m trucks 1 m apart across: IoU 1/3 as they are (suppressed at 0.2), 1/6 with both shrunk by 0.7."""
    h = _put(_put(_empty(), 1, 0, 0.5, 0.5, (4.0, 2.0, 2.0), logit=3.0), 1, 0, 0.5, 1.5, (4.0, 2.0, 2.0), logit=2.0)
    boxes, scores, labels, counts = _ref(h, _cfg())
    assert counts.tolist() == [0, 2, 0, 0, 0, 0] and labels.tolist() == [1, 1] and scores[0] > scores[1]
    np.testing.assert_allclose(boxes[:, 3:6], [[4.0, 2.0, 2.0]] * 2, rtol=2e-7)   # written unscaled
    _, _, _, counts = _ref(h, _cfg(nms_rescale_factor=_factors(1, [1.0, 1.0])))
    assert counts.tolist() == [0, 1, 0, 0, 0, 0]


def test_pedestrian_cone_overlap_only_when_scaled(oracle_mod):
    """A 0.6 m pedestrian and a 0.4 m cone 0.5 m apart touch at an edge; scaled by 4.5 and 9.0 their IoU is 0.546 > 0.5."""
    h = _put(_put(_empty(), 5, 0, 0.5, 0.5, (0.6, 0.6, 1.7), logit=3.0), 5, 1, 1.0, 0.5, (0.4, 0.4, 1.0), logit=2.0)
    _, _, labels, counts = _ref(h, _cfg())
    assert counts.tolist() == [0, 0, 0, 0, 0, 1] and labels.tolist() == [8]
    _, _, labels, counts = _ref(h, _cfg(nms_rescale_factor=_factors(5, 1.0)))
    assert counts.tolist() == [0, 0, 0, 0, 0, 2] and labels.tolist() == [8, 9]


@pytest.mark.parametrize("dx,kept", [(0.5, 1), (1.0, 1), (1.0 + 2.0 ** -10, 2)])
def test_barrier_circle_radius(oracle_mod, dx, kept):
    """circle_nms compares the SQUARED distance with min_radius (1 for barriers): 0.25 and exactly 1.0 suppress, just
    past 1.0 does not."""
    h = _put(_put(_empty(), 3, 0, 0.75, 0.5, logit=3.0), 3, 0, 0.75 + dx, 0.5, logit=2.0)
    boxes, _, labels, counts = _ref(h, _cfg())
    assert counts.tolist() == [0, 0, 0, kept, 0, 0] and labels.tolist() == [5] * kept
    assert boxes[0, 0] == np.float32(0.75)


def test_both_classes_of_one_cell(oracle_mod):
    """One cell over the threshold as pedestrian and as cone is two candidates (not the cell's arg-max); the same box
    scaled by 4.5 and by 9.0 has IoU 0.25, so both survive."""
    h = _put(_put(_empty(), 5, 0, 0.5, 0.5, logit=1.0), 5, 1, 0.5, 0.5, logit=3.0)
    boxes, scores, labels, counts = _ref(h, _cfg())
    assert counts[5] == 2 and labels.tolist() == [9, 8] and scores[0] > scores[1]
    assert np.array_equal(boxes[0], boxes[1])
    # in a task whose classes share a factor the second is suppressed (IoU 1)
    h = _put(_put(_empty(), 4, 0, 0.5, 0.5, logit=1.0), 4, 1, 0.5, 0.5, logit=3.0)
    assert _ref(h, _cfg())[2].tolist() == [7]


def test_range_is_tested_on_the_decoded_centre(oracle_mod):
    """With the range cut to +-4 m: a centre at x = 6 m (offset 0.5: inside as a raw value) is dropped, and a centre at
    x = 1 m written as cell 4 + offset 5 (outside as a raw value) is kept."""
    cfg = _cfg(post_center_limit_range=[-4.0, -4.0, -10.0, 4.0, 4.0, 10.0])
    h = _put(_empty(), 0, 0, 6.5, 0.5)
    assert _ref(h, cfg)[3].sum() == 0 and _ref(h, _cfg())[3].sum() == 1
    h = _put(_empty(), 0, 0, -3.5, 0.5, reg=(5.0, 0.5))
    boxes, _, _, counts = _ref(h, cfg)
    assert counts.tolist() == [1, 0, 0, 0, 0, 0] and boxes[0, 0] == 1.0
    # both ends inclusive
    h = _put(_put(_empty(), 0, 0, 4.0, 0.0), 0, 0, -4.0, -4.0)
    assert _ref(h, cfg)[3][0] == 2


def test_rows_empty_tasks_bottom_centre_and_labels(oracle_mod):
    h = _empty()
    boxes, scores, labels, counts = _ref(h, _cfg())
    assert boxes.shape == (0, 9) and not len(scores) and not len(labels) and not counts.any()   # no fake row
    for t, c in ((0, 0), (1, 1), (2, 0), (3, 0), (4, 1), (5, 1)):
        _put(h, t, c, -6.5 + 2 * t, 0.5, (2.0, 1.0, 3.0), z=-1.0, yaw=0.3)
    boxes, scores, labels, counts = _ref(h, _cfg())
    assert counts.tolist() == [1] * 6 and labels.tolist() == [0, 2, 3, 5, 7, 9]
    np.testing.assert_allclose(boxes[:, 2], -2.5, rtol=1e-6)   # z - dz / 2
    np.testing.assert_allclose(boxes[:, 6], 0.3, rtol=1e-6)
    np.testing.assert_allclose(boxes[:, 7:], [[0.5, -0.25]] * 6)
    np.testing.assert_allclose(scores, 1 / (1 + np.exp(-2.0)), rtol=1e-6)
    # a score at the threshold is not a candidate (strict >); post_max_size cuts the kept list
    h = _put(_put(_empty(), 0, 0, 0.5, 0.5, logit=3.0), 0, 0, 5.5, 0.5, logit=2.0)
    assert _ref(h, _cfg(score_threshold=float(np.float32(1) / (np.float32(1) + np.exp(np.float32(-2))))))[3][0] == 1
    assert _ref(h, _cfg(post_max_size=1))[3][0] == 1 and _ref(h, _cfg())[3][0] == 2


def test_per_class_then_global_topk_is_the_thresholded_topk(oracle_mod):
    """The reference's selection order (top-K per class, top-K of those, threshold after the decode) against the op's
    formulation (threshold, then the best max_num by (score desc, class * H*W + cell asc)) on tied and untied planes."""
    from bevdet_postprocess_oracle import task_selection
    from paddle3d_b200 import synth
    cfg = _cfg(max_num=40)
    for seed, quant in ((0, None), (1, 4.0)):
        h = synth.centerpoint_head_outputs(seed, T_CH, H, W, hm_mean=-1.5)
        for t, C in enumerate(T_CH):
            hm = h["hm"][t] if quant is None else np.round(h["hm"][t] * quant) / np.float32(quant)
            _, s, cls, flat = task_selection(hm, h["reg"][t], h["height"][t], h["dim"][t], h["vel"][t], h["rot"][t],
                                             dict(cfg, post_center_limit_range=[-1e9] * 3 + [1e9] * 3))
            sc = (np.float32(1) / (np.float32(1) + np.exp(-hm.reshape(-1), dtype=np.float32))).astype(np.float32)
            cand = np.nonzero(sc > np.float32(cfg["score_threshold"]))[0]
            want = cand[np.lexsort((cand, -sc[cand]))][:40]
            assert len(cand) > 40 and np.array_equal(flat, want) and np.array_equal(cls, want // (H * W))
            assert np.array_equal(s, sc[want])


# ------------------------------------------------------------------------------------------------------------ the ABI
def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib


def test_symbols_and_signatures():
    L = _lib()
    lib = ctypes.CDLL(L.LIB_PATH)
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "p3d_b200.h")).read(), flags=re.S)
    for name in ("p3d_bevdet_postprocess_workspace_bytes", "p3d_bevdet_postprocess"):
        assert hasattr(lib, name)
        decl = re.search(r"\b(\w+)\s+%s\s*\(([^;]*)\)\s*;" % name, src)
        params = [p.strip() for p in decl.group(2).split(",")]
        res, args = L.SIGNATURES[name]
        assert len(args) == len(params), name
        assert res is (ctypes.c_size_t if decl.group(1) == "size_t" else ctypes.c_int)
        for a, p in zip(args, params):
            want = (ctypes.c_void_p if "*" in p or p.startswith("p3d_stream_t") else ctypes.c_float if p.startswith("float")
                    else ctypes.c_size_t if p.startswith("size_t") else ctypes.c_int)
            assert a is want, (name, p)
    assert "#define P3D_BEVDET_NMS_ROTATE 0" in src and "#define P3D_BEVDET_NMS_CIRCLE 1" in src


def test_invalid_arguments_are_refused_before_any_launch():
    L = _lib()
    lib = L.lib()
    ints, floats = L.host_ints, L.host_floats
    ch = ints(T_CH)
    size = lib.p3d_bevdet_postprocess_workspace_bytes
    need = size(6, ch, 128, 128, 500)
    assert need >= 10 * 16384 * 8 + 6 * 500 * (8 + 8 + 36 + 4 + 4 + 64 + 4)
    assert size(0, ch, 128, 128, 500) == 0 and size(6, None, 128, 128, 500) == 0 and size(6, ch, 0, 128, 500) == 0
    assert size(6, ch, 128, 128, 0) == 0 and size(6, ints([1, 2, 0, 1, 2, 2]), 128, 128, 500) == 0
    assert size(17, ints([1] * 17), 8, 8, 10) == 0

    buf = ctypes.create_string_buffer(64)
    p = ctypes.addressof(buf)   # a non-null address, never dereferenced: every call below is refused on the host
    P6 = (ctypes.c_void_p * 6)(*[p] * 6)
    ok = dict(T=6, hm=P6, ch=ch, H=128, W=128, osf=8, thr=0.1, max_num=500, pre=1000, post=500,
              types=ints([0, 0, 0, 1, 0, 0]), nms_thr=floats([0.2] * 6), radius=floats([4, 12, 10, 1, 0.85, 0.175]),
              rescale=floats([1.0] * 10), off=ints(OFF), out=p, ws=p, ws_bytes=need)

    def call(**over):
        a = dict(ok, **over)
        return lib.p3d_bevdet_postprocess(
            a["T"], a["hm"], a["ch"], P6, P6, P6, P6, P6, a["H"], a["W"], floats([0.1, 0.1]), floats([-51.2] * 3 + [51.2] * 3),
            floats([-61.2, -61.2, -10, 61.2, 61.2, 10]), a["osf"], a["thr"], a["max_num"], a["pre"], a["post"], a["types"],
            a["nms_thr"], a["radius"], a["rescale"], a["off"], a["out"], p, p, p, a["ws"], a["ws_bytes"], None)
    assert call(T=0) == -1
    assert call(T=17) == -4
    assert call(ch=ints([1, 2, 0, 1, 2, 2])) == -1            # a channel count < 1
    assert call(max_num=0) == -1 and call(pre=0) == -1 and call(post=0) == -1
    assert call(H=0) == -1 and call(osf=0) == -1
    assert call(types=ints([0, 0, 2, 1, 0, 0])) == -1          # unknown NMS type
    assert call(rescale=floats([1.0] * 9 + [0.0])) == -1       # non-positive factor
    assert call(rescale=floats([1.0, -0.7] + [1.0] * 8)) == -1
    assert call(rescale=floats([float("nan")] + [1.0] * 9)) == -1
    assert call(radius=floats([4, 12, 10, -1, 0.85, 0.175])) == -1
    assert call(hm=(ctypes.c_void_p * 6)(p, p, None, p, p, p)) == -1
    assert call(out=None) == -1 and call(types=None) == -1 and call(rescale=None) == -1
    assert call(ch=ints([40, 30, 1, 1, 1, 1])) == -4           # more than 64 classes
    assert call(ws_bytes=need - 1) == -2 and call(ws=None) == -2


def test_python_layer_argument_checks():
    import torch
    L = _lib()
    from paddle3d_b200 import ops
    from paddle3d_b200.bevdet import TEST_CFG_BEVDET as tc
    from paddle3d_b200.ops.bevdet_postprocess import bevdet_postprocess_heads, task_attrs
    assert ops.bevdet_postprocess.bevdet_postprocess_device and ops.bevdet_postprocess.bevdet_postprocess
    types, thr, radius, rescale = task_attrs(6, T_CH, tc["nms_type"], tc["nms_thr"], tc["nms_rescale_factor"], tc["min_radius"])
    assert types == [0, 0, 0, 1, 0, 0] and thr == [0.2] * 5 + [0.5] and radius == [4, 12, 10, 1, 0.85, 0.175]
    assert rescale == [1.0, 0.7, 0.7, 0.4, 0.55, 1.1, 1.0, 1.0, 4.5, 9.0]
    assert task_attrs(6, T_CH, "rotate", 0.2, 1.0, 0.0) == ([0] * 6, [0.2] * 6, [0.0] * 6, [1.0] * 10)   # scalars
    args = dict(nms_type=tc["nms_type"], nms_thr=tc["nms_thr"], nms_rescale_factor=tc["nms_rescale_factor"],
                min_radius=tc["min_radius"])
    for bad in (dict(nms_type=["rotate"] * 5), dict(nms_thr=[0.2] * 7), dict(min_radius=[1.0] * 2),
                dict(nms_rescale_factor=[1.0] * 5), dict(nms_rescale_factor=_factors(1, [0.7, 0.7, 0.7])),
                dict(nms_rescale_factor=_factors(0, [1.0, 1.0])), dict(nms_type=["rotate"] * 5 + ["nms_gpu"]),
                dict(nms_rescale_factor=_factors(2, [0.4, 0.0])), dict(min_radius=[4, 12, 10, -1, 0.85, 0.175])):
        with pytest.raises(ValueError):
            task_attrs(6, T_CH, **dict(args, **bad))
    h = {k: [torch.from_numpy(a) for a in v] for k, v in _empty().items()}
    with pytest.raises(L.P3DError):
        bevdet_postprocess_heads(h, _cfg(), OFF)   # CPU tensors: there is no CPU path


def test_configs_select_the_decode():
    from paddle3d_b200 import bevdet as bd
    assert "nms_type" not in bd.CONFIG["test"] and "nms_type" not in bd.CONFIG_4D["test"]
    for cfg, base in ((bd.CONFIG_BEVDET_NMS, bd.CONFIG), (bd.CONFIG_4D_BEVDET_NMS, bd.CONFIG_4D)):
        assert cfg["test"] is bd.TEST_CFG_BEVDET and {k: v for k, v in cfg.items() if k != "test"} == \
            {k: v for k, v in base.items() if k != "test"}
    assert bd.BEVDet(bd.CONFIG_BEVDET_NMS, device="cpu").result_rows() == 3000
    assert bd.BEVDet4D(bd.CONFIG_4D_BEVDET_NMS, device="cpu").result_rows() == 3000
    assert bd.BEVDet(device="cpu").result_rows() == 498 and bd.BEVDet4D(device="cpu").result_rows() == 498


def test_paddle_registration():
    glue = os.path.join(ROOT, "paddle_ext", "p3d_paddle_ops.cc")
    r = subprocess.run(["g++", "-std=c++17", "-fsyntax-only", "-I", os.path.join(ROOT, "oracle", "stub"), "-I",
                        os.path.join(ROOT, "include"), glue], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    assert "PD_BUILD_OP(p3d_bevdet_postprocess)" in open(glue).read()
