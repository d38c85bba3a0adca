"""Paddle3D checkpoints without a GPU: the `.pdparams` reader (the forms paddle.save writes, and a file that names any
global other than an ndarray's or a dict's is refused before that global is called), the name tables of the four LiDAR
models (keys and Paddle layouts), and load_state_dict's checks (every error reported, the model untouched)."""
import collections
import os
import pickle

import numpy as np
import pytest

from paddle3d_b200 import centerpoint_pillars as cpp
from paddle3d_b200 import checkpoint
from paddle3d_b200 import pointpillars as pp
from paddle3d_b200 import synth


def _voxel(seed=0):
    from paddle3d_b200.dense_head import DenseRPNHead
    from paddle3d_b200.layers import SparseResNet3D
    net = SparseResNet3D(synth.C3["point_dim"], synth.C3["voxel_size"], synth.C3["point_cloud_range"])
    net.init_weight(seed=seed, device="cpu")
    dense = DenseRPNHead(in_channels=128 * 2).init_weight(seed=seed + 1, device=None)
    return checkpoint.centerpoint_voxel(net, dense)


def _tables():
    """(name, table, model with state_dict / load_state_dict or None) of the four models, numpy / CPU parameters."""
    car = pp.PointPillars().init_weight(seed=1, device=None)
    pc = pp.PointPillars(synth.C2_PED_CYCLIST, pp.CONFIG_PED_CYCLIST).init_weight(seed=1, device=None)
    cpm = cpp.CenterPointPillars().init_weight(seed=1, device=None)
    return [("centerpoint_voxel", _voxel(), None), ("centerpoint_pillars", checkpoint.centerpoint_pillars(cpm), cpm),
            ("pointpillars_car", checkpoint.pointpillars(car), car),
            ("pointpillars_cyclist_pedestrian", checkpoint.pointpillars(pc), pc)]


def _save(path, sd, form="dict"):
    names = {k: "param_%d" % i for i, k in enumerate(sd)}
    if form == "tuple":
        obj = {k: (names[k], v) for k, v in sd.items()}
    elif form == "ordered":
        obj = collections.OrderedDict(sd)
    else:
        obj = dict(sd)
    obj[checkpoint.STRUCTURED_NAMES] = names
    with open(path, "wb") as f:
        pickle.dump(obj, f, protocol=4)


def _same(a, b):
    return list(a) == list(b) and all(a[k].dtype == b[k].dtype and np.array_equal(a[k], b[k]) for k in a)


@pytest.mark.parametrize("form", ["dict", "tuple", "ordered"])
def test_reader_accepts_the_forms_paddle_save_writes(tmp_path, form):
    m = pp.PointPillars().init_weight(seed=3, device=None)
    sd = m.state_dict()
    sd_int = dict(sd, **{"global_step": np.array([7], np.int64)})
    _save(tmp_path / "m.pdparams", sd_int, form)
    got = checkpoint.read_pdparams(str(tmp_path / "m.pdparams"))
    assert checkpoint.STRUCTURED_NAMES not in got
    assert _same({k: got[k] for k in sd}, sd) and got["global_step"].dtype == np.int64
    with open(tmp_path / "m.pdparams", "rb") as f:  # a file object as well as a path
        assert list(checkpoint.read_pdparams(f)) == list(got)
    # the integer entry is not a parameter: the load ignores it
    m2 = pp.PointPillars().load_state_dict(got, None)
    assert _same(m2.state_dict(), sd)


class _Payload:
    def __init__(self, *call):
        self.call = call

    def __reduce__(self):
        return self.call


@pytest.mark.parametrize("call", ["os.system", "builtins.eval", "numpy.load"])
def test_reader_refuses_other_globals_without_running_them(tmp_path, call):
    marker = tmp_path / "ran"
    cmd = "touch %s" % marker
    fn = {"os.system": (os.system, (cmd,)), "builtins.eval": (eval, ("open(%r, 'w').close()" % str(marker),)),
          "numpy.load": (np.load, (str(tmp_path / "nothing.npy"),))}[call]
    sd = {"a.weight": np.ones((2, 2), np.float32), "b.weight": _Payload(*fn)}
    path = tmp_path / "evil.pdparams"
    with open(path, "wb") as f:
        pickle.dump(sd, f, protocol=4)
    with pytest.raises(pickle.UnpicklingError) as e:
        checkpoint.read_pdparams(str(path))
    assert fn[0].__name__ in str(e.value) and "refusing global" in str(e.value)
    assert not marker.exists()


@pytest.mark.parametrize("bad", ["float64", "float16", "nan", "inf", "object"])
def test_reader_refuses_values_and_names_the_key(tmp_path, bad):
    a = {"float64": np.ones(3, np.float64), "float16": np.ones(3, np.float16),
         "nan": np.array([1.0, np.nan], np.float32), "inf": np.array([np.inf], np.float32),
         "object": [1.0, 2.0]}[bad]
    path = tmp_path / "m.pdparams"
    with open(path, "wb") as f:
        pickle.dump({"good.weight": np.ones(2, np.float32), "neck.deblocks.0.1._mean": a}, f, protocol=4)
    with pytest.raises((ValueError, pickle.UnpicklingError)) as e:
        checkpoint.read_pdparams(str(path))
    assert "neck.deblocks.0.1._mean" in str(e.value) or bad == "object"


@pytest.mark.parametrize("which", range(4), ids=["centerpoint_voxel", "centerpoint_pillars", "pointpillars_car",
                                                 "pointpillars_cyclist_pedestrian"])
def test_state_dict_keys_are_the_table_in_paddle_layouts(which):
    name, table, model = _tables()[which]
    sd = checkpoint.state_dict(table)
    shapes = collections.OrderedDict()
    for g in table:
        shapes.update(g.shapes())
    assert list(sd) == list(shapes) and len(sd) == len(set(sd))
    if model is not None:
        assert _same(model.state_dict(), sd)
    for k, v in sd.items():
        assert v.dtype == np.float32 and v.flags["C_CONTIGUOUS"] and v.shape == tuple(shapes[k]), k
        bn_weight = k.endswith(".weight") and k[:-len("weight")] + "_mean" in sd
        if k.endswith(("._mean", "._variance", ".bias")) or bn_weight:
            assert v.ndim == 1, k
        elif k.startswith("middle_encoder.") and v.ndim != 1:
            assert v.ndim == 5, k        # sparse conv [kD, kH, kW, Cin, Cout]
        elif k.endswith("linear.weight"):
            assert v.ndim == 2, k        # Linear [in, out]
        elif v.ndim != 1:
            assert v.ndim == 4, k        # Conv2D [Cout, Cin, k, k] / Conv2DTranspose [Cin, Cout, k, k]
    expect = {
        "centerpoint_voxel": {"middle_encoder.conv_input.0.weight": (3, 3, 3, 5, 16),
                              "middle_encoder.conv1.0.conv1.weight": (3, 3, 3, 16, 16),
                              "middle_encoder.conv4.0.weight": (3, 3, 3, 64, 128),
                              "middle_encoder.extra_conv.0.weight": (3, 1, 1, 128, 128),
                              "middle_encoder.extra_conv.1._mean": (128,),
                              "backbone.blocks.0.3.weight": (128, 128, 3, 3),
                              "backbone.blocks.1.0.weight": (256, 128, 3, 3),
                              "neck.deblocks.0.0.weight": (256, 128, 1, 1),      # stride 1: Conv2D k = 1
                              "neck.deblocks.1.0.weight": (256, 256, 2, 2),      # Conv2DTranspose [Cin, Cout, k, k]
                              "bbox_head.shared_conv.0.weight": (64, 512, 3, 3),
                              "bbox_head.tasks.0.hm.3.bias": (1,), "bbox_head.tasks.1.hm.3.weight": (2, 64, 3, 3),
                              "bbox_head.tasks.5.vel.1._variance": (64,)},
        "centerpoint_pillars": {"voxel_encoder.pfn_layers.0.linear.weight": (10, 32),
                                "voxel_encoder.pfn_layers.1.linear.weight": (64, 64),
                                "backbone.blocks.0.0.weight": (64, 64, 3, 3),
                                "neck.deblocks.0.0.weight": (128, 64, 2, 2),     # stride 0.5: Conv2D k = 2
                                "neck.deblocks.2.0.weight": (256, 128, 2, 2),    # Conv2DTranspose [Cin, Cout, k, k]
                                "bbox_head.shared_conv.0.weight": (64, 384, 3, 3)},
        "pointpillars_car": {"pillar_encoder.pfn_layers.0.linear.weight": (9, 64),
                             "neck.deblocks.0.0.weight": (64, 128, 1, 1),       # Conv2DTranspose k = 1
                             "neck.deblocks.2.0.weight": (256, 128, 4, 4),
                             "head.cls_head.weight": (2, 384, 1, 1), "head.box_head.weight": (14, 384, 1, 1),
                             "head.dir_head.bias": (4,)},
        "pointpillars_cyclist_pedestrian": {"head.cls_head.weight": (8, 384, 1, 1), "head.box_head.bias": (28,),
                                            "head.dir_head.weight": (8, 384, 1, 1)},
    }[name]
    for k, s in expect.items():
        assert sd[k].shape == s, (k, sd[k].shape)
    if name.startswith("pointpillars"):  # the one head conv is cls | box | dir
        m = model.head.np
        np.testing.assert_array_equal(np.concatenate([sd["head.cls_head.weight"], sd["head.box_head.weight"],
                                                      sd["head.dir_head.weight"]]), m["weight"])
        np.testing.assert_array_equal(np.concatenate([sd["head.cls_head.bias"], sd["head.box_head.bias"],
                                                      sd["head.dir_head.bias"]]), m["bias"])


@pytest.mark.parametrize("make", [lambda: pp.PointPillars(), lambda: cpp.CenterPointPillars(),
                                  lambda: pp.PointPillars(synth.C2_PED_CYCLIST, pp.CONFIG_PED_CYCLIST)],
                         ids=["pointpillars_car", "centerpoint_pillars", "pointpillars_cyclist_pedestrian"])
def test_numpy_round_trip_into_an_unseeded_model(tmp_path, make):
    """A's parameters through a file into a model that was never initialised, and into one of another seed: the same
    state dict and the same export_numpy (what the CPU arms read), bit for bit."""
    a = make().init_weight(seed=4, device=None)
    _save(tmp_path / "a.pdparams", a.state_dict(), "tuple")
    sd = checkpoint.read_pdparams(tmp_path / "a.pdparams")
    for b in (make(), make().init_weight(seed=9, device=None)):
        b.load_state_dict(sd, None)
        assert _same(b.state_dict(), a.state_dict())
        ea, eb = a.export_numpy(), b.export_numpy()

        def flat(x, out):
            if isinstance(x, dict):
                for k in sorted(x):
                    flat(x[k], out)
            elif isinstance(x, (list, tuple)):
                for v in x:
                    flat(v, out)
            elif isinstance(x, np.ndarray):
                out.append(x)
            return out
        fa, fb = flat(ea, []), flat(eb, [])
        assert len(fa) == len(fb) and all(np.array_equal(x, y) for x, y in zip(fa, fb))


def _errors_cases(sd):
    k_conv = next(k for k, v in sd.items() if v.ndim == 4 and v.shape[0] != v.shape[1])
    k_bn, k_nan = [k for k in sd if k.endswith("._mean")][:2]
    k_w = next(k for k in sd if k.endswith(".bias"))
    return {
        "missing": (lambda d: d.pop(k_bn), [k_bn, "missing"]),
        "unexpected": (lambda d: d.__setitem__("bbox_head.extra.weight", np.ones(3, np.float32)),
                       ["bbox_head.extra.weight", "unexpected"]),
        "transposed": (lambda d: d.__setitem__(k_conv, np.ascontiguousarray(d[k_conv].swapaxes(0, 1))), [k_conv, "shape"]),
        "float64": (lambda d: d.__setitem__(k_w, d[k_w].astype(np.float64)), [k_w, "float64"]),
        "nan": (lambda d: d[k_nan].__setitem__(0, np.nan), [k_nan, "non-finite"]),
    }


@pytest.mark.parametrize("which", range(4), ids=["centerpoint_voxel", "centerpoint_pillars", "pointpillars_car",
                                                 "pointpillars_cyclist_pedestrian"])
@pytest.mark.parametrize("case", ["missing", "unexpected", "transposed", "float64", "nan", "all"])
def test_load_errors_name_the_key_and_leave_the_model_untouched(which, case):
    _, table, _ = _tables()[which]
    before = checkpoint.state_dict(table)
    cases = _errors_cases(before)
    sd = {k: v.copy() for k, v in before.items()}
    sd = {k: v * np.float32(1.5) for k, v in sd.items()}  # a load that got through would change every value
    want = []
    for name, (edit, words) in cases.items():
        if case in (name, "all"):
            edit(sd)
            want += words
    with pytest.raises(ValueError) as e:
        checkpoint.load_state_dict(table, sd, None)
    for w in want:
        assert w in str(e.value), (w, str(e.value))
    assert _same(checkpoint.state_dict(table), before)


def test_calibration_refuses_loaded_weights():
    from paddle3d_b200.dense_head import DenseRPNHead
    car = pp.PointPillars().init_weight(seed=1, device=None)
    car2 = pp.PointPillars().load_state_dict(car.state_dict(), None)
    assert not car.loaded and car2.loaded
    with pytest.raises(RuntimeError, match="loaded from a checkpoint"):
        car2.calibrate_cls_bias(None)
    cpm = cpp.CenterPointPillars().load_state_dict(cpp.CenterPointPillars().init_weight(1, None).state_dict(), None)
    with pytest.raises(RuntimeError, match="loaded from a checkpoint"):
        cpm.calibrate_heatmap_bias(None)
    assert not DenseRPNHead().loaded
