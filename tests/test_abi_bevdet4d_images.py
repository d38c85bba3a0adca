"""CPU suite for BEVDet4D from camera images: the model's config checks, its seeded weights against both parents', its
FLOP count, and the pose bookkeeping of a drive (bevdet.drive_mats) against sensor2keyegos chains and the oracle's
shift matrix."""
import numpy as np
import pytest

from bevdet4d_oracle import shift_matrix


@pytest.mark.parametrize("bad,match", [(dict(num_adj=2), "num_adj"), (dict(input_size=(250, 704)), "multiple of 32"),
                                       (dict(input_size=(256, 700)), "multiple of 32"), (dict(downsample=8), "downsample")])
def test_config_checks(bad, match):
    from paddle3d_b200.bevdet import CONFIG_4D_IMG, BEVDet4DFromImages
    with pytest.raises(ValueError, match=match):
        BEVDet4DFromImages(dict(CONFIG_4D_IMG, **bad), device="cpu")


def test_crop_must_match_input_size():
    from paddle3d_b200.bevdet import CONFIG_4D_IMG, DATA_CONFIG, BEVDet4DFromImages
    with pytest.raises(ValueError, match="crops"):
        BEVDet4DFromImages(dict(CONFIG_4D_IMG, data_config=dict(DATA_CONFIG, input_size=(128, 352))), device="cpu")


def _equal(a, b, path="w"):
    """Nested dicts / lists / arrays equal, element for element."""
    if isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            _equal(a[k], b[k], "%s.%s" % (path, k))
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _equal(x, y, "%s[%d]" % (path, i))
    elif isinstance(a, np.ndarray):
        assert a.dtype == b.dtype and np.array_equal(a, b), path
    else:
        assert a == b, path


def test_seeded_weights_equal_both_parents():
    from paddle3d_b200.bevdet import BEVDet4D, BEVDet4DFromImages, BEVDetFromImages
    seed = 5
    m = BEVDet4DFromImages(device="cpu").init_weight(seed=seed, bn_gain=1.5, device=False)
    w = m.export_numpy()
    assert "pre_process" in w and "image_encoder" in w
    w4 = BEVDet4D(device="cpu").init_weight(seed=seed, bn_gain=1.5, device=False).export_numpy()
    wi = BEVDetFromImages(device="cpu").init_weight(seed=seed, bn_gain=1.5, device=False).export_numpy()
    _equal(w["image_encoder"], wi["image_encoder"], "image_encoder")
    _equal({k: v for k, v in w.items() if k != "image_encoder"}, w4)
    other = BEVDet4DFromImages(device="cpu").init_weight(seed=seed + 1, device=False).export_numpy()
    assert not np.array_equal(other["image_encoder"]["stem"]["weight"], w["image_encoder"]["stem"]["weight"])


def test_flops_frame_total():
    from paddle3d_b200.bevdet import CONFIG_4D, CONFIG_IMG, BEVDet4D, BEVDet4DFromImages, BEVDetFromImages
    fl = BEVDet4DFromImages(device="cpu").flops()
    four = BEVDet4D(CONFIG_4D, device="cpu").flops()
    img = BEVDetFromImages(CONFIG_IMG, device="cpu").flops()
    assert fl["frame_total"] == four["total"] + img["img_total"]
    for k, v in four.items():
        assert fl[k] == v, k
    for k in ("img_stem", "img_layers", "img_backbone", "img_neck", "depth_net", "img_total"):
        assert fl[k] == img[k], k


def _drive(n, rig_seed=3, speed=9.0, yaw_rate=0.25):
    from paddle3d_b200 import synth
    rig = synth.camera_rig(rig_seed, bda=False)
    poses = synth.ego_poses(n, speed=speed, yaw_rate=yaw_rate)
    s2e, k = rig["sensor2ego"][0], rig["cam2imgs"][0]
    return [(None, s2e, np.broadcast_to(p, (6, 4, 4)).copy(), k) for p in poses]


def test_drive_mats():
    """First frame new_sequence; mats[0] and prev_sensor2keyego equal sensor2keyegos chains written out here; the
    shift descriptor of consecutive frames equals rows 0-1 of the oracle's shift matrix; mats[1:] are test_mats'."""
    from paddle3d_b200.bevdet import BEVDet4DFromImages, drive_mats
    from paddle3d_b200.ops import bev_pool_v2 as bp
    m = BEVDet4DFromImages(device="cpu")
    items = _drive(5)
    out = list(drive_mats(iter(items), m.test_mats))
    assert [s[2] for s in out] == [True, False, False, False, False]
    assert out[0][1] is None
    lower, interval, _ = m.vt.grid_args()
    for j, (mats, prev, _) in enumerate(out):
        _, s2e, e2g, k = items[j]
        key = np.linalg.inv(e2g[0].astype(np.float64))
        curr = np.stack([key @ e2g[c] @ s2e[c].astype(np.float64) for c in range(6)])[None]
        np.testing.assert_allclose(mats[0], curr, rtol=0, atol=1e-12)
        np.testing.assert_array_equal(mats[1], k[None])
        want = m.test_mats(curr, k[None], np.eye(3, dtype=np.float32)[None])
        for g, w in zip(mats[2:], want[2:]):
            np.testing.assert_array_equal(g, w)
        np.testing.assert_array_equal(mats[4], np.eye(3)[None])
        if j == 0:
            continue
        _, s2e_p, e2g_p, _ = items[j - 1]
        want_prev = np.stack([key @ e2g_p[c] @ s2e_p[c].astype(np.float64) for c in range(6)])[None]
        np.testing.assert_allclose(prev, want_prev, rtol=0, atol=1e-12)
        tf = shift_matrix(curr, want_prev, mats[4], lower, interval)
        tf6 = m.shift_desc(mats, prev)
        assert np.array_equal(tf6, bp.pack_shift(mats[0], prev, mats[4], lower, interval))
        # pack_shift rounds the fp64 matrix to fp32 once
        np.testing.assert_allclose(tf6, tf[:, :2].reshape(1, 6), rtol=0, atol=1e-6 * max(1.0, np.abs(tf).max()))
        assert np.abs(tf[0, :2, 2]).max() > 1.0  # the ego moved by more than a BEV cell


def test_drive_mats_is_lazy():
    """One item in, one step out: the bookkeeping streams (infer_stream pulls items as the drive goes)."""
    from paddle3d_b200.bevdet import BEVDet4DFromImages, drive_mats
    m = BEVDet4DFromImages(device="cpu")
    items = _drive(3)
    pulled = []

    def gen():
        for it in items:
            pulled.append(1)
            yield it
    g = drive_mats(gen(), m.test_mats)
    next(g)
    assert len(pulled) == 1
    next(g)
    assert len(pulled) == 2
