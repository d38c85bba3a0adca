"""CPU suite for BEVDet4D: host-side argument checks of p3d_bev_shift_h16 (every call here is refused before it reaches
the device), the oracle's shift_feature against a torch fp64 restatement of BEVDet4D's gen_grid + F.grid_sample, the
kernel's fp32 restatement and pack_shift against it, and the model's shapes and FLOP count."""
import ctypes

import numpy as np
import pytest

from bevdet4d_oracle import shift_feature, shift_h16_fp32


def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib.lib()


def test_shift_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16  # 16-byte aligned host pointer, never dereferenced
    f = L.p3d_bev_shift_h16

    def call(inp=p, B=1, h=8, w=8, in_c=96, c=80, tf=p, out=p, out_c=160, c0=80):
        return f(inp, B, h, w, in_c, c, tf, out, out_c, c0, None, None)
    assert call(c=72) == -1             # C % 16
    assert call(c=0) == -1
    assert call(c=112) == -1            # more channels than the input rows hold
    assert call(in_c=80) == -1          # input rows of whole 32-channel groups
    assert call(out_c=144) == -1        # out_C % 32
    assert call(c0=72) == -1            # out_c0 % 16
    assert call(c0=96) == -1            # past out_C
    assert call(h=1) == -1 and call(w=1) == -1 and call(B=0) == -1
    assert call(inp=p + 8) == -1 and call(out=p + 8) == -1 and call(tf=p + 2) == -1  # alignment
    assert call(inp=None) == -1 and call(out=None) == -1 and call(tf=None) == -1


# ------------------------------------------------------------------------------------------------ the shift's maths
def _torch_shift(feat, curr, prev, bda, lower, interval):
    """BEVDet4D.shift_feature / gen_grid as BEVDet writes it, in torch fp64."""
    import torch
    import torch.nn.functional as F
    feat, curr, prev, bda = [torch.from_numpy(np.asarray(a, np.float64)) for a in (feat, curr, prev, bda)]
    n, c, h, w = feat.shape
    xs = torch.linspace(0, w - 1, w, dtype=feat.dtype).view(1, w).expand(h, w)
    ys = torch.linspace(0, h - 1, h, dtype=feat.dtype).view(h, 1).expand(h, w)
    grid = torch.stack((xs, ys, torch.ones_like(xs)), -1).view(1, h, w, 3).expand(n, h, w, 3).view(n, h, w, 3, 1)
    bda_ = torch.zeros((n, 1, 4, 4), dtype=grid.dtype)
    bda_[:, :, :3, :3] = bda.unsqueeze(1)
    bda_[:, :, 3, 3] = 1
    c02l0 = bda_.matmul(curr[:, 0:1])
    c12l0 = bda_.matmul(prev[:, 0:1])
    l02l1 = c02l0.matmul(torch.inverse(c12l0))[:, 0, :, :].view(n, 1, 1, 4, 4)
    keep = [True, True, False, True]
    l02l1 = l02l1[:, :, :, keep, :][:, :, :, :, keep]
    feat2bev = torch.zeros((3, 3), dtype=grid.dtype)
    feat2bev[0, 0], feat2bev[1, 1] = interval[0], interval[1]
    feat2bev[0, 2], feat2bev[1, 2] = lower[0], lower[1]
    feat2bev[2, 2] = 1
    tf = torch.inverse(feat2bev.view(1, 3, 3)).matmul(l02l1).matmul(feat2bev.view(1, 3, 3))
    grid = tf.matmul(grid)
    norm = torch.tensor([w - 1.0, h - 1.0], dtype=feat.dtype)
    grid = grid[:, :, :, :2, 0] / norm.view(1, 1, 1, 2) * 2.0 - 1.0
    return F.grid_sample(feat, grid, mode="bilinear", padding_mode="zeros", align_corners=True).numpy(), tf[:, 0, 0].numpy()


def _drives():
    """(name, sensor2keyego curr, prev [1, N, 4, 4], bda [1, 3, 3]) from a camera rig and synth.ego_poses motions."""
    from paddle3d_b200 import synth
    from paddle3d_b200.ops import bev_pool_v2 as bp
    out = []
    for name, seed, bda, speed, yaw_rate in (("identity", 1, False, 0.0, 0.0), ("sub-cell", 2, False, 0.5, 0.0),
                                             ("yaw 5 deg + 2 m", 3, False, 4.0, np.radians(10.0)),
                                             ("bda flip / rotation", 4, True, 7.0, 0.2),
                                             ("half out", 5, True, 16.0, 0.1)):
        rig = synth.camera_rig(seed, bda=bda)
        poses = synth.ego_poses(2, speed=speed, yaw_rate=yaw_rate)
        e2g = [np.broadcast_to(p, (1, 6, 4, 4)) for p in poses]
        s2e = rig["sensor2ego"].astype(np.float64)
        curr = bp.sensor2keyegos(s2e, e2g[1], e2g[1])
        prev = bp.sensor2keyegos(s2e, e2g[0], e2g[1])
        out.append((name, curr, prev, rig["bda"].astype(np.float64)))
    return out


GRID = ((-8.0, -6.4), (0.8, 0.8))  # a 20 x 16 BEV of 0.8 m cells


@pytest.mark.parametrize("k", range(5))
def test_oracle_shift_matches_torch(k):
    name, curr, prev, bda = _drives()[k]
    rng = np.random.default_rng(k)
    feat = rng.normal(size=(1, 5, 16, 20))
    want, _ = _torch_shift(feat, curr, prev, bda, *GRID)
    got = shift_feature(feat, curr, prev, bda, *GRID)
    np.testing.assert_allclose(got, want, rtol=0, atol=1e-12, err_msg=name)
    if name == "identity":
        np.testing.assert_allclose(got, feat, atol=1e-12)
    if name == "half out":
        zero = np.all(want == 0, axis=1)
        assert 0.2 < zero.mean() < 0.9, zero.mean()
    # the kernel's fp32 order at pack_shift's descriptor: within fp32 rounding of the coordinates (a few 1e-6 pixel
    # moves a sample by that fraction of the local gradient, bounded by 2 max |x| per pixel)
    from paddle3d_b200.ops import bev_pool_v2 as bp
    tf6 = bp.pack_shift(curr, prev, bda, *GRID)
    f32 = feat.astype(np.float32)
    got32 = shift_h16_fp32(f32.transpose(0, 2, 3, 1), tf6).transpose(0, 3, 1, 2)
    want32 = shift_feature(f32, curr, prev, bda, *GRID)
    assert np.abs(got32 - want32).max() <= 1e-4 * np.abs(f32).max(), (name, np.abs(got32 - want32).max())


def test_pack_shift_matches_torch_chain():
    from paddle3d_b200.ops import bev_pool_v2 as bp
    for name, curr, prev, bda in _drives():
        _, tf = _torch_shift(np.zeros((1, 1, 16, 20)), curr, prev, bda, *GRID)
        np.testing.assert_allclose(bp.shift_matrix(curr, prev, bda, *GRID), tf, rtol=0, atol=1e-9, err_msg=name)
        tf6 = bp.pack_shift(curr, prev, bda, *GRID)
        assert tf6.dtype == np.float32 and tf6.shape == (1, 6)
        assert np.array_equal(tf6, tf[:, :2].reshape(1, 6).astype(np.float32)) or \
            np.abs(tf6 - tf[:, :2].reshape(1, 6)).max() <= 1e-6 * max(1.0, np.abs(tf).max()), name


def test_shift_fp32_special_cases():
    """A huge or NaN translation gives zeros; the start frame's transform (prev = curr) is the identity to fp32."""
    from paddle3d_b200.ops import bev_pool_v2 as bp
    x = np.random.default_rng(0).normal(size=(1, 16, 20, 16)).astype(np.float32)
    for t in (1e30, np.nan, -np.inf):
        tf6 = np.array([[1, 0, t, 0, 1, 0]], np.float32)
        assert not shift_h16_fp32(x, tf6).any()
    _, curr, _, bda = _drives()[3]
    tf6 = bp.pack_shift(curr, curr, bda, *GRID)
    np.testing.assert_allclose(tf6, [[1, 0, 0, 0, 1, 0]], atol=1e-12)
    # the fp32 normalise / unnormalise round trip moves a sample by up to a few 1e-6 pixel (grid_sample's own rounding)
    np.testing.assert_allclose(shift_h16_fp32(x, tf6), x, rtol=0, atol=2e-5 * np.abs(x).max())


def test_model_shapes_and_flops(oracle_mod):
    from bevdet4d_oracle import CpuBEVDet4D
    from paddle3d_b200.bevdet import CONFIG_4D, BEVDet, BEVDet4D
    m = BEVDet4D(device="cpu").init_weight(seed=3, device=False)
    assert m.image_shape == (1, 128, 128, 96) and m.enc_shape == (1, 128, 128, 160)
    assert (m.bev_C, m.hist_C) == (80, 96)
    fl = m.flops()
    pre = 5 * 2.0 * 128 * 128 * 9 * 80 * 80
    bb = 0.0
    cin = 160
    for s, cout in enumerate((160, 320, 640)):
        px = (64 >> s) ** 2
        bb += 2.0 * px * 9 * (2 * cin * cout + 3 * cout * cout)
        cin = cout
    assert fl["pre_process"] == pytest.approx(pre) and fl["backbone"] == pytest.approx(bb)
    single = BEVDet(device="cpu").flops()
    assert fl["fpn"] == pytest.approx(single["fpn"]) and fl["head"] == pytest.approx(single["head"])
    assert fl["total"] == pytest.approx(single["total"] + pre + 2.0 * 64 * 64 * 9 * 2 * 80 * 160)
    assert 170e9 < fl["total"] < 178e9
    w = m.export_numpy()
    assert [[b["down"] is not None for b in st] for st in w["pre_process"]] == [[True, False]]
    assert w["pre_process"][0][0]["conv1"]["weight"].shape == (80, 80, 3, 3)
    assert w["backbone"][0][0]["conv1"]["weight"].shape == (160, 160, 3, 3)
    assert all(c.cin_pad == 96 for c in m.pre_process.convs())
    with pytest.raises(ValueError, match="num_adj"):
        BEVDet4D(dict(CONFIG_4D, num_adj=2), device="cpu")
    # the oracle's pre_process keeps 80 channels at the BEV's size, ReLU after the residual
    cpu = CpuBEVDet4D(w, m.test_cfg, m.label_off)
    bev = np.random.default_rng(0).normal(size=(1, 80, 16, 16)).astype(np.float32)
    y = cpu.pre_process(bev)
    assert y.shape == (1, 80, 16, 16) and y.min() >= 0.0
    feats = cpu.backbone(np.concatenate([y, y], 1))
    assert [f.shape for f in feats] == [(1, 160, 8, 8), (1, 320, 4, 4), (1, 640, 2, 2)]
