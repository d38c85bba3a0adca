"""CPU: the KITTI geometry and formats of paddle3d_b200/kitti.py - the calib reader, the camera frustum planes, the host
cull (the device cull's oracle) against a numba restatement of points_in_convex_polygon_3d_jit, and to_kitti's labels."""
import numpy as np
import pytest

from paddle3d_b200 import kitti, synth


def _calib():
    return kitti.parse_calib(synth.KITTI_CALIB)


def test_read_calib(tmp_path):
    p = tmp_path / "000000.txt"
    p.write_text(synth.KITTI_CALIB)
    c = kitti.read_calib(p)
    assert set(c) == {"P0", "P1", "P2", "P3", "R0_rect", "Tr_velo_to_cam"}
    assert all(m.shape == (4, 4) and m.dtype == np.float64 for m in c.values())
    assert c["P2"][0, 0] == 721.5377 and c["P2"][2, 3] == 2.745884e-03 and np.array_equal(c["P2"][3], [0, 0, 0, 1])
    assert c["R0_rect"][3, 3] == 1.0 and c["R0_rect"][0, 1] == 9.837760e-03 and c["R0_rect"][0, 3] == 0.0
    assert c["Tr_velo_to_cam"][2, 3] == -2.717806e-01
    lines = synth.KITTI_CALIB.splitlines()
    for key in ("R0_rect", "Tr_velo_to_cam", "P2"):
        p.write_text("\n".join(line for line in lines if not line.startswith(key + ":")))
        with pytest.raises(ValueError, match=key):
            kitti.read_calib(p)
    p.write_text("\n".join(line + " 1.0" if line.startswith("P2:") else line for line in lines))
    with pytest.raises(ValueError, match="P2"):
        kitti.read_calib(p)


def test_image_shape(tmp_path):
    import struct
    import zlib
    p = tmp_path / "a.png"
    ihdr = struct.pack(">IIBBBBB", 1224, 370, 8, 2, 0, 0, 0)
    p.write_bytes(b"\x89PNG\r\n\x1a\n" + struct.pack(">I", 13) + b"IHDR" + ihdr +
                  struct.pack(">I", zlib.crc32(b"IHDR" + ihdr)))
    assert kitti.image_shape(p) == (370, 1224)
    assert kitti.image_shape(None) == (375, 1242)
    (tmp_path / "b.png").write_bytes(b"GIF89a" + bytes(20))
    with pytest.raises(ValueError):
        kitti.image_shape(tmp_path / "b.png")


@pytest.mark.parametrize("shape", [(375, 1242), (370, 1224), (512, 1392)])
def test_frustum_corners_project_to_image_corners(shape):
    c = _calib()
    corners = kitti.frustum_corners(c, shape)
    m = c["P2"] @ c["R0_rect"] @ c["Tr_velo_to_cam"]
    h = np.concatenate([corners, np.ones((8, 1))], 1) @ m.T
    uv, depth = h[:, :2] / h[:, 2:3], h[:, 2]
    H, W = shape
    want = np.array([[0, 0], [0, H], [W, H], [W, 0]] * 2, np.float64)
    assert np.abs(uv - want).max() <= 1e-9 * max(H, W)
    assert np.allclose(depth[:4], kitti.NEAR_CLIP, rtol=1e-9, atol=0) and np.allclose(depth[4:], kitti.FAR_CLIP, rtol=1e-9)


def _cam_to_lidar(c, xyz_rect):
    return kitti.camera_to_lidar(np.asarray(xyz_rect, np.float64).reshape(-1, 3), c["R0_rect"], c["Tr_velo_to_cam"])


def test_cull_keeps_the_view_and_drops_the_rest():
    c = _calib()
    shape = (375, 1242)
    planes = kitti.frustum_planes(c, shape)
    C, R, T = kitti.projection_matrix_to_crt(c["P2"])

    def pixel_point(u, v, depth):
        """The LiDAR point that the reference's camera model places at pixel (u, v) and the given depth."""
        x = (np.array([u, v]) - C[0:2, 2]) * depth / np.array([C[0, 0], C[1, 1]])
        cam = np.linalg.inv(R) @ (np.array([x[0], x[1], depth]) - T)
        return _cam_to_lidar(c, cam)[0]

    ahead = np.array([[10.0, 0.0, 0.0, 0.5]], np.float32)  # on the optical axis (LiDAR x), 10 m ahead
    assert kitti.camera_visible_mask(ahead, planes).all()
    H, W = shape
    eps = 1e-3
    dropped = [[-10.0, 0.0, 0.0], [-0.5, 0.0, 0.0], [0.0, 0.0, 0.0]]  # behind the camera, at the sensor
    for u, v in ((-eps, H / 2), (W + eps, H / 2), (W / 2, -eps), (W / 2, H + eps)):
        dropped.append(pixel_point(u, v, 10.0))  # just past each image edge
    dropped.append(pixel_point(W / 2, H / 2, 100.5))  # beyond the far plane
    pts = np.concatenate([np.array(dropped, np.float32), np.zeros((len(dropped), 1), np.float32)], 1)
    assert not kitti.camera_visible_mask(pts, planes).any()
    inside = [pixel_point(u, v, 10.0) for u, v in ((eps * 10, H / 2), (W - eps * 10, H / 2), (W / 2, 1.0))]
    assert kitti.camera_visible_mask(np.array(inside, np.float32), planes).all()
    # exactly on each plane (value 0 in float64) is dropped, a hair inside is kept
    pt = np.array([[3.0, 0.0, 0.0, 0.0]], np.float32)
    for j in range(6):
        on = np.zeros((6, 4))
        on[:, 3] = -1.0
        on[j] = (1.0, 0.0, 0.0, -3.0)
        assert not kitti.camera_visible_mask(pt, on)[0]
        on[j, 3] = -3.0 - 1e-9
        assert kitti.camera_visible_mask(pt, on)[0]
    nan = np.array([[np.nan, 0, 0, 0], [0, np.nan, 0, 0], [0, 0, np.nan, 0]], np.float32)
    assert kitti.camera_visible_mask(nan, planes).all()  # the reference's `sign >= 0` is false on NaN
    inf = np.array([[np.inf, 0, 0, 0], [-np.inf, 0, 0, 0], [0, np.inf, 0, 0]], np.float32)
    assert not kitti.camera_visible_mask(inf, planes).any()


def test_cull_equals_numba_points_in_convex_polygon():
    """remove_camera_invisible bit for bit against points_in_convex_polygon_3d_jit restated under numba, on a 115k-point
    raw scan: the fp64 promotion of fp32 points and the unfused arithmetic are pinned."""
    numba = pytest.importorskip("numba")

    @numba.njit
    def points_in_convex_polygon_3d_jit(points, normal_vec, d):
        n = points.shape[0]
        ret = np.ones(n, dtype=np.bool_)
        for i in range(n):
            for k in range(normal_vec.shape[0]):
                sign = (points[i, 0] * normal_vec[k, 0] + points[i, 1] * normal_vec[k, 1] +
                        points[i, 2] * normal_vec[k, 2] + d[k])
                if sign >= 0:
                    ret[i] = False
                    break
        return ret

    cloud, c, shape = synth.kitti_raw_cloud(5)
    assert len(cloud) > 100000
    planes = kitti.frustum_planes(c, shape)
    rng = np.random.default_rng(0)
    want = points_in_convex_polygon_3d_jit(cloud[:, :3], np.ascontiguousarray(planes[:, :3]),
                                           np.ascontiguousarray(planes[:, 3]))
    got = kitti.camera_visible_mask(cloud, planes)
    assert np.array_equal(got, want) and 10000 < got.sum() < 30000
    assert np.array_equal(kitti.remove_camera_invisible(cloud, planes), cloud[want])
    # rounding-sensitive rows: fp32 points on the frustum's edges and faces, within a few ulps of its planes
    corners = kitti.frustum_corners(c, shape)
    t = rng.uniform(0, 1, size=(20000, 1))
    a, b = corners[rng.integers(0, 8, 20000)], corners[rng.integers(0, 8, 20000)]
    edge = (a + t * (b - a)).astype(np.float32)
    edge = np.concatenate([edge, np.zeros((len(edge), 1), np.float32)], 1)
    want = points_in_convex_polygon_3d_jit(edge[:, :3], np.ascontiguousarray(planes[:, :3]),
                                           np.ascontiguousarray(planes[:, 3]))
    assert np.array_equal(kitti.camera_visible_mask(edge, planes), want)
    assert 0 < want.sum() < len(want)


def test_to_kitti_hand_computed():
    c = _calib()
    shape = (375, 1242)
    # box straight ahead: 20 m in front, on the ground, facing along the LiDAR x axis
    boxes = np.array([[20.0, 0.0, -0.9, 1.6, 3.9, 1.56, 0.3],      # ahead
                      [8.0, 7.0, -0.9, 1.6, 3.9, 1.56, 0.0],       # straddles the left image edge
                      [10.0, 30.0, -0.9, 1.6, 3.9, 1.56, 0.0]],    # far to the left: wholly outside the image
                     np.float32)
    scores = np.array([0.9, 0.5, 0.7], np.float32)
    labels = np.array([0, 0, 0])
    a = kitti.to_kitti(boxes, scores, labels, c, shape, ("Car",))
    assert list(a["name"]) == ["Car", "Car"] and np.allclose(a["score"], [0.9, 0.5])
    # location: the box centre through R0_rect . Tr_velo_to_cam (the bottom centre in the camera frame is the LiDAR
    # centre: SECOND keeps the LiDAR z as given)
    m = c["R0_rect"] @ c["Tr_velo_to_cam"]
    for i in range(2):
        loc = (m @ np.append(boxes[i, :3].astype(np.float64), 1.0))[:3]
        assert np.allclose(a["location"][i], loc, rtol=0, atol=1e-12)
        assert np.allclose(a["dimensions"][i], boxes[i, [5, 3, 4]])  # h w l
        assert a["rotation_y"][i] == np.float64(boxes[i, 6])
        assert np.isclose(a["alpha"][i], -np.arctan2(-float(boxes[i, 1]), float(boxes[i, 0])) + float(boxes[i, 6]))
        back = kitti.camera_to_lidar(a["location"][i:i + 1], c["R0_rect"], c["Tr_velo_to_cam"])[0]
        assert np.allclose(back, boxes[i, :3], atol=1e-9)  # lidar -> camera -> lidar
    # the 2-D box of the box ahead: min / max of its eight corners projected through P2, inside the image
    cam = kitti.box_lidar_to_camera(boxes[:1].astype(np.float64), c["R0_rect"], c["Tr_velo_to_cam"])
    x, y, z, l, h, w, r = cam[0]
    corners = []
    for dx, dy, dz in [(sx, sy, sz) for sx in (-0.5, 0.5) for sy in (-1.0, 0.0) for sz in (-0.5, 0.5)]:
        px, py, pz = dx * l, dy * h, dz * w
        corners.append([x + np.cos(r) * px + np.sin(r) * pz, y + py, z - np.sin(r) * px + np.cos(r) * pz])
    uvw = np.concatenate([np.array(corners), np.ones((8, 1))], 1) @ c["P2"][:3].T
    uv = uvw[:, :2] / uvw[:, 2:]
    assert np.allclose(a["bbox"][0], [uv[:, 0].min(), uv[:, 1].min(), uv[:, 0].max(), uv[:, 1].max()], atol=1e-9)
    assert 0 < a["bbox"][0, 0] < a["bbox"][0, 2] < 1242 and 0 < a["bbox"][0, 1] < a["bbox"][0, 3] < 375
    # the box to the left is clipped at u = 0
    assert a["bbox"][1, 0] == 0.0 and a["bbox"][1, 2] > 0
    assert np.isclose(a["alpha"][1], -np.arctan2(-7.0, 8.0))
    empty = kitti.to_kitti(np.zeros((0, 7)), np.zeros(0), np.zeros(0, int), c, shape)
    assert len(empty["name"]) == 0 and kitti.format_label_lines(empty) == []


def test_label_line_format(tmp_path):
    annos = dict(name=np.array(["Pedestrian"], dtype=object), alpha=np.array([-1.2345678]),
                 bbox=np.array([[712.4, 143.0, 810.73, 307.92]]), dimensions=np.array([[1.89, 0.48, 1.2]]),
                 location=np.array([[1.84, 1.47, 8.41]]), rotation_y=np.array([0.01]), score=np.array([0.87654321]))
    want = "Pedestrian 0.0000 0 -1.2346 712.4000 143.0000 810.7300 307.9200 1.8900 0.4800 1.2000 1.8400 1.4700 " \
           "8.4100 0.0100 0.8765"
    assert kitti.format_label_lines(annos) == [want]
    assert len(want.split()) == 16
    kitti.write_label_file(tmp_path / "000001.txt", annos)
    assert (tmp_path / "000001.txt").read_text() == want + "\n"
