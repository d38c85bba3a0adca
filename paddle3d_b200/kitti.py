"""KITTI object-split geometry and formats around the PointPillars and CenterPoint-pillars KITTI frames (numpy, float64).

PARITY UNPINNED: every convention here is recalled from the references below, not checked against a checkout of them.

  read_calib               SECOND kitti_common.get_kitti_image_info (calib part, extend_matrix): P0..P3, R0_rect and
                           Tr_velo_to_cam of a `calib/*.txt`, padded to 4 x 4.
  image_shape              the (H, W) that Paddle3D's RemoveCameraInvisiblePointsKITTI reads with cv2.imread(...).shape[:2],
                           here from the PNG IHDR chunk (the pixels are never decoded); DEFAULT_IMAGE_SHAPE without one.
  frustum_planes           SECOND box_np_ops.remove_outside_points (Paddle3D transforms RemoveCameraInvisiblePointsKITTI):
                           projection_matrix_to_CRT_kitti -> get_frustum -> camera_to_lidar -> corner_to_surfaces_3d ->
                           surface_equ_3d_jitv2.
  remove_camera_invisible  points_in_convex_polygon_3d_jit: the host cull, and the oracle of the device cull
                           (csrc/sweep_merge.cu, p3d_merge_sweeps_frustum).
  to_kitti                 SECOND's convert_detection_to_kitti_annos / Paddle3D's KITTI result conversion:
                           box_lidar_to_camera, center_to_corner_box3d (origin (0.5, 1.0, 0.5), axis 1), the 2-D box of
                           the corners projected through P2 (homogeneous coordinate 1), dropped when wholly outside the
                           image and clipped to it, alpha = -arctan2(-y_lidar, x_lidar) + r.
  centerpoint_to_lidar_boxes
                           Paddle3D CenterPoint._parse_results_to_sample (paddle3d/models/detection/centerpoint/
                           centerpoint.py) and the KITTI metric's box conversion: the centerpoint_postprocess op's
                           (x, y, z_centre, d0, d1, d2, rot) with dims[0:2] swapped, rot -> -(rot + pi / 2) and the box
                           declared centred (origin (0.5, 0.5, 0.5)), so z drops by h / 2 to the bottom face.
  format_label_lines       kitti_common.kitti_result_line (4 decimals): the 16-field KITTI result line; truncation and
                           occlusion are written as 0.
"""
import struct

import numpy as np

DEFAULT_IMAGE_SHAPE = (375, 1242)  # (H, W) the reference assumes when no image is read
NEAR_CLIP, FAR_CLIP = 0.001, 100.0
# KITTI type names in label order of the two PointPillars models and of CenterPoint-pillars KITTI (tasks [Car],
# [Pedestrian, Cyclist]: synth.CP_PILLARS_KITTI_TASKS)
CLASS_NAMES = {"car": ("Car",), "ped_cyclist": ("Cyclist", "Pedestrian"), "centerpoint": ("Car", "Pedestrian", "Cyclist")}

_CALIB_KEYS = {"P0": (3, 4), "P1": (3, 4), "P2": (3, 4), "P3": (3, 4), "R0_rect": (3, 3), "Tr_velo_to_cam": (3, 4)}


def _extend(m):
    out = np.eye(4, dtype=np.float64)
    out[:m.shape[0], :m.shape[1]] = m
    return out


def parse_calib(text, source="calib"):
    """read_calib on the file's text."""
    vals = {}
    for line in text.splitlines():
        if ":" in line:
            k, v = line.split(":", 1)
            vals[k.strip()] = v.split()
    calib = {}
    for key, shape in _CALIB_KEYS.items():
        if key not in vals:
            raise ValueError("%s: no %s" % (source, key))
        try:
            m = np.array([float(x) for x in vals[key]], np.float64)
        except ValueError:
            raise ValueError("%s: %s is not a list of numbers" % (source, key)) from None
        if m.size != shape[0] * shape[1]:
            raise ValueError("%s: %s has %d values, expected %d" % (source, key, m.size, shape[0] * shape[1]))
        calib[key] = _extend(m.reshape(shape))
    return calib


def read_calib(path):
    """A KITTI object calib file -> {"P0".."P3", "R0_rect", "Tr_velo_to_cam": 4 x 4 float64}.  A missing or misshapen
    key raises ValueError naming it."""
    with open(path) as f:
        return parse_calib(f.read(), str(path))


def image_shape(png_path=None):
    """(H, W) of a PNG from its IHDR chunk; DEFAULT_IMAGE_SHAPE when png_path is None."""
    if png_path is None:
        return DEFAULT_IMAGE_SHAPE
    with open(png_path, "rb") as f:
        head = f.read(24)
    if len(head) < 24 or head[:8] != b"\x89PNG\r\n\x1a\n" or head[12:16] != b"IHDR":
        raise ValueError("%s: not a PNG file" % png_path)
    w, h = struct.unpack(">II", head[16:24])
    return int(h), int(w)


def projection_matrix_to_crt(proj):
    """P = C [R | T] with C upper triangular (QR of inv(P[:3, :3])).  Returns (C, R, T)."""
    cr, ct = proj[0:3, 0:3], proj[0:3, 3]
    rinv, cinv = np.linalg.qr(np.linalg.inv(cr))
    return np.linalg.inv(cinv), np.linalg.inv(rinv), cinv @ ct


def get_frustum(bbox_image, C, near_clip=NEAR_CLIP, far_clip=FAR_CLIP):
    """The 8 corners [8, 3] of the image box's view frustum in the rectified camera frame (near 4, then far 4)."""
    fku, fkv = C[0, 0], -C[1, 1]
    u0v0 = C[0:2, 2]
    z = np.array([near_clip] * 4 + [far_clip] * 4, dtype=C.dtype)[:, np.newaxis]
    b = bbox_image
    box = np.array([[b[0], b[1]], [b[0], b[3]], [b[2], b[3]], [b[2], b[1]]], dtype=C.dtype)
    near = (box - u0v0) / np.array([fku / near_clip, -fkv / near_clip], dtype=C.dtype)
    far = (box - u0v0) / np.array([fku / far_clip, -fkv / far_clip], dtype=C.dtype)
    return np.concatenate([np.concatenate([near, far], axis=0), z], axis=1)


def lidar_to_camera(points, r_rect, velo2cam):
    p = np.concatenate([points, np.ones(points.shape[:-1] + (1,))], axis=-1)
    return (p @ (r_rect @ velo2cam).T)[..., :3]


def camera_to_lidar(points, r_rect, velo2cam):
    p = np.concatenate([points, np.ones(points.shape[:-1] + (1,))], axis=-1)
    return (p @ np.linalg.inv((r_rect @ velo2cam).T))[..., :3]


def frustum_corners(calib, shape=DEFAULT_IMAGE_SHAPE):
    """The 8 frustum corners [8, 3] in the LiDAR frame (remove_outside_points up to corner_to_surfaces_3d)."""
    C, R, T = projection_matrix_to_crt(calib["P2"])
    fr = get_frustum([0, 0, shape[1], shape[0]], C)
    fr = fr - T
    fr = (np.linalg.inv(R) @ fr.T).T
    return camera_to_lidar(fr, calib["R0_rect"], calib["Tr_velo_to_cam"])


# corner_to_surfaces_3d: the corner indices of each of the six faces
_SURFACES = ((0, 1, 2, 3), (7, 6, 5, 4), (0, 3, 7, 4), (1, 5, 6, 2), (0, 4, 5, 1), (3, 2, 6, 7))


def frustum_planes(calib, shape=DEFAULT_IMAGE_SHAPE):
    """Six planes [6, 4] float64 (a, b, c, d), normals outward: a LiDAR point (x, y, z) is inside the camera's view iff
    ((x a + y b) + z c) + d < 0 for every plane.  surface_equ_3d_jitv2's arithmetic, one operation at a time."""
    corners = frustum_corners(calib, shape)
    out = np.zeros((6, 4), np.float64)
    for j, idx in enumerate(_SURFACES):
        s0, s1, s2 = (corners[i] for i in idx[:3])
        sv0 = [float(s0[k]) - float(s1[k]) for k in range(3)]
        sv1 = [float(s1[k]) - float(s2[k]) for k in range(3)]
        n = (sv0[1] * sv1[2] - sv0[2] * sv1[1], sv0[2] * sv1[0] - sv0[0] * sv1[2], sv0[0] * sv1[1] - sv0[1] * sv1[0])
        d = -float(s0[0]) * n[0] - float(s0[1]) * n[1] - float(s0[2]) * n[2]
        out[j] = (n[0], n[1], n[2], d)
    return out


def check_planes(planes):
    """planes as a finite [6, 4] float64 array (ValueError otherwise)."""
    p = np.asarray(planes, np.float64)
    if p.shape != (6, 4) or not np.isfinite(p).all():
        raise ValueError("frustum planes must be a finite [6, 4] array, got shape %s" % (p.shape,))
    return np.ascontiguousarray(p)


def camera_visible_mask(points, planes):
    """The keep mask of remove_camera_invisible.  fp32 x, y, z are widened to float64 (numba's promotion against the
    float64 normals), each product and sum rounded on its own; a row is dropped when any plane gives >= 0, so a NaN row is
    kept (the voxeliser drops it) and a row on a plane is dropped."""
    p = np.asarray(points)
    planes = check_planes(planes)
    x, y, z = (p[:, k].astype(np.float64) for k in range(3))
    keep = np.ones(len(p), bool)
    for a, b, c, d in planes:
        v = ((x * a + y * b) + z * c) + d
        keep &= ~(v >= 0)
    return keep


def remove_camera_invisible(points, planes):
    """points [n, >= 3] -> the rows inside the camera frustum, in order (Paddle3D RemoveCameraInvisiblePointsKITTI)."""
    return np.asarray(points)[camera_visible_mask(points, planes)]


def box_lidar_to_camera(boxes, r_rect, velo2cam):
    """LiDAR (x, y, z, w, l, h, r) -> camera (x, y, z, l, h, w, r)."""
    xyz = lidar_to_camera(boxes[:, 0:3], r_rect, velo2cam)
    w, l, h, r = boxes[:, 3:4], boxes[:, 4:5], boxes[:, 5:6], boxes[:, 6:7]
    return np.concatenate([xyz, l, h, w, r], axis=1)


def camera_box_corners(boxes_cam, origin=(0.5, 1.0, 0.5)):
    """center_to_corner_box3d(locs, (l, h, w), r, origin, axis=1) -> [N, 8, 3]."""
    dims = boxes_cam[:, 3:6]
    norm = np.stack(np.unravel_index(np.arange(8), [2] * 3), axis=1).astype(np.float64)[[0, 1, 3, 2, 4, 5, 7, 6]]
    corners = dims.reshape(-1, 1, 3) * (norm - np.array(origin, np.float64)).reshape(1, 8, 3)
    s, c = np.sin(boxes_cam[:, 6]), np.cos(boxes_cam[:, 6])
    zeros, ones = np.zeros_like(c), np.ones_like(c)
    rot_t = np.stack([[c, zeros, -s], [zeros, ones, zeros], [s, zeros, c]])
    return np.einsum("aij,jka->aik", corners, rot_t) + boxes_cam[:, :3].reshape(-1, 1, 3)


def project_to_image(points, proj):
    p = np.concatenate([points, np.ones(points.shape[:-1] + (1,))], axis=-1) @ proj.T
    return p[..., :2] / p[..., 2:3]


def to_kitti(boxes, scores, labels, calib, shape=DEFAULT_IMAGE_SHAPE, class_names=CLASS_NAMES["car"]):
    """LiDAR-frame detections (boxes [K, 7] (x, y, z, w, l, h, theta), scores [K], labels [K]) -> KITTI annotations: a
    dict of arrays name, alpha, bbox [K', 4] (left, top, right, bottom), dimensions [K', 3] (h, w, l), location [K', 3]
    (camera frame, bottom centre), rotation_y, score.  A box whose projected 2-D box lies wholly outside the image is
    dropped; the others are clipped to it."""
    boxes = np.asarray(boxes, np.float64).reshape(-1, 7)
    scores = np.asarray(scores, np.float64).reshape(-1)
    labels = np.asarray(labels).reshape(-1)
    cam = box_lidar_to_camera(boxes, calib["R0_rect"], calib["Tr_velo_to_cam"])
    uv = project_to_image(camera_box_corners(cam), calib["P2"])
    bbox = np.concatenate([uv.min(axis=1), uv.max(axis=1)], axis=1) if len(boxes) else np.zeros((0, 4))
    H, W = shape
    keep = ~((bbox[:, 0] > W) | (bbox[:, 1] > H) | (bbox[:, 2] < 0) | (bbox[:, 3] < 0))
    bbox = bbox[keep]
    bbox[:, 2:] = np.minimum(bbox[:, 2:], [W, H])
    bbox[:, :2] = np.maximum(bbox[:, :2], 0.0)
    cam, lid = cam[keep], boxes[keep]
    return dict(name=np.array([class_names[int(c)] for c in labels[keep]], dtype=object),
                alpha=-np.arctan2(-lid[:, 1], lid[:, 0]) + cam[:, 6], bbox=bbox, dimensions=cam[:, [4, 5, 3]],
                location=cam[:, :3], rotation_y=cam[:, 6], score=scores[keep])


def centerpoint_to_lidar_boxes(boxes):
    """CenterPoint boxes [K, 7] (x, y, z_centre, d0, d1, d2, rot), as the centerpoint_postprocess op and the velocity-free
    CenterPoint-pillars KITTI frame return them, -> the LiDAR boxes [K, 7] (x, y, z_bottom, w, l, h, theta) to_kitti
    takes: (x, y, z - d2 / 2, d1, d0, d2, -(rot + pi / 2)), float64."""
    b = np.asarray(boxes, np.float64).reshape(-1, 7)
    return np.stack([b[:, 0], b[:, 1], b[:, 2] - b[:, 5] / 2, b[:, 4], b[:, 3], b[:, 5], -(b[:, 6] + np.pi / 2)], axis=1)


def format_label_lines(annos):
    """KITTI result lines: type truncated occluded alpha left top right bottom h w l x y z rotation_y score."""
    lines = []
    for i in range(len(annos["name"])):
        vals = [annos["alpha"][i], *annos["bbox"][i], *annos["dimensions"][i], *annos["location"][i],
                annos["rotation_y"][i], annos["score"][i]]
        lines.append(" ".join([annos["name"][i], "0.0000", "0"] + ["%.4f" % float(v) for v in vals]))
    return lines


def write_label_file(path, annos):
    """One KITTI result file (one line per detection; empty without detections)."""
    lines = format_label_lines(annos)
    with open(path, "w") as f:
        f.write("".join(line + "\n" for line in lines))
