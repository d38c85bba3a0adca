"""GPU tests of BEVDet and BEVDet4D from JPEG camera files: BEVDetJpegHotPath's boxes bit-equal to BEVDetFrameHotPath fed
Pillow's decode of the same files under both box decodes, captured == eager, lanes in flight == one lane, accelerate;
BEVDet4DJpegHotPath.infer_stream over a drive with a restart == BEVDet4DFrameHotPath.infer_stream on the decoded frames;
a corrupt file failing its frame's result() by camera while the lane's next frame succeeds; and rejections raised
before anything is enqueued."""
import io

import numpy as np
import pytest

from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu
BN_GAIN = 6.0 ** 0.5


def _pil_frames(jpegs):
    """Pillow's decode of the files: uint8 [N, H, W, 3] pinned."""
    import torch
    from PIL import Image
    return torch.from_numpy(np.stack([np.asarray(Image.open(io.BytesIO(f)).convert("RGB")) for f in jpegs])).pin_memory()


def _args(rig):
    return rig["sensor2ego"], rig["cam2imgs"], rig["bda"]


def _equal(a, b):
    import torch
    return len(a) == len(b) and all(torch.equal(x, y) for x, y in zip(a, b))


def _clone(r):
    return [t.clone() for t in r]


@pytest.fixture(scope="module")
def model(cuda):
    """A seeded BEVDetFromImages at 256 x 704 calibrated on the images of Pillow's decode of its first files."""
    import torch
    from paddle3d_b200.bevdet import BEVDetFromImages
    m = BEVDetFromImages(device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    rig = synth.camera_rig(31)
    jpegs = synth.camera_jpegs(7, quality=95)
    imgs = m.images_from_frames(_pil_frames(jpegs).to(cuda))
    m.calibrate_heatmap_bias(m.test_mats(*_args(rig)), imgs)
    torch.cuda.synchronize()
    return dict(m=m, rig=rig, jpegs=jpegs)


@pytest.mark.parametrize("decode", ["default", "bevdet_nms"])
def test_jpeg_lane_equals_frame_lane(cuda, model, decode):
    from paddle3d_b200.bevdet import CONFIG_IMG_BEVDET_NMS, BEVDetFromImages, BEVDetFrameHotPath, BEVDetJpegHotPath
    m = model["m"]
    if decode == "bevdet_nms":
        base = m
        m = BEVDetFromImages(CONFIG_IMG_BEVDET_NMS, device=cuda)
        m.encoder, m.head, m.image_encoder, m.prep_plan = base.encoder, base.head, base.image_encoder, base.prep_plan
    rig, jpegs = model["rig"], model["jpegs"]
    ref = BEVDetFrameHotPath(m, device=cuda).capture(count_nodes=True)
    want = _clone(ref.infer_frames(*_args(rig), _pil_frames(jpegs)))
    hot = BEVDetJpegHotPath(m, device=cuda).capture(count_nodes=True)
    got = _clone(hot.infer_jpegs(*_args(rig), jpegs))
    assert len(want[0]) > 0 and _equal(got, want)
    assert int(hot.h_status[0]) == 0 and not hot.h_jpeg_status.any()
    plan = m.prep_plan
    assert np.array_equal(hot.band.cpu().numpy(), _pil_frames(jpegs).numpy()[:, plan.band[0]:plan.band[1]])
    print("graph nodes: jpeg lane %s, frame lane %s" % (hot.graph_nodes, ref.graph_nodes))


def test_jpeg_lane_eager_lanes_accelerate(cuda, model):
    """Captured == eager (forward_frames on Pillow's decode) with files of other qualities, tables and restart intervals
    on every replay; three lanes sharing the model in flight == one lane; accelerate == full."""
    import torch
    from paddle3d_b200.bevdet import BEVDetFromImages, BEVDetJpegHotPath
    m = model["m"]
    rigs = [synth.camera_rig(40 + i) for i in range(3)]
    files = [synth.camera_jpegs(50, quality=75, optimize=True), synth.camera_jpegs(51, quality=95, restart_marker_blocks=7),
             synth.camera_jpegs(52, quality=90, subsampling=0)]
    hot = BEVDetJpegHotPath(m, device=cuda).capture()
    want = []
    for r, f in zip(rigs, files):
        boxes, scores, labels, counts = m.forward_frames(*_args(r), _pil_frames(f).to(cuda))
        k = int(counts[-1])
        eager = [boxes[:k].cpu(), scores[:k].cpu(), labels[:k].cpu()]
        got = _clone(hot.infer_jpegs(*_args(r), f))
        assert len(eager[0]) > 0 and _equal(got, eager)
        want.append(eager)
    assert not torch.equal(want[0][0], want[1][0])
    lanes = [BEVDetJpegHotPath(m, device=cuda).capture().share_model(hot) for _ in range(3)]
    for rep in range(2):  # the second round deals the frames to other lanes
        for i, lane in enumerate(lanes):
            j = (i + rep) % 3
            lane.launch_jpegs(*_args(rigs[j]), files[j])
        for i, lane in enumerate(lanes):
            assert _equal(lane.result(), want[(i + rep) % 3]), (rep, i)
    acc_model = BEVDetFromImages(accelerate=True, device=cuda)
    acc_model.encoder, acc_model.head, acc_model.image_encoder = m.encoder, m.head, m.image_encoder
    acc_model.prep_plan = m.prep_plan
    acc = BEVDetJpegHotPath(acc_model, device=cuda).capture()
    for i in (0, 0, 1, 0):
        assert _equal(acc.infer_jpegs(*_args(rigs[i]), files[i]), want[i])


def test_corrupt_file_fails_its_frame_only(cuda, model):
    """Truncation after the SOS, random bytes in the entropy-coded segment and an undefined code: the frame's result()
    raises naming the JPEG decode and the camera; the lane's next frame equals a fresh lane's."""
    from paddle3d_b200.bevdet import BEVDetJpegHotPath
    from paddle3d_b200.ops import jpeg
    m, rig, good = model["m"], model["rig"], model["jpegs"]
    fresh = _clone(BEVDetJpegHotPath(m, device=cuda).capture().infer_jpegs(*_args(rig), good))
    lane = BEVDetJpegHotPath(m, device=cuda).capture()
    a = [jpeg.parse(f).ecs[0] for f in good]
    junk = np.random.default_rng(0).integers(0, 256, 4096, dtype=np.uint8).tobytes()
    corrupt = [(2, good[2][:a[2] + 1000] + b"\xff\xd9"),
               (4, good[4][:a[4] + 5000] + junk + good[4][a[4] + 9096:]),
               (1, good[1][:a[1]] + b"\xff\x00" * 8 + good[1][a[1] + 16:])]
    for cam, bad in corrupt:
        files = list(good)
        files[cam] = bad
        lane.launch_jpegs(*_args(rig), files)
        with pytest.raises(RuntimeError, match="JPEG decode failed: camera %d" % cam):
            lane.result()
        assert _equal(lane.infer_jpegs(*_args(rig), good), fresh)


def test_rejections_before_enqueue(cuda, model):
    """Capacity overflow, a rejected header, a wrong size or count: ValueError, and the lane's next frame is unaffected."""
    from paddle3d_b200.bevdet import BEVDetJpegHotPath
    m, rig, good = model["m"], model["rig"], model["jpegs"]
    small = BEVDetJpegHotPath(m, device=cuda, max_bytes=max(len(f) for f in good)).capture()
    want = _clone(small.infer_jpegs(*_args(rig), good))
    big = synth.camera_jpegs(7, quality=100, subsampling=0)
    with pytest.raises(ValueError, match="capacity"):
        small.launch_jpegs(*_args(rig), big)
    prog = list(good)
    buf = io.BytesIO()
    from PIL import Image
    Image.fromarray(synth.camera_frames(7, 1)[0]).save(buf, "JPEG", progressive=True)
    prog[3] = buf.getvalue()
    with pytest.raises(ValueError, match="progressive"):
        small.launch_jpegs(*_args(rig), prog)
    with pytest.raises(ValueError, match="want 900 x 1600"):
        small.launch_jpegs(*_args(rig), synth.camera_jpegs(7, H=450, W=800))
    with pytest.raises(ValueError, match="want 6"):
        small.launch_jpegs(*_args(rig), good[:5])
    assert _equal(small.infer_jpegs(*_args(rig), good), want)


def test_4d_infer_stream(cuda):
    """A drive of four key frames on one lane (the second drive restarts the sequence) from JPEG files with different
    encodings == BEVDet4DFrameHotPath.infer_stream on Pillow's decode of the same files."""
    import torch
    from paddle3d_b200.bevdet import BEVDet4DFrameHotPath, BEVDet4DFromImages, BEVDet4DJpegHotPath, drive_mats
    m = BEVDet4DFromImages(device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    rig = synth.camera_rig(34, bda=False)
    kws = [dict(quality=95), dict(quality=75, optimize=True), dict(quality=90, restart_marker_rows=1),
           dict(quality=95, subsampling=1)]
    jpegs = [synth.camera_jpegs(30 + k, **kw) for k, kw in enumerate(kws)]
    poses = synth.ego_poses(len(kws), speed=8.0, yaw_rate=0.2)
    items = [(j, rig["sensor2ego"][0], np.broadcast_to(p, (m.N, 4, 4)).copy(), rig["cam2imgs"][0])
             for j, p in zip(jpegs, poses)]
    frame_items = [(_pil_frames(j),) + it[1:] for j, it in zip(jpegs, items)]
    mats0, _, _ = next(drive_mats(frame_items, m.test_mats))
    m.calibrate_heatmap_bias(mats0, m.images_from_frames(frame_items[0][0].to(cuda)))
    ref = BEVDet4DFrameHotPath(m, device=cuda).capture()
    want = list(ref.infer_stream(iter(frame_items)))
    assert len(want[0][0]) > 0 and not torch.equal(want[0][0], want[1][0])
    hot = BEVDet4DJpegHotPath(m, device=cuda).capture()
    for rep in range(2):
        got = list(hot.infer_stream(iter(items)))
        assert len(got) == len(items)
        for k, (g, w) in enumerate(zip(got, want)):
            assert _equal(g, w), (rep, k)
    # launch_jpegs + result per item with drive_mats' matrices: the same
    one = BEVDet4DJpegHotPath(m, device=cuda).capture()
    for item, (mats, prev, new), w in zip(items, drive_mats(items, m.test_mats), want):
        assert _equal(one.infer_jpegs(mats[0], mats[1], mats[4], item[0], prev, new), w)
