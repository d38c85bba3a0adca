"""GPU tests of BEVDet from decoded camera frames: p3d_image_prep_u8 bit-equal to the host pipeline (image_prep_oracle,
itself checked against Pillow + OpenCV in test_image_prep_oracle.py, and against Pillow + OpenCV directly where they are
installed) at BEVDet's sizes, upscaling, scale 1 and 8, crops past the image and partial tiles, writing its output and
nothing else and reading only the band; and the captured frame (BEVDetFrameHotPath) bit-equal to BEVDetImageHotPath on
the host-prepared images, eager, lanes, accelerate, pinned and device input."""
import numpy as np
import pytest

from image_prep_oracle import pipeline, pipeline_pil_cv2
from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu
BN_GAIN = 6.0 ** 0.5
MEAN, STD = (123.675, 116.28, 103.53), (58.395, 57.12, 57.375)


def _frames(seed, n, H, W):
    if (H, W) == (900, 1600):
        return synth.camera_frames(seed, n)
    return np.random.default_rng([seed, H, W]).integers(0, 256, (n, H, W, 3), dtype=np.uint8)


def _run(cuda, plan, frames_dev):
    """image_prep_u8 into a NaN-poisoned buffer with a guard tail; returns (output, tail)."""
    import torch
    from paddle3d_b200.ops.image_prep import image_prep_u8
    shape = plan.out_shape(frames_dev.shape[0])
    n = int(np.prod(shape))
    buf = torch.full((n + 1024,), float("nan"), dtype=torch.float32, device=cuda)
    out = buf[:n].view(shape)
    got = image_prep_u8(frames_dev, plan, out=out)
    torch.cuda.synchronize()
    assert got.data_ptr() == out.data_ptr()
    return out.cpu().numpy(), buf[n:].cpu().numpy()


CASES = [  # N, (H0, W0), resize (W, H), crop box, swap_rb
    (6, (900, 1600), (704, 396), (0, 140, 704, 396), True),      # BEVDet-R50
    (1, (900, 1600), (704, 396), (0, 140, 704, 396), False),
    (1, (900, 1600), (1408, 792), (0, 280, 1408, 792), True),    # the 512 x 1408 configs
    (1, (900, 1600), (704, 396), (-10, 300, 714, 428), True),    # past the resized image on three sides; fW % 4 != 0
    (2, (50, 60), (90, 80), (3, 5, 83, 77), False),              # upscaling
    (1, (41, 43), (43, 41), (0, 0, 43, 41), True),               # scale 1
    (3, (37, 53), (31, 20), (1, 2, 30, 19), False),              # odd sizes, partial tiles
    (1, (64, 96), (12, 8), (0, 0, 12, 8), True),                 # scale 8: 33 taps
    (1, (900, 1600), (704, 396), (0, 400, 704, 420), True),      # no kept row: all normalise(0)
]


@pytest.mark.parametrize("N,src,dims,box,swap", CASES)
def test_bit_equal_to_host_pipeline(cuda, N, src, dims, box, swap):
    import torch
    from paddle3d_b200.ops.image_prep import ImagePrepPlan
    fr = _frames(N + src[0], N, *src)
    plan = ImagePrepPlan(src, dims, box, MEAN, STD, swap, device=cuda)
    got, tail = _run(cuda, plan, torch.from_numpy(fr).to(cuda))
    want = pipeline(fr, dims, box, MEAN, STD, swap)
    assert got.shape == want.shape and np.array_equal(got.view(np.int32), want.view(np.int32))
    assert np.isnan(tail).all()


def test_bit_equal_to_pillow_cv2(cuda):
    """The kernel against Pillow and OpenCV themselves at BEVDet-R50's config, six cameras."""
    import torch
    pytest.importorskip("cv2")
    pytest.importorskip("PIL.Image")
    from paddle3d_b200.bevdet import DATA_CONFIG
    from paddle3d_b200.ops.image_prep import ImagePrepPlan, test_augmentation
    fr = synth.camera_frames(5)
    a = test_augmentation(DATA_CONFIG)
    plan = ImagePrepPlan.from_data_config(DATA_CONFIG, device=cuda)
    got, _ = _run(cuda, plan, torch.from_numpy(fr).to(cuda))
    want = pipeline_pil_cv2(fr, a["resize_dims"], a["crop"], DATA_CONFIG["mean"], DATA_CONFIG["std"])
    assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_reads_only_the_band(cuda):
    """Garbage outside the band leaves the output unchanged; the band's first and last rows both change it."""
    import torch
    from paddle3d_b200.bevdet import DATA_CONFIG
    from paddle3d_b200.ops.image_prep import ImagePrepPlan
    plan = ImagePrepPlan.from_data_config(DATA_CONFIG, device=cuda)
    y0, y1 = plan.band
    fr = torch.from_numpy(synth.camera_frames(9, 2)).to(cuda)
    ref, _ = _run(cuda, plan, fr)
    junk = fr.clone()
    junk[:, :y0] = torch.randint(0, 256, junk[:, :y0].shape, dtype=torch.uint8, device=cuda)
    junk[:, y1:] = torch.randint(0, 256, junk[:, y1:].shape, dtype=torch.uint8, device=cuda)
    got, _ = _run(cuda, plan, junk)
    assert np.array_equal(got.view(np.int32), ref.view(np.int32))
    band, _ = _run(cuda, plan, fr[:, y0:y1].contiguous())  # the band alone
    assert np.array_equal(band.view(np.int32), ref.view(np.int32))
    for row in (y0, y1 - 1):
        hit = fr.clone()
        hit[:, row] = 255 - hit[:, row]
        got, _ = _run(cuda, plan, hit)
        assert not np.array_equal(got.view(np.int32), ref.view(np.int32)), row


_PROFILE = """
import json, sys
import torch
from torch.profiler import ProfilerActivity, profile
sys.path.insert(0, sys.argv[1])
from paddle3d_b200 import synth
from paddle3d_b200.bevdet import DATA_CONFIG
from paddle3d_b200.ops.image_prep import ImagePrepPlan, image_prep_u8
plan = ImagePrepPlan.from_data_config(DATA_CONFIG, device="cuda")
fr = torch.from_numpy(synth.camera_frames(1, 1)).cuda()
image_prep_u8(fr, plan)
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as prof:
    image_prep_u8(fr, plan)
    torch.cuda.synchronize()
print("KERNELS " + json.dumps([e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]))
"""


def test_profiler_sees_the_kernel(cuda):
    """One call under torch.profiler sees image_prep_u8_kernel by name.  In a process of its own: a profiler session
    opened earlier in the same process (test_gpu_camera_pool.py opens one) leaves later sessions without kernel records."""
    import json
    import subprocess
    import sys
    from conftest import ROOT
    r = subprocess.run([sys.executable, "-c", _PROFILE, ROOT], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-2000:]
    names = json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("KERNELS ")][-1][8:])
    if not names:
        pytest.skip("torch.profiler reported no CUDA kernels on this device")
    assert any("image_prep_u8" in n for n in names), sorted(set(names))


# ---------------------------------------------------------------------------------------------------- the frame
@pytest.fixture(scope="module")
def frame(cuda):
    """A seeded BEVDetFromImages at 256 x 704 calibrated on the host-prepared images of its first frames."""
    import torch
    from paddle3d_b200.bevdet import BEVDetFromImages
    m = BEVDetFromImages(device=cuda).init_weight(seed=0, bn_gain=BN_GAIN)
    rig = synth.camera_rig(31)
    fr = synth.camera_frames(7)
    dc = m.data_config
    a = m.augmentation
    imgs = pipeline(fr, a["resize_dims"], a["crop"], dc["mean"], dc["std"], dc["to_rgb"])
    m.calibrate_heatmap_bias(m.test_mats(rig["sensor2ego"], rig["cam2imgs"], rig["bda"]), torch.from_numpy(imgs).to(cuda))
    return dict(m=m, rig=rig, frames=fr, imgs=imgs)


def _args(rig):
    return rig["sensor2ego"], rig["cam2imgs"], rig["bda"]


def _equal(a, b):
    import torch
    return all(torch.equal(x, y) for x, y in zip(a, b))


@pytest.mark.parametrize("decode", ["default", "bevdet_nms"])
def test_frame_equals_image_frame(cuda, frame, decode):
    """Boxes, scores and labels bit-equal to BEVDetImageHotPath on the host-prepared images; one more kernel node; status
    word 0; pinned host input."""
    import torch
    from paddle3d_b200.bevdet import CONFIG_IMG_BEVDET_NMS, BEVDetFromImages, BEVDetFrameHotPath, BEVDetImageHotPath
    m = frame["m"]
    if decode == "bevdet_nms":
        base = m
        m = BEVDetFromImages(CONFIG_IMG_BEVDET_NMS, device=cuda)
        m.encoder, m.head, m.image_encoder, m.prep_plan = base.encoder, base.head, base.image_encoder, base.prep_plan
    rig = frame["rig"]
    ref = BEVDetImageHotPath(m, device=cuda).capture(count_nodes=True)
    want = [t.clone() for t in ref.infer(m.test_mats(*_args(rig)), torch.from_numpy(frame["imgs"]).to(cuda))]
    hot = BEVDetFrameHotPath(m, device=cuda).capture(count_nodes=True)
    got = [t.clone() for t in hot.infer_frames(*_args(rig), torch.from_numpy(frame["frames"]).pin_memory())]
    assert len(want[0]) > 0 and _equal(got, want)
    assert int(hot.h_status[0]) == 0
    assert torch.equal(hot.imgs.cpu(), torch.from_numpy(frame["imgs"]))
    g, r = hot.graph_nodes, ref.graph_nodes
    assert g == dict(r, kernel=r["kernel"] + 1), (g, r)


def test_frame_eager_lanes_accelerate_inputs(cuda, frame):
    """Captured == eager (forward_frames) with new frames and rigs on every replay; three lanes sharing the model == one
    lane; accelerate == full; device input == pinned input; pageable host input refused."""
    import torch
    from paddle3d_b200.bevdet import BEVDetFromImages, BEVDetFrameHotPath
    m = frame["m"]
    rigs = [synth.camera_rig(40 + i) for i in range(3)]
    host = [torch.from_numpy(synth.camera_frames(50 + i)).pin_memory() for i in range(3)]
    dev = [h.to(cuda) for h in host]
    hot = BEVDetFrameHotPath(m, device=cuda).capture()
    want = []
    for r, d in zip(rigs, dev):
        boxes, scores, labels, counts = m.forward_frames(*_args(r), d)
        k = int(counts[-1])
        eager = [boxes[:k].cpu(), scores[:k].cpu(), labels[:k].cpu()]
        got = [t.clone() for t in hot.infer_frames(*_args(r), d)]
        assert k > 0 and _equal(got, eager)
        assert _equal([t.clone() for t in hot.infer_frames(*_args(r), host[len(want)])], eager)
        want.append(eager)
    assert not torch.equal(want[0][0], want[1][0])
    lanes = [BEVDetFrameHotPath(m, device=cuda).capture().share_model(hot) for _ in range(3)]
    for rep in range(2):
        for i, lane in enumerate(lanes):
            lane.launch_frames(*_args(rigs[i]), host[i] if rep else dev[i])
        for i, lane in enumerate(lanes):
            assert _equal(lane.result(), want[i]), "lane %d" % i
    acc_model = BEVDetFromImages(accelerate=True, device=cuda)
    acc_model.encoder, acc_model.head, acc_model.image_encoder = m.encoder, m.head, m.image_encoder
    acc_model.prep_plan = m.prep_plan
    acc = BEVDetFrameHotPath(acc_model, device=cuda).capture()
    for i in (0, 0, 1, 0):
        assert _equal(acc.infer_frames(*_args(rigs[i]), host[i]), want[i])
    with pytest.raises(ValueError, match="pageable"):
        hot.launch_frames(*_args(rigs[0]), torch.from_numpy(frame["frames"]))
    with pytest.raises(ValueError, match="uint8"):
        hot.launch_frames(*_args(rigs[0]), dev[0].float())
    with pytest.raises(ValueError, match="uint8"):
        hot.launch_frames(*_args(rigs[0]), dev[0][:, :450].contiguous())
