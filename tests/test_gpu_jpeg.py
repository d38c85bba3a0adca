"""GPU tests of the device JPEG decoder (p3d_jpeg_decode_u8): byte-equal to np.asarray(Image.open(f).convert("RGB"))
on small images over subsampling x quality x optimize x restart markers, on full-size camera frames, odd sizes, a flat
image, white noise, bands and N = 1 / 6; one captured graph over frames of different lengths and tables; and corrupt
data (truncation, random bytes, an undefined code, restart markers out of sequence) setting that image's status word
while the other images of the call decode normally."""
import io
import itertools

import numpy as np
import pytest

from paddle3d_b200 import synth

pytestmark = pytest.mark.gpu


def _encode(img, **kw):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "JPEG", **kw)
    return buf.getvalue()


def _pil(f):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))


def _decode(cuda, files, rows=None, expect_status=0):
    """Decode files on the device into a poisoned buffer with a guard tail; returns (images, status)."""
    import torch
    from paddle3d_b200.ops import jpeg
    data, desc, hdrs = jpeg.batch(files)
    H, W = hdrs[0].height, hdrs[0].width
    y0, y1 = rows or (0, H)
    n = len(files)
    size = n * (y1 - y0) * W * 3
    buf = torch.full((size + 4096,), 0xA5, dtype=torch.uint8, device=cuda)
    out = buf[:size].view(n, y1 - y0, W, 3)
    status = torch.zeros(n, dtype=torch.int32, device=cuda)
    jpeg.jpeg_decode_u8(torch.from_numpy(data).to(cuda), torch.from_numpy(desc.view(np.uint8)).to(cuda), n, (H, W),
                        rows=(y0, y1), out=out, status=status,
                        max_bytes=max(int(d) for d in desc["length"]))
    torch.cuda.synchronize()
    assert (buf[size:] == 0xA5).all(), "wrote past the output"
    st = status.cpu().tolist()
    if expect_status is not None:
        assert st == [expect_status] * n, "status %s" % st
    return out.cpu().numpy(), st


def _check(cuda, files, rows=None):
    got, _ = _decode(cuda, files, rows)
    for i, f in enumerate(files):
        want = _pil(f)
        if rows:
            want = want[rows[0]:rows[1]]
        assert np.array_equal(got[i], want), "image %d differs at %d pixels" % (i, int((got[i] != want).any(-1).sum()))


SMALL = [(1, 1), (8, 8), (9, 17), (33, 31), (64, 100)]


@pytest.mark.parametrize("size", SMALL)
@pytest.mark.parametrize("subsampling", [0, 1, 2])
def test_small_grid(cuda, size, subsampling):
    """quality 50 / 75 / 95 / 100 x optimize x (no restart, restart_marker_blocks=1, restart_marker_rows=1): one batch."""
    rng = np.random.default_rng([size[0], size[1], subsampling])
    files = []
    for q, opt, rst in itertools.product([50, 75, 95, 100], [False, True], [None, "blocks", "rows"]):
        img = np.clip(rng.normal(128, 60, size + (3,)), 0, 255).astype(np.uint8)
        kw = dict(quality=q, subsampling=subsampling, optimize=opt)
        if rst:
            kw["restart_marker_" + rst] = 1
        files.append(_encode(img, **kw))
    _check(cuda, files)


CAMERA = [dict(quality=q, subsampling=s) for q in (75, 95, 100) for s in (2, 1, 0)] + [
    dict(quality=95, subsampling=2, optimize=True),
    dict(quality=95, subsampling=2, restart_marker_blocks=16),
    dict(quality=75, subsampling=1, restart_marker_rows=1, optimize=True),
    dict(quality=100, subsampling=0, restart_marker_blocks=5),
]


@pytest.mark.parametrize("kw", CAMERA, ids=lambda kw: "-".join("%s%s" % (k[:4], v) for k, v in kw.items()))
def test_camera_frames(cuda, kw):
    _check(cuda, synth.camera_jpegs(3, **kw))


@pytest.mark.parametrize("size,subsampling", [((899, 1599), 2), ((899, 1599), 1), ((1, 4096), 2), ((1, 4096), 0),
                                              ((4096, 1), 2)])
def test_odd_sizes(cuda, size, subsampling):
    img = synth.camera_frames(5, 1, *size)[0] if min(size) > 1 else \
        np.random.default_rng(size).integers(0, 256, size + (3,), dtype=np.uint8)
    _check(cuda, [_encode(img, quality=90, subsampling=subsampling)])


def test_flat_grey(cuda):
    """Long EOB runs: many blocks in one subsequence."""
    img = np.full((900, 1600, 3), 128, np.uint8)
    _check(cuda, [_encode(img, quality=q, subsampling=s) for q, s in ((75, 2), (95, 0), (50, 1))])


def test_white_noise_q100_444(cuda):
    """The longest codes at their densest."""
    img = np.random.default_rng(1).integers(0, 256, (2, 900, 1600, 3), dtype=np.uint8)
    _check(cuda, [_encode(im, quality=100, subsampling=0) for im in img])


@pytest.mark.parametrize("rows", [(355, 900), (1, 899), (13, 14), (17, 31), (0, 16), (884, 900)])
@pytest.mark.parametrize("subsampling", [2, 1, 0])
def test_band(cuda, rows, subsampling):
    """Rows of BEVDet's prep band (355, 900) and rows starting and ending inside an MCU row."""
    _check(cuda, synth.camera_jpegs(4, 2, quality=95, subsampling=subsampling), rows)


def test_band_of_prep_plan(cuda):
    from paddle3d_b200 import bevdet
    from paddle3d_b200.ops.image_prep import ImagePrepPlan
    plan = ImagePrepPlan.from_data_config(bevdet.DATA_CONFIG, device=cuda)
    _check(cuda, synth.camera_jpegs(6, quality=95), plan.band)


@pytest.mark.parametrize("n", [1, 6])
def test_batch_sizes(cuda, n):
    _check(cuda, synth.camera_jpegs(7, n, quality=90))


def test_one_graph_serves_any_stream(cuda):
    """One captured decode replayed over frames of other compressed lengths, tables and restart intervals."""
    import torch
    from paddle3d_b200.ops import jpeg
    variants = [dict(quality=75), dict(quality=95), dict(quality=95, optimize=True),
                dict(quality=90, restart_marker_blocks=3), dict(quality=100, subsampling=0),
                dict(quality=85, subsampling=1, restart_marker_rows=2)]
    frames = [synth.camera_jpegs(10 + i, 3, **kw) for i, kw in enumerate(variants)]
    cap = max(len(f) for fr in frames for f in fr)
    data_dev = torch.zeros(3 * cap, dtype=torch.uint8, device=cuda)
    desc_dev = torch.zeros(3 * jpeg.DESC_DTYPE.itemsize, dtype=torch.uint8, device=cuda)
    out = torch.empty((3, 900, 1600, 3), dtype=torch.uint8, device=cuda)
    status = torch.zeros(3, dtype=torch.int32, device=cuda)

    def stage(files):
        data, desc, _ = jpeg.batch(files)
        data_dev[:len(data)].copy_(torch.from_numpy(data))
        desc_dev.copy_(torch.from_numpy(desc.view(np.uint8)))

    stage(frames[0])
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        jpeg.jpeg_decode_u8(data_dev, desc_dev, 3, (900, 1600), out=out, status=status, max_bytes=cap)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        jpeg.jpeg_decode_u8(data_dev, desc_dev, 3, (900, 1600), out=out, status=status, max_bytes=cap)
    for files in frames[::-1] + frames:
        stage(files)
        status.zero_()
        g.replay()
        torch.cuda.synchronize()
        assert status.cpu().tolist() == [0, 0, 0]
        got = out.cpu().numpy()
        for i, f in enumerate(files):
            assert np.array_equal(got[i], _pil(f))


def _ecs(f):
    from paddle3d_b200.ops import jpeg
    return jpeg.parse(f).ecs


def test_corrupt_truncated(cuda):
    from paddle3d_b200.ops import jpeg
    good = synth.camera_jpegs(8, 2, quality=90)
    a, b = _ecs(good[0])
    cut = good[0][:a + (b - a) // 3] + b"\xff\xd9"
    got, st = _decode(cuda, [cut, good[1]], expect_status=None)
    assert st[0] & jpeg.STATUS_TRUNCATED and st[1] == 0 and np.array_equal(got[1], _pil(good[1]))
    cut = good[0][:a] + b"\xff\xd9"  # nothing after the SOS
    _, st = _decode(cuda, [good[1], cut], expect_status=None)
    assert st[0] == 0 and st[1] & jpeg.STATUS_TRUNCATED


def test_corrupt_random_bytes(cuda):
    good = synth.camera_jpegs(8, 1, quality=90)[0]
    a, b = _ecs(good)
    rng = np.random.default_rng(0)
    for pos in (a, a + (b - a) // 2, b - 5000):
        junk = rng.integers(0, 256, 4096, dtype=np.uint8).tobytes()
        bad = good[:pos] + junk + good[pos + 4096:]
        _, st = _decode(cuda, [bad], expect_status=None)
        assert st[0] != 0


def test_corrupt_undefined_code(cuda):
    """Sixteen one-bits are never a code (the all-ones code is reserved)."""
    from paddle3d_b200.ops import jpeg
    good = synth.camera_jpegs(8, 1, quality=90)[0]
    a, b = _ecs(good)
    bad = good[:a] + b"\xff\x00" * 8 + good[a + 16:]
    _, st = _decode(cuda, [bad], expect_status=None)
    assert st[0] & jpeg.STATUS_BAD_CODE


def test_corrupt_restart_sequence(cuda):
    from paddle3d_b200.ops import jpeg
    good = synth.camera_jpegs(8, 1, quality=90, restart_marker_blocks=8)[0]
    a, b = _ecs(good)
    i = good.index(b"\xff\xd3", a)
    bad = good[:i] + b"\xff\xd5" + good[i + 2:]
    _, st = _decode(cuda, [bad], expect_status=None)
    assert st[0] & jpeg.STATUS_BAD_RESTART
