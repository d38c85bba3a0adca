"""CPU suite: the numpy JPEG decoder (jpeg_oracle) against Pillow bit for bit over subsampling x quality x optimize x
restart markers x sizes; the same streams decoded by Pillow with libjpeg-turbo's SIMD paths disabled (so the bits are
those of the C algorithms the oracle restates); and ops/jpeg.parse on the supported set, its descriptor, and every
rejection with its reason."""
import io
import itertools
import os
import subprocess
import sys

import numpy as np
import pytest

import jpeg_oracle as jo
from paddle3d_b200.ops import jpeg

SIZES = [(1, 1), (8, 8), (9, 17), (33, 31), (64, 100)]
QUALITIES = [50, 75, 95, 100]
RESTARTS = [None, "blocks", "rows"]


def _encode(img, **kw):
    from PIL import Image
    buf = io.BytesIO()
    Image.fromarray(img).save(buf, "JPEG", **kw)
    return buf.getvalue()


def _pil(f):
    from PIL import Image
    return np.asarray(Image.open(io.BytesIO(f)).convert("RGB"))


def _grid(subsampling):
    rng = np.random.default_rng([subsampling, 11])
    for size, q, opt, rst in itertools.product(SIZES, QUALITIES, [False, True], RESTARTS):
        img = np.clip(rng.normal(128, 60, size + (3,)), 0, 255).astype(np.uint8)
        kw = dict(quality=q, subsampling=subsampling, optimize=opt)
        if rst:
            kw["restart_marker_" + rst] = 1
        yield (size, q, opt, rst), _encode(img, **kw)


@pytest.mark.parametrize("subsampling", [0, 1, 2], ids=["444", "422", "420"])
def test_oracle_equals_pillow(subsampling):
    for case, f in _grid(subsampling):
        assert np.array_equal(jo.decode(f), _pil(f)), case


def test_pillow_without_simd_decodes_the_same(tmp_path):
    """JSIMD_FORCENONE=1 makes libjpeg-turbo take its C paths (jidctint.c, jdsample.c, jdcolor.c): the same bytes."""
    files = [f for s in (0, 1, 2) for i, (_, f) in enumerate(_grid(s)) if i % 9 == 0]
    for i, f in enumerate(files):
        (tmp_path / ("%03d.jpg" % i)).write_bytes(f)
    code = ("import sys, glob, io, numpy as np\nfrom PIL import Image\n"
            "for p in sorted(glob.glob(sys.argv[1] + '/*.jpg')):\n"
            "    np.save(p[:-4] + '.npy', np.asarray(Image.open(p).convert('RGB')))\n")
    env = dict(os.environ, JSIMD_FORCENONE="1")
    subprocess.run([sys.executable, "-c", code, str(tmp_path)], check=True, env=env, timeout=120)
    for i, f in enumerate(files):
        c_paths = np.load(tmp_path / ("%03d.npy" % i))
        assert np.array_equal(c_paths, _pil(f)) and np.array_equal(c_paths, jo.decode(f)), i


def test_parse_supported_set():
    from PIL import Image
    img = np.random.default_rng(3).integers(0, 256, (37, 45, 3), dtype=np.uint8)
    for subsampling, samp in ((0, (1, 1)), (1, (2, 1)), (2, (2, 2))):
        for kw in (dict(quality=80), dict(quality=60, optimize=True), dict(quality=90, restart_marker_blocks=3)):
            f = _encode(img, subsampling=subsampling, **kw)
            h = jpeg.parse(f)
            im = Image.open(io.BytesIO(f))
            assert (h.height, h.width) == (37, 45) and h.sampling == [samp, (1, 1), (1, 1)]
            for c, (_, _, _, tq) in enumerate(im.layer):
                assert np.array_equal(h.quant[c], np.asarray(im.quantization[tq]))
            assert h.restart_interval == (3 if "restart_marker_blocks" in kw else 0)
            assert f[h.ecs[1]:h.ecs[1] + 2] == b"\xff\xd9" and f[h.ecs[0] - 1] == 0  # Ah/Al closes the SOS header
            assert np.array_equal(jo.decode(f), _pil(f))


def test_descriptor_matches_the_header():
    files = [_encode(np.full((16, 24, 3), v, np.uint8), quality=q, subsampling=s)
             for v, q, s in ((10, 75, 2), (200, 95, 0), (99, 50, 1))]
    data, desc, hdrs = jpeg.batch(files)
    assert desc.dtype == jpeg.DESC_DTYPE and len(desc) == 3
    off = 0
    for f, d, h in zip(files, desc, hdrs):
        assert d["offset"] == off + h.ecs[0] and d["length"] == h.ecs[1] - h.ecs[0]
        assert bytes(data[d["offset"]:d["offset"] + d["length"]]) == f[h.ecs[0]:h.ecs[1]]
        assert (d["height"], d["width"], d["hs"], d["vs"]) == (16, 24, h.hs, h.vs)
        assert np.array_equal(d["quant"], h.quant)
        for c in range(3):
            assert np.array_equal(d["dc_bits"][c], h.dc[c][0]) and np.array_equal(d["ac_bits"][c], h.ac[c][0])
            assert np.array_equal(d["dc_vals"][c, :len(h.dc[c][1])], h.dc[c][1])
            assert np.array_equal(d["ac_vals"][c, :len(h.ac[c][1])], h.ac[c][1])
        # the oracle decodes the same image from the descriptor's tables
        assert np.array_equal(jo.decode(f), _pil(f))
        off += len(f)
    with pytest.raises(ValueError, match="want"):
        jpeg.batch([files[0], _encode(np.zeros((8, 8, 3), np.uint8))])


def _segment(f, marker):
    """(start, end) of the first segment with this marker byte, marker included."""
    i = 2
    while True:
        m = f[i + 1]
        ln = (f[i + 2] << 8) | f[i + 3]
        if m == marker:
            return i, i + 2 + ln
        i += 2 + ln


def _patch(f, i, b):
    return f[:i] + bytes([b]) + f[i + 1:]


@pytest.fixture(scope="module")
def base():
    return _encode(np.random.default_rng(5).integers(0, 256, (20, 30, 3), dtype=np.uint8), quality=85)


def test_parse_rejections(base):
    from PIL import Image
    img = np.random.default_rng(6).integers(0, 256, (20, 30, 3), dtype=np.uint8)
    sof, _ = _segment(base, 0xC0)
    cmyk = io.BytesIO()
    Image.fromarray(np.zeros((8, 8, 4), np.uint8), "CMYK").save(cmyk, "JPEG")
    dht = _segment(base, 0xC4)
    # SOF0 segment: FF C0, length, precision (+4), height (+5), width (+7), Nf (+9), then (id, hv, tq) per component
    cases = [
        ("progressive", _encode(img, progressive=True)),
        ("arithmetic", _patch(base, sof + 1, 0xC9)),
        ("12-bit", _patch(base, sof + 4, 12)),
        ("1 components", _encode(img[..., 0])),                                 # grayscale
        ("4 components", cmyk.getvalue()),                                      # CMYK
        ("missing DC Huffman table 0", base[:dht[0]] + base[dht[1]:]),
        ("missing quantisation table 3", _patch(base, sof + 12, 3)),
        ("truncated", base[:40]),
        ("over the limit", _patch(_patch(base, sof + 5, 0x23), sof + 6, 0x29)),  # 9001 rows
        ("sampling", _patch(base, sof + 14, 0x21)),                              # Cb at 2 x 1
        ("no SOI", base[2:]),
    ]
    for reason, f in cases:
        with pytest.raises(ValueError, match=reason):
            jpeg.parse(f)


def test_parse_rejects_an_all_ones_code(base):
    """A DC table whose codes fill their length (the last code is all ones) is not a T.81 table."""
    s, e = _segment(base, 0xC4)
    # two codes of length 1: '0' and '1' (all ones)
    full = bytes([0xFF, 0xC4, 0, 2 + 17 + 2, 0x00, 2] + [0] * 15 + [0, 1])
    with pytest.raises(ValueError, match="all-ones"):
        jpeg.parse(base[:s] + full + base[s:])


def test_camera_jpegs_round_trip():
    from paddle3d_b200 import synth
    files = synth.camera_jpegs(0, 2, 48, 64, quality=90)
    frames = synth.camera_frames(0, 2, 48, 64)
    assert len(files) == 2
    for f, fr in zip(files, frames):
        got = _pil(f)
        assert got.shape == fr.shape and np.abs(got.astype(int) - fr).mean() < 16  # lossy, not garbage
        assert np.array_equal(jo.decode(f), got)
