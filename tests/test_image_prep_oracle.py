"""CPU suite for BEVDet's image prep: the numpy restatement of Pillow's 8-bit BICUBIC resample (image_prep_oracle, which
the device kernel is tested against) equals PIL.Image.resize bit for bit; the kernel's normalisation expression equals
mmcv.imnormalize's steps through OpenCV; the test augmentation gives camera_rig's post_rots / post_trans; the image
prep plan's band; and BEVDetFromImages' data_config checks."""
import numpy as np
import pytest

from image_prep_oracle import crop, normalize, pipeline, pipeline_pil_cv2, resize
from paddle3d_b200 import synth
from paddle3d_b200.ops import image_prep as ip

MEAN, STD = (123.675, 116.28, 103.53), (58.395, 57.12, 57.375)


def _img(seed, H, W):
    if (H, W) == (900, 1600):
        return synth.camera_frames(seed, 1)[0]
    return np.random.default_rng([seed, H, W]).integers(0, 256, (H, W, 3), dtype=np.uint8)


@pytest.mark.parametrize("src,dst", [
    ((900, 1600), (396, 704)),    # BEVDet-R50
    ((900, 1600), (792, 1408)),   # the 512 x 1408 configs
    ((396, 704), (900, 1600)),    # nuScenes sizes the other way
    ((37, 53), (20, 31)),         # odd / prime sizes
    ((53, 37), (31, 20)),
    ((50, 60), (80, 90)),         # upscaling
    ((41, 43), (41, 43)),         # scale exactly 1 (Pillow copies)
    ((41, 43), (20, 43)),         # one axis at scale 1
    ((64, 96), (8, 12)),          # scale 8: 33 taps
    ((97, 13), (13, 97)),         # down on one axis, up on the other
])
def test_resample_matches_pillow(src, dst):
    Image = pytest.importorskip("PIL.Image")
    img = _img(1, *src)
    want = np.array(Image.fromarray(img).resize((dst[1], dst[0])))
    assert np.array_equal(resize(img, (dst[1], dst[0])), want)


def test_crop_matches_pillow():
    Image = pytest.importorskip("PIL.Image")
    img = _img(2, 37, 53)
    for box in ((0, 5, 53, 37), (-3, -4, 20, 10), (40, 30, 70, 45), (60, 40, 70, 50)):
        assert np.array_equal(crop(img, box), np.array(Image.fromarray(img).crop(box))), box


def test_coefficients():
    """Tap counts 2 ceil(2 max(scale, 1)) + 1, each row's weights summing to ~2^22, the BEVDet band's rows."""
    for i, o, k in ((1600, 704, 11), (900, 396, 11), (1600, 1408, 7), (60, 90, 5), (64, 8, 33)):
        kk, b = ip.resize_coeffs(i, o)
        assert kk.shape == (o, k) and b.shape == (o, 2) and b[:, 1].min() >= 1 and (b.sum(1) <= i).all()
        assert np.abs(kk.sum(1) - (1 << 22)).max() <= k
    kv, yb = ip.resize_coeffs(900, 396)
    assert tuple(yb[140]) == (315, 9) and yb[395].sum() == 900


@pytest.mark.parametrize("swap_rb", [True, False])
def test_normalisation_matches_cv2(swap_rb):
    """fp32(fp64(v -_fp32 mean) * (1 / fp64 std)) over every uint8 value equals imnormalize's cv2 steps."""
    pytest.importorskip("cv2")
    pytest.importorskip("PIL.Image")
    v = np.arange(256, dtype=np.uint8)
    img = np.stack([v, v[::-1], np.roll(v, 77)], -1).reshape(16, 16, 3)
    box = (0, 0, 16, 16)
    got = pipeline(img[None], (16, 16), box, MEAN, STD, swap_rb)
    want = pipeline_pil_cv2(img[None], (16, 16), box, MEAN, STD, swap_rb)
    assert np.array_equal(got.view(np.int32), want.view(np.int32))
    # the fp64 product rounded once is not the fp32 product: the expression is not a restatement of a plain fp32 one
    x = (img.astype(np.float32)[..., ::-1] if swap_rb else img.astype(np.float32)) - np.float32(MEAN)
    plain = (x * (np.float32(1) / np.float32(STD))).transpose(2, 0, 1)
    assert not np.array_equal(plain.view(np.int32), normalize(img, MEAN, STD, swap_rb).view(np.int32))


def test_pipeline_matches_pillow_cv2_bevdet():
    """The whole test pipeline of BEVDet-R50 on two seeded nuScenes-size frames, and a crop reaching past the image."""
    pytest.importorskip("cv2")
    pytest.importorskip("PIL.Image")
    fr = synth.camera_frames(3, 2)
    for dims, box, swap in (((704, 396), (0, 140, 704, 396), True), ((704, 396), (-8, 300, 720, 420), False)):
        got = pipeline(fr, dims, box, MEAN, STD, swap)
        want = pipeline_pil_cv2(fr, dims, box, MEAN, STD, swap)
        assert np.array_equal(got.view(np.int32), want.view(np.int32))


def test_camera_frames():
    fr = synth.camera_frames(0, 2, 90, 160)
    assert fr.shape == (2, 90, 160, 3) and fr.dtype == np.uint8 and fr.flags["C_CONTIGUOUS"]
    assert (fr == 0).mean() > 0.005 and (fr == 255).mean() > 0.005 and len(np.unique(fr)) == 256
    assert np.array_equal(fr, synth.camera_frames(0, 2, 90, 160)) and not np.array_equal(fr, synth.camera_frames(1, 2, 90,
                                                                                                                  160))


def test_augmentation_matches_camera_rig():
    from paddle3d_b200.bevdet import DATA_CONFIG
    a = ip.test_augmentation(DATA_CONFIG)
    assert a["resize_dims"] == (704, 396) and a["crop"] == (0, 140, 704, 396)
    rig = synth.camera_rig(0)
    assert np.array_equal(a["post_rot"], rig["post_rots"][0, 0]) and np.array_equal(a["post_tran"], rig["post_trans"][0, 0])
    b = ip.test_augmentation(dict(DATA_CONFIG, input_size=(512, 1408)))
    assert b["resize_dims"] == (1408, 792) and b["crop"] == (0, 280, 1408, 792)


def test_plan_band():
    """The band is exactly the source rows the kept rows' taps read; crops past the image."""
    from paddle3d_b200.bevdet import DATA_CONFIG
    p = ip.ImagePrepPlan.from_data_config(DATA_CONFIG, device="cpu")
    assert p.band == (315, 900) and p.band_rows == 585 and p.out_size == (256, 704) and p.crop_origin == (0, 140)
    assert p.yb[140, 0] == 0 and p.yb[395].sum() == 585
    assert p.band_bytes(6) == 6 * 585 * 1600 * 3 and p.out_bytes(6) == 6 * 3 * 256 * 704 * 4
    q = ip.ImagePrepPlan((900, 1600), (704, 396), (0, 380, 704, 420), MEAN, STD, device="cpu")
    assert q.band[1] == 900 and q.out_size == (40, 704)
    r = ip.ImagePrepPlan((900, 1600), (704, 396), (0, 400, 704, 420), MEAN, STD, device="cpu")
    assert r.band_rows == 1  # no kept row: every output pixel is the normalised 0
    with pytest.raises(ValueError, match="more than 8"):
        ip.ImagePrepPlan((900, 1600), (704, 100), (0, 0, 704, 100), MEAN, STD, device="cpu")


def test_model_data_config_checks():
    from paddle3d_b200.bevdet import CONFIG_IMG, DATA_CONFIG, BEVDetFromImages
    m = BEVDetFromImages(device="cpu")
    assert m.data_config["input_size"] == (256, 704)
    mats = m.test_mats(np.zeros((1, 6, 4, 4), np.float32), np.zeros((1, 6, 3, 3), np.float32), np.eye(3)[None])
    rig = synth.camera_rig(0)
    assert np.array_equal(mats[2], rig["post_rots"]) and np.array_equal(mats[3], rig["post_trans"])
    small = BEVDetFromImages(dict(CONFIG_IMG, input_size=(128, 352)), device="cpu")  # DATA_CONFIG at its input_size
    assert small.augmentation["crop"] == (0, 70, 352, 198)
    with pytest.raises(ValueError, match="crops"):
        BEVDetFromImages(dict(CONFIG_IMG, data_config=dict(DATA_CONFIG, input_size=(256, 640))), device="cpu")
    with pytest.raises(ValueError, match="crops"):
        BEVDetFromImages(dict(CONFIG_IMG, input_size=(128, 352), data_config=DATA_CONFIG), device="cpu")
