"""numpy restatement of BEVDet's test-time image pipeline, what paddle3d_b200.ops.image_prep computes on the device:
Pillow's 8-bit BICUBIC resample (ImagingResample: horizontal pass on the rows the vertical taps need, rounded to uint8,
then the vertical pass), Pillow's crop (zero outside the resized image) and mmcv.imnormalize (float32, BGR2RGB swap,
subtract the fp32 mean in fp32, multiply by 1 / std in fp64 and round once).  test_image_prep_oracle.py checks it
against Pillow and OpenCV themselves."""
import numpy as np

from paddle3d_b200.ops.image_prep import PRECISION_BITS, resize_coeffs


def _pass(x, kk, bounds, axis):
    """One 8-bit pass along axis (0: rows, 1: columns) of x [h, w, 3] uint8 -> uint8, int64 accumulation from 1 << 21
    (int32 never overflows at these weights), >> 22, clamped to [0, 255]."""
    out_n = len(bounds)
    acc = np.full((out_n, x.shape[1 - axis], 3), 1 << (PRECISION_BITS - 1), np.int64)
    xs = np.moveaxis(x, axis, 0).astype(np.int64)
    for k in range(kk.shape[1]):
        idx = bounds[:, 0] + k
        live = k < bounds[:, 1]
        w = np.where(live, kk[:, k], 0).astype(np.int64)
        acc += w[:, None, None] * xs[np.minimum(idx, xs.shape[0] - 1)]
    v = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(v, 0, axis)


def resize(img, size):
    """PIL.Image.fromarray(img).resize(size) (BICUBIC, size = (W, H)) for img [H0, W0, 3] uint8."""
    H0, W0 = img.shape[:2]
    W, H = size
    kh, xb = resize_coeffs(W0, W)
    kv, yb = resize_coeffs(H0, H)
    y0, y1 = int(yb[0, 0]), int(yb[-1].sum())
    tmp = _pass(img[y0:y1], kh, xb, 1) if W != W0 else img[y0:y1]
    yb = yb.copy()
    yb[:, 0] -= y0
    return _pass(tmp, kv, yb, 0) if H != H0 else tmp


def crop(img, box):
    """PIL.Image.crop(box) of img [H, W, 3]: pixels outside the image are 0."""
    x0, y0, x1, y1 = box
    out = np.zeros((y1 - y0, x1 - x0, 3), np.uint8)
    H, W = img.shape[:2]
    sy0, sy1, sx0, sx1 = max(y0, 0), min(y1, H), max(x0, 0), min(x1, W)
    if sy0 < sy1 and sx0 < sx1:
        out[sy0 - y0:sy1 - y0, sx0 - x0:sx1 - x0] = img[sy0:sy1, sx0:sx1]
    return out


def normalize(img, mean, std, swap_rb=True):
    """mmcv.imnormalize(img, mean, std, to_rgb=swap_rb) with BEVDet's float32 mean / std, as the kernel computes it:
    fp32(fp64(fp32(v - fp32 mean)) * (1 / fp64 std)), output channel c from input channel 2 - c when swapped; [H, W, 3]
    uint8 -> [3, H, W] float32."""
    x = img.astype(np.float32)
    if swap_rb:
        x = x[..., ::-1]
    m = np.asarray(mean, np.float32).reshape(1, 1, 3)
    s = 1.0 / np.asarray(std, np.float32).astype(np.float64).reshape(1, 1, 3)
    y = ((x - m).astype(np.float64) * s).astype(np.float32)
    return np.ascontiguousarray(y.transpose(2, 0, 1))


def pipeline(frames, resize_dims, box, mean, std, swap_rb=True):
    """frames [N, H0, W0, 3] uint8 -> [N, 3, fH, fW] float32: resize, crop, normalize per frame."""
    return np.stack([normalize(crop(resize(f, resize_dims), box), mean, std, swap_rb) for f in frames])


def pipeline_pil_cv2(frames, resize_dims, box, mean, std, swap_rb=True):
    """The same through Pillow and OpenCV themselves (mmcv.imnormalize's steps, BEVDet's mmlabNormalize arrays)."""
    import cv2
    from PIL import Image
    out = []
    mean = np.asarray(mean, np.float32)
    std = np.asarray(std, np.float32)
    for f in frames:
        img = np.array(Image.fromarray(f).resize(tuple(resize_dims)).crop(tuple(box))).astype(np.float32)
        m64 = np.float64(mean.reshape(1, -1))
        stdinv = 1 / np.float64(std.reshape(1, -1))
        if swap_rb:
            cv2.cvtColor(img, cv2.COLOR_BGR2RGB, img)
        cv2.subtract(img, m64, img)
        cv2.multiply(img, stdinv, img)
        out.append(img.transpose(2, 0, 1))
    return np.ascontiguousarray(np.stack(out))
