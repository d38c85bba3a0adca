"""BEVDet's test-time image pipeline on the device (csrc/image_prep.cu): PrepareImageInputs.img_transform (a Pillow
BICUBIC resize, then a crop) and mmlabNormalize (mmcv.imnormalize with to_rgb=True) of decoded uint8 RGB frames, as one
kernel that writes what the host pipeline writes, bit for bit.  The reference has no op for it (it is a data
transform); tests/image_prep_oracle.py restates it in numpy and checks that restatement against Pillow and OpenCV."""
import ctypes as C
import math

import numpy as np
import torch

from .._lib import check, fptr, host_floats, lib
from .._mem import ptr, require_cuda, stream

PRECISION_BITS = 22   # Pillow's fixed-point coefficients on 8-bit images (Resample.c: 32 - 8 - 2)
MAX_SCALE = 8         # in / out per axis: at most 2 * ceil(2 * 8) + 1 = 33 taps


def _bicubic(x):
    """Pillow's bicubic_filter, a = -0.5."""
    a = -0.5
    x = abs(x)
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def resize_coeffs(in_size, out_size):
    """Pillow's precompute_coeffs + normalize_coeffs_8bpc for BICUBIC on one axis of a resize from in_size to out_size
    pixels (box [0, in_size)), in Python double with Resample.c's expression order: (kk int32 [out_size, ksize],
    bounds int32 [out_size, 2] = (xmin, n): output i reads inputs [xmin, xmin + n) with weights kk[i, :n])."""
    in_size, out_size = int(in_size), int(out_size)
    if in_size < 1 or out_size < 1:
        raise ValueError("resize_coeffs: sizes %d -> %d" % (in_size, out_size))
    scale = filterscale = float(in_size) / out_size
    if filterscale < 1.0:
        filterscale = 1.0
    support = 2.0 * filterscale
    ksize = int(math.ceil(support)) * 2 + 1
    kk = np.zeros((out_size, ksize), np.int32)
    bounds = np.zeros((out_size, 2), np.int32)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        w = [_bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for v in w:
            ww += v
        for x in range(xmax):
            v = w[x] / ww if ww != 0.0 else w[x]
            kk[xx, x] = int(-0.5 + v * (1 << PRECISION_BITS)) if v < 0 else int(0.5 + v * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return kk, bounds


def test_augmentation(data_config):
    """BEVDet's sample_augmentation + img_transform with train=False (no flip, no rotation): dict(resize, resize_dims
    (W, H), crop (x0, y0, x1, y1) of the resized image, post_rot [3, 3] and post_tran [3] float32)."""
    H, W = (int(v) for v in data_config["src_size"])
    fH, fW = (int(v) for v in data_config["input_size"])
    resize = float(fW) / float(W) + data_config.get("resize_test", 0.0)
    resize_dims = (int(W * resize), int(H * resize))
    newW, newH = resize_dims
    if newW < 1 or newH < 1 or fH < 1 or fW < 1:
        raise ValueError("test_augmentation: resize %s to %s, input_size %s" % ((W, H), resize_dims, (fH, fW)))
    crop_h = int((1 - np.mean(data_config["crop_h"])) * newH) - fH
    crop_w = int(max(0, newW - fW) / 2)
    post_rot = np.diag([resize, resize, 1.0]).astype(np.float32)
    post_tran = np.array([-crop_w, -crop_h, 0.0], np.float32)
    return dict(resize=resize, resize_dims=resize_dims, crop=(crop_w, crop_h, crop_w + fW, crop_h + fH),
                post_rot=post_rot, post_tran=post_tran)


class ImagePrepPlan:
    """What p3d_image_prep_u8 reads for one data config, built once: the coefficient tables of both axes on the device,
    the source row band [y0, y1) the crop's rows need (the vertical xmin relative to y0), the crop origin, the output
    size (fH, fW), and mean (fp32) / 1 / std (fp64) per output channel.  mean / std: mmcv.imnormalize's, given in the
    order of its output channels; swap_rb (its to_rgb): output channel c reads input channel 2 - c."""

    def __init__(self, src_size, resize_dims, crop, mean, std, swap_rb=True, device="cuda"):
        self.src_size = H0, W0 = tuple(int(v) for v in src_size)
        self.resize_dims = rW, rH = tuple(int(v) for v in resize_dims)
        x0, y0c, x1, y1c = (int(v) for v in crop)
        self.crop_origin = (x0, y0c)
        self.out_size = fH, fW = (y1c - y0c, x1 - x0)
        if fH < 1 or fW < 1:
            raise ValueError("ImagePrepPlan: crop %s is empty" % (tuple(crop),))
        if W0 > MAX_SCALE * rW or H0 > MAX_SCALE * rH:
            raise ValueError("ImagePrepPlan: %s -> %s reduces by more than %d" % ((W0, H0), (rW, rH), MAX_SCALE))
        self.kh, self.xb = resize_coeffs(W0, rW)
        kv, yb = resize_coeffs(H0, rH)
        rows = [r for r in range(y0c, y0c + fH) if 0 <= r < rH]  # the resized rows the crop keeps
        if rows:
            self.band = (int(yb[rows[0], 0]), int(yb[rows[-1]].sum()))
        else:  # the crop misses the resized image: every output pixel is normalise(0); one row keeps the shapes valid
            self.band = (0, 1)
        self.kv, self.yb = kv, yb.copy()
        self.yb[:, 0] -= self.band[0]
        self.band_rows = self.band[1] - self.band[0]
        self.mean = np.asarray(mean, np.float32).reshape(3)
        self.std_inv = 1.0 / np.asarray(std, np.float32).astype(np.float64).reshape(3)
        self.swap_rb = bool(swap_rb)
        dev = torch.device(device)
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
        self.dev = dict(kh=t(self.kh), xb=t(self.xb), kv=t(self.kv), yb=t(self.yb))
        self._mean_host = host_floats(self.mean)
        self._std_inv_host = (C.c_double * 3)(*[float(v) for v in self.std_inv])

    @classmethod
    def from_data_config(cls, data_config, device="cuda"):
        aug = test_augmentation(data_config)
        return cls(data_config["src_size"], aug["resize_dims"], aug["crop"], data_config["mean"], data_config["std"],
                   data_config.get("to_rgb", True), device)

    def out_shape(self, n):
        return (n, 3) + self.out_size

    def band_bytes(self, n):
        """Bytes of the band of n frames: what the kernel reads and what a frame copies to the device."""
        return n * self.band_rows * self.src_size[1] * 3

    def out_bytes(self, n):
        return n * 3 * self.out_size[0] * self.out_size[1] * 4


def image_prep_u8(frames, plan, out=None):
    """Resize, crop and normalise uint8 RGB frames on the device (p3d_image_prep_u8): frames [N, H0, W0, 3] (whole
    frames; the band is sliced out) or [N, band_rows, W0, 3] (the plan's band) -> fp32 [N, 3, fH, fW], bit-identical
    to Pillow's resize and crop followed by mmcv.imnormalize."""
    frames = require_cuda(frames, "frames", torch.uint8)
    H0, W0 = plan.src_size
    if frames.dim() != 4 or frames.shape[3] != 3 or frames.shape[2] != W0 or frames.shape[1] not in (H0, plan.band_rows):
        raise ValueError("image_prep_u8: frames %s, want [N, %d or %d, %d, 3] uint8"
                         % (tuple(frames.shape), H0, plan.band_rows, W0))
    if frames.shape[1] != plan.band_rows:
        frames = frames[:, plan.band[0]:plan.band[1]].contiguous()
    n = frames.shape[0]
    if out is None:
        out = torch.empty(plan.out_shape(n), dtype=torch.float32, device=frames.device)
    elif out.dtype != torch.float32 or tuple(out.shape) != plan.out_shape(n) or not out.is_contiguous():
        raise ValueError("image_prep_u8: out %s %s, want contiguous float32 %s" % (tuple(out.shape), out.dtype,
                                                                                  plan.out_shape(n)))
    d = plan.dev
    rW, rH = plan.resize_dims
    fH, fW = plan.out_size
    check(lib().p3d_image_prep_u8(ptr(frames), n, plan.band_rows, H0, W0, ptr(d["kh"]), ptr(d["xb"]), d["kh"].shape[1],
                                  rW, ptr(d["kv"]), ptr(d["yb"]), d["kv"].shape[1], rH, plan.crop_origin[0],
                                  plan.crop_origin[1], fH, fW, fptr(plan._mean_host), fptr(plan._std_inv_host), int(plan.swap_rb),
                                  ptr(out), stream(frames.device)), "image_prep_u8")
    return out
