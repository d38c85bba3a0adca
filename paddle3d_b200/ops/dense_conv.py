"""SURVEY.md §8f-1: dense 2-D convolutions of the RPN / neck / CenterHead on wgmma.  Default: the fp16-pair kernels of
`csrc/dense_conv_f16.cu` (second half of this file; per-layer timings: tools/dense_bench.py).  The first
half drives the tf32-pair kernels (`csrc/dense_conv_tc.cu`, images as "pixel split rows" [B*H*W, 2*C] fp32), kept
for models whose activations leave fp16's range.  Weights are given in Paddle's layouts (Conv2D [Cout, Cin, kH, kW],
Conv2DTranspose [Cin, Cout, k, k])."""
import torch

from .._lib import check, lib
from .._mem import ptr, require_cuda, stream


def n_tile_for(cout):
    """Output-channel tile of the kernel: 128 for wide layers, 64, or 16 for the 1-3 channel head outputs."""
    return 128 if cout >= 128 else (64 if cout > 16 else 16)


def nchw_to_pixel_split(x):
    x = require_cuda(x, "x", torch.float32)
    b, c, h, w = x.shape
    out = torch.empty((b * h * w, 2 * c), dtype=torch.float32, device=x.device)
    check(lib().p3d_nchw_to_pixel_split(ptr(x), b, c, h, w, ptr(out), stream(x.device)), "nchw_to_pixel_split")
    return out


def _pack(w_tci, n_tile):
    """w_tci [taps, Cin, Cout] fp32 on the device -> per-N-tile packed images, concatenated."""
    L = lib()
    taps, cin, cout = w_tci.shape
    tiles = (cout + n_tile - 1) // n_tile
    total = L.p3d_dense_conv2d_packed_weight_bytes(taps, cin, cout, n_tile)
    if not total:
        raise ValueError("unsupported dense conv shape: taps %d Cin %d Cout %d" % (taps, cin, cout))
    packed = torch.zeros((total // 4,), dtype=torch.float32, device=w_tci.device)
    padded = torch.zeros((taps, cin, tiles * n_tile), dtype=torch.float32, device=w_tci.device)
    padded[:, :, :cout] = w_tci
    block = taps * cin * 2 * n_tile
    for t in range(tiles):
        wt = padded[:, :, t * n_tile:(t + 1) * n_tile].contiguous()
        dst = packed[t * block:(t + 1) * block]
        check(L.p3d_sparse_conv_pack_weights(ptr(wt), taps, cin, n_tile, ptr(dst), stream(wt.device)),
              "sparse_conv_pack_weights")
    return packed


def pack_conv_weight(weight, n_tile):
    """paddle.nn.Conv2D weight [Cout, Cin, kH, kW] -> packed (tap = dy * kW + dx)."""
    weight = require_cuda(weight, "weight", torch.float32)
    cout, cin, kh, kw = weight.shape
    return _pack(weight.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout).contiguous(), n_tile)


def pack_deconv_weight(weight, n_tile):
    """paddle.nn.Conv2DTranspose weight [Cin, Cout, k, k] -> packed (tap = dy * k + dx)."""
    weight = require_cuda(weight, "weight", torch.float32)
    cin, cout, k, k2 = weight.shape
    return _pack(weight.permute(2, 3, 0, 1).reshape(k * k2, cin, cout).contiguous(), n_tile)


def dense_conv2d(x_split, shape, packed, cout, n_tile, kernel, stride=1, padding=0, up=1, scale=None, shift=None,
                 relu=False, out_split=None, out_channels=None, out_c0=0, want_nchw=False):
    """x_split [B*H*W, 2*Cin]; shape = (B, H, W, Cin).  Returns (out_split or None, out_nchw or None, (B, oH, oW)).

    out_split: an existing [B*oH*oW, 2*out_channels] buffer to write columns [out_c0, out_c0 + cout) of (channel
    concat), or None to allocate one of `out_channels` (default cout) channels; want_nchw adds fp32 planes."""
    x_split = require_cuda(x_split, "x_split", torch.float32)
    b, h, w, cin = [int(v) for v in shape]
    if up > 1:
        oh, ow = h * up, w * up
        kh = kw = st = up
        pd = 0
    else:
        kh = kw = int(kernel)
        st, pd = int(stride), int(padding)
        oh, ow = (h + 2 * pd - kh) // st + 1, (w + 2 * pd - kw) // st + 1
    dev = x_split.device
    oc = int(out_channels or cout)
    if out_split is None and not want_nchw:
        out_split = torch.empty((b * oh * ow, 2 * oc), dtype=torch.float32, device=dev)
    out_nchw = torch.empty((b, cout, oh, ow), dtype=torch.float32, device=dev) if want_nchw else None
    check(lib().p3d_dense_conv2d_split(ptr(x_split), b, h, w, cin, ptr(packed), int(cout), int(n_tile), kh, kw, st, pd,
                                       int(up), ptr(scale), ptr(shift), int(relu), ptr(out_split), oc, int(out_c0),
                                       ptr(out_nchw), stream(dev)), "dense_conv2d_split")
    return out_split, out_nchw, (b, oh, ow)


# ---------------------------------------------------------------------------------------------------------------------
# fp16-pair ("H16") path (csrc/dense_conv_f16.cu): the default of DenseRPNHead.  Images are pixel H16 rows
# [B*H*W, 2*C] float16 = per pixel, groups of 32 channels [hi 32 | lo' 32]; x = hi + lo' * 2^-11.
def n_tile_for_f16(cout):
    """Output-channel tile.  P3D_DENSE_NTILE (tuning hook) forces 64 or 128 for the wide layers."""
    import os
    forced = os.environ.get("P3D_DENSE_NTILE")
    if forced and cout >= 128:
        return int(forced)
    return 128 if cout >= 128 else 64


def _status(dev):
    from . import sparse_nn as sp
    return sp.status_tensor(dev)


def nchw_to_pixel_h16(x):
    x = require_cuda(x, "x", torch.float32)
    b, c, h, w = x.shape
    out = torch.empty((b * h * w, 2 * c), dtype=torch.float16, device=x.device)
    check(lib().p3d_nchw_to_pixel_h16(ptr(x), b, c, h, w, ptr(out), ptr(_status(x.device)), stream(x.device)),
          "nchw_to_pixel_h16")
    return out


def pixel_h16_to_nchw(x_h16, shape):
    b, h, w, c = [int(v) for v in shape]
    out = torch.empty((b, c, h, w), dtype=torch.float32, device=x_h16.device)
    check(lib().p3d_pixel_h16_to_nchw(ptr(x_h16), b, c, h, w, ptr(out), stream(x_h16.device)), "pixel_h16_to_nchw")
    return out


def _pack_f16(w_tci, n_tile):
    """w_tci [taps, Cin, Cout] fp32 on the device -> per-N-tile fp16-pair k-block images, concatenated."""
    L = lib()
    taps, cin, cout = w_tci.shape
    tiles = (cout + n_tile - 1) // n_tile
    total = L.p3d_dense_conv2d_f16_packed_weight_bytes(taps, cin, cout, n_tile)
    if not total:
        raise ValueError("unsupported dense conv shape: taps %d Cin %d Cout %d" % (taps, cin, cout))
    packed = torch.zeros((total,), dtype=torch.uint8, device=w_tci.device)
    padded = torch.zeros((taps, cin, tiles * n_tile), dtype=torch.float32, device=w_tci.device)
    padded[:, :, :cout] = w_tci
    block = taps * cin * n_tile * 4
    for t in range(tiles):
        wt = padded[:, :, t * n_tile:(t + 1) * n_tile].contiguous()
        dst = packed[t * block:(t + 1) * block]
        check(L.p3d_dense_conv2d_f16_pack_weights(ptr(wt), taps, cin, n_tile, ptr(dst), ptr(_status(wt.device)),
                                                  stream(wt.device)), "dense_conv2d_f16_pack_weights")
    return packed


def pack_conv_weight_f16(weight, n_tile):
    weight = require_cuda(weight, "weight", torch.float32)
    cout, cin, kh, kw = weight.shape
    return _pack_f16(weight.permute(2, 3, 1, 0).reshape(kh * kw, cin, cout).contiguous(), n_tile)


def pack_deconv_weight_f16(weight, n_tile):
    weight = require_cuda(weight, "weight", torch.float32)
    cin, cout, k, k2 = weight.shape
    return _pack_f16(weight.permute(2, 3, 0, 1).reshape(k * k2, cin, cout).contiguous(), n_tile)


def dense_conv2d_f16(x_h16, shape, packed, cout, n_tile, kernel, stride=1, padding=0, up=1, scale=None, shift=None,
                     relu=False, out_h16=None, out_channels=None, out_c0=0, want_nchw=False, mode=0, m_tiles=0,
                     residual=None, res_channels=None):
    """x_h16 [B*H*W, 2*Cin] float16 pixel H16 rows; shape = (B, H, W, Cin).  Returns (out_h16 or None, out_nchw or None,
    (B, oH, oW)).  out_h16: an existing [B*oH*oW, 2*out_channels] buffer to write channels [out_c0, out_c0 + cout) of
    (channel concat), or None to allocate one; want_nchw adds fp32 planes.  mode 1 forces per-tap loads.  residual: pixel
    H16 rows [B*oH*oW, 2*res_channels] (default cout channels) whose channels [0, cout) are added before ReLU
    (p3d_dense_conv2d_f16_residual: H16 output only)."""
    x_h16 = require_cuda(x_h16, "x_h16", torch.float16)
    b, h, w, cin = [int(v) for v in shape]
    if up > 1:
        oh, ow = h * up, w * up
        kh = kw = st = up
        pd = 0
    else:
        kh = kw = int(kernel)
        st, pd = int(stride), int(padding)
        oh, ow = (h + 2 * pd - kh) // st + 1, (w + 2 * pd - kw) // st + 1
    dev = x_h16.device
    oc = int(out_channels or cout)
    if out_h16 is None and not want_nchw:
        out_h16 = torch.empty((b * oh * ow, 2 * oc), dtype=torch.float16, device=dev)
    out_nchw = torch.empty((b, cout, oh, ow), dtype=torch.float32, device=dev) if want_nchw else None
    if residual is not None:
        residual = require_cuda(residual, "residual", torch.float16)
        rc = int(res_channels or cout)
        if tuple(residual.shape) != (b * oh * ow, 2 * rc):
            raise ValueError("residual rows %s, want (%d, %d)" % (tuple(residual.shape), b * oh * ow, 2 * rc))
        check(lib().p3d_dense_conv2d_f16_residual(
            ptr(x_h16), b, h, w, cin, ptr(packed), int(cout), int(n_tile), kh, kw, st, pd, int(up), ptr(scale), ptr(shift),
            int(relu), ptr(out_h16), oc, int(out_c0), ptr(out_nchw), ptr(residual), rc, int(mode), int(m_tiles),
            ptr(_status(dev)), stream(dev)), "dense_conv2d_f16_residual")
        return out_h16, out_nchw, (b, oh, ow)
    check(lib().p3d_dense_conv2d_f16(ptr(x_h16), b, h, w, cin, ptr(packed), int(cout), int(n_tile), kh, kw, st, pd, int(up),
                                     ptr(scale), ptr(shift), int(relu), ptr(out_h16), oc, int(out_c0), ptr(out_nchw),
                                     int(mode), int(m_tiles), ptr(_status(dev)), stream(dev)), "dense_conv2d_f16")
    return out_h16, out_nchw, (b, oh, ow)


def upsample_bilinear_h16(x_h16, shape, scale, out_h16=None, out_channels=None, out_c0=0):
    """nn.Upsample(scale_factor=scale, mode='bilinear', align_corners=True) on pixel H16 rows x_h16 [B*h*w, 2*C], shape =
    (B, h, w, C) (p3d_upsample_bilinear_h16; scale 1 copies).  Writes channels [out_c0, out_c0 + C) of out_h16 [B*sh*sw,
    2*out_channels] (None: a new C-channel image).  Returns (out_h16, (B, s h, s w))."""
    x_h16 = require_cuda(x_h16, "x_h16", torch.float16)
    b, h, w, c = [int(v) for v in shape]
    s = int(scale)
    oc = int(out_channels or c)
    dev = x_h16.device
    if out_h16 is None:
        out_h16 = torch.empty((b * h * s * w * s, 2 * oc), dtype=torch.float16, device=dev)
    check(lib().p3d_upsample_bilinear_h16(ptr(x_h16), b, h, w, c, s, ptr(out_h16), oc, int(out_c0), ptr(_status(dev)),
                                          stream(dev)), "upsample_bilinear_h16")
    return out_h16, (b, h * s, w * s)


def upsample_nearest_h16(x_h16, shape, scale, out_h16=None, out_channels=None, out_c0=0):
    """F.interpolate(mode='nearest') to scale x the size on pixel H16 rows x_h16 [B*h*w, 2*C], shape = (B, h, w, C)
    (p3d_upsample_nearest_h16: the pairs are copied).  Writes channels [out_c0, out_c0 + C) of out_h16 [B*sh*sw,
    2*out_channels] (None: a new C-channel image).  Returns (out_h16, (B, s h, s w))."""
    x_h16 = require_cuda(x_h16, "x_h16", torch.float16)
    b, h, w, c = [int(v) for v in shape]
    s = int(scale)
    oc = int(out_channels or c)
    dev = x_h16.device
    if out_h16 is None:
        out_h16 = torch.empty((b * h * s * w * s, 2 * oc), dtype=torch.float16, device=dev)
    check(lib().p3d_upsample_nearest_h16(ptr(x_h16), b, h, w, c, s, ptr(out_h16), oc, int(out_c0), stream(dev)),
          "upsample_nearest_h16")
    return out_h16, (b, h * s, w * s)


def pack_stem_weight(weight):
    """ResNet stem weight [64, 3, 7, 7] fp32 -> the mma fragment image p3d_resnet_stem_h16 reads."""
    weight = require_cuda(weight, "weight", torch.float32).contiguous()
    if tuple(weight.shape) != (64, 3, 7, 7):
        raise ValueError("resnet stem weight %s, want (64, 3, 7, 7)" % (tuple(weight.shape),))
    L = lib()
    packed = torch.empty((L.p3d_resnet_stem_packed_weight_bytes(),), dtype=torch.uint8, device=weight.device)
    check(L.p3d_resnet_stem_pack_weights(ptr(weight), ptr(packed), ptr(_status(weight.device)), stream(weight.device)),
          "resnet_stem_pack_weights")
    return packed


def stem_shape(h, w):
    """(pH, pW) of the stem's output: conv 7x7 s2 p3, then MaxPool2d(3, 2, 1)."""
    ch, cw = (h - 1) // 2 + 1, (w - 1) // 2 + 1
    return (ch - 1) // 2 + 1, (cw - 1) // 2 + 1


def resnet_stem_h16(x, packed, scale, shift, out_h16=None):
    """MaxPool2d(3, 2, 1)(ReLU(BN(conv7x7 s2 p3))) of fp32 images x [B, 3, H, W] (p3d_resnet_stem_h16) -> (pixel H16 rows
    [B*pH*pW, 2*64], (B, pH, pW, 64)).  packed: pack_stem_weight; scale / shift [64]: the folded BatchNorm."""
    x = require_cuda(x, "x", torch.float32)
    b, c, h, w = x.shape
    if c != 3:
        raise ValueError("resnet_stem_h16 takes 3-channel images, got %d" % c)
    ph, pw = stem_shape(h, w)
    if out_h16 is None:
        out_h16 = torch.empty((b * ph * pw, 128), dtype=torch.float16, device=x.device)
    check(lib().p3d_resnet_stem_h16(ptr(x), b, h, w, ptr(packed), ptr(scale), ptr(shift), ptr(out_h16),
                                    ptr(_status(x.device)), stream(x.device)), "resnet_stem_h16")
    return out_h16, (b, ph, pw, 64)
