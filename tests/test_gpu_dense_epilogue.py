"""The dense fp16-pair conv's epilogue warps (csrc/dense_conv_f16.cu): one launch that writes both the pixel H16 image
(at a channel offset inside a wider image) and the fp32 NCHW planes gives the same bits as two launches that write one
each, leaves the image's other channels alone, and raises the fp16-overflow status bit when an output saturates."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _t(cuda, a):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(cuda)


@pytest.mark.parametrize("cin,cout,k,stride,pad,up,h,w,m_tiles", [
    (32, 64, 3, 1, 1, 1, 20, 23, 2),    # haloed tiles, two M tiles, ragged edges
    (64, 128, 3, 2, 1, 1, 21, 34, 1),   # per-tap loads, N tile 128
    (64, 64, 2, 2, 0, 2, 9, 11, 1),     # transposed conv: the tap picks the output pixel
])
def test_h16_and_nchw_in_one_launch(cuda, cin, cout, k, stride, pad, up, h, w, m_tiles):
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(cin * 3 + cout)
    x = rng.normal(size=(2, cin, h, w)).astype(np.float32)
    wshape = (cin, cout, k, k) if up > 1 else (cout, cin, k, k)
    wt = (rng.normal(size=wshape) / np.sqrt(cin * k * k)).astype(np.float32)
    scale = _t(cuda, rng.uniform(0.5, 1.5, cout).astype(np.float32))
    shift = _t(cuda, rng.normal(size=cout).astype(np.float32))
    nt = dc.n_tile_for_f16(cout)
    packed = (dc.pack_deconv_weight_f16 if up > 1 else dc.pack_conv_weight_f16)(_t(cuda, wt), nt)
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    oh, ow = (h * up, w * up) if up > 1 else ((h + 2 * pad - k) // stride + 1, (w + 2 * pad - k) // stride + 1)
    oc, c0 = cout + 64, 32  # the layer's channels sit at [32, 32 + cout) of a wider image
    sentinel = torch.full((2 * oh * ow, 2 * oc), 7.0, dtype=torch.float16, device=cuda)
    both = sentinel.clone()
    _, nchw_both, _ = dc.dense_conv2d_f16(xs, (2, h, w, cin), packed, cout, nt, k, stride, pad, up, scale, shift, True,
                                          out_h16=both, out_channels=oc, out_c0=c0, want_nchw=True, m_tiles=m_tiles)
    alone = sentinel.clone()
    dc.dense_conv2d_f16(xs, (2, h, w, cin), packed, cout, nt, k, stride, pad, up, scale, shift, True, out_h16=alone,
                        out_channels=oc, out_c0=c0, m_tiles=m_tiles)
    _, nchw_alone, _ = dc.dense_conv2d_f16(xs, (2, h, w, cin), packed, cout, nt, k, stride, pad, up, scale, shift, True,
                                           want_nchw=True, m_tiles=m_tiles)
    torch.cuda.synchronize()
    assert torch.equal(both, alone)
    assert torch.equal(nchw_both, nchw_alone)
    img = dc.pixel_h16_to_nchw(both, (2, oh, ow, oc))
    # the pair carries 22 of the fp32 value's 24 bits
    np.testing.assert_allclose(img[:, c0:c0 + cout].cpu().numpy(), nchw_both.cpu().numpy(), rtol=2.0 ** -21, atol=2.0 ** -30)
    untouched = torch.cat([img[:, :c0], img[:, c0 + cout:]], 1)
    assert torch.all(untouched == 7.0 + 7.0 / 2048)


def test_overflow_sets_status_bit(cuda):
    import torch
    from paddle3d_b200.ops import dense_conv as dc
    rng = np.random.default_rng(9)
    cin, cout, h, w = 32, 64, 12, 16
    x = rng.normal(size=(1, cin, h, w)).astype(np.float32)
    wt = (rng.normal(size=(cout, cin, 3, 3)) / np.sqrt(cin * 9)).astype(np.float32)
    packed = dc.pack_conv_weight_f16(_t(cuda, wt), 64)
    xs = dc.nchw_to_pixel_h16(_t(cuda, x))
    status = dc._status(cuda)
    status.zero_()
    ones = _t(cuda, np.ones(cout, np.float32))
    zeros = _t(cuda, np.zeros(cout, np.float32))
    dc.dense_conv2d_f16(xs, (1, h, w, cin), packed, cout, 64, 3, 1, 1, 1, ones, zeros, False)
    torch.cuda.synchronize()
    assert int(status.item()) == 0
    big = _t(cuda, np.full(cout, 1e6, np.float32))
    out, _, _ = dc.dense_conv2d_f16(xs, (1, h, w, cin), packed, cout, 64, 3, 1, 1, 1, big, zeros, False)
    torch.cuda.synchronize()
    assert int(status.item()) & 1
    status.zero_()
    assert float(out.float().abs().max()) <= 65504.0
