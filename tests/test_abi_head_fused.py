"""CPU suite: host-side argument checks of the fused CenterHead entry points (p3d_head_conv_p_f16, p3d_head_tap_sum).
Every call here is refused before it reaches the device."""
import ctypes


def test_head_fused_argument_checks():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    L = _lib.lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16  # 16-byte aligned host pointer, never dereferenced
    odd = p + 4
    conv = L.p3d_head_conv_p_f16
    # missing W2 images / P buffer, empty image, misaligned P buffer
    assert conv(p, 1, 8, 8, 64, p, 256, p, p, None, p, None, None) == -1
    assert conv(p, 1, 8, 8, 64, p, 256, p, p, p, None, None, None) == -1
    assert conv(p, 0, 8, 8, 64, p, 256, p, p, p, p, None, None) == -1
    assert conv(p, 1, 8, 8, 64, p, 256, p, p, p, odd, None, None) == -1
    # input channels not a multiple of 32, heads that do not fill whole 128-channel N tiles
    assert conv(p, 1, 8, 8, 48, p, 256, p, p, p, p, None, None) == -4
    assert conv(p, 1, 8, 8, 64, p, 192, p, p, p, p, None, None) == -4
    tap = L.p3d_head_tap_sum
    assert tap(None, 1, 8, 8, 4, p, p, p, 8, p, None) == -1
    assert tap(p, 1, 8, 8, 0, p, p, p, 8, p, None) == -1
    assert tap(p, 1, 8, 8, 4, p, p, None, 8, p, None) == -1
    assert tap(odd, 1, 8, 8, 4, p, p, p, 8, p, None) == -1
