"""CPU suite: host-side argument checks of p3d_jpeg_decode_u8 and its workspace size (every call here is refused before
it reaches the device)."""
import ctypes


def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib.lib()


def test_jpeg_workspace_bytes():
    L = _lib()
    ws = L.p3d_jpeg_decode_workspace_bytes
    assert ws(6, 900, 1600, 1 << 20) > 6 * 900 * 1600 * 3  # at least the coefficient planes of 4:4:4
    assert ws(6, 900, 1600, 1 << 21) > ws(6, 900, 1600, 1 << 20) > ws(1, 900, 1600, 1 << 20)
    for args in ((0, 900, 1600, 1), (6, 0, 1600, 1), (6, 900, 0, 1), (6, 900, 1600, 0), (65, 8, 8, 1), (1, 8193, 8, 1),
                 (1, 8, 8193, 1), (1, 8, 8, (1 << 28) + 1)):
        assert ws(*args) == 0, args
    assert ws(64, 8192, 8192, 1 << 28) > 0


def test_jpeg_decode_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf)  # host pointer, never dereferenced
    f = L.p3d_jpeg_decode_u8
    big = L.p3d_jpeg_decode_workspace_bytes(6, 900, 1600, 1 << 20)

    def call(data=p, nbytes=1 << 20, desc=p, N=6, H=900, W=1600, y0=0, y1=900, max_bytes=1 << 20, out=p, status=p, ws=p,
             ws_bytes=big):
        return f(data, nbytes, desc, N, H, W, y0, y1, max_bytes, out, status, ws, ws_bytes, None)
    for k in ("data", "desc", "out", "status", "ws"):
        assert call(**{k: None}) == -1, k
    for k in ("nbytes", "N", "H", "W", "max_bytes"):
        assert call(**{k: 0}) == -1, k
    assert call(y0=-1) == -1 and call(y1=0) == -1 and call(y0=5, y1=5) == -1 and call(y1=901) == -1
    assert call(N=65) == -4
    assert call(H=8193, y1=8193) == -4 and call(W=8193) == -4
    assert call(max_bytes=(1 << 28) + 1) == -4
    assert call(ws_bytes=big - 1) == -2                       # workspace smaller than p3d_jpeg_decode_workspace_bytes
