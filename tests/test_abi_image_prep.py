"""CPU suite: host-side argument checks of p3d_image_prep_u8 (every call here is refused before it reaches the device)."""
import ctypes


def _lib():
    import __graft_entry__ as g
    g.build()
    from paddle3d_b200 import _lib
    return _lib.lib()


def test_image_prep_argument_checks():
    L = _lib()
    buf = ctypes.create_string_buffer(256)
    p = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 16  # 16-byte aligned host pointer, never dereferenced
    mean = (ctypes.c_float * 3)(1, 2, 3)
    sinv = (ctypes.c_double * 3)(1, 1, 1)
    f = L.p3d_image_prep_u8

    def call(fr=p, N=6, band=585, H0=900, W0=1600, kh=p, xb=p, khs=11, rW=704, kv=p, yb=p, kvs=11, rH=396, cx=0, cy=140,
             fH=256, fW=704, m=mean, s=sinv, out=p):
        return f(fr, N, band, H0, W0, kh, xb, khs, rW, kv, yb, kvs, rH, cx, cy, fH, fW, ctypes.cast(m, ctypes.c_void_p)
                 if m is not None else None, ctypes.cast(s, ctypes.c_void_p) if s is not None else None, 1, out, None)
    for k in ("fr", "kh", "xb", "kv", "yb", "m", "s", "out"):
        assert call(**{k: None}) == -1, k
    for k in ("N", "band", "H0", "W0", "khs", "rW", "kvs", "rH", "fH", "fW"):
        assert call(**{k: 0}) == -1, k
    assert call(band=901) == -1                     # the band is part of the source
    assert call(out=p + 4) == -1                    # 16-byte stores
    assert call(khs=9) == -1 and call(kvs=13) == -1  # tables inconsistent with their sizes
    assert call(rW=1600, khs=11) == -1              # scale 1: 5 taps
    assert call(cy=1 << 29) == -1 and call(cx=-(1 << 29)) == -1
    assert call(rW=2000, khs=7) == -1               # upscaling: 5 taps
    assert call(rW=199, khs=35) == -4               # a reduction by more than 8: more than 33 taps
    assert call(rH=112, kvs=35) == -4
    assert call(N=65536) == -4
    assert call(N=6, fH=20000, fW=20000) == -4      # N * 3 * fH * fW past int32
