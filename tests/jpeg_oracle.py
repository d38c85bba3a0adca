"""numpy restatement of the device JPEG decoder (csrc/jpeg_decode.cu), stage by stage, written against libjpeg-turbo's C
code paths that Pillow's Image.open runs: the sequential Huffman decode (jdhuff.c, restart handling of jdmarker.c), the
DC prediction, jpeg_idct_islow (jidctint.c) with its range_limit table (jdmaster.c), h2v1 / h2v2 fancy upsampling and the
plain replication used below three chroma columns (jdsample.c) with the context rows of jdmainct.c, and ycc_rgb_convert
(jdcolor.c).  It is sequential and slow; it is the reference, not a product path."""
import numpy as np

from paddle3d_b200.ops.jpeg import ZIGZAG, parse


# ---------------------------------------------------------------- entropy decode


def _segments(ecs):
    """Unstuff the entropy-coded segment and split it at its RSTn markers: [(marker number or None, bytes)]."""
    out, cur, num = [], bytearray(), None
    i, n = 0, len(ecs)
    while i < n:
        b = ecs[i]
        if b != 0xFF:
            cur.append(b)
            i += 1
            continue
        if i + 1 >= n:
            raise ValueError("oracle: 0xFF at the end of the data")
        m = ecs[i + 1]
        if m == 0x00:
            cur.append(0xFF)
        elif 0xD0 <= m <= 0xD7:
            out.append((num, bytes(cur)))
            cur, num = bytearray(), m - 0xD0
        else:
            raise ValueError("oracle: marker 0x%02X inside the scan" % m)
        i += 2
    out.append((num, bytes(cur)))
    return out


class _Bits:
    def __init__(self, data):
        self.v = int.from_bytes(data, "big") if data else 0
        self.n = 8 * len(data)
        self.p = 0

    def get(self, k):
        if k == 0:
            return 0
        if self.p + k > self.n:
            raise ValueError("oracle: data ends before the last MCU")
        r = (self.v >> (self.n - self.p - k)) & ((1 << k) - 1)
        self.p += k
        return r


def _table(bits, vals):
    """code length -> {code: symbol} (canonical codes of T.81 Annex C)."""
    t, code, j = {}, 0, 0
    for length in range(1, 17):
        d = {}
        for _ in range(int(bits[length - 1])):
            d[code] = int(vals[j])
            code += 1
            j += 1
        t[length] = d
        code <<= 1
    return t


def _decode_symbol(br, tab):
    code = 0
    for length in range(1, 17):
        code = (code << 1) | br.get(1)
        s = tab[length].get(code)
        if s is not None:
            return s
    raise ValueError("oracle: undefined Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def entropy_decode(data, hdr=None):
    """Coefficients of every component: [bh, bw, 64] int64 in natural (row-major) order, DC undifferenced, quantised
    (bh x bw = the MCU grid's blocks of the component, padding blocks included)."""
    hdr = hdr or parse(data)
    data = bytes(data)
    mr, mc = hdr.mcus
    samp = hdr.sampling
    coef = [np.zeros((mr * v, mc * h, 64), np.int64) for h, v in samp]
    dct = [_table(*t) for t in hdr.dc]
    act = [_table(*t) for t in hdr.ac]
    segs = _segments(data[hdr.ecs[0]:hdr.ecs[1]])
    ri = hdr.restart_interval or mr * mc
    total = mr * mc
    if len(segs) != -(-total // ri):
        raise ValueError("oracle: %d restart intervals, want %d" % (len(segs), -(-total // ri)))
    for r, (num, seg) in enumerate(segs):
        if r and num != (r - 1) % 8:
            raise ValueError("oracle: restart marker out of sequence")
        br = _Bits(seg)
        pred = [0, 0, 0]
        for m in range(r * ri, min(total, (r + 1) * ri)):
            my, mx = divmod(m, mc)
            for c, (h, v) in enumerate(samp):
                for by in range(v):
                    for bx in range(h):
                        blk = coef[c][my * v + by, mx * h + bx]
                        s = _decode_symbol(br, dct[c])
                        pred[c] += _extend(br.get(s), s)
                        blk[0] = pred[c]
                        k = 1
                        while k < 64:
                            rs = _decode_symbol(br, act[c])
                            run, s = rs >> 4, rs & 15
                            if s:
                                k += run
                                if k > 63:
                                    raise ValueError("oracle: run past coefficient 63")
                                blk[ZIGZAG[k]] = _extend(br.get(s), s)
                                k += 1
                            elif run == 15:
                                k += 16
                            else:
                                break
    return coef


# ---------------------------------------------------------------- islow IDCT

CONST_BITS, PASS1_BITS = 13, 2
FIX_0_298631336, FIX_0_390180644, FIX_0_541196100, FIX_0_765366865 = 2446, 3196, 4433, 6270
FIX_0_899976223, FIX_1_175875602, FIX_1_501321110, FIX_1_847759065 = 7373, 9633, 12299, 15137
FIX_1_961570560, FIX_2_053119869, FIX_2_562915447, FIX_3_072711026 = 16069, 16819, 20995, 25172


def _descale(x, n):
    return (x + (1 << (n - 1))) >> n


def _idct_1d(i0, i1, i2, i3, i4, i5, i6, i7):
    """One pass of jpeg_idct_islow before its descale: outputs 0..7."""
    z1 = (i2 + i6) * FIX_0_541196100
    tmp2 = z1 + i6 * -FIX_1_847759065
    tmp3 = z1 + i2 * FIX_0_765366865
    tmp0 = (i0 + i4) << CONST_BITS
    tmp1 = (i0 - i4) << CONST_BITS
    tmp10, tmp13, tmp11, tmp12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    t0, t1, t2, t3 = i7, i5, i3, i1
    z1, z2, z3, z4 = t0 + t3, t1 + t2, t0 + t2, t1 + t3
    z5 = (z3 + z4) * FIX_1_175875602
    t0, t1, t2, t3 = t0 * FIX_0_298631336, t1 * FIX_2_053119869, t2 * FIX_3_072711026, t3 * FIX_1_501321110
    z1, z2 = z1 * -FIX_0_899976223, z2 * -FIX_2_562915447
    z3, z4 = z3 * -FIX_1_961570560 + z5, z4 * -FIX_0_390180644 + z5
    t0 += z1 + z3
    t1 += z2 + z4
    t2 += z2 + z3
    t3 += z1 + z4
    return [tmp10 + t3, tmp11 + t2, tmp12 + t1, tmp13 + t0, tmp13 - t0, tmp12 - t1, tmp11 - t2, tmp10 - t3]


def range_limit_idct(x):
    """IDCT_range_limit(cinfo)[x & RANGE_MASK]: the 10-bit wrap, then the clamp of the shifted sample."""
    s = ((x + 512) & 1023) - 512
    return np.clip(s + 128, 0, 255)


def idct_islow(coef, quant):
    """coef [..., 64] quantised (natural order), quant [64] -> uint8 [..., 8, 8]."""
    c = coef.reshape(-1, 8, 8).astype(np.int64) * quant.reshape(8, 8).astype(np.int64)
    ws = np.stack(_idct_1d(*[c[:, r, :] for r in range(8)]), axis=1)          # pass 1 over columns: [b, row, col]
    ws = _descale(ws, CONST_BITS - PASS1_BITS)
    ws = ((ws + (1 << 31)) % (1 << 32)) - (1 << 31)                            # the int workspace
    out = np.stack(_idct_1d(*[ws[:, :, j] for j in range(8)]), axis=2)        # pass 2 over rows
    out = range_limit_idct(_descale(out, CONST_BITS + PASS1_BITS + 3))
    return out.astype(np.uint8).reshape(coef.shape[:-1] + (8, 8))


def planes(coef, quant):
    """Component sample planes uint8 [bh * 8, bw * 8] (MCU-padded)."""
    out = []
    for c, q in zip(coef, quant):
        bh, bw = c.shape[:2]
        px = idct_islow(c, q)
        out.append(np.ascontiguousarray(px.transpose(0, 2, 1, 3).reshape(bh * 8, bw * 8)))
    return out


# ---------------------------------------------------------------- upsampling and colour


def upsample(plane, dh, dw, hs, vs, H, W):
    """A chroma plane (real size dh x dw in its top-left) to H x W, as jdsample.c does for luma sampling hs x vs."""
    p = plane[:dh, :dw].astype(np.int32)
    if vs == 2:
        fancy = dw > 2
        if fancy:
            ys = np.arange(H)
            near = ys // 2
            far = np.clip(np.where(ys % 2 == 0, near - 1, near + 1), 0, dh - 1)  # context rows: the last real row
            cs = 3 * p[near] + p[far]                                         # column sums [H, dw]
            xs = np.arange(W)
            i = xs // 2
            left = np.maximum(i - 1, 0)
            right = np.minimum(i + 1, dw - 1)
            even = (3 * cs[:, i] + cs[:, left] + 8) >> 4
            odd = (3 * cs[:, i] + cs[:, right] + 7) >> 4
            return np.where(xs % 2 == 0, even, odd).astype(np.uint8)
        return p[np.arange(H) // 2][:, np.arange(W) // 2].astype(np.uint8)
    if hs == 2:
        rows = p[:H]
        if dw > 2:
            xs = np.arange(W)
            i = xs // 2
            left = np.maximum(i - 1, 0)
            right = np.minimum(i + 1, dw - 1)
            even = (3 * rows[:, i] + rows[:, left] + 1) >> 2
            odd = (3 * rows[:, i] + rows[:, right] + 2) >> 2
            return np.where(xs % 2 == 0, even, odd).astype(np.uint8)
        return rows[:, np.arange(W) // 2].astype(np.uint8)
    return p[:H, :W].astype(np.uint8)


SCALEBITS = 16
ONE_HALF = 1 << (SCALEBITS - 1)
FIX_1_40200, FIX_1_77200, FIX_0_71414, FIX_0_34414 = 91881, 116130, 46802, 22554


def ycc_to_rgb(y, cb, cr):
    y, cb, cr = (a.astype(np.int64) for a in (y, cb, cr))
    x_cb, x_cr = cb - 128, cr - 128
    r = y + ((FIX_1_40200 * x_cr + ONE_HALF) >> SCALEBITS)
    g = y + ((-FIX_0_34414 * x_cb + ONE_HALF + -FIX_0_71414 * x_cr) >> SCALEBITS)
    b = y + ((FIX_1_77200 * x_cb + ONE_HALF) >> SCALEBITS)
    return np.clip(np.stack([r, g, b], -1), 0, 255).astype(np.uint8)


def decode(data):
    """uint8 [H, W, 3]: what np.asarray(Image.open(f).convert("RGB")) gives."""
    hdr = parse(data)
    coef = entropy_decode(data, hdr)
    pl = planes(coef, hdr.quant)
    H, W, hs, vs = hdr.height, hdr.width, hdr.hs, hdr.vs
    dh, dw = -(-H // vs), -(-W // hs)
    y = pl[0][:H, :W]
    cb = upsample(pl[1], dh, dw, hs, vs, H, W)
    cr = upsample(pl[2], dh, dw, hs, vs, H, W)
    return ycc_to_rgb(y, cb, cr)
