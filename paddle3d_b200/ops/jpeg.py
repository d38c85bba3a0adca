"""Baseline JPEG decoding on the device (csrc/jpeg_decode.cu): the uint8 RGB rows np.asarray(Image.open(f).convert("RGB"))
gives for Pillow's libjpeg-turbo, bit for bit (islow IDCT, fancy upsampling, YCbCr -> RGB of its C code paths).

The host reads the markers (parse) and packs one descriptor per image; it never walks the entropy-coded bytes.  The
device unstuffs them, finds the restart markers, Huffman-decodes the bitstream in parallel, and runs IDCT, upsampling
and colour conversion on the rows asked for.  tests/jpeg_oracle.py restates the decoder in numpy and checks it against
Pillow."""
import functools

import numpy as np
import torch

from .._lib import check, lib
from .._mem import ptr, require_cuda, stream, workspace

MAX_IMAGES = 64
MAX_SIDE = 8192

# One image of a batch: its entropy-coded segment (offset into the concatenated bytes, length up to the EOI marker),
# its geometry (luma sampling hs x vs; chroma is 1 x 1), its restart interval in MCUs (0 = none), and per component
# (Y, Cb, Cr) the quantisation table in natural order and the raw BITS / HUFFVAL of its DC and AC Huffman tables.
DESC_DTYPE = np.dtype([("offset", "<i8"), ("length", "<i4"), ("height", "<i4"), ("width", "<i4"), ("hs", "<i4"),
                       ("vs", "<i4"), ("restart_interval", "<i4"), ("quant", "<u2", (3, 64)),
                       ("dc_bits", "<u1", (3, 16)), ("dc_vals", "<u1", (3, 16)), ("ac_bits", "<u1", (3, 16)),
                       ("ac_vals", "<u1", (3, 256))])
assert DESC_DTYPE.itemsize == 1328

# bits of the status word
STATUS_BAD_CODE = 1      # a code the table does not define, or a run past coefficient 63
STATUS_BAD_RESTART = 2   # a restart marker out of sequence, missing or misplaced
STATUS_TRUNCATED = 4     # the data ends before the last MCU
STATUS_BAD_MARKER = 8    # a marker other than RSTn (or a fill byte) inside the entropy-coded segment
STATUS_BAD_DESC = 16     # a descriptor disagrees with the call (that image is not decoded)

ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6,
                   7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31,
                   39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int32)  # zig-zag index k -> natural (row-major) index

_SOF_NAMES = {0xC2: "progressive DCT (SOF2)", 0xC3: "lossless (SOF3)", 0xC5: "differential sequential (SOF5)",
              0xC6: "differential progressive (SOF6)", 0xC7: "differential lossless (SOF7)",
              0xC9: "arithmetic coding (SOF9)", 0xCA: "arithmetic progressive (SOF10)", 0xCB: "arithmetic lossless (SOF11)",
              0xCD: "arithmetic differential (SOF13)", 0xCE: "arithmetic differential progressive (SOF14)",
              0xCF: "arithmetic differential lossless (SOF15)"}


class JpegHeader:
    """What parse() reads: height, width, sampling [(h, v)] * 3, quant [3, 64] uint16 (natural order, per component),
    dc / ac [(bits uint8 [16], vals uint8 [n])] * 3 (per component), restart_interval (MCUs, 0 = none), ecs (start, end)
    byte range of the entropy-coded segment."""

    __slots__ = ("height", "width", "sampling", "quant", "dc", "ac", "restart_interval", "ecs")

    @property
    def hs(self):
        return self.sampling[0][0]

    @property
    def vs(self):
        return self.sampling[0][1]

    @property
    def mcus(self):
        """(MCU rows, MCU columns)."""
        return (-(-self.height // (8 * self.vs)), -(-self.width // (8 * self.hs)))


def _u16(data, i):
    return (data[i] << 8) | data[i + 1]


def _check_huffman(bits, vals, kind, tid):
    """Canonical codes of BITS must fit their lengths, and no code may be all ones (T.81 Annex C reserves it): a decoder
    reading the < 8 one-bits that pad a restart interval then never completes a symbol there."""
    code = 0
    for length in range(1, 17):
        code += int(bits[length - 1])  # one past the last code of this length
        if code > (1 << length):
            raise ValueError("jpeg: Huffman table %s%d has more codes than %d-bit lengths allow" % (kind, tid, length))
        if code == (1 << length):
            raise ValueError("jpeg: Huffman table %s%d uses the all-ones code" % (kind, tid))
        code <<= 1
    if kind == "DC" and len(vals) and vals.max() > 11:
        raise ValueError("jpeg: DC table %d has a category above 11 (8-bit samples)" % tid)
    if kind == "AC" and len(vals) and (vals & 15).max() > 10:
        raise ValueError("jpeg: AC table %d has a size above 10 (8-bit samples)" % tid)


@functools.lru_cache(maxsize=256)
def _huffman_table(raw, tc, th):
    """(BITS, HUFFVAL) of one DHT table from its 16 + n bytes, checked; cached, since a camera's encoder repeats its
    tables in every file."""
    bits = np.frombuffer(raw[:16], np.uint8)
    vals = np.frombuffer(raw[16:], np.uint8)
    _check_huffman(bits, vals, "AC" if tc else "DC", th)
    return bits, vals


def parse(data):
    """Read the markers of one JPEG file (bytes, bytearray, memoryview or uint8 numpy array) and return its
    JpegHeader.  Raises ValueError naming the reason for anything outside the supported set: baseline / extended
    sequential Huffman DCT, 8-bit, three components Y Cb Cr in one interleaved scan, chroma 1 x 1 and luma 1 x 1, 2 x 1
    or 2 x 2, at most 8192 x 8192."""
    if isinstance(data, np.ndarray):
        data = data.tobytes()
    elif not isinstance(data, bytes):
        data = bytes(data)
    n = len(data)
    if n < 4 or data[0] != 0xFF or data[1] != 0xD8:
        raise ValueError("jpeg: no SOI marker")
    qt = {}
    dht = {}
    sof = None
    ri = 0
    jfif = adobe = False
    adobe_transform = None
    i = 2
    while True:
        if i + 4 > n:
            raise ValueError("jpeg: truncated header")
        if data[i] != 0xFF:
            raise ValueError("jpeg: expected a marker at byte %d" % i)
        while i < n and data[i] == 0xFF:
            i += 1
        if i + 3 > n:
            raise ValueError("jpeg: truncated header")
        m = data[i]
        i += 1
        if m in (0xD8, 0xD9) or 0xD0 <= m <= 0xD7 or m == 0x01:
            raise ValueError("jpeg: marker 0x%02X before the scan" % m)
        length = _u16(data, i)
        if length < 2 or i + length > n:
            raise ValueError("jpeg: truncated header (marker 0x%02X)" % m)
        seg = data[i + 2:i + length]
        start = i + length
        i = start
        if 0xE0 <= m <= 0xEF or m == 0xFE:
            if m == 0xE0 and seg[:5] == b"JFIF\0":
                jfif = True
            if m == 0xEE and seg[:5] == b"Adobe" and len(seg) >= 12:
                adobe, adobe_transform = True, seg[11]
            continue
        if m == 0xDB:
            j = 0
            while j < len(seg):
                pq, tq = seg[j] >> 4, seg[j] & 15
                if pq > 1 or tq > 3:
                    raise ValueError("jpeg: bad DQT table %d precision %d" % (tq, pq))
                size = 64 * (pq + 1)
                if j + 1 + size > len(seg):
                    raise ValueError("jpeg: truncated header (DQT)")
                raw = np.frombuffer(seg[j + 1:j + 1 + size], np.uint8 if pq == 0 else ">u2").astype(np.uint16)
                tab = np.zeros(64, np.uint16)
                tab[ZIGZAG] = raw
                qt[tq] = tab
                j += 1 + size
            continue
        if m == 0xC4:
            j = 0
            while j < len(seg):
                if j + 17 > len(seg):
                    raise ValueError("jpeg: truncated header (DHT)")
                tc, th = seg[j] >> 4, seg[j] & 15
                if tc > 1 or th > 3:
                    raise ValueError("jpeg: bad DHT class %d id %d" % (tc, th))
                cnt = sum(seg[j + 1:j + 17])
                if cnt > 256 or j + 17 + cnt > len(seg):
                    raise ValueError("jpeg: truncated or oversized DHT table")
                dht[(tc, th)] = _huffman_table(seg[j + 1:j + 17 + cnt], tc, th)
                j += 17 + cnt
            continue
        if m == 0xDD:
            if length != 4:
                raise ValueError("jpeg: bad DRI length")
            ri = _u16(data, start - 2)
            continue
        if m in (0xC0, 0xC1):
            if sof is not None:
                raise ValueError("jpeg: second SOF marker")
            if len(seg) < 6:
                raise ValueError("jpeg: truncated header (SOF)")
            if seg[0] != 8:
                raise ValueError("jpeg: %d-bit samples (only 8-bit are supported)" % seg[0])
            H, W, nf = _u16(seg, 1), _u16(seg, 3), seg[5]
            if nf != 3:
                raise ValueError("jpeg: %d components (only three, Y Cb Cr, are supported: no grayscale or CMYK)" % nf)
            if len(seg) < 6 + 3 * nf:
                raise ValueError("jpeg: truncated header (SOF)")
            comps = [(seg[6 + 3 * c], seg[7 + 3 * c] >> 4, seg[7 + 3 * c] & 15, seg[8 + 3 * c]) for c in range(nf)]
            if H == 0 or W == 0:
                raise ValueError("jpeg: image size %d x %d (a DNL-defined height is not supported)" % (H, W))
            if H > MAX_SIDE or W > MAX_SIDE:
                raise ValueError("jpeg: image size %d x %d is over the limit of %d" % (H, W, MAX_SIDE))
            samp = [(c[1], c[2]) for c in comps]
            if samp[1] != (1, 1) or samp[2] != (1, 1) or samp[0] not in ((1, 1), (2, 1), (2, 2)):
                raise ValueError("jpeg: sampling %s (supported: chroma 1x1, luma 1x1, 2x1 or 2x2)" % (samp,))
            sof = (H, W, comps)
            continue
        if m in _SOF_NAMES:
            raise ValueError("jpeg: %s is not supported" % _SOF_NAMES[m])
        if m == 0xCC:
            raise ValueError("jpeg: arithmetic coding (DAC) is not supported")
        if m == 0xDA:
            if sof is None:
                raise ValueError("jpeg: SOS before SOF")
            H, W, comps = sof
            ns = seg[0] if seg else 0
            if ns != 3 or len(seg) < 1 + 2 * ns + 3:
                raise ValueError("jpeg: the scan holds %d components (one interleaved scan of three is supported)" % ns)
            sel = [(seg[1 + 2 * c], seg[2 + 2 * c] >> 4, seg[2 + 2 * c] & 15) for c in range(ns)]
            ss, se, ahl = seg[1 + 2 * ns], seg[2 + 2 * ns], seg[3 + 2 * ns]
            if ss != 0 or se != 63 or ahl != 0:
                raise ValueError("jpeg: scan parameters Ss=%d Se=%d Ah/Al=%d (not a sequential scan)" % (ss, se, ahl))
            if [s[0] for s in sel] != [c[0] for c in comps]:
                raise ValueError("jpeg: scan component order differs from the frame's")
            ids = [c[0] for c in comps]
            if adobe and adobe_transform != 1:
                raise ValueError("jpeg: Adobe transform %d (only YCbCr is supported)" % adobe_transform)
            if not jfif and not adobe and ids == [82, 71, 66]:
                raise ValueError("jpeg: RGB components (only YCbCr is supported)")
            hdr = JpegHeader()
            hdr.height, hdr.width = H, W
            hdr.sampling = [(c[1], c[2]) for c in comps]
            hdr.restart_interval = ri
            q, dc, ac = [], [], []
            for c, s in zip(comps, sel):
                if c[3] not in qt:
                    raise ValueError("jpeg: missing quantisation table %d" % c[3])
                if (0, s[1]) not in dht:
                    raise ValueError("jpeg: missing DC Huffman table %d" % s[1])
                if (1, s[2]) not in dht:
                    raise ValueError("jpeg: missing AC Huffman table %d" % s[2])
                q.append(qt[c[3]])
                dc.append(dht[(0, s[1])])
                ac.append(dht[(1, s[2])])
            hdr.quant = np.stack(q)
            hdr.dc, hdr.ac = dc, ac
            end = data.rfind(b"\xff\xd9")
            if end < start:
                raise ValueError("jpeg: no EOI marker after the scan")
            hdr.ecs = (start, end)
            return hdr
        raise ValueError("jpeg: unsupported marker 0x%02X" % m)


def pack(headers, offsets, desc=None):
    """Descriptors (DESC_DTYPE [N]) of images whose files start at offsets[i] in the concatenated bytes."""
    desc = np.zeros(len(headers), DESC_DTYPE) if desc is None else desc
    for i, (h, off) in enumerate(zip(headers, offsets)):
        d = desc[i]
        d["offset"] = int(off) + h.ecs[0]
        d["length"] = h.ecs[1] - h.ecs[0]
        d["height"], d["width"] = h.height, h.width
        d["hs"], d["vs"] = h.hs, h.vs
        d["restart_interval"] = h.restart_interval
        d["quant"] = h.quant
        d["dc_bits"] = 0
        d["dc_vals"] = 0
        d["ac_bits"] = 0
        d["ac_vals"] = 0
        for c in range(3):
            d["dc_bits"][c] = h.dc[c][0]
            d["dc_vals"][c, :len(h.dc[c][1])] = h.dc[c][1]
            d["ac_bits"][c] = h.ac[c][0]
            d["ac_vals"][c, :len(h.ac[c][1])] = h.ac[c][1]
    return desc


def batch(files, size=None, out=None):
    """Parse N files and concatenate them: (data uint8 numpy [sum of lengths], desc DESC_DTYPE [N], headers).  size
    (H, W): every image must have it (ValueError otherwise); None takes the first image's.  out: a uint8 numpy array to
    concatenate into (data is then its first bytes; ValueError when the files do not fit)."""
    blobs = [f if isinstance(f, bytes) else (f.tobytes() if isinstance(f, np.ndarray) else bytes(f)) for f in files]
    headers = [parse(b) for b in blobs]
    if not headers:
        raise ValueError("jpeg: no images")
    if size is None:
        size = (headers[0].height, headers[0].width)
    for i, h in enumerate(headers):
        if (h.height, h.width) != tuple(size):
            raise ValueError("jpeg: image %d is %d x %d, want %d x %d" % (i, h.height, h.width, size[0], size[1]))
    offsets = np.cumsum([0] + [len(b) for b in blobs])
    if out is None:
        out = np.empty(int(offsets[-1]), np.uint8)
    elif len(out) < offsets[-1]:
        raise ValueError("jpeg: %d bytes do not fit in %d" % (offsets[-1], len(out)))
    for b, o in zip(blobs, offsets):
        out[o:o + len(b)] = np.frombuffer(b, np.uint8)
    return out[:offsets[-1]], pack(headers, offsets[:-1]), headers


def workspace_bytes(n, size, max_bytes):
    return lib().p3d_jpeg_decode_workspace_bytes(int(n), int(size[0]), int(size[1]), int(max_bytes))


def jpeg_decode_u8(data_dev, desc_dev, n, size, rows=None, out=None, status=None, max_bytes=None):
    """Decode n JPEG images of size (H, W) on the device (p3d_jpeg_decode_u8): data_dev uint8 (the concatenated
    files), desc_dev uint8 (n DESC_DTYPE records, as batch() builds them) -> uint8 [n, y1 - y0, W, 3], rows [y0, y1)
    of every image (default: all).  status: int32 [n] on the device (one word per image, bits OR-ed in), or None for
    a fresh one that is checked here (RuntimeError naming the image on corrupt data, which synchronises); a caller that
    passes its own reads it later.  max_bytes: the
    largest entropy-coded segment the workspace is sized for (default: all of data_dev)."""
    data_dev = require_cuda(data_dev, "data", torch.uint8)
    desc_dev = require_cuda(desc_dev, "desc", torch.uint8)
    H, W = (int(v) for v in size)
    y0, y1 = (0, H) if rows is None else (int(rows[0]), int(rows[1]))
    if not 0 <= y0 < y1 <= H:
        raise ValueError("jpeg_decode_u8: rows %s outside [0, %d)" % ((y0, y1), H))
    if desc_dev.numel() < n * DESC_DTYPE.itemsize:
        raise ValueError("jpeg_decode_u8: descriptor holds %d bytes, want %d" % (desc_dev.numel(),
                                                                                 n * DESC_DTYPE.itemsize))
    shape = (n, y1 - y0, W, 3)
    if out is None:
        out = torch.empty(shape, dtype=torch.uint8, device=data_dev.device)
    elif out.dtype != torch.uint8 or tuple(out.shape) != shape or not out.is_contiguous():
        raise ValueError("jpeg_decode_u8: out %s %s, want contiguous uint8 %s" % (tuple(out.shape), out.dtype, shape))
    own_status = status is None
    if own_status:
        status = torch.zeros(n, dtype=torch.int32, device=data_dev.device)
    elif status.dtype != torch.int32 or status.numel() < n or not status.is_contiguous():
        raise ValueError("jpeg_decode_u8: status %s %s, want contiguous int32 [%d]" % (tuple(status.shape), status.dtype, n))
    max_bytes = data_dev.numel() if max_bytes is None else int(max_bytes)
    L = lib()
    ws = workspace(L.p3d_jpeg_decode_workspace_bytes(n, H, W, max_bytes), data_dev.device, "jpeg")
    check(L.p3d_jpeg_decode_u8(ptr(data_dev), data_dev.numel(), ptr(desc_dev), n, H, W, y0, y1, max_bytes, ptr(out),
                               ptr(status), ptr(ws), ws.numel(), stream(data_dev.device)), "jpeg_decode_u8")
    if own_status:
        for i, s in enumerate(status.cpu().tolist()):
            if s:
                raise RuntimeError("jpeg_decode_u8: image %d: corrupt JPEG data (status 0x%x: %s)" % (i, s, status_reason(s)))
    return out


def status_reason(s):
    names = [(STATUS_BAD_CODE, "bad Huffman code"), (STATUS_BAD_RESTART, "restart marker out of sequence"),
             (STATUS_TRUNCATED, "data ends before the last MCU"), (STATUS_BAD_MARKER, "unexpected marker"),
             (STATUS_BAD_DESC, "descriptor disagrees with the call")]
    return ", ".join(t for b, t in names if s & b) or "none"
