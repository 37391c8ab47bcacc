"""CPU reference of the JPEG decode of csrc/jpeg.cu, restated sequentially in numpy from ITU T.81 and libjpeg-turbo's
documented default decompression: the marker segments come from virtex_b200.jpeg.parse; everything after SOS is
decoded here one symbol at a time, the way libjpeg's Huffman decoder reads the stream (FF00 unstuffing, zero bits
after a marker, RSTn resets the DC predictors), then islow IDCT, fancy upsampling, table-driven YCbCr -> RGB and
OpenCV's EXIF orientation.  decode(buf) is meant to equal cv2.cvtColor(cv2.imdecode(buf, IMREAD_COLOR), BGR2RGB)."""
import numpy as np

from virtex_b200 import jpeg as J


class _Bits:
    def __init__(self, b, pos):
        self.b, self.pos, self.acc, self.n, self.marker = b, pos, 0, 0, None

    def _byte(self):
        if self.marker is not None or self.pos >= len(self.b):
            return 0
        c = self.b[self.pos]
        self.pos += 1
        if c != 0xFF:
            return c
        while self.pos < len(self.b) and self.b[self.pos] == 0xFF:
            self.pos += 1
        c2 = self.b[self.pos] if self.pos < len(self.b) else 0xD9
        self.pos += 1
        if c2 == 0:
            return 0xFF
        self.marker = c2
        return 0

    def bit(self):
        if self.n == 0:
            self.acc, self.n = self._byte(), 8
        self.n -= 1
        return (self.acc >> self.n) & 1

    def bits(self, s):
        v = 0
        for _ in range(s):
            v = (v << 1) | self.bit()
        return v

    def restart(self, k):
        self.n = 0
        while self.marker is None and self.pos < len(self.b):  # find the marker the data stops at
            self._byte()
        if self.marker != 0xD0 + (k & 7):
            raise ValueError(f"expected RST{k & 7}, found {self.marker}")
        self.marker = None


class _Huff:
    def __init__(self, counts, vals):
        self.maxcode, self.valptr, self.mincode = [-1] * 17, [0] * 17, [0] * 17
        self.vals = vals
        code = k = 0
        for length in range(1, 17):
            c = counts[length - 1]
            if c:
                self.valptr[length], self.mincode[length] = k, code
                code += c
                k += c
                self.maxcode[length] = code - 1
            code <<= 1

    def decode(self, br):
        code = 0
        for length in range(1, 17):
            code = (code << 1) | br.bit()
            if code <= self.maxcode[length]:
                return self.vals[self.valptr[length] + code - self.mincode[length]]
        raise ValueError("bad Huffman code")


def _extend(v, s):
    return v - (1 << s) + 1 if s and v < (1 << (s - 1)) else v


def coefficients(h, b):
    """Entropy decode: per component, int64 [by, bx, 64] coefficients in natural order (absolute DC)."""
    nf = len(h.comps)
    geo = [(1, 1)] if nf == 1 else [(h.comps[0][1], h.comps[0][2]), (1, 1), (1, 1)]
    hmax, vmax = geo[0]
    mcux, mcuy = -(-h.frame_w // (8 * hmax)), -(-h.frame_h // (8 * vmax))
    planes = [np.zeros((mcuy * v, mcux * hh, 64), np.int64) for hh, v in geo]
    dc_t = [_Huff(*h.dc[s[1]]) for s in h.scan]
    ac_t = [_Huff(*h.ac[s[2]]) for s in h.scan]
    br = _Bits(b, h.scan_off)
    pred = [0] * nf
    nrst = 0
    for m in range(mcux * mcuy):
        if h.ri and m and m % h.ri == 0:
            br.restart(nrst)
            nrst += 1
            pred = [0] * nf
        my, mx = divmod(m, mcux)
        for c, (hh, v) in enumerate(geo):
            for dy in range(v):
                for dx in range(hh):
                    blk = planes[c][my * v + dy, mx * hh + dx]
                    s = dc_t[c].decode(br)
                    pred[c] += _extend(br.bits(s), s)
                    blk[0] = np.int16(pred[c])  # libjpeg stores the predictor's sum as a 16-bit coefficient
                    k = 1
                    while k < 64:
                        rs = ac_t[c].decode(br)
                        r, s = rs >> 4, rs & 15
                        if s:
                            k += r
                            if k > 63:
                                raise ValueError("coefficient run past 63")
                            blk[J.ZIGZAG[k]] = _extend(br.bits(s), s)
                            k += 1
                        elif r == 15:
                            k += 16
                        else:
                            break
    return planes, geo


_C = dict(F0298=2446, F0390=3196, F0541=4433, F0765=6270, F0899=7373, F1175=9633, F1501=12299, F1847=15137,
          F1961=16069, F2053=16819, F2562=20995, F3072=25172)


def _idct8(x, shift):
    """islow 8-point pass over the last axis of int64 x [..., 8]."""
    c = _C
    z2, z3 = x[..., 2], x[..., 6]
    z1 = (z2 + z3) * c["F0541"]
    tmp2, tmp3 = z1 - z3 * c["F1847"], z1 + z2 * c["F0765"]
    tmp0, tmp1 = (x[..., 0] + x[..., 4]) << 13, (x[..., 0] - x[..., 4]) << 13
    t10, t13, t11, t12 = tmp0 + tmp3, tmp0 - tmp3, tmp1 + tmp2, tmp1 - tmp2
    tmp0, tmp1, tmp2, tmp3 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
    z1, z2, z3, z4 = tmp0 + tmp3, tmp1 + tmp2, tmp0 + tmp2, tmp1 + tmp3
    z5 = (z3 + z4) * c["F1175"]
    tmp0, tmp1, tmp2, tmp3 = tmp0 * c["F0298"], tmp1 * c["F2053"], tmp2 * c["F3072"], tmp3 * c["F1501"]
    z1, z2, z3, z4 = -z1 * c["F0899"], -z2 * c["F2562"], -z3 * c["F1961"] + z5, -z4 * c["F0390"] + z5
    tmp0, tmp1, tmp2, tmp3 = tmp0 + z1 + z3, tmp1 + z2 + z4, tmp2 + z2 + z3, tmp3 + z1 + z4
    r = 1 << (shift - 1)
    out = [t10 + tmp3, t11 + tmp2, t12 + tmp1, t13 + tmp0, t13 - tmp0, t12 - tmp1, t11 - tmp2, t10 - tmp3]
    return np.stack([(o + r) >> shift for o in out], -1)


def idct_islow(coef, q):
    """coef int64 [..., 64] natural order, q [64] -> uint8 [..., 8, 8] with libjpeg's wrap-around range limit."""
    x = (coef * q).reshape(coef.shape[:-1] + (8, 8))
    ws = _idct8(np.swapaxes(x, -1, -2), 13 - 2)            # columns
    ws = np.swapaxes(ws, -1, -2).astype(np.int32).astype(np.int64)
    out = _idct8(ws, 13 + 2 + 3)                             # rows
    return np.clip(((out + 512) & 1023) - 512 + 128, 0, 255).astype(np.uint8)


def _plane(blocks):
    by, bx = blocks.shape[:2]
    return blocks.transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)


def _upsample(p, h0, v0, H, W):
    """libjpeg-turbo's fancy upsampling of a chroma plane (real size ceil(H / v0) x ceil(W / h0)) to H x W."""
    ch, cw = -(-H // v0), -(-W // h0)
    p = p[:ch, :cw].astype(np.int64)
    if (h0, v0) == (1, 1):
        return p
    if h0 == 2 and cw <= 2:  # h2v1 / h2v2 on a plane at most 2 wide: box replication
        return np.repeat(np.repeat(p, 2, 1), v0, 0)[:H, :W]
    up = np.r_[0, np.arange(ch - 1)]
    dn = np.r_[np.arange(1, ch), ch - 1]
    lf = np.r_[0, np.arange(cw - 1)]
    rt = np.r_[np.arange(1, cw), cw - 1]
    if (h0, v0) == (2, 1):
        out = np.empty((ch, 2 * cw), np.int64)
        out[:, 0::2] = (3 * p + p[:, lf] + 1) >> 2
        out[:, 1::2] = (3 * p + p[:, rt] + 2) >> 2
    elif (h0, v0) == (1, 2):
        out = np.empty((2 * ch, cw), np.int64)
        out[0::2] = (3 * p + p[up] + 1) >> 2
        out[1::2] = (3 * p + p[dn] + 2) >> 2
    else:
        out = np.empty((2 * ch, 2 * cw), np.int64)
        for dy, nb in ((0, up), (1, dn)):
            s = 3 * p + p[nb]
            out[dy::2, 0::2] = (3 * s + s[:, lf] + 8) >> 4
            out[dy::2, 1::2] = (3 * s + s[:, rt] + 7) >> 4
    return out[:H, :W]


def orient(img, o):
    """OpenCV's ApplyExifOrientation."""
    if o in (5, 6, 7, 8):
        img = img.transpose(1, 0, 2)
    if o in (2, 6):
        img = img[:, ::-1]
    elif o in (3, 7):
        img = img[::-1, ::-1]
    elif o in (4, 8):
        img = img[::-1]
    return np.ascontiguousarray(img)


def decode(buf):
    """uint8 (H, W, 3) RGB of a JPEG the device path supports (virtex_b200.jpeg.parse(buf).supported)."""
    b = J._as_bytes(buf)
    h = J.parse(b)
    if not h.supported:
        raise ValueError(f"not on the device path: {h.reason}")
    blocks, geo = coefficients(h, b)
    H, W = h.frame_h, h.frame_w
    planes = [_plane(idct_islow(bl, h.qt[h.comps[c][3]])) for c, bl in enumerate(blocks)]
    y = planes[0][:H, :W].astype(np.int64)
    if len(planes) == 1:
        rgb = np.stack([y, y, y], -1)
    else:
        h0, v0 = geo[0]
        cb = _upsample(planes[1], h0, v0, H, W) - 128
        cr = _upsample(planes[2], h0, v0, H, W) - 128
        r = y + ((91881 * cr + 32768) >> 16)
        g = y + ((-46802 * cr - 22554 * cb + 32768) >> 16)
        bl = y + ((116130 * cb + 32768) >> 16)
        rgb = np.stack([r, g, bl], -1)
    return orient(np.clip(rgb, 0, 255).astype(np.uint8), h.orientation)
