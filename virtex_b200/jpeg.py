"""JPEG decoding on the GPU, bit-exact with the reference's image reads.

Every dataset of the reference reads its images with `cv2.imread(path)` + `cv2.cvtColor(image, cv2.COLOR_BGR2RGB)`
(virtex/data/datasets/captioning.py, classification.py, downstream.py).  `decode(buffers, device)` gives the same
uint8 HWC RGB pixels from the compressed bytes, computed by the kernels of csrc/jpeg.cu:

    images = jpeg.decode([open(p, "rb").read() for p in paths], "cuda")   # list of (H, W, 3) uint8 CUDA tensors

The host parses the marker segments up to SOS (this module) and hands the kernels a small table per image.  The
device path covers baseline / extended sequential Huffman JPEGs, 8-bit, one interleaved scan, grey or YCbCr with luma
sampling 1x1, 2x1, 1x2 or 2x2 and 1x1 chroma, with or without restart markers, and every EXIF orientation.  Anything
else -- progressive, arithmetic, 12-bit, CMYK / YCCK / RGB, multi-scan, other sampling, EXIF blocks this parser does
not fully understand, a missing EOI, data that is not a JPEG, and streams whose entropy data the device finds corrupt
-- is decoded by cv2 on the host, so the output equals the reference's by construction.  Only a fallback needed while
cv2 is not importable raises (ValueError naming the image).
"""
import struct
from typing import List, Optional, Sequence

import numpy as np
import torch

from .ops import _stream, call

# include/virtex_b200.h
NI, N64, HUFF_BYTES = 48, 8, 1536
I_H, I_W, I_ORIENT, I_NCOMP, I_MCUX, I_MCUY, I_RI, I_BPM, I_NSEG = range(9)
I_SEG_BASE, I_CHUNK_BASE, I_CHUNK_CAP, I_OH, I_OW, I_COMP = 9, 10, 11, 12, 13, 16
Q_ENT_SRC, Q_ENT_LEN, Q_ENT_DST, Q_COEF, Q_PLANE, Q_OUT = 0, 1, 2, 3, 4, 7
ST_MARKER, ST_BADCODE, ST_RUN, ST_OUT, ST_UNSYNCED = 1, 2, 4, 8, 16

CHUNK_BITS = 1024     # bits per self-synchronising decode chunk
# rounds launched before the first status read: 640x480 q90 4:2:0 images need 4-9 (H100 run of scripts/bench_jpeg.py),
# and a round in which a chunk's predecessor did not change only copies its state
SYNC_ROUNDS = 16

# zig-zag index -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13,
                   6, 7, 14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38,
                   31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63], np.int64)

_SOF_NAMES = {0xC0: "baseline", 0xC1: "extended sequential", 0xC2: "progressive", 0xC3: "lossless",
              0xC5: "differential sequential", 0xC6: "differential progressive", 0xC7: "differential lossless",
              0xC9: "arithmetic sequential", 0xCA: "arithmetic progressive", 0xCB: "arithmetic lossless",
              0xCD: "differential arithmetic sequential", 0xCE: "differential arithmetic progressive",
              0xCF: "differential arithmetic lossless"}
MAX_DIMENSION = 65500  # libjpeg's JPEG_MAX_DIMENSION


class JpegHeader:
    """What the marker segments up to SOS say about one image.  `supported` is False with a `reason` when the image
    has to be decoded on the host; `height` / `width` are the oriented size the decode returns."""
    __slots__ = ("supported", "reason", "frame_h", "frame_w", "orientation", "height", "width", "precision", "sof",
                 "comps", "qt", "dc", "ac", "scan", "ss_se_ah_al", "ri", "scan_off", "eoi", "jfif", "adobe")

    def __init__(self):
        self.supported, self.reason = True, ""
        self.frame_h = self.frame_w = self.height = self.width = 0
        self.orientation, self.precision, self.sof, self.ri = 1, 8, None, 0
        self.comps, self.scan, self.ss_se_ah_al = [], [], None
        self.qt, self.dc, self.ac = {}, {}, {}
        self.scan_off = self.eoi = -1
        self.jfif, self.adobe = False, None

    def _reject(self, reason):
        if self.supported:
            self.supported, self.reason = False, reason


def _as_bytes(buf) -> bytes:
    if isinstance(buf, bytes):
        return buf
    if torch.is_tensor(buf):
        buf = buf.cpu().numpy()
    if isinstance(buf, np.ndarray):
        if buf.dtype != np.uint8 or buf.ndim != 1:
            raise ValueError("an encoded image is a 1-D uint8 array")
        return buf.tobytes()
    return bytes(buf)


def is_encoded(x) -> bool:
    """True for what the decoders take as compressed bytes: bytes, bytearray, memoryview or a 1-D uint8 array."""
    if isinstance(x, (bytes, bytearray, memoryview)):
        return True
    if isinstance(x, np.ndarray) or torch.is_tensor(x):
        return x.ndim == 1 and x.dtype in (np.uint8, torch.uint8)
    return False


def _exif_orientation(d: bytes) -> Optional[int]:
    """Orientation tag of IFD0 of an APP1 'Exif' payload; 1 when absent, None when the block is not well formed."""
    t = d[6:]
    if len(t) < 8 or t[:2] not in (b"II", b"MM"):
        return None
    e = "<" if t[:2] == b"II" else ">"
    if struct.unpack(e + "H", t[2:4])[0] != 42:
        return None
    off = struct.unpack(e + "I", t[4:8])[0]
    if off < 8 or off + 2 > len(t):
        return None
    cnt = struct.unpack(e + "H", t[off:off + 2])[0]
    if off + 2 + 12 * cnt > len(t):
        return None
    for k in range(cnt):
        p = off + 2 + 12 * k
        tag, typ, count = struct.unpack(e + "HHI", t[p:p + 8])
        if tag == 0x0112:
            if typ != 3 or count != 1:
                return None
            v = struct.unpack(e + "H", t[p + 8:p + 10])[0]
            return v if 1 <= v <= 8 else None
    return 1


def _huff_check(counts):
    """libjpeg's table check: the codes of each length fit in that many bits, and none is all ones."""
    code = 0
    for length in range(1, 17):
        code += counts[length - 1]
        if counts[length - 1] and code >= (1 << length):
            raise ValueError("bad Huffman table (over-subscribed code space)")
        code <<= 1


def parse(buf) -> JpegHeader:
    """Parses the marker segments up to SOS.  Raises ValueError for malformed segments (truncated, bad table ids or
    counts, zero or oversized dimensions); returns an unsupported header for data that is not a JPEG."""
    b = _as_bytes(buf)
    h = JpegHeader()
    n = len(b)
    if n < 4 or b[0] != 0xFF or b[1] != 0xD8:
        h._reject("not a JPEG (no SOI)")
        return h
    i, app1_seen = 2, False
    while True:
        if i >= n:
            raise ValueError("JPEG truncated before SOS")
        if b[i] != 0xFF:
            raise ValueError(f"JPEG: expected a marker at byte {i}")
        while i < n and b[i] == 0xFF:
            i += 1
        if i >= n:
            raise ValueError("JPEG truncated before SOS")
        m = b[i]
        i += 1
        if m == 0xD9 or m == 0xD8 or 0xD0 <= m <= 0xD7 or m == 0x01 or m == 0x00:
            raise ValueError(f"JPEG: unexpected marker 0x{m:02X} before SOS")
        if i + 2 > n:
            raise ValueError("JPEG truncated in a marker segment")
        L = (b[i] << 8) | b[i + 1]
        if L < 2 or i + L > n:
            raise ValueError(f"JPEG: truncated marker segment 0x{m:02X}")
        s = b[i + 2:i + L]
        i += L
        if m == 0xE0:
            if len(s) >= 14 and s[:5] == b"JFIF\0":
                h.jfif = True
        elif m == 0xE1:
            if not app1_seen:  # OpenCV reads the orientation from the first APP1 segment
                app1_seen = True
                o = _exif_orientation(s) if s[:6] == b"Exif\0\0" else None
                if o is None:
                    h._reject("APP1 / EXIF block not understood")
                else:
                    h.orientation = o
        elif m == 0xEE:
            if len(s) >= 12 and s[:5] == b"Adobe":
                h.adobe = s[11]
        elif m == 0xDB:
            p = 0
            while p < len(s):
                pq, tq = s[p] >> 4, s[p] & 15
                if pq > 1 or tq > 3:
                    raise ValueError("JPEG: bad DQT table id or precision")
                size = 64 * (1 + pq)
                if p + 1 + size > len(s):
                    raise ValueError("JPEG: truncated DQT")
                v = np.frombuffer(s, np.uint8 if pq == 0 else ">u2", 64, p + 1).astype(np.int64)
                nat = np.zeros(64, np.int64)
                nat[ZIGZAG] = v
                h.qt[tq] = nat
                p += 1 + size
        elif m == 0xC4:
            p = 0
            while p < len(s):
                if p + 17 > len(s):
                    raise ValueError("JPEG: truncated DHT")
                tc, th = s[p] >> 4, s[p] & 15
                if tc > 1 or th > 3:
                    raise ValueError("JPEG: bad DHT table class or id")
                counts = tuple(s[p + 1:p + 17])
                total = sum(counts)
                if total > 256 or p + 17 + total > len(s):
                    raise ValueError("JPEG: bad DHT symbol count")
                vals = bytes(s[p + 17:p + 17 + total])
                _huff_check(counts)
                (h.dc if tc == 0 else h.ac)[th] = (counts, vals)
                p += 17 + total
        elif m in _SOF_NAMES:
            if h.sof is not None:
                raise ValueError("JPEG: more than one SOF")
            if len(s) < 6:
                raise ValueError("JPEG: truncated SOF")
            h.sof, h.precision = m, s[0]
            h.frame_h, h.frame_w, nf = (s[1] << 8) | s[2], (s[3] << 8) | s[4], s[5]
            if len(s) != 6 + 3 * nf or nf == 0:
                raise ValueError("JPEG: bad SOF component count")
            if not (0 < h.frame_h <= MAX_DIMENSION and 0 < h.frame_w <= MAX_DIMENSION):
                raise ValueError(f"JPEG: bad frame size {h.frame_h}x{h.frame_w}")
            for c in range(nf):
                cid, hv, tq = s[6 + 3 * c], s[7 + 3 * c], s[8 + 3 * c]
                hs, vs = hv >> 4, hv & 15
                if not (1 <= hs <= 4 and 1 <= vs <= 4) or tq > 3:
                    raise ValueError("JPEG: bad SOF sampling factor or table id")
                h.comps.append((cid, hs, vs, tq))
        elif m == 0xDD:
            if len(s) != 2:
                raise ValueError("JPEG: bad DRI length")
            h.ri = (s[0] << 8) | s[1]
        elif m == 0xDA:
            if h.sof is None:
                raise ValueError("JPEG: SOS before SOF")
            ns = s[0] if s else 0
            if ns == 0 or len(s) != 1 + 2 * ns + 3:
                raise ValueError("JPEG: bad SOS length")
            for k in range(ns):
                cs, t = s[1 + 2 * k], s[2 + 2 * k]
                if (t >> 4) > 3 or (t & 15) > 3:
                    raise ValueError("JPEG: bad SOS table id")
                h.scan.append((cs, t >> 4, t & 15))
            h.ss_se_ah_al = (s[1 + 2 * ns], s[2 + 2 * ns], s[3 + 2 * ns] >> 4, s[3 + 2 * ns] & 15)
            h.scan_off = i
            break
        elif m == 0xCC:
            h._reject("arithmetic coding")
    swap = h.orientation >= 5
    h.height, h.width = (h.frame_w, h.frame_h) if swap else (h.frame_h, h.frame_w)
    _classify(h, b)
    return h


def _classify(h: JpegHeader, b: bytes):
    if h.sof not in (0xC0, 0xC1):
        h._reject(f"{_SOF_NAMES[h.sof]} JPEG")
    if h.precision != 8:
        h._reject(f"{h.precision}-bit samples")
    nf = len(h.comps)
    if nf == 3:
        ids = tuple(c[0] for c in h.comps)
        if not h.jfif and h.adobe is not None and h.adobe != 1:
            h._reject("Adobe transform %d (RGB / CMYK)" % h.adobe)
        elif not h.jfif and h.adobe is None and ids == (82, 71, 66):
            h._reject("RGB-coded components")
        if tuple(c[1:3] for c in h.comps[1:]) != ((1, 1), (1, 1)) or h.comps[0][1:3] not in ((1, 1), (2, 1), (1, 2), (2, 2)):
            h._reject("sampling factors %s" % [c[1:3] for c in h.comps])
    elif nf != 1:
        h._reject(f"{nf} components")
    if len(h.scan) != nf or [s[0] for s in h.scan] != [c[0] for c in h.comps]:
        h._reject("not one interleaved scan of every component")
    if h.ss_se_ah_al != (0, 63, 0, 0):
        h._reject("scan parameters of a non-sequential scan")
    for (cid, _, _, tq), sc in zip(h.comps, h.scan):
        if tq not in h.qt or int(h.qt[tq].max()) > 32767:
            h._reject("missing or out-of-range quantisation table")
        elif sc[1] not in h.dc or sc[2] not in h.ac:
            h._reject("missing Huffman table")
        elif max(h.dc[sc[1]][1], default=0) > 15:
            h._reject("DC table symbol above 15")
    if h.supported:
        eoi = b.rfind(b"\xff\xd9")
        if eoi < h.scan_off:
            h._reject("no EOI (truncated)")
        h.eoi = eoi


def image_size(buf):
    """(H, W) of the RGB image `decode` returns (after the EXIF orientation), from the headers alone."""
    h = parse(buf)
    if h.sof is None:
        raise ValueError("not a JPEG")
    return h.height, h.width


# ------------------------------------------------------------------------------------------------- device tables
_huff_cache = {}


def _huff_table(counts, vals) -> np.ndarray:
    key = (counts, vals)
    t = _huff_cache.get(key)
    if t is None:
        look = np.zeros(512, np.uint16)
        maxcode = np.full(18, -1, np.int32)
        valoff = np.zeros(17, np.int32)
        code = k = 0
        for length in range(1, 17):
            c = counts[length - 1]
            if c:
                valoff[length] = k - code
                for _ in range(c):
                    if length <= 9:
                        look[code << (9 - length):(code + 1) << (9 - length)] = (length << 8) | vals[k]
                    code += 1
                    k += 1
                maxcode[length] = code - 1
            code <<= 1
        v = np.zeros(256, np.uint8)
        v[:len(vals)] = np.frombuffer(vals, np.uint8)
        t = np.zeros(HUFF_BYTES, np.uint8)
        t[:1024] = look.view(np.uint8)
        t[1024:1096] = maxcode.view(np.uint8)
        t[1096:1164] = valoff.view(np.uint8)
        t[1164:1420] = v
        if len(_huff_cache) > 4096:
            _huff_cache.clear()
        _huff_cache[key] = t
    return t


def _align(x, a=16):
    return (x + a - 1) // a * a


class Plan:
    """Per-batch tables of the kernels for supported headers; src_off[n] = where image n's bytes start in the device
    source buffer, out_off[n] = where its RGB pixels go in the output buffer."""

    def __init__(self, headers: Sequence[JpegHeader], src_off, out_off, chunk_bits=CHUNK_BITS):
        B = len(headers)
        self.B, self.chunk_bits = B, chunk_bits
        info = np.zeros((B, NI), np.int32)
        info64 = np.zeros((B, N64), np.int64)
        qtabs, qidx, htabs, hidx = [], {}, [], {}

        def qid(v):
            key = v.tobytes()
            if key not in qidx:
                qidx[key] = len(qtabs)
                qtabs.append(v.astype(np.uint16))
            return qidx[key]

        def hid(t):
            if t not in hidx:
                hidx[t] = len(htabs)
                htabs.append(_huff_table(*t))
            return hidx[t]

        ent = seg = slot = blk = plane = 0
        self.max_pixels = 0
        for n, h in enumerate(headers):
            H, W = h.frame_h, h.frame_w
            nf = len(h.comps)
            if nf == 1:
                hmax = vmax = 1
                geo = [(1, 1)]
            else:
                hmax, vmax = h.comps[0][1], h.comps[0][2]
                geo = [(hmax, vmax), (1, 1), (1, 1)]
            mcux, mcuy = -(-W // (8 * hmax)), -(-H // (8 * vmax))
            bpm = sum(a * c for a, c in geo)
            nmcu = mcux * mcuy
            nseg = -(-nmcu // h.ri) if h.ri else 1
            L = h.eoi - h.scan_off
            cap = -(-L * 8 // chunk_bits) + nseg
            r = info[n]
            r[[I_H, I_W, I_ORIENT, I_NCOMP, I_MCUX, I_MCUY, I_RI, I_BPM, I_NSEG]] = (
                H, W, h.orientation, nf, mcux, mcuy, h.ri, bpm, nseg)
            r[[I_SEG_BASE, I_CHUNK_BASE, I_CHUNK_CAP, I_OH, I_OW]] = (seg, slot, cap, h.height, h.width)
            b0 = 0
            q = info64[n]
            q[[Q_ENT_SRC, Q_ENT_LEN, Q_ENT_DST, Q_COEF, Q_OUT]] = (src_off[n] + h.scan_off, L, ent, blk, out_off[n])
            for c, ((cid, _, _, tq), sc) in enumerate(zip(h.comps, h.scan)):
                hs, vs = geo[c]
                bw, bh = mcux * hs, mcuy * vs
                r[I_COMP + 8 * c:I_COMP + 8 * c + 8] = (hs, vs, qid(h.qt[tq]), hid(h.dc[sc[1]]), hid(h.ac[sc[2]]),
                                                       bw, bh, b0)
                b0 += hs * vs
                q[Q_PLANE + c] = plane
                plane += _align(bw * bh * 64)
            ent += _align(L)
            seg += nseg
            slot += cap
            blk += nmcu * bpm
            self.max_pixels = max(self.max_pixels, h.height * h.width)
        self.info, self.info64 = info, info64
        self.quant = np.stack(qtabs) if qtabs else np.zeros((1, 64), np.uint16)
        self.huff = np.stack(htabs) if htabs else np.zeros((1, HUFF_BYTES), np.uint8)
        self.n_ent, self.n_seg, self.n_slots, self.n_blocks, self.n_plane = ent, seg, slot, blk, plane
        self.max_chunks = int(info[:, I_CHUNK_CAP].max()) if B else 0

    def tables(self):
        return [self.info, self.info64, self.quant, self.huff]


class GpuJpegDecoder:
    """Runs the kernels of csrc/jpeg.cu over one Plan; workspaces grow on demand and are reused across calls."""

    def __init__(self, device):
        self.device = torch.device(device)
        self._buf = {}
        self.stage_events = None   # a list: (name, torch.cuda.Event) appended after each stage (bench_jpeg.py)
        self.last_rounds = None    # np.int32 [B]: the last synchronisation round that changed a chunk, per image

    def _ws(self, name, numel, dtype):
        t = self._buf.get(name)
        if t is None or t.numel() < numel:
            t = torch.empty(max(int(numel * 1.25), 64), dtype=dtype, device=self.device)
            self._buf[name] = t
        return t

    def _mark(self, name):
        if self.stage_events is not None:
            e = torch.cuda.Event(enable_timing=True)
            e.record()
            self.stage_events.append((name, e))

    def run(self, plan: Plan, src_ptr: int, tab_ptrs, out_ptr: int) -> np.ndarray:
        """Decodes every image of the plan into out_ptr; returns the per-image status words (one D2H read when the
        first SYNC_ROUNDS rounds synchronise every chunk).  While an image is UNSYNCED its other bits may come from
        chunks decoded from stale entries, so more rounds run -- continuing from the state reached -- and the
        coefficients are decoded again, until no image is UNSYNCED (at most as many rounds as chunks)."""
        B, cb, s = plan.B, plan.chunk_bits, _stream()
        info, info64, quant, huff = tab_ptrs
        i32 = torch.int32
        flags = self._ws("flags", 3 * B, i32)[:3 * B]
        flags.zero_()
        status, rnd, nchunks = flags[:B], flags[B:2 * B], flags[2 * B:]
        ent = self._ws("ent", plan.n_ent, torch.uint8)
        segs = self._ws("segs", 3 * plan.n_seg, i32)
        seg_start, seg_len, seg_chunk0 = (segs[k * plan.n_seg:].data_ptr() for k in range(3))
        state = self._ws("state", 8 * plan.n_slots, i32)
        st = [state.data_ptr(), state[4 * plan.n_slots:].data_ptr()]
        excl = self._ws("excl", plan.n_slots, i32)
        coef = self._ws("coef", plan.n_blocks * 64, torch.int16)[:plan.n_blocks * 64]
        planes = self._ws("planes", plan.n_plane, torch.uint8)
        self._mark("start")
        call("vtx_jpeg_unstuff", src_ptr, info, info64, B, ent.data_ptr(), seg_start, seg_len, seg_chunk0,
             nchunks.data_ptr(), status.data_ptr(), cb, s)
        self._mark("unstuff")
        segargs = (ent.data_ptr(), info, info64, huff, seg_start, seg_len, seg_chunk0, nchunks.data_ptr(), B,
                   plan.n_slots)
        done, rounds = -1, SYNC_ROUNDS
        while True:
            for r in range(done + 1, rounds + 1):
                call("vtx_jpeg_sync", *segargs, st[(r - 1) & 1] if r else None, st[r & 1], r, rnd.data_ptr(), cb, s)
            done = rounds
            self._mark("sync")
            coef.zero_()
            status.bitwise_and_(ST_MARKER)  # unstuffing errors stay; the decode's are recomputed
            call("vtx_jpeg_count_scan", info, nchunks.data_ptr(), st[rounds & 1], excl.data_ptr(), B, s)
            call("vtx_jpeg_coefs", *segargs, st[rounds & 1], excl.data_ptr(), coef.data_ptr(), status.data_ptr(),
                 cb, s)
            self._mark("coefs")
            call("vtx_jpeg_dc_scan", info, info64, coef.data_ptr(), B, s)
            call("vtx_jpeg_idct", info, info64, coef.data_ptr(), quant, planes.data_ptr(), B, plan.n_blocks, s)
            self._mark("idct")
            call("vtx_jpeg_color", info, info64, planes.data_ptr(), out_ptr, B, plan.max_pixels, s)
            self._mark("color")
            host = flags[:2 * B].cpu().numpy()
            st_host, self.last_rounds = host[:B], host[B:]
            if not (st_host & ST_UNSYNCED).any() or rounds >= plan.max_chunks:
                return st_host
            rounds *= 2


# --------------------------------------------------------------------------------------------------- host fallback
def host_decode(buf, what="image") -> np.ndarray:
    """cv2.cvtColor(cv2.imdecode(buf, IMREAD_COLOR), COLOR_BGR2RGB): the reference's read, for what the device path
    does not reproduce.  Raises ValueError naming `what` when cv2 is not importable or cannot decode the data."""
    try:
        import cv2
    except ImportError as e:
        raise ValueError(f"{what} needs the host JPEG decoder, but cv2 is not importable ({e})") from None
    a = np.frombuffer(_as_bytes(buf), np.uint8)
    img = cv2.imdecode(a, cv2.IMREAD_COLOR) if a.size else None
    if img is None:
        raise ValueError(f"{what}: cv2 cannot decode it")
    return np.ascontiguousarray(cv2.cvtColor(img, cv2.COLOR_BGR2RGB))


def parse_or_none(buf, what="image"):
    """(header or None when the image goes to the host decoder, bytes)."""
    b = _as_bytes(buf)
    try:
        h = parse(b)
    except ValueError:
        return None, b
    return (h if h.supported else None), b


# ------------------------------------------------------------------------------------------------------ public API
_decoders = {}


def decoder_for(device) -> GpuJpegDecoder:
    device = torch.device(device)
    if device.type == "cuda" and device.index is None:
        device = torch.device("cuda", torch.cuda.current_device())
    d = _decoders.get(device)
    if d is None:
        d = _decoders[device] = GpuJpegDecoder(device)
    return d


class DecodeResult(list):
    """The decoded images (list of uint8 (H, W, 3) CUDA tensors); `fallbacks` = how many the host decoded."""
    fallbacks = 0


def decode(buffers: Sequence, device="cuda", chunk_bits: int = CHUNK_BITS) -> List[torch.Tensor]:
    """Compressed JPEG bytes -> uint8 (H, W, 3) RGB CUDA tensors, views into one packed tensor, equal to
    cv2.cvtColor(cv2.imdecode(buf, cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB).  `fallbacks` on the returned list counts the
    images cv2 decoded on the host.  chunk_bits: the Huffman decoder's chunk size (a multiple of 8, >= 64)."""
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("jpeg.decode runs on a CUDA device")
    B = len(buffers)
    heads, data, host = [], [], {}
    for n, buf in enumerate(buffers):
        h, b = parse_or_none(buf)
        heads.append(h)
        data.append(b)
        if h is None:
            host[n] = host_decode(b, f"image {n}")
    shapes = [(h.height, h.width) if h is not None else host[n].shape[:2] for n, h in enumerate(heads)]
    out_off = np.zeros(B + 1, np.int64)
    out_off[1:] = np.cumsum([_align(hh * ww * 3) for hh, ww in shapes])
    out = torch.empty(max(int(out_off[-1]), 16), dtype=torch.uint8, device=device)
    views = DecodeResult(out[out_off[n]:out_off[n] + hh * ww * 3].view(hh, ww, 3) for n, (hh, ww) in enumerate(shapes))
    dev_idx = [n for n, h in enumerate(heads) if h is not None]
    if dev_idx:
        with torch.cuda.device(device):
            src_off = np.zeros(len(dev_idx) + 1, np.int64)
            src_off[1:] = np.cumsum([_align(len(data[n])) for n in dev_idx])
            plan = Plan([heads[n] for n in dev_idx], src_off, out_off[dev_idx], chunk_bits)
            tabs = plan.tables()
            tab_off, cur = [], int(src_off[-1])
            for t in tabs:
                tab_off.append(cur)
                cur += _align(t.nbytes)
            staging = torch.empty(cur, dtype=torch.uint8).pin_memory()
            hs = staging.numpy()
            for k, n in enumerate(dev_idx):
                hs[src_off[k]:src_off[k] + len(data[n])] = np.frombuffer(data[n], np.uint8)
            for o, t in zip(tab_off, tabs):
                hs[o:o + t.nbytes] = np.frombuffer(t.tobytes(), np.uint8)
            dev = staging.to(device, non_blocking=True)
            base = dev.data_ptr()
            status = decoder_for(device).run(plan, base, [base + o for o in tab_off], out.data_ptr())
            for k, n in enumerate(dev_idx):
                if status[k]:
                    host[n] = host_decode(data[n], f"image {n}")
    for n, a in host.items():
        if a.shape[:2] != shapes[n]:
            raise ValueError(f"image {n}: cv2 decoded {a.shape[:2]}, the headers say {shapes[n]}")
        views[n].copy_(torch.from_numpy(a))
    views.fallbacks = len(host)
    return views
