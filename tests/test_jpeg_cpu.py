"""JPEG decoding, CPU side: the numpy restatement of the decode (tests/jpeg_oracle.py) against cv2.imdecode itself on
a corpus made here with cv2.imencode and Pillow, the header parser's classification, and the golden file the GPU
tests read (scripts/make_jpeg_golden.py)."""
import hashlib
import io
import os

import numpy as np
import pytest

from tests import jpeg_oracle as O
from virtex_b200 import jpeg as J

cv2 = pytest.importorskip("cv2")

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_decode.npz")


def _gen():
    from scripts import make_jpeg_golden as M
    return M


def _ref(buf):
    return cv2.cvtColor(cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR), cv2.COLOR_BGR2RGB)


@pytest.mark.parametrize("sf", ["444", "422", "420", "440"])
def test_oracle_is_bit_exact_against_cv2(sf):
    M = _gen()
    for q in (10, 30, 50, 75, 90, 95, 100):
        for ri in (0, 1, 3):
            for h, w in ((1, 1), (1, 9), (9, 1), (17, 9), (9, 17), (24, 40), (33, 19)):
                buf = M.cv2_jpeg(M.synth(h, w, q + ri + h), q, sf, ri)
                assert J.parse(buf).supported
                assert np.array_equal(O.decode(buf), _ref(buf)), (sf, q, ri, h, w)
    buf = M.cv2_jpeg(M.synth(40, 31, 2), 85, sf, optimize=True)
    assert np.array_equal(O.decode(buf), _ref(buf))


def test_oracle_grey_pillow_and_range_limit_corner():
    M = _gen()
    for q in (10, 60, 100):
        for ri in (0, 2):
            buf = M.cv2_jpeg(M.synth(21, 35, q)[..., 0], q, ri=ri)
            assert J.parse(buf).supported and len(J.parse(buf).comps) == 1
            assert np.array_equal(O.decode(buf), _ref(buf)), (q, ri)
    for sub in (0, 1, 2):
        buf = M.pil_jpeg(M.synth(26, 19, sub), quality=92, subsampling=sub)
        assert np.array_equal(O.decode(buf), _ref(buf)), sub
    # full-range noise at quality 100: IDCT outputs beyond 0..255 go through the wrap-around range limit
    rng = np.random.default_rng(0)
    for sf in ("444", "420"):
        buf = M.cv2_jpeg(rng.integers(0, 256, (32, 32, 3), np.uint8), 100, sf)
        assert np.array_equal(O.decode(buf), _ref(buf)), sf


def test_oracle_applies_every_exif_orientation_as_opencv_does():
    M = _gen()
    base = M.pil_jpeg(M.synth(23, 37, 1), quality=88, subsampling=2)
    for o in range(1, 9):
        buf = M.with_orientation(base, o)
        h = J.parse(buf)
        assert h.supported and h.orientation == o
        ref = _ref(buf)
        assert J.image_size(buf) == ref.shape[:2]
        assert np.array_equal(O.decode(buf), ref), o


def test_parser_classifies_what_the_device_path_cannot_reproduce():
    M = _gen()
    from PIL import Image
    img = M.synth(20, 24, 3)
    assert J.parse(M.pil_jpeg(img, quality=80, progressive=True)).reason == "progressive JPEG"
    f = io.BytesIO()
    Image.fromarray(img).convert("CMYK").save(f, "JPEG")
    assert not J.parse(f.getvalue()).supported
    assert not J.parse(M.cv2_jpeg(img, 90, "411")).supported
    assert not J.parse(b"\x89PNG\r\n\x1a\n" + bytes(40)).supported
    full = M.cv2_jpeg(img, 90)
    big = M.cv2_jpeg(M.synth(64, 64, 3), 95)
    assert "EOI" in J.parse(big[:len(big) - 200]).reason
    bad_exif = full[:2] + b"\xff\xe1\x00\x10Exif\0\0MM\0*\0\0\0\x40" + full[2:]
    assert not J.parse(bad_exif).supported
    # an RGB-coded (Adobe transform 0) file
    f = io.BytesIO()
    Image.fromarray(img).save(f, "JPEG", quality=90, subsampling=0, keep_rgb=True)
    assert not J.parse(f.getvalue()).supported
    # encoded inputs of every accepted type
    for x in (full, bytearray(full), memoryview(full), np.frombuffer(full, np.uint8)):
        assert J.is_encoded(x) and J.image_size(x) == (20, 24)
    assert not J.is_encoded(np.zeros((4, 4, 3), np.uint8))


def test_parser_rejects_malformed_marker_segments():
    M = _gen()
    good = M.cv2_jpeg(M.synth(16, 16, 0), 90)
    sof = good.index(b"\xff\xc0")
    dqt = good.index(b"\xff\xdb")
    dht = good.index(b"\xff\xc4")
    cases = {
        "truncated segment": good[:sof + 6],
        "zero height": good[:sof + 5] + b"\x00\x00" + good[sof + 7:],
        "zero width": good[:sof + 7] + b"\x00\x00" + good[sof + 9:],
        "bad DQT id": good[:dqt + 4] + b"\x07" + good[dqt + 5:],
        "bad DHT class": good[:dht + 4] + b"\x20" + good[dht + 5:],
        "segment length past the end": good[:dqt + 2] + b"\xff\xff" + good[dqt + 4:],
        "bad component count": good[:sof + 9] + b"\x05" + good[sof + 10:],
    }
    for what, buf in cases.items():
        with pytest.raises(ValueError):
            J.parse(buf)
            pytest.fail(what)


def test_huffman_tables_and_plan_layout():
    M = _gen()
    buf = M.cv2_jpeg(M.synth(35, 50, 1), 90, "420", 2)
    h = J.parse(buf)
    plan = J.Plan([h, h], [0, 4096], [0, 35 * 50 * 3])
    assert plan.info.shape == (2, J.NI) and plan.info64.shape == (2, J.N64)
    assert plan.quant.shape[0] == 2 and plan.huff.shape == (4, J.HUFF_BYTES)  # shared across the two images
    r = plan.info[0]
    assert (r[J.I_MCUX], r[J.I_MCUY], r[J.I_BPM], r[J.I_RI]) == (4, 3, 6, 2)
    assert r[J.I_NSEG] == 6 and plan.info[1, J.I_SEG_BASE] == 6
    assert plan.info64[1, J.Q_COEF] == 72 and plan.n_blocks == 144
    assert plan.info64[1, J.Q_ENT_SRC] == 4096 + h.scan_off
    # every code of the lookup table decodes to the canonical symbol
    counts, vals = h.ac[0]
    t = plan.huff[1]
    look = t[:1024].view(np.uint16)
    code = k = 0
    for length in range(1, 10):
        for _ in range(counts[length - 1]):
            e = look[code << (9 - length)]
            assert (e >> 8, e & 255) == (length, vals[k])
            code, k = code + 1, k + 1
        code <<= 1


def test_golden_file_matches_cv2_and_the_oracle():
    z = np.load(GOLD)
    for i in range(int(z["n"])):
        buf = z[f"buf{i}"].tobytes()
        name = str(z[f"name{i}"])
        try:
            h = J.parse(buf)
            supported = h.supported
        except ValueError:
            supported = False
        assert supported == bool(z[f"device{i}"]), name
        if z[f"shape{i}"][0] < 0:
            continue
        ref = _ref(buf)
        if f"rgb{i}" in z:
            assert np.array_equal(z[f"rgb{i}"], ref), name
            if supported and not name.startswith("corrupt"):
                assert np.array_equal(O.decode(buf), ref), name
        else:
            assert hashlib.sha256(ref.tobytes()).hexdigest() == str(z[f"sha{i}"]), name
