"""Writes tests/golden/jpeg_decode.npz: JPEG files made with cv2.imencode and Pillow, each with what the reference
reads from it, cv2.cvtColor(cv2.imdecode(buf, IMREAD_COLOR), COLOR_BGR2RGB) (the full pixels for small images, a
SHA-256 of them for the 640x480 ones), so that the GPU tests need neither cv2 nor Pillow to know the answer.

    python scripts/make_jpeg_golden.py
"""
import hashlib
import io
import os
import struct

import cv2
import numpy as np
from PIL import Image

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "jpeg_decode.npz")
SF = {"444": 0x111111, "422": 0x211111, "420": 0x221111, "440": 0x121111, "411": 0x411111}


def synth(h, w, seed, noise=25.0):
    """Gradients, a few soft discs and noise: natural-ish spectra at every size."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float64)
    img = np.stack([x * 255 / max(w - 1, 1), y * 255 / max(h - 1, 1), (x + y) * 127 / max(h + w - 2, 1) + 64], -1)
    for _ in range(4):
        cy, cx, r = rng.uniform(0, h), rng.uniform(0, w), rng.uniform(2, max(h, w) / 2 + 3)
        img += rng.uniform(-90, 90, 3) * np.exp(-((y - cy) ** 2 + (x - cx) ** 2) / (2 * r * r))[..., None]
    img += rng.normal(0, noise, img.shape)
    return np.clip(img, 0, 255).astype(np.uint8)


def cv2_jpeg(rgb, q=90, sf="420", ri=0, optimize=False):
    params = [cv2.IMWRITE_JPEG_QUALITY, q, cv2.IMWRITE_JPEG_RST_INTERVAL, ri, cv2.IMWRITE_JPEG_OPTIMIZE, int(optimize)]
    if rgb.ndim == 3:
        params += [cv2.IMWRITE_JPEG_SAMPLING_FACTOR, SF[sf]]
        rgb = cv2.cvtColor(rgb, cv2.COLOR_RGB2BGR)
    ok, enc = cv2.imencode(".jpg", rgb, params)
    assert ok
    return enc.tobytes()


def pil_jpeg(rgb, **kw):
    f = io.BytesIO()
    Image.fromarray(rgb).save(f, "JPEG", **kw)
    return f.getvalue()


def with_orientation(buf, o):
    """Inserts a little-endian EXIF APP1 block with IFD0 = {Orientation: o} after SOI."""
    tiff = b"II*\0" + struct.pack("<I", 8) + struct.pack("<H", 1) + struct.pack("<HHIHH", 0x0112, 3, 1, o, 0) + \
        struct.pack("<I", 0)
    seg = b"Exif\0\0" + tiff
    return buf[:2] + b"\xff\xe1" + struct.pack(">H", len(seg) + 2) + seg + buf[2:]


def reference(buf):
    img = cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)
    return cv2.cvtColor(img, cv2.COLOR_BGR2RGB)


def corpus():
    """(name, bytes, expected on the device path)"""
    out = []
    for sf in ("444", "422", "420", "440"):
        for q in (10, 50, 90, 100):
            out.append((f"{sf}_q{q}_37x53", cv2_jpeg(synth(37, 53, q), q, sf), True))
        for ri in (1, 3):
            out.append((f"{sf}_q75_rst{ri}_29x45", cv2_jpeg(synth(29, 45, ri), 75, sf, ri), True))
        for h, w in ((1, 1), (1, 13), (11, 1), (17, 9), (2, 3)):
            out.append((f"{sf}_q85_{h}x{w}", cv2_jpeg(synth(h, w, h * w), 85, sf), True))
        out.append((f"{sf}_q80_optimized_40x31", cv2_jpeg(synth(40, 31, 5), 80, sf, optimize=True), True))
    for h, w, q, ri in ((1, 1, 90, 0), (17, 9, 10, 0), (40, 33, 100, 0), (40, 33, 70, 2)):
        out.append((f"gray_q{q}_rst{ri}_{h}x{w}", cv2_jpeg(synth(h, w, 9)[..., 0], q, ri=ri), True))
    out.append(("q100_noise_24x24", cv2_jpeg(np.random.default_rng(1).integers(0, 256, (24, 24, 3), np.uint8), 100,
                                             "444"), True))
    base = pil_jpeg(synth(23, 37, 11), quality=88, subsampling=2)
    for o in range(1, 9):
        out.append((f"exif_orientation{o}_23x37", with_orientation(base, o), True))
    bad_exif = base[:2] + b"\xff\xe1\x00\x10Exif\0\0MM\0*\0\0\0\x40" + base[2:]  # IFD0 offset past the block
    out.append(("exif_malformed", bad_exif, False))
    out.append(("pil_422_q95_31x20", pil_jpeg(synth(31, 20, 4), quality=95, subsampling=1), True))
    out.append(("progressive_33x27", pil_jpeg(synth(33, 27, 6), quality=80, progressive=True), False))
    cmyk = Image.fromarray(synth(19, 21, 7)).convert("CMYK")
    f = io.BytesIO()
    cmyk.save(f, "JPEG", quality=85)
    out.append(("cmyk_19x21", f.getvalue(), False))
    out.append(("411_q90_32x48", cv2_jpeg(synth(32, 48, 8), 90, "411"), False))
    full = cv2_jpeg(synth(48, 64, 12), 90, "420")
    out.append(("truncated_48x64", full[:len(full) // 2], False))
    sos = full.index(b"\xff\xda")
    mid = sos + (len(full) - sos) // 2
    out.append(("corrupt_stray_marker_48x64", full[:mid] + b"\xff\xd3" + full[mid:], True))
    out.append(("corrupt_cut_entropy_48x64", full[:mid] + full[-2:], True))
    out.append(("not_a_jpeg", b"GIF89a" + bytes(range(64)), False))
    out.append(("large_640x480_q90_420", cv2_jpeg(synth(480, 640, 22, noise=4.0), 90, "420"), True))
    out.append(("large_480x640_q90_422_rst8", cv2_jpeg(synth(640, 480, 23, noise=4.0), 90, "422", 8), True))
    return out


def main():
    z = {}
    items = corpus()
    for i, (name, buf, dev) in enumerate(items):
        z[f"name{i}"] = np.array(name)
        z[f"buf{i}"] = np.frombuffer(buf, np.uint8)
        z[f"device{i}"] = np.array(dev)
        img = cv2.imdecode(np.frombuffer(buf, np.uint8), cv2.IMREAD_COLOR)
        if img is None:
            z[f"shape{i}"] = np.array([-1, -1, -1])
            continue
        rgb = reference(buf)
        z[f"shape{i}"] = np.array(rgb.shape)
        if rgb.size > 64 * 64 * 3:
            z[f"sha{i}"] = np.array(hashlib.sha256(rgb.tobytes()).hexdigest())
        else:
            z[f"rgb{i}"] = rgb
    z["n"] = np.array(len(items))
    np.savez_compressed(OUT, **z)
    print(f"wrote {OUT}: {len(items)} files, {os.path.getsize(OUT)} bytes")


if __name__ == "__main__":
    main()
