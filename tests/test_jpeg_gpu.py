"""JPEG decoding on the H100 (csrc/jpeg.cu through virtex_b200.jpeg), bit-exact against what cv2.imdecode returns,
read from tests/golden/jpeg_decode.npz (scripts/make_jpeg_golden.py) so that no encoder is needed here.  Images the
device path leaves to cv2 need cv2 at run time; those checks skip without it."""
import hashlib
import os

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "jpeg_decode.npz")


def _need_cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _golden():
    z = np.load(GOLD)
    out = []
    for i in range(int(z["n"])):
        out.append(dict(name=str(z[f"name{i}"]), buf=z[f"buf{i}"].tobytes(), device=bool(z[f"device{i}"]),
                        shape=tuple(int(v) for v in z[f"shape{i}"]),
                        rgb=z[f"rgb{i}"] if f"rgb{i}" in z else None,
                        sha=str(z[f"sha{i}"]) if f"sha{i}" in z else None))
    return out


def _check(item, got):
    a = got.cpu().numpy()
    assert a.shape == item["shape"], item["name"]
    if item["rgb"] is not None:
        d = np.abs(a.astype(int) - item["rgb"].astype(int))
        assert d.max() == 0, (item["name"], d.max(), int((d > 0).sum()))
    else:
        assert hashlib.sha256(a.tobytes()).hexdigest() == item["sha"], item["name"]


def _on_device(items):
    return [g for g in items if g["device"] and not g["name"].startswith("corrupt")]


def test_decode_is_bit_exact_on_the_golden_corpus():
    _need_cuda()
    from virtex_b200 import jpeg
    items = _on_device(_golden())
    out = jpeg.decode([g["buf"] for g in items], "cuda")
    assert out.fallbacks == 0
    for g, t in zip(items, out):
        assert t.is_cuda and t.dtype == torch.uint8
        _check(g, t)


def test_batch_of_256_mixed_sizes():
    _need_cuda()
    from virtex_b200 import jpeg
    items = _on_device(_golden())
    large = [g for g in items if g["name"].startswith("large")]
    rng = np.random.default_rng(0)
    batch = []
    for k in range(256):  # every 4th a 640x480 / 480x640 file, the rest drawn from the corpus
        batch.append(large[k // 4 % len(large)] if k % 4 == 0 else items[int(rng.integers(len(items)))])
    out = jpeg.decode([g["buf"] for g in batch], "cuda")
    assert out.fallbacks == 0
    for g, t in zip(batch, out):
        _check(g, t)
    rounds = jpeg.decoder_for("cuda").last_rounds
    print("synchronisation rounds (images per round):", np.bincount(rounds))


@pytest.mark.parametrize("chunk_bits", ["shorter", "exact", 64, 256])
def test_segment_lengths_against_the_chunk_size(chunk_bits):
    """One chunk longer than the segment, exactly one chunk, and many chunks per segment."""
    _need_cuda()
    from virtex_b200 import jpeg
    items = {g["name"]: g for g in _golden()}
    names = ["gray_q90_rst0_1x1", "420_q90_37x53", "444_q75_rst1_29x45", "large_480x640_q90_422_rst8"]
    if chunk_bits == "shorter":
        bits = 1 << 20
    elif chunk_bits == "exact":
        # the unstuffed entropy length of a file without restarts: its only segment is exactly one chunk
        names = names[1:2]
        h = jpeg.parse(items[names[0]]["buf"])
        seg = items[names[0]]["buf"][h.scan_off:h.eoi].replace(b"\xff\x00", b"\xff")
        bits = len(seg) * 8
    else:
        bits = chunk_bits
    out = jpeg.decode([items[n]["buf"] for n in names], "cuda", chunk_bits=bits)
    assert out.fallbacks == 0
    for n, t in zip(names, out):
        _check(items[n], t)


def test_pipeline_fed_jpeg_bytes_equals_the_pipeline_fed_decoded_arrays():
    _need_cuda()
    pytest.importorskip("cv2")  # the progressive / CMYK / truncated items are decoded by cv2
    from virtex_b200 import jpeg
    from virtex_b200.data_gpu import GpuInputPipeline
    g = {x["name"]: x for x in _golden()}
    # a file without EOI goes to cv2 too; OpenCV 4.13 returns None for it, so the batch names the image
    with pytest.raises(ValueError, match="image 1"):
        GpuInputPipeline("cuda")([g["large_640x480_q90_420"]["buf"], g["truncated_48x64"]["buf"]],
                                 [GpuInputPipeline("cuda").val_params(480, 640)] * 2)
    names = ["large_640x480_q90_420", "exif_orientation6_23x37", "progressive_33x27", "cmyk_19x21",
             "corrupt_stray_marker_48x64", "420_q75_rst3_29x45", "large_480x640_q90_422_rst8", "gray_q70_rst2_40x33",
             "exif_malformed", "pil_422_q95_31x20"]
    bufs = [g[n]["buf"] for n in names]
    bufs[1] = np.frombuffer(bufs[1], np.uint8)       # a 1-D uint8 array
    bufs[5] = bytearray(bufs[5])
    bufs[7] = memoryview(bufs[7])
    arrays = [jpeg.host_decode(b) for b in bufs]
    pipe = GpuInputPipeline("cuda")
    for mode in ("train", "val"):
        rng = np.random.default_rng(5)
        sizes = [jpeg.image_size(b) for b in bufs]
        assert sizes == [a.shape[:2] for a in arrays]
        if mode == "train":
            params = [pipe.sample_train_params(rng, *hw) for hw in sizes]
        else:
            params = [pipe.val_params(*hw) for hw in sizes[:1] + sizes[6:7]]
        sel = range(len(bufs)) if mode == "train" else (0, 6)
        toks = [[1, 5, 6, 2]] * len(params)
        # mixed: decoded arrays and encoded bytes in one batch
        mixed = [arrays[k] if k % 3 == 2 else bufs[k] for k in sel]
        ref = pipe([arrays[k] for k in sel], params, toks)
        ref = {k: v.clone() for k, v in ref.items()}
        got = pipe(mixed, params, toks)
        n_fallback = sum(1 for k in sel if k % 3 != 2 and (not g[names[k]]["device"] or "corrupt" in names[k]))
        assert int(got["_jpeg_fallbacks"]) == n_fallback
        assert "_jpeg_fallbacks" not in ref
        assert torch.equal(got["_image_u8"], ref["_image_u8"]), mode
        assert torch.equal(got["image"], ref["image"]), mode
        assert torch.equal(got["caption_tokens"], ref["caption_tokens"])


def test_corrupt_entropy_data_falls_back_to_cv2_and_the_next_call_works():
    _need_cuda()
    pytest.importorskip("cv2")
    from virtex_b200 import jpeg
    g = {x["name"]: x for x in _golden()}
    for name in ("corrupt_stray_marker_48x64", "corrupt_cut_entropy_48x64"):
        bad, good = g[name], g["420_q90_37x53"]
        out = jpeg.decode([good["buf"], bad["buf"], good["buf"]], "cuda")
        assert out.fallbacks == 1, name
        for item, t in zip((good, bad, good), out):
            _check(item, t)
        nxt = jpeg.decode([good["buf"], g["large_640x480_q90_420"]["buf"]], "cuda")
        assert nxt.fallbacks == 0
        _check(good, nxt[0])
        _check(g["large_640x480_q90_420"], nxt[1])
