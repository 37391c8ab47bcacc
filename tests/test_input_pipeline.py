"""Input pipeline (SURVEY section 8 row f-3).  CPU: the numpy oracle (oracle/input_pipeline.py) against golden vectors
produced by OpenCV itself (oracle/make_input_golden.py; geometry bit-exact, colour-jitter compositions within the
float-order noise of cv2's HSV2RGB: <= 4 LSB on < 0.1 % of values) and against torch's own collate.  GPU: the CUDA
kernels against the oracle, BIT-EXACT (uint8 stage and fp32 output), through the C ABI.
The COMPOSITION of albumentations' ColorJitter is restated from its published algorithm (the package is not installed):
parity unpinned for that composition, pinned for every cv2 primitive it is built from."""
import os

import numpy as np
import pytest
import torch

from oracle import input_pipeline as P

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "input_pipeline.npz")


def _golden():
    z = np.load(GOLD)
    items = []
    for i in range(int(z["n"])):
        j = z[f"jit{i}"]
        jit = None if j[0] < 0 else (float(j[0]), float(j[1]), float(j[2]), float(j[3]), tuple(int(v) for v in j[4:]))
        items.append((z[f"img{i}"], tuple(int(v) for v in z[f"box{i}"]), bool(z[f"flip{i}"]), jit, z[f"train{i}"]))
    return items


def _oracle_u8(img, box, flip, jit):
    y0, x0, h, w = box
    out = P.resize_linear_u8(img[y0:y0 + h, x0:x0 + w], 224, 224)
    if flip:
        out = out[:, ::-1]
    return P.color_jitter(out, *jit) if jit is not None else out


def test_oracle_matches_opencv_golden_vectors():
    for img, box, flip, jit, ref in _golden():
        d = np.abs(_oracle_u8(img, box, flip, jit).astype(int) - ref.astype(int))
        if jit is None:
            assert d.max() == 0  # crop + cv2.resize + cv2.flip: bit-exact
        else:
            assert d.max() <= 4 and (d > 0).mean() < 1e-3, (d.max(), (d > 0).mean())


def test_oracle_collate_matches_the_reference_collate():
    """captioning.py:68-100: [SOS] .. [EOS] trimmed to max_len, `pad_sequence(batch_first, padding_value)`, flipped copy."""
    rng = np.random.default_rng(0)
    lists = [[1] + list(rng.integers(4, 10000, n)) + [2] for n in (3, 28, 40, 9, 0)]
    cap, rev, lens = P.collate_captions(lists, max_len=30, pad=0)
    trimmed = [torch.tensor(t[:30]) for t in lists]
    ref_cap = torch.nn.utils.rnn.pad_sequence(trimmed, batch_first=True, padding_value=0)
    ref_rev = torch.nn.utils.rnn.pad_sequence([t.flip(0) for t in trimmed], batch_first=True, padding_value=0)
    assert np.array_equal(cap, ref_cap.numpy()) and np.array_equal(rev, ref_rev.numpy())
    assert lens.tolist() == [len(t) for t in trimmed]


def test_oracle_val_geometry_and_normalisation():
    assert P.val_geometry(480, 640) == (256, 341, 16, 58)
    assert P.val_geometry(640, 427) == (384, 256, 80, 16)
    img = np.full((4, 5, 3), 128, np.uint8)
    out = P.normalize_chw(img)
    assert out.shape == (3, 4, 5) and out.dtype == np.float32
    ref = (128 / 255.0 - np.array(P.IMAGENET_MEAN)) / np.array(P.IMAGENET_STD)
    assert np.allclose(out[:, 0, 0], ref, atol=1e-6)


# ------------------------------------------------------------------------------------------------------------- GPU
@pytest.mark.gpu
def test_gpu_train_transform_is_bit_exact_against_the_oracle():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200.data_gpu import GpuInputPipeline, ImageParams
    pipe = GpuInputPipeline("cuda")
    gold = _golden()
    rng = np.random.default_rng(7)
    images, params, expect_u8 = [], [], []
    for img, box, flip, jit, _ in gold:
        images.append(img)
        params.append(ImageParams(box, (224, 224), (0, 0), flip, jit))
        expect_u8.append(_oracle_u8(img, box, flip, jit))
    # more boxes / jitters than the fixture holds, every jitter op order and the degenerate factors
    base = gold[0][0]
    orders = [(0, 1, 2, 3), (3, 2, 1, 0), (1, 0, 3, 2), (2, 3, 0, 1)]
    for k in range(8):
        p = pipe.sample_train_params(rng, *base.shape[:2], jitter_p=1.0)
        jit = list(p.jitter)
        jit[4] = orders[k % 4]
        if k == 5:
            jit[1] = 0.0   # contrast 0: every pixel becomes the grey mean
        if k == 6:
            jit[2] = 0.0   # saturation 0: grey image
        if k == 7:
            jit[0], jit[1], jit[2], jit[3] = 1.0, 1.0, 1.0, 0.0   # identities
        p.jitter = tuple(jit)
        images.append(base)
        params.append(p)
        expect_u8.append(_oracle_u8(base, p.region, p.flip, p.jitter))
    tokens = [[1] + list(rng.integers(4, 10000, n)) + [2] for n in rng.integers(0, 40, len(images))]
    batch = pipe(images, params, tokens)
    torch.cuda.synchronize()
    # resample + flip stage: bit-exact vs the oracle of cv2.resize
    for n, (img, p) in enumerate(zip(images, params)):
        y0, x0, h, w = p.region
        ref = P.resize_linear_u8(img[y0:y0 + h, x0:x0 + w], 224, 224)
        ref = ref[:, ::-1] if p.flip else ref
        assert np.array_equal(batch["_image_u8"][n].cpu().numpy(), ref), n
    # full transform: bit-exact fp32 vs the oracle
    out = batch["image"].cpu().numpy()
    for n, u8 in enumerate(expect_u8):
        ref = P.normalize_chw(u8)
        assert np.array_equal(out[n], ref), (n, np.abs(out[n] - ref).max(), params[n].jitter)
    cap, rev, lens = P.collate_captions(tokens, 30, 0)
    assert np.array_equal(batch["caption_tokens"].cpu().numpy(), cap)
    assert np.array_equal(batch["noitpac_tokens"].cpu().numpy(), rev)
    assert np.array_equal(batch["caption_lengths"].cpu().numpy(), lens)


@pytest.mark.gpu
def test_gpu_val_transform_and_model_consumes_the_batch():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from virtex_b200.data_gpu import GpuInputPipeline
    pipe = GpuInputPipeline("cuda")
    rng = np.random.default_rng(3)
    images = [rng.integers(0, 256, s, dtype=np.uint8) for s in ((480, 640, 3), (640, 427, 3), (256, 256, 3), (300, 225, 3))]
    params = [pipe.val_params(*im.shape[:2]) for im in images]
    batch = pipe(images, params, [[1, 5, 6, 2], [1, 9, 2], [1, 2], [1, 7, 8, 9, 10, 2]])
    out = batch["image"].cpu().numpy()
    for n, im in enumerate(images):
        assert np.array_equal(out[n], P.val_transform(im)), n
    # the batch dict is what CaptioningModel.forward takes (captioning.py:71-77)
    from oracle import virtex_oracle as O
    from tests.helpers import build_model
    spec = O.Spec(hidden=128, layers=1, heads=2, ffn=256)
    model = build_model(spec, O.synth_state(spec, 3, bn3_gain=0.25)).eval()
    del batch["_image_u8"]
    with torch.no_grad():
        res = model(batch)
    cpu_batch = {k: v.cpu() for k, v in batch.items()}
    with torch.no_grad():
        ref = O.model_forward(O.synth_state(spec, 3, bn3_gain=0.25), cpu_batch, spec, training=False)
    assert abs(res["loss"].item() - ref["loss"].item()) < 2e-3 * ref["loss"].item()
