"""CPU tests of nucleus-sampling captioning: the float64 restatement of the sampler against the fixture written from the
reference's own model and sampler, the engine's launch schedule of a sampling run (dry run against the C-ABI
prototypes) and its input limits, the kernel's uniforms, and the decoder's factory and model dispatch."""
import functools
import os

import numpy as np
import pytest
import torch

from tests import captioning_oracle as C
from tests import nucleus_oracle as N
from tests.dropout_replica import as_u64
from tests.test_captioning_cpu import _captioning_model, dry  # noqa: F401  (dry: the dry-run fixture)


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, N.GOLDEN))


@functools.lru_cache(maxsize=None)
def _step(case):
    spec = N.case_spec(case)
    vf, P = C.visual_features(N.case_state(case), N.case_image(case), spec)
    return C.head_step(P, spec, vf)


@pytest.mark.parametrize("case", list(N.CASES))
def test_oracle_sampler_equals_reference_fixture(golden, case):
    c, g = N.CASES[case], golden[case]
    r = N.nucleus_sampling(_step(case), c["B"], c["p"], c["max_steps"], torch.Generator().manual_seed(c["rng"]))
    assert torch.equal(r["predictions"], g["predictions"])
    for mine, ref in zip(r["sizes"], g["sizes"]):
        assert torch.equal(mine, ref)
    for mine, ref in zip(r["banned_alone"], g["banned_alone"]):
        assert torch.equal(mine, ref)
    for mine, ref in zip(r["margins"], g["margins"]):
        assert (mine - ref).abs().max() <= 1e-9


def test_fixtures_cover_the_sampler_rules(golden):
    peaked = golden["post_h128_peaked"]
    # rule 3 / 4: single-token nuclei that are never the last token (a caption independent of the draws) ...
    assert all(bool((s == 1).all()) for s in peaked["sizes"]) and not any(bool(a.any()) for a in peaked["banned_alone"])
    assert peaked["predictions"].shape == (3, N.CASES["post_h128_peaked"]["max_steps"])
    # ... and nuclei of many tokens
    assert max(int(s.max()) for s in golden["post_h128_spread"]["sizes"]) > 1000
    assert any(bool(((s > 1) & (s < 1000)).any()) for s in golden["pre_h256_spread"]["sizes"])
    # rule 1 / 6 / 7: the batch stops early, EOS repeats after a caption's first EOS, captions end at different steps
    stop = golden["post_h128_eos_stop"]["predictions"]
    assert stop.shape[1] < N.CASES["post_h128_eos_stop"]["max_steps"] and (stop[:, -1] == N.EOS).all()
    first = (stop == N.EOS).int().argmax(1)
    assert len(set(first.tolist())) > 1
    for b in range(stop.shape[0]):
        assert (stop[b, first[b]:] == N.EOS).all()
    # rule 5: the nucleus is the banned last token alone (SOS at step 0), and the reference samples uniformly
    alone = golden["post_h128_banned_alone"]
    assert alone["banned_alone"][0].all() and (alone["predictions"][:, 0] != N.SOS).all()


def test_uniform_replica_is_the_hash_statement():
    """uniform24 (vectorised) equals the kernel's arithmetic written out in Python integers."""
    mask = (1 << 64) - 1
    K1, K2 = 0x9E3779B97F4A7C15, 0xD6E8FEB86659FD93
    for seed in (0, 12345, -7, 2 ** 63 + 11):
        for s, R in ((0, 3), (7, 256), (29, 1)):
            got = N.uniform24(seed, s, R, np.arange(R))
            for row in range(R):
                x = as_u64(seed) ^ ((K1 * (N.SITE + 1)) & mask) ^ (((s * R + row) * K2) & mask)
                for _ in range(2):
                    x ^= x >> 32
                    x = (x * K2) & mask
                x ^= x >> 32
                assert int(got[row]) == x >> 40 < 2 ** 24


# ---------------------------------------------------------------------------------------------------------- dry run
@pytest.mark.parametrize("layers,hidden,norm_first", [(1, 128, False), (4, 128, False), (1, 256, True), (4, 128, True)])
def test_nucleus_schedule(dry, layers, hidden, norm_first):  # noqa: F811
    B, steps = 2, 30
    eng = _captioning_model(layers, hidden, norm_first).engine
    st = eng.nucleus_start(torch.zeros(B, 3, 224, 224), 0.9, steps, 1, 2, 1234)
    start = list(dry.calls)
    for _ in range(steps - 1):
        eng.nucleus_step(st)
    assert st.L == steps and st.tokens().shape == (B, steps)
    names = [c[0] for c in dry.calls]
    ln = 6 if norm_first else 3
    per_step = 1 + layers * (3 + ln) + (1 if norm_first else 0) + 1  # ... and one sampling launch
    gemms_per_step = layers * (3 + 2 + 2) + 1
    assert names.count("vtx_nucleus_sample") == steps and "vtx_beam_rows" not in names
    assert names.count("vtx_attn_decode") == 2 * layers * steps
    assert names.count("vtx_embed_fwd") == steps and "vtx_attn_fwd" not in names
    assert len([n for n in names if n != "gemm"]) - len([c for c in start if c[0] != "gemm"]) == per_step * (steps - 1)
    assert names.count("gemm") - [c[0] for c in start].count("gemm") == gemms_per_step * (steps - 1)
    for c in dry.calls:  # every dropout-carrying launch runs with p = 0
        if c[0] in ("vtx_embed_fwd", "vtx_add_ln_fwd", "vtx_gelu_dropout_fwd"):
            assert c[{"vtx_embed_fwd": -4, "vtx_add_ln_fwd": -5, "vtx_gelu_dropout_fwd": -4}[c[0]]] == 0.0
    # step t: self-attention over t + 1 keys of the row's own cache (no index table); cross-attention group 1
    attn = [c for c in dry.calls if c[0] == "vtx_attn_decode"]
    for t in range(steps):
        self_a, cross_a = attn[2 * layers * t], attn[2 * layers * t + 1]
        assert self_a[7] == 0 and self_a[13] == 1 and self_a[14] == t + 1 and self_a[11] == B
        assert cross_a[7] == 0 and cross_a[13] == 1 and cross_a[14] == 49 and cross_a[11] == B
    # the sampling launches: B rows, step index t, nucleus size, eos, and the sampler's own seed buffer
    samp = [c for c in dry.calls if c[0] == "vtx_nucleus_sample"]
    assert [c[9] for c in samp] == list(range(steps))
    assert all(c[3] == B and c[4] == 10000 and c[6] == 2 and abs(c[7] - 0.9) < 1e-7 for c in samp)
    assert all(c[8] == eng.ws.flat["ns.seed"].data_ptr() != eng.seed.data_ptr() for c in samp)
    assert int(eng.ws.flat["ns.seed"][0]) == 1234
    assert eng.generation == 0 and eng._tape is None
    assert not any(k.startswith(("textual.", "head.", "hb.", "bs.")) for k in eng.ws.flat)


def test_nucleus_rejects_runs_that_do_not_fit(dry):  # noqa: F811
    eng = _captioning_model(1, 128, False).engine
    dry.calls.clear()
    with pytest.raises(ValueError):  # 31 positions; the head has 30 (beam search of 31 steps needs 30 and fits)
        eng.nucleus_start(torch.zeros(2, 3, 224, 224), 0.9, 31, 1, 2, 0)
    with pytest.raises(ValueError):  # 9 x 9 feature positions: more than the attention kernel's 64 keys
        eng.nucleus_start(torch.zeros(2, 3, 288, 288), 0.9, 30, 1, 2, 0)
    with pytest.raises(ValueError):
        eng.nucleus_start(torch.zeros(2, 3, 224, 224), 1.5, 30, 1, 2, 0)
    assert not dry.calls
    eng.nucleus_start(torch.zeros(2, 3, 256, 256), 0.9, 30, 1, 2, 0)
    eng.beam_start(torch.zeros(2, 3, 224, 224), 5, 2, 31, 1, 2)


# ---------------------------------------------------------------------------------------------------------- factories
def test_factory_builds_a_model_that_dispatches_to_the_sampler(monkeypatch):
    from virtex_b200 import models
    from virtex_b200.config import Config
    from virtex_b200.factories import CaptionDecoderFactory, PretrainingModelFactory
    cfg = Config(None, ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256",
                        "MODEL.DECODER.NAME", "nucleus_sampling"])
    dec = CaptionDecoderFactory.from_config(cfg)
    assert dec.name == "nucleus_sampling"
    assert (dec.nucleus_size, dec.max_steps, dec.eos_index) == (
        cfg.MODEL.DECODER.NUCLEUS_SIZE, cfg.MODEL.DECODER.MAX_DECODING_STEPS, cfg.DATA.EOS_INDEX)
    model = PretrainingModelFactory.from_config(cfg)
    assert model.decoder.name == "nucleus_sampling"
    seen = []
    monkeypatch.setattr(models.CaptioningModel, "_nucleus_sampling", lambda self, image: seen.append(image) or "caps")
    monkeypatch.setattr(models.CaptioningModel, "_beam_search", lambda self, image: pytest.fail("beam search ran"))
    image = torch.zeros(1, 3, 224, 224)
    assert model.eval()({"image": image}) == {"predictions": "caps"} and seen[0] is image


def test_sampler_needs_eval_mode_and_a_cuda_image():
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone("resnet50", visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, 10000, 128, 1, 2, 256)
    nucleus = CaptionDecoderFactory.create("nucleus_sampling", eos_index=2, max_steps=30, nucleus_size=0.9)
    model = ForwardCaptioningModel(visual, textual, decoder=nucleus)
    with pytest.raises(RuntimeError):
        model.train()({"image": torch.zeros(1, 3, 224, 224)})
    with pytest.raises(NotImplementedError):
        model.eval()({"image": torch.zeros(1, 3, 224, 224)})
