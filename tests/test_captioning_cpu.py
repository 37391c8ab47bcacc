"""CPU tests of beam-search captioning: the float64 restatement of the search against the fixtures written from the
reference's own model and search, the engine's launch schedule of a search (dry run against the C-ABI prototypes), and
the decoder's factory parameters."""
import functools
import os

import pytest
import torch

from oracle import virtex_oracle as O
from tests import captioning_oracle as C
from tests.test_engine_dryrun import Recorder, _check_gemm


@functools.lru_cache(maxsize=None)
def _features(seed, batch_seed, contrast):
    """The backbone part of a state depends only on its seed, so cases that share seed and images share features."""
    case = next(c for c in C.CASES if (C.CASES[c]["seed"], C.CASES[c]["batch_seed"], C.CASES[c]["contrast"]) ==
                (seed, batch_seed, contrast))
    return C.visual_features(C.case_state(case), C.case_image(case), C.case_spec(case))[0]


@pytest.fixture(scope="module")
def golden(golden_dir):
    return torch.load(os.path.join(golden_dir, C.GOLDEN))


@pytest.mark.parametrize("case", list(C.CASES))
def test_oracle_search_equals_reference_fixture(golden, case):
    c, spec = C.CASES[case], C.case_spec(case)
    state = C.case_state(case)
    P = {k: (v.double() if v.is_floating_point() else v) for k, v in state.items()}
    r = C.beam_search(C.head_step(P, spec, _features(c["seed"], c["batch_seed"], c["contrast"])), c["B"], c["beam"], c["max_steps"])
    g = golden[case]
    assert torch.equal(r["predictions"], g["beams"])
    assert torch.equal(r["predictions"].reshape(c["B"], c["beam"], -1)[:, 0], g["predictions"])
    assert (r["scores"] - g["scores"]).abs().max() <= 1e-12
    for mine, ref in zip(r["node_gaps"] + r["image_gaps"], g["node_gaps"] + g["image_gaps"]):
        finite = torch.isfinite(ref)
        assert torch.equal(finite, torch.isfinite(mine))
        assert (mine[finite] - ref[finite]).abs().max() <= 1e-9


def test_fixtures_cover_the_search_rules(golden):
    # rule 1: beam 1 with every first token EOS returns one column; rule 3: an early stop of the whole batch; a
    # predicted padding token (embedded as a zero row at the next step)
    assert golden["post_h128_beam1_all_eos"]["predictions"].shape == (3, 1)
    assert golden["post_h128_early_stop"]["predictions"].shape[1] < C.CASES["post_h128_early_stop"]["max_steps"]
    assert (golden["post_h128_token0"]["beams"][..., :-1] == 0).any()
    assert golden["pre_h256_beam5"]["predictions"].shape == (3, 12)
    # the images differ enough that beam search gives them different captions
    assert len({tuple(p) for p in golden["pre_h256_beam5"]["predictions"].tolist()}) > 1


def test_caption_score_is_the_search_score(golden):
    case = "post_h128_early_stop"
    c, spec = C.CASES[case], C.case_spec(case)
    P = {k: (v.double() if v.is_floating_point() else v) for k, v in C.case_state(case).items()}
    step = C.head_step(P, spec, _features(c["seed"], c["batch_seed"], c["contrast"]))
    beams = golden[case]["beams"]
    got = C.caption_score(step, beams[:, 0].contiguous())
    assert (got - golden[case]["scores"][:, 0]).abs().max() <= 1e-9


# ---------------------------------------------------------------------------------------------------------- dry run
@pytest.fixture
def dry(monkeypatch):
    from virtex_b200 import engine as E, ops
    rec = Recorder()

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), (name, len(args), len(ops._PROTOS[name]))
        rec.calls.append((name,) + tuple(args))

    def fake_gemm(A, B, D, M, N, K, col_scale=None, col_shift=None, **kw):
        _check_gemm(A, B, D, M, N, K, **kw)
        rec.calls.append(("gemm", M, N, K))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 132)
    return rec


def _captioning_model(layers, hidden, norm_first):
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone("resnet50", visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, 10000, hidden, layers, hidden // 64, 4 * hidden, dropout=0.1,
                                            norm_first=norm_first)
    decoder = CaptionDecoderFactory.create("beam_search", eos_index=2, max_steps=30, beam_size=5)
    return ForwardCaptioningModel(visual, textual, decoder=decoder)


@pytest.mark.parametrize("layers,hidden,norm_first", [(1, 128, False), (4, 128, False), (1, 256, True), (4, 128, True)])
def test_beam_search_schedule(dry, layers, hidden, norm_first):
    B, beam, steps = 2, 5, 30
    eng = _captioning_model(layers, hidden, norm_first).engine
    st = eng.beam_start(torch.zeros(B, 3, 224, 224), beam, 2, steps, 1, 2)
    start = list(dry.calls)
    for _ in range(steps - 1):
        eng.beam_step(st)
    assert st.L == steps and st.best().shape == (B, steps)
    names = [c[0] for c in dry.calls]
    ln = 6 if norm_first else 3  # add + LayerNorm launches per layer: pre-norm runs the LN and the residual add apart
    # embedding, per layer two attentions + GELU + the LayerNorms, the final LayerNorm (pre-norm), two beam-step halves
    per_step = 1 + layers * (3 + ln) + (1 if norm_first else 0) + 2
    gemms_per_step = layers * (3 + 2 + 2) + 1
    assert names.count("vtx_attn_decode") == 2 * layers * steps
    assert names.count("vtx_beam_rows") == names.count("vtx_beam_select") == steps
    assert names.count("vtx_embed_fwd") == steps and "vtx_attn_fwd" not in names
    assert len([n for n in names if n != "gemm"]) - len([c for c in start if c[0] != "gemm"]) == per_step * (steps - 1)
    assert names.count("gemm") - [c[0] for c in start].count("gemm") == gemms_per_step * (steps - 1)
    # every dropout-carrying launch of the search runs with p = 0
    for c in dry.calls:
        if c[0] in ("vtx_embed_fwd", "vtx_add_ln_fwd", "vtx_gelu_dropout_fwd"):
            assert c[{"vtx_embed_fwd": -4, "vtx_add_ln_fwd": -5, "vtx_gelu_dropout_fwd": -4}[c[0]]] == 0.0
    # self-attention of step t reads t keys through the index table; cross-attention 49 keys, one block per image
    attn = [c for c in dry.calls if c[0] == "vtx_attn_decode"]
    last_step = attn[-2 * layers:]
    self_a, cross_a = last_step[0], last_step[1]
    assert self_a[7] != 0 and self_a[13] == 1 and self_a[14] == steps - 1 and self_a[11] == B * beam
    assert cross_a[7] == 0 and cross_a[13] == beam and cross_a[14] == 49 and cross_a[11] == B
    # the search's buffers are its own workspace keys; no training tape is touched, the generation is unchanged
    assert eng.generation == 0 and eng._tape is None
    assert not any(k.startswith(("textual.", "head.", "hb.")) for k in eng.ws.flat)
    # step 0: B rows, top-beam first tokens of one parent row; later steps: per-node 2 of beam parents
    sel = [c for c in dry.calls if c[0] == "vtx_beam_select"]
    assert sel[0][3:6] == (1, beam, beam) and sel[1][3:6] == (beam, 2, beam)


def test_beam_search_rejects_more_steps_than_positions(dry):
    eng = _captioning_model(1, 128, False).engine
    with pytest.raises(ValueError):
        eng.beam_start(torch.zeros(2, 3, 224, 224), 5, 2, 32, 1, 2)
    # the attention kernel attends over at most 64 keys: a 288 x 288 image has 9 x 9 feature positions; rejected before
    # any launch
    dry.calls.clear()
    with pytest.raises(ValueError):
        eng.beam_start(torch.zeros(2, 3, 288, 288), 5, 2, 30, 1, 2)
    assert not dry.calls
    eng.beam_start(torch.zeros(2, 3, 256, 256), 5, 2, 30, 1, 2)


# ---------------------------------------------------------------------------------------------------------- factories
def test_decoder_factory_parameters():
    from virtex_b200.config import Config
    from virtex_b200.factories import CaptionDecoderFactory, PretrainingModelFactory
    cfg = Config(None, ["MODEL.TEXTUAL.NAME", "transdec_postnorm::L1_H128_A2_F256"])
    dec = CaptionDecoderFactory.from_config(cfg)
    assert dec.name == "beam_search"
    assert (dec.beam_size, dec.per_node_beam_size, dec.max_steps, dec.eos_index) == (
        cfg.MODEL.DECODER.BEAM_SIZE, 2, cfg.MODEL.DECODER.MAX_DECODING_STEPS, cfg.DATA.EOS_INDEX)
    model = PretrainingModelFactory.from_config(cfg)
    assert model.decoder.per_node_beam_size == 2 and model.sos_index == cfg.DATA.SOS_INDEX
    nucleus = CaptionDecoderFactory.create("nucleus_sampling", eos_index=2, max_steps=30, nucleus_size=0.9)
    assert not hasattr(nucleus, "per_node_beam_size")


def test_caption_without_tokens_needs_a_beam_search_decoder():
    from virtex_b200.factories import CaptionDecoderFactory
    from virtex_b200.models import ForwardCaptioningModel
    from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
    visual = TorchvisionVisualBackbone("resnet50", visual_feature_size=2048)
    textual = TransformerDecoderTextualHead(2048, 10000, 128, 1, 2, 256)
    batch = {"image": torch.zeros(1, 3, 224, 224)}
    with pytest.raises(ValueError):
        ForwardCaptioningModel(visual, textual).eval()(batch)
    nucleus = CaptionDecoderFactory.create("nucleus_sampling", eos_index=2, max_steps=30, nucleus_size=0.9)
    with pytest.raises(NotImplementedError):
        ForwardCaptioningModel(visual, textual, decoder=nucleus).eval()(batch)
    beam = CaptionDecoderFactory.create("beam_search", eos_index=2, max_steps=30, beam_size=5)
    with pytest.raises(RuntimeError):  # train mode
        ForwardCaptioningModel(visual, textual, decoder=beam).train()(batch)
