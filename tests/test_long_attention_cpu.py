"""Host side of attention past 32 queries and 64 keys: the dropout-index layout of the host replica, the engine's
schedule at crop 320 and 48 tokens on the dry run of tests/test_engine_dryrun.py, the limits it enforces before any
launch, and Config overrides of DATA.IMAGE_CROP_SIZE / MAX_CAPTION_LENGTH through the factories."""
import numpy as np
import pytest
import torch

from oracle import virtex_oracle as O
from tests import attention_replica as AR
from tests import dropout_replica as R
from tests.test_engine_dryrun import _REPLAY, _check_gemm, _model, _record_dropout, _run, Recorder


def test_attn_index_is_unchanged_for_the_one_warp_shapes():
    """The generalised layout equals tests/dropout_replica.py's (Qs = 32, Ks = 64) wherever the one-warp kernels run."""
    for B, heads in ((1, 1), (2, 3), (3, 2)):
        for Tq in range(1, 33):
            for Tk in range(1, 65):
                assert np.array_equal(AR.attn_index(B, heads, Tq, Tk), R.attn_index(B, heads, Tq, Tk)), (B, heads,
                                                                                                          Tq, Tk)


@pytest.mark.parametrize("B,heads,Tq,Tk", [(2, 3, 100, 400), (3, 2, 33, 33), (2, 2, 32, 65), (1, 2, 1024, 1024),
                                           (2, 16, 64, 144)])
def test_attn_index_is_injective_for_long_shapes(B, heads, Tq, Tk):
    idx = AR.attn_index(B, heads, Tq, Tk)
    Qs, Ks = AR.attn_rows(Tq, Tk)
    assert np.unique(idx).size == idx.size
    assert int(idx.max()) < B * heads * Qs * Ks
    # each row starts a 4-element hash group: the kernels hash the two keys (j, j + 1), j even, of a lane together
    assert (idx[..., 0] % 4 == 0).all()


@pytest.fixture
def dry_args(monkeypatch):
    """tests/test_engine_dryrun.py's recorder, keeping every call's arguments."""
    from virtex_b200 import engine as E, ops
    rec = Recorder()
    rec.args = []

    def fake_call(name, *args):
        assert len(args) == len(ops._PROTOS[name]), (name, len(args), len(ops._PROTOS[name]))
        rec.calls.append(name)
        rec.args.append((name, args))
        _record_dropout(rec, name, args)

    def fake_gemm(A, B, D, M, N, K, **kw):
        _check_gemm(A, B, D, M, N, K, **kw)
        rec.calls.append(("gemm", M, N, K, kw.get("conv_mode", 0), kw.get("bnr") is not None))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 148)
    return rec


def test_engine_schedule_at_crop_320_and_48_tokens(dry_args):
    """A 10 x 10 grid and T = 48: self-attention launches with Tq = Tk = 48, cross-attention with Tq = 48, Tk = 100;
    the LSE workspaces hold B * A * 64 rows; every forward dropout site is replayed exactly once in backward."""
    spec = O.Spec(hidden=128, layers=2, heads=2, ffn=256, max_len=48)
    model = _model(spec)
    B = 3
    eng = _run(model, O.synth_batch(B, seed=4, max_len=48, ragged=True, image_size=320))
    shapes = {"vtx_attn_fwd": [], "vtx_attn_bwd": []}
    for name, args in dry_args.args:
        if name == "vtx_attn_fwd":
            shapes[name].append((args[9], args[10], args[11], args[12]))   # B, heads, Tq, Tk
        elif name == "vtx_attn_bwd":
            shapes[name].append((args[15], args[16], args[17], args[18]))
    for name in shapes:
        assert sorted(set(shapes[name])) == [(B, 2, 48, 48), (B, 2, 48, 100)], (name, shapes[name])
        assert len(shapes[name]) == 2 * 2 * spec.layers
    for rec in eng._recs:
        for lr in rec["layers"]:
            assert lr["lse_s"].numel() == B * 2 * 64 and lr["lse_c"].numel() == B * 2 * 64
    fwd = [d for d in dry_args.drops if d[0] in _REPLAY]
    bwd = [d for d in dry_args.drops if d[0] not in _REPLAY]
    assert len(fwd) == 2 * (1 + 6 * spec.layers)
    assert sorted(bwd) == sorted((_REPLAY[name][0], site, p) for name, site, p in fwd)


@pytest.mark.parametrize("max_len,image_size", [(1025, 224), (30, 1056)])
def test_engine_rejects_attention_past_the_limit_before_any_launch(dry_args, max_len, image_size):
    """T = 1025 tokens, or a 1056 x 1056 image (a 33 x 33 = 1089-position grid): ValueError, nothing launched."""
    from virtex_b200.engine import ATTN_MAX_T
    assert ATTN_MAX_T == 1024
    spec = O.Spec(**dict(hidden=128, layers=1, heads=2, ffn=256, max_len=max_len))
    model = _model(spec)
    batch = O.synth_batch(1, seed=1, max_len=max_len, image_size=image_size)
    with pytest.raises(ValueError, match="at most 1024"):
        _run(model, batch)
    assert dry_args.calls == []


def test_head_logits_rejects_attention_past_the_limit_before_any_launch(dry_args):
    from virtex_b200.engine import head_logits
    from virtex_b200.modules import TransformerDecoderTextualHead
    head = TransformerDecoderTextualHead(2048, 100, 128, 1, 2, 256, max_caption_length=30)
    feats = torch.zeros(1, 2048, 33, 33)
    with pytest.raises(ValueError, match="at most 1024"):
        head_logits(head, feats, torch.ones(1, 5, dtype=torch.int64), torch.full((1,), 5))
    assert dry_args.calls == []


@pytest.mark.parametrize("crop,max_len", [(320, 48), (384, 64), (288, 40)])
def test_config_overrides_build_the_model_and_pipeline(crop, max_len, monkeypatch):
    """DATA.IMAGE_CROP_SIZE / MAX_CAPTION_LENGTH overrides reach the head's positional table and the input pipeline."""
    from virtex_b200 import data_gpu
    from virtex_b200.config import Config
    from virtex_b200.factories import PretrainingModelFactory
    cfg = Config(None, ["DATA.IMAGE_CROP_SIZE", crop, "DATA.MAX_CAPTION_LENGTH", max_len])
    model = PretrainingModelFactory.from_config(cfg)
    assert model.textual.embedding.positions.weight.shape[0] == max_len
    seen = {}   # the pipeline itself needs a CUDA device: record what from_config hands its constructor
    monkeypatch.setattr(data_gpu.GpuInputPipeline, "__init__", lambda self, device, **kw: seen.update(kw))
    data_gpu.GpuInputPipeline.from_config(cfg, "cuda")
    assert (seen["crop_size"], seen["max_caption_length"]) == (crop, max_len)
