"""Token / multilabel classification pretext models on the CPU: the oracle against fixtures written by the reference's
own models (scripts/make_classification_golden.py), the config -> factory -> model path with reference-keyed
state_dicts, and a dry run of the engine's classification schedule with every launch checked against its prototype in
include/virtex_b200.h."""
import os
import re

import pytest
import torch

from oracle import virtex_oracle as O
from tests import classification_oracle as CO
from tests.test_engine_dryrun import _check_gemm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
BF16, F32 = torch.bfloat16, torch.float32


def _golden(golden_dir, name):
    return torch.load(os.path.join(golden_dir, CO.CASES[name][0] + ".pt"), weights_only=False)


def _inputs(g, **kw):
    state = CO.synth_classification_state(g["vocab"], g["seed"])
    batch = CO.synth_label_batch(3, seed=g["batch_seed"], vocab=g["vocab"], ignore=g["ignore"], **kw)
    return state, batch


def _assert_grads_match(grads, ref):
    names = ref["names"]
    assert sorted(grads) == names
    norm = torch.tensor([grads[n].norm().item() for n in names], dtype=torch.float64)
    ssum = torch.tensor([grads[n].sum().item() for n in names], dtype=torch.float64)
    assert torch.isfinite(norm).all()
    assert torch.allclose(norm, ref["norm"], rtol=1e-7, atol=1e-12)
    assert ((ssum - ref["sum"]).abs() <= 1e-6 * ref["sum"].abs() + 1e-9 * (1 + norm)).all()


# ------------------------------------------------------------------------------------------------------ oracle vs golden
@pytest.mark.parametrize("name", list(CO.CASES))
def test_classification_oracle_matches_the_reference(golden_dir, name):
    """float64 oracle == float64 reference model: loss, every gradient's norm, sum and probe, eval loss and top-10."""
    g = _golden(golden_dir, name)
    state, batch = _inputs(g)
    assert all(len(set(r.tolist()) - set(g["ignore"])) < (r != 0).sum() for r in batch["labels"])  # dups / ignored ids
    assert (batch["labels"] == 0).any(dim=1).sum() >= 2  # ragged padding
    out, grads = CO.loss_and_grads(state, batch, g["ignore"], torch.float64)
    ref = g["f64"]
    assert abs(out["loss"].item() - ref["loss"].item()) < 1e-9
    _assert_grads_match(grads, ref["grads"])
    for k, probe in ref["grad_probe"].items():
        assert torch.allclose(grads[k].flatten()[:64], probe, rtol=1e-7, atol=1e-12), k
    ev = CO.eval_forward(state, batch, g["ignore"], torch.float64)
    assert abs(ev["loss"].item() - ref["eval_loss"].item()) < 1e-9
    assert torch.equal(ev["predictions"], ref["eval_predictions"])
    assert ev["predictions"].dtype == torch.int64 and tuple(ev["predictions"].shape) == (3, 10)
    # float32 oracle against both reference runs
    out32, _ = CO.loss_and_grads(state, batch, g["ignore"], torch.float32)
    for tag in ("f32", "f64"):
        assert abs(out32["loss"].item() - g[tag]["loss"].item()) < 2e-6 * g[tag]["loss"].item()


@pytest.mark.parametrize("name", list(CO.CASES))
def test_empty_label_set_gives_nan_loss_and_no_gradient(golden_dir, name):
    """An image whose labels are all ignored: NaN loss (the reference's mean over an empty set), yet every gradient is
    finite and equal to the reference's, and that image's logits receive exactly zero gradient."""
    g = _golden(golden_dir, name)
    state, batch = _inputs(g, empty_rows=(CO.EMPTY_ROW,))
    assert set(batch["labels"][CO.EMPTY_ROW].tolist()) <= set(g["ignore"])
    out, grads = CO.loss_and_grads(state, batch, g["ignore"], torch.float64)
    ref = g["f64"]["empty_row"]
    assert torch.isnan(out["loss"]) and torch.isnan(ref["loss"])
    _assert_grads_match(grads, ref["grads"])
    logits = out["logits"].clone().requires_grad_(True)
    CO.khot_loss_rows(logits, batch["labels"], g["ignore"]).mean().backward()
    assert torch.equal(logits.grad[CO.EMPTY_ROW], torch.zeros_like(logits.grad[CO.EMPTY_ROW]))
    assert logits.grad[[r for r in range(3) if r != CO.EMPTY_ROW]].abs().sum() > 0


# ------------------------------------------------------------------------------------------------- config and factories
def _config(name, extra=()):
    from virtex_b200.config import Config
    return Config("_base_bicaptioning_R_50_L1_H1024.yaml",
                  ["MODEL.NAME", name, "MODEL.TEXTUAL.NAME", "none", "OPTIM.NO_DECAY", "none", *extra])


@pytest.mark.parametrize("name,extra,cls_name,vocab,ignore", [
    ("token_classification", (), "TokenClassificationModel", 10000, [0, 1, 2, 3]),
    ("multilabel_classification", ("DATA.VOCAB_SIZE", 81), "MultiLabelClassificationModel", 81, [0]),
])
def test_factories_build_the_reference_models(name, extra, cls_name, vocab, ignore):
    from virtex_b200 import modules
    from virtex_b200.factories import PretrainingModelFactory, TextualHeadFactory, param_group_hparams
    cfg = _config(name, extra)
    head = TextualHeadFactory.from_config(cfg)
    assert isinstance(head, modules.LinearTextualHead)
    assert (head.visual_feature_size, head.vocab_size, head.hidden_size, head.textual_feature_size) == (2048, vocab, 2048, 2048)
    model = PretrainingModelFactory.from_config(cfg)
    assert type(model).__name__ == cls_name and model.ignore_indices == ignore
    assert isinstance(model.textual, modules.LinearTextualHead)
    # the reference's key set: the backbone plus textual.output.{weight,bias}; its checkpoints load strictly
    keys = set(model.state_dict())
    assert {k for k in keys if not k.startswith("visual.")} == {"textual.output.weight", "textual.output.bias"}
    assert keys == set(O.backbone_param_shapes(CO.SPEC)) | {"textual.output.weight", "textual.output.bias"}
    sd = CO.synth_classification_state(vocab, 3)
    model.load_state_dict(sd, strict=True)
    assert torch.equal(model.textual.output.weight, sd["textual.output.weight"])
    # OPTIM.NO_DECAY "none" matches no parameter name: weight decay everywhere, CNN_LR on the backbone only
    assert param_group_hparams(cfg, "textual.output.bias") == (cfg.OPTIM.LR, cfg.OPTIM.WEIGHT_DECAY)
    assert param_group_hparams(cfg, "visual.cnn.bn1.bias") == (cfg.OPTIM.CNN_LR, cfg.OPTIM.WEIGHT_DECAY)


def test_linear_head_keeps_the_reference_init_and_signature():
    from virtex_b200.modules import LinearTextualHead
    torch.manual_seed(0)
    head = LinearTextualHead(visual_feature_size=2048, vocab_size=81, hidden_size=999)  # extra kwargs are ignored
    bound = 1 / 2048 ** 0.5
    assert head.output.weight.abs().max() <= bound and head.output.bias.abs().max() <= bound
    assert head.output.weight.std() > 0.5 * bound
    with pytest.raises(ValueError):
        from virtex_b200.models import TokenClassificationModel
        from virtex_b200.modules import TorchvisionVisualBackbone, TransformerDecoderTextualHead
        TokenClassificationModel(TorchvisionVisualBackbone(), TransformerDecoderTextualHead(2048, 100, 128, 1, 2, 256),
                                 [0])


class _Tokenizer:
    def id_to_token(self, i):
        return f"t{i}"

    def decode(self, ids):
        return " ".join(map(str, ids))


def test_log_predictions_formats_like_the_reference(monkeypatch):
    """log_predictions is pure Python over the eval-mode predictions (stubbed here: there is no CPU forward)."""
    from virtex_b200 import models
    from virtex_b200.modules import LinearTextualHead, TorchvisionVisualBackbone
    preds = torch.arange(20).view(2, 10)
    monkeypatch.setattr(models.ClassificationModel, "_eval_predictions", lambda self, batch: preds)
    batch = {"caption_tokens": torch.tensor([[5, 0, 3, 0], [7, 9, 1, 0]])}
    tok = models.TokenClassificationModel(TorchvisionVisualBackbone(), LinearTextualHead(2048, 100), [0, 1, 2, 3])
    text = tok.log_predictions(batch, _Tokenizer())
    assert "Caption tokens : 5 0 3 0\n" in text and "Predictions (f): t0 t1 t2 t3 t4 t5 t6 t7 t8 t9\n" in text
    ml = models.MultiLabelClassificationModel(TorchvisionVisualBackbone(), LinearTextualHead(2048, 81), [0])
    text = ml.log_predictions(batch)
    assert "COCO Instance IDs (GT)   : [3, 5]\n" in text and "COCO Instance IDs (Pred) : [0, 1]\n" in text
    assert "COCO Instance IDs (GT)   : [1, 7, 9]\n" in text and "COCO Instance IDs (Pred) : [10, 11, 12]\n" in text


# ------------------------------------------------------------------------------------------------------------ dry run
def _header_arity():
    """Number of parameters of every vtx_* function declared in include/virtex_b200.h."""
    header = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "virtex_b200.h")).read(), flags=re.S)
    return {m.group(1): len([a for a in m.group(2).split(",") if a.strip() and a.strip() != "void"])
            for m in re.finditer(r"\bint\s+(vtx_[a-z0-9_]+)\s*\(([^)]*)\)", header)}


@pytest.fixture
def recorder(monkeypatch):
    """Replace the engine's launchers with recorders that check each call against the header prototype and each GEMM
    against the buffer sizes its operands imply."""
    from virtex_b200 import engine as E, ops
    arity = _header_arity()
    calls = []

    def fake_call(name, *args):
        assert len(args) == arity[name] == len(ops._PROTOS[name]), (name, len(args), arity.get(name))
        calls.append((name,) + args)

    def fake_gemm(A, B, D, M, N, K, **kw):
        _check_gemm(A, B, D, M, N, K, **kw)
        calls.append(("gemm", M, N, K, D, kw))

    monkeypatch.setattr(E, "call", fake_call)
    monkeypatch.setattr(E, "gemm", fake_gemm)
    monkeypatch.setattr(E, "_stream", lambda: 0)
    monkeypatch.setattr(E, "_require_cuda", lambda dev: None)
    monkeypatch.setattr(ops, "num_sms", lambda: 132)
    return calls


def _names(calls):
    return [c[0] for c in calls]


def _cls_model(vocab, ignore, frozen=False):
    from virtex_b200.models import MultiLabelClassificationModel, TokenClassificationModel
    from virtex_b200.modules import LinearTextualHead, TorchvisionVisualBackbone
    cls = TokenClassificationModel if vocab == 10000 else MultiLabelClassificationModel
    return cls(TorchvisionVisualBackbone("resnet50", frozen=frozen), LinearTextualHead(2048, vocab), ignore)


@pytest.mark.parametrize("vocab,ignore,B", [(10000, [0, 1, 2, 3], 3), (81, [0], 5)])
def test_classification_training_schedule(recorder, vocab, ignore, B):
    model = _cls_model(vocab, ignore)
    eng = model.engine
    assert eng.classify and eng.pad == 0 and eng.ignore.tolist() == ignore
    batch = CO.synth_label_batch(B, seed=1, vocab=vocab, ignore=ignore, image_size=224)
    loss = eng.forward(batch["image"], None, None, None, training=True, with_grad=True, labels=batch["labels"])
    assert tuple(loss.shape) == (2,)
    tags = []
    eng.backward(zero_grads=True, bucket_cb=tags.append)
    assert tags == ["head", "layer4", "layer3", "layer2", "rest"]
    names = _names(recorder)
    for n in ("vtx_group_mean_fwd", "vtx_khot_xent", "vtx_group_mean_bwd", "vtx_colsum"):
        assert names.count(n) == 1, n
    assert "vtx_topk_rows" not in names and "vtx_cross_entropy" not in names and "vtx_embed_fwd" not in names
    ld = (vocab + 7) // 8 * 8
    assert eng._cls["logits"].shape == (B, ld) and eng._cls["logits"].dtype == BF16 and eng._cls["logits_f32"] is None
    if vocab == 81:
        assert ld == 88
    head = [c for c in recorder if c[0] == "gemm"]
    fwd = [c for c in head if c[1:4] == (B, vocab, 2048)]
    assert len(fwd) == 1 and fwd[0][4].dtype == BF16 and fwd[0][4].stride(0) == ld and fwd[0][5]["bias"] is not None
    dgrad = [c for c in head if c[1:4] == (B, 2048, vocab)]
    assert len(dgrad) == 1 and dgrad[0][5]["b_mn"] == 1
    wgrad = [c for c in head if c[1:4] == (vocab, 2048, B)]
    assert len(wgrad) == 1 and wgrad[0][5]["atomic"] and wgrad[0][5]["a_mn"] == 1
    khot = next(c for c in recorder if c[0] == "vtx_khot_xent")
    # (logits, ldl, labels, ldlab, B, L, V, ignore, n_ignore, loss, write_grad, stream)
    assert khot[2] == ld and khot[5:8] == (B, batch["labels"].shape[1], vocab) and khot[9] == len(ignore) and khot[11] == 1
    mean_bwd = next(c for c in recorder if c[0] == "vtx_group_mean_bwd")
    assert mean_bwd[3:6] == (B, 49, 2048)
    # the pool's adjoint feeds the backbone backward: its first launch comes after it
    assert names.index("vtx_group_mean_bwd") < names.index("vtx_bn_bwd_reduce")


def test_classification_eval_frozen_and_tape(recorder):
    model = _cls_model(81, [0])
    eng = model.engine
    batch = CO.synth_label_batch(2, seed=2, vocab=81, ignore=[0], image_size=224)
    eng.forward(batch["image"], None, None, None, training=False, with_grad=False, labels=batch["labels"])
    f32 = [c for c in recorder if c[0] == "gemm" and c[4].dtype == F32]
    assert len(f32) == 1 and f32[0][1:4] == (2, 81, 2048) and f32[0][4].stride(0) == 88
    assert next(c for c in recorder if c[0] == "vtx_khot_xent")[11] == 0
    with pytest.raises(RuntimeError):
        eng.backward()  # no dlogits were written
    assert "vtx_topk_rows" not in _names(recorder)
    out = eng.predictions()
    assert out.shape == (2, 10) and out.dtype == torch.int64
    topk = next(c for c in recorder if c[0] == "vtx_topk_rows")
    assert topk[2:6] == (88, 2, 81, 10)
    # frozen backbone: the linear layer's gradients only -- no dgrad, no pool adjoint, no backbone backward
    recorder.clear()
    eng = _cls_model(10000, [0, 1, 2, 3], frozen=True).engine
    eng.forward(batch["image"], None, None, None, training=True, with_grad=True, labels=batch["labels"])
    tags = []
    eng.backward(bucket_cb=tags.append)
    names = _names(recorder)
    assert tags == ["head", "rest"]
    assert "vtx_group_mean_bwd" not in names and not any(n.startswith("vtx_bn_bwd") for n in names)
    assert not any(c[0] == "gemm" and c[1:4] == (2, 2048, 10000) for c in recorder)
    assert names.count("vtx_colsum") == 1
